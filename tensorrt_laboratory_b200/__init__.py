"""H100-native replacement for the per-request inference hot path of trtlab/tensorrt.

Python side: model front-ends (Caffe prototxt / ONNX-lite), deterministic weights, engine-blob builder
and a ctypes binding of the C-ABI ``libb200infer.so`` (see ``include/b200infer.h``).  All compute is
in ``csrc/`` (hand-written sm_90a CUDA); there is no CPU fallback.
"""
__version__ = "0.1.0"
