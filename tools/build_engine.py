#!/usr/bin/env python
"""Build a B2ENGINE plan file -- the step the reference performs with `trtexec` (reference models/setup.py:32-56,
examples/ONNX/resnet50/build.py:35-67).

  python tools/build_engine.py --model resnet50 --precision fp16 --batch 8 -o rn50_b8_fp16.plan
  python tools/build_engine.py --prototxt /path/ResNet-152-deploy.prototxt --precision fp16 --batch 32 -o rn152.plan
  python tools/build_engine.py --model mnist --precision fp32 --batch 1 -o mnist.plan
  python tools/build_engine.py --prototxt deploy.prototxt --caffemodel weights.caffemodel --precision int8 --batch 32 -o rn.plan
  python tools/build_engine.py --model resnet50 --precision fp8 --batch 8 -o rn50_fp8.plan  (E4M3 bottleneck convolutions)
  python tools/build_engine.py --model resnet50 --batch 8 --tune -o rn50_tuned.plan      (on a GPU box: tactics in the file)
  python tools/build_engine.py --model resnext50 --precision fp16 --batch 8 --tune -o rx50.plan  (ResNeXt-50 32x4d)
  python tools/build_engine.py --model resnext50 --precision int8 --batch 8 -o rx50_int8.plan  (grouped 1-byte convolutions)
  python tools/build_engine.py --model bert-base --seq 128 --batch 16 [--weights bert.npz] --tune -o bert.plan  (fp16)
  python tools/build_engine.py --model bert-base --seq 384 --batch 16 --remove-padding -o bert_packed.plan  (masked tokens skipped)
  python tools/build_engine.py --model vit-b16 --batch 8 [--weights vit.npz] --tune -o vit.plan  (ViT-B/16, also vit-b32 / vit-l16; fp16)
  python tools/build_engine.py --model googlenet --batch 8 [--caffemodel bvlc_googlenet.caffemodel] --tune -o googlenet.plan  (fp16)
  python tools/build_engine.py --model densenet121 --batch 8 [--caffemodel F | --weights tv.npz] --tune -o densenet.plan  (fp16;
      also densenet169 / densenet201; --weights: a torchvision densenetNNN state_dict saved as .npz)
  python tools/build_engine.py --model vgg16 --batch 8 [--caffemodel VGG_ILSVRC_16_layers.caffemodel | --weights tv.npz] --tune
      -o vgg16.plan  (fp16; also vgg19; --weights: a torchvision vggNN state_dict saved as .npz)
Weights: deterministic synthetic weights (the reference's benchmark engines are weightless too, models/README.md:6-7),
unless --caffemodel names a binary NetParameter (trtexec --model=...); MNIST and --onnx carry their own weights.
--precision int8 / fp8: post-training quantization (fp8: E4M3), max-abs calibration on --calib (an .npy [N,C,H,W] fp32) or on
synthetic images.  Grouped convolutions are quantized too when Cin/g == Cout/g divides 128 or is a multiple of 128; a
model with any other grouped geometry builds in fp16 or fp32 only.
--tune: time the kernel configurations on this machine's GPU (what trtexec does while building) and store the tactic table
in the plan file; an engine deserialized from it never tunes at load.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tensorrt_laboratory_b200 import builder, graph, weights  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", choices=["resnet50", "resnet152", "resnext50", "mnist", "bert-base", "vit-b16", "vit-b32", "vit-l16", "googlenet",
                                        "densenet121", "densenet169", "densenet201", "vgg16", "vgg19"])
    ap.add_argument("--seq", type=int, default=128, help="bert-base: the sequence length of the plan (64, 128, 256, 384 or 512)")
    ap.add_argument("--weights", help="bert-base / vit-*: .npz of Hugging Face BertModel / ViTForImageClassification parameters; "
                                        "densenet* / vgg*: .npz of a torchvision state_dict (default: seeded weights)")
    ap.add_argument("--remove-padding", action="store_true",
                    help="bert-base: a packed plan that computes only the tokens with input_mask != 0 (same bindings)")
    ap.add_argument("--prototxt")
    ap.add_argument("--onnx", help="ONNX CNN classifier (Conv / BatchNormalization / Relu / Add / MaxPool / AveragePool / "
                                   "GlobalAveragePool / Flatten / Reshape / Gemm / MatMul / Softmax), e.g. an ONNX-zoo ResNet")
    ap.add_argument("--precision", choices=["fp16", "fp32", "int8", "fp8"], default="fp16")
    ap.add_argument("--caffemodel", help="binary caffe NetParameter with the weights of --prototxt / --model resnetNN")
    ap.add_argument("--calib", help="int8 / fp8: .npy of calibration inputs [N, C, H, W] fp32 (default: 8 synthetic images)")
    ap.add_argument("--tune", action="store_true", help="needs a GPU: tune kernel tactics now and embed them in the plan")
    ap.add_argument("--tune-all-batches", action="store_true", help="with --tune: one tactic set per batch size 1..max")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("-o", "--output", required=True)
    a = ap.parse_args()
    prec = {"fp16": builder.PREC_FP16, "fp32": builder.PREC_FP32, "int8": builder.PREC_INT8, "fp8": builder.PREC_FP8}[a.precision]

    def weights_for(net):
        if a.caffemodel:
            from tensorrt_laboratory_b200 import caffemodel
            return caffemodel.load_caffemodel(a.caffemodel, net)
        return weights.random_weights(net, a.seed)

    if a.model == "bert-base":  # its own builder: int32 token bindings, fp16 only
        from tensorrt_laboratory_b200 import bert
        cfg = bert.BertConfig(seq=a.seq)
        blob = builder.build_bert_plan(cfg, a.weights, a.batch, seed=a.seed, precision=prec, remove_padding=a.remove_padding)
        net = {"name": f"bert-base S={a.seq}" + (" packed" if a.remove_padding else "")}
    elif a.model in ("vit-b16", "vit-b32", "vit-l16"):  # its own builder: patch and token ops, fp16 only
        from tensorrt_laboratory_b200 import vit
        cfg = {"vit-b16": vit.VIT_B16, "vit-b32": vit.VIT_B32, "vit-l16": vit.VIT_L16}[a.model]
        blob = builder.build_vit_plan(cfg, a.weights, a.batch, seed=a.seed, precision=prec)
        net = {"name": a.model}
    elif a.prototxt:
        with open(a.prototxt) as f:
            net = graph.parse_prototxt(f.read())
        wts = weights_for(net)
    elif a.onnx:
        from tensorrt_laboratory_b200 import onnx_import, onnx_lite
        net, wts = onnx_import.import_onnx(onnx_lite.load_model(a.onnx), name=os.path.splitext(os.path.basename(a.onnx))[0])
    elif a.model == "mnist":
        sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
        from tests import helpers
        net, wts, _, _ = helpers.load_mnist_golden()
    elif a.model == "googlenet":  # BVLC GoogLeNet (no auxiliary classifiers): Concat and LRN, fp16 only
        net = graph.googlenet_caffe()
        wts = weights_for(net)
    elif a.model.startswith("densenet"):  # pre-activation 1x1s and growing concatenations, fp16 only
        net = graph.densenet_caffe(int(a.model[8:]))
        if prec != builder.PREC_FP16:
            raise SystemExit("DenseNet builds in fp16 only")
        if a.weights:
            from tensorrt_laboratory_b200 import densenet
            wts = densenet.load_weights(a.weights, int(a.model[8:]))
        else:
            wts = weights_for(net)
    elif a.model in ("vgg16", "vgg19"):  # hidden FC layers on the streaming tensor-core FC kernel, fp16 only
        net = graph.vgg_caffe(int(a.model[3:]))
        if prec != builder.PREC_FP16:
            raise SystemExit("VGG builds in fp16 only")
        if a.weights:
            from tensorrt_laboratory_b200 import vgg
            wts = vgg.load_weights(a.weights, int(a.model[3:]))
        else:
            wts = weights_for(net)
    elif a.model == "resnext50":  # 32x4d: grouped 3x3 convolutions, cpg 4 ... 32 (every precision)
        net = graph.resnext_caffe(50)
        wts = weights_for(net)
    else:
        net = graph.resnet_caffe(int(a.model[6:]))
        wts = weights_for(net)
    if a.model not in ("bert-base", "vit-b16", "vit-b32", "vit-l16"):
        low = graph.lower(net, wts)
        if prec in (builder.PREC_INT8, builder.PREC_FP8):
            import numpy as np
            from tensorrt_laboratory_b200 import quantize
            if a.calib:
                calib = np.load(a.calib).astype(np.float32)
            else:
                calib = weights.synthetic_input(8, chw=tuple(net["input_dims"][1:]), seed=4321)
            low = quantize.quantize_lowered(low, calib, fmt="e4m3" if prec == builder.PREC_FP8 else "int8", grouped=True)
        blob = builder.build_plan(low, prec, a.batch)
    if a.tune:
        from tensorrt_laboratory_b200 import capi
        eng = capi.Engine(blob)
        n = eng.tune(streams=4, all_batches=a.tune_all_batches)
        blob = builder.attach_tactics(blob, eng.tactics())
        print(f"tuned {n} tactics on this GPU")
    with open(a.output, "wb") as f:
        f.write(blob)
    print(f"wrote {a.output}: {len(blob) / 1e6:.1f} MB, {net['name']}, {a.precision}, max batch {a.batch}")


if __name__ == "__main__":
    main()
