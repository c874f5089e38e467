"""Small CNN layer lists (test infrastructure only) in the layer names and forms of the full generators in ``graph``, for
per-op and whole-net tests of GoogLeNet, DenseNet and VGG."""
from __future__ import annotations

from typing import Optional, Sequence


def inception_net(cin: int = 64, hw: int = 14, widths=(16, 32, 48, 96), reduce=(24, 16), lrn: Optional[dict] = None,
                  pool_proj: bool = True, name: str = "inception") -> dict:
    """A small inception module in the BVLC names: [LRN ->] 1x1 | 3x3 reduce -> 3x3 | 5x5 reduce -> 5x5 | pool -> pool proj,
    concatenated.  ``widths``: the four branch outputs (the last is the pool projection)."""
    L = []

    def conv(lname, bottom, nout, k, pad=0):
        L.append(dict(name=lname, type="Convolution", bottoms=[bottom], tops=[lname], num_output=nout, kernel_size=k, pad=pad,
                      stride=1, bias_term=True))
        L.append(dict(name=lname + "_relu", type="ReLU", bottoms=[lname], tops=[lname]))

    prev = "data"
    if lrn:
        L.append(dict(name="norm", type="LRN", bottoms=["data"], tops=["norm"], **lrn))
        prev = "norm"
    conv("b/1x1", prev, widths[0], 1)
    conv("b/3x3_reduce", prev, reduce[0], 1)
    conv("b/3x3", "b/3x3_reduce", widths[1], 3, 1)
    conv("b/5x5_reduce", prev, reduce[1], 1)
    conv("b/5x5", "b/5x5_reduce", widths[2], 5, 2)
    L.append(dict(name="b/pool", type="Pooling", bottoms=[prev], tops=["b/pool"], pool="MAX", kernel_size=3, stride=1, pad=1))
    conv("b/pool_proj", "b/pool", widths[3], 1)
    L.append(dict(name="b/output", type="Concat", bottoms=["b/1x1", "b/3x3", "b/5x5", "b/pool_proj"], tops=["b/output"], axis=1))
    return {"name": name, "input": "data", "input_dims": [1, cin, hw, hw], "layers": L}


def dense_net(cin: int = 64, hw: int = 16, layers: int = 3, growth: int = 32, bottleneck: int = 128, classes: int = 16) -> dict:
    """A small DenseNet in the layer names and form of ``graph.densenet_caffe``: a 1x1 stem convolution (+ BN, ReLU) of
    ``cin`` channels, the 3x3/2 pad-1 max pool (FLOOR) that starts block 2, ``layers`` dense layers, a transition
    (BN-ReLU-1x1-AVE 2x2/2) into block 3 with ``layers`` more, then BN-ReLU, the global average pool, fc6 and prob."""
    L = []

    def conv(name, bottom, nout, k, pad=0):
        L.append(dict(name=name, type="Convolution", bottoms=[bottom], tops=[name], num_output=nout, kernel_size=k, pad=pad, stride=1,
                      bias_term=False))

    def bsr(prefix, relu, bottom):
        bn = prefix + "/bn"
        L.append(dict(name=bn, type="BatchNorm", bottoms=[bottom], tops=[bn], use_global_stats=True, eps=1e-5))
        L.append(dict(name=prefix + "/scale", type="Scale", bottoms=[bn], tops=[bn], bias_term=True))
        L.append(dict(name=relu, type="ReLU", bottoms=[bn], tops=[bn]))
        return bn

    conv("conv1", "data", cin, 1)
    L.append(dict(name="pool1", type="Pooling", bottoms=[bsr("conv1", "relu1", "conv1")], tops=["pool1"], pool="MAX", kernel_size=3,
                  stride=2, pad=1, ceil_mode=False))
    prev, c = "pool1", cin
    for b in (2, 3):
        for l in range(1, layers + 1):
            x1, x2 = f"conv{b}_{l}/x1", f"conv{b}_{l}/x2"
            conv(x1, bsr(x1, f"relu{b}_{l}/x1", prev), bottleneck, 1)
            conv(x2, bsr(x2, f"relu{b}_{l}/x2", x1), growth, 3, 1)
            L.append(dict(name=f"concat_{b}_{l}", type="Concat", bottoms=[prev, x2], tops=[f"concat_{b}_{l}"], axis=1))
            prev, c = f"concat_{b}_{l}", c + growth
        if b == 2:
            c //= 2
            conv("conv2_blk", bsr("conv2_blk", "relu2_blk", prev), c, 1)
            L.append(dict(name="pool2", type="Pooling", bottoms=["conv2_blk"], tops=["pool2"], pool="AVE", kernel_size=2, stride=2, pad=0))
            prev = "pool2"
    L.append(dict(name="pool5", type="Pooling", bottoms=[bsr("conv5_blk", "relu5_blk", prev)], tops=["pool5"], pool="AVE",
                  kernel_size=hw // 4, stride=1, pad=0))
    L.append(dict(name="fc6", type="InnerProduct", bottoms=["pool5"], tops=["fc6"], num_output=classes, bias_term=True))
    L.append(dict(name="prob", type="Softmax", bottoms=["fc6"], tops=["prob"]))
    return {"name": "dense", "input": "data", "input_dims": [1, 3, hw, hw], "layers": L}


def fc_net(chw: Sequence[int], couts: Sequence[int], relus: Sequence[bool], name: Optional[str] = None) -> dict:
    """data [C, H, W] -> fc1 (-> relu1) [-> fc2 (-> relu2)]: one or two InnerProduct layers, no softmax, so every FC output
    can be bound."""
    L, prev = [], "data"
    for i, (c, r) in enumerate(zip(couts, relus), 1):
        L.append(dict(name=f"fc{i}", type="InnerProduct", bottoms=[prev], tops=[f"fc{i}"], num_output=c, bias_term=True))
        if r:
            L.append(dict(name=f"relu{i}", type="ReLU", bottoms=[f"fc{i}"], tops=[f"fc{i}"]))
        prev = f"fc{i}"
    tag = "_".join(f"{c}{'r' if r else ''}" for c, r in zip(couts, relus))
    return {"name": name or f"fc_{'x'.join(map(str, chw))}_{tag}", "input": "data", "input_dims": [1, *chw], "layers": L}
