"""Plan builder: lowered graph (+ folded weights) -> B2ENGINE blob.

This is the offline step the reference performs with ``trtexec`` (reference ``models/setup.py:32-56``,
``examples/ONNX/resnet50/build.py:35-67``): it fixes precision and max batch, lays weights out in the
kernel-native format and writes one self-contained file that ``Runtime::DeserializeEngine`` loads
(reference ``trtlab/tensorrt/src/runtime.cc:62-95``).  Binary layout: ``csrc/plan_format.h``.
"""
from __future__ import annotations

import struct
from typing import Dict, List, Optional, Sequence

import numpy as np

from . import graph as G

PREC_FP32, PREC_FP16, PREC_INT8, PREC_FP8 = 0, 1, 2, 3
OP_INPUT_CAST, OP_CONV, OP_MAXPOOL, OP_AVGPOOL, OP_FC, OP_SOFTMAX, OP_OUTPUT_CAST, OP_QUANTIZE = range(8)
OP_EMBED_LN, OP_LAYERNORM, OP_ATTENTION, OP_POOLER = range(8, 12)   # transformer ops (version-3 plans)
OP_PATCHIFY, OP_TOKENS, OP_CLS_HEAD = range(12, 15)                  # Vision Transformer ops (version-3 plans)
OP_LRN = 15                                                          # local response normalisation (version-4 plans)
CONV_RELU, CONV_PACKED, CONV_INT8, CONV_GELU = 1, 2, 4, 8            # OpRec.relu bits of a convolution
CONV_PREACT = 16  # OpRec.relu bit of a convolution or average pool: BatchNorm + ReLU input prologue (version-4 plans)
FC_STREAM = 32    # OpRec.relu bit of an FC: streaming tensor-core FC layer, packed weights (version-4 fp16 plans; bit 0 = ReLU)
FLAG_ROWS_OUT, FLAG_PACKED = 1, 2  # OpRecV3.flags: channels-last output cast; op on packed (padding-free) rows
T_ACT, T_VEC = 0, 1
MAGIC = b"B2ENGINE"
VERSION = 1           # plans without grouped convolutions: 176-byte op records
VERSION_GROUPED = 2   # a plan with at least one grouped convolution: 192-byte op records (+ groups)
VERSION_TRANSFORMER = 3  # a plan with transformer ops or a GELU convolution: 224-byte op records (plan_format.h OpRecV3)
VERSION_CONCAT = 4    # a plan with channel-slice convolutions or LRN: 192-byte op records (+ groups, out_c0, out_cw)

_HEADER = struct.Struct("<8sIIIIIIQQ64s16x")
_TENSOR = struct.Struct("<64sIIIIIif4x")  # ... binding, scale (INT8 tensors: real value = q * scale; 0 = fp16 / fp32 tensor)
_OP = struct.Struct("<64sIiiiiIIIIIIIIIIIQQQQIIII")
_OP_V2 = struct.Struct("<64sIiiiiIIIIIIIIIIIQQQQIIIII12x")  # version 2: _OP + groups + 12 reserved bytes
# version 3: _OP + groups, heads, vocab, positions, types, binding2, binding3, out2, eps, flags + 8 reserved bytes
_OP_V3 = struct.Struct("<64sIiiiiIIIIIIIIIIIQQQQIIIIIIIIIiiifI8x")
_OP_V4 = struct.Struct("<64sIiiiiIIIIIIIIIIIQQQQIIIIIII4x")  # version 4: _OP + groups, out_c0, out_cw + 4 reserved bytes
_BINDING = struct.Struct("<64sIIiI8i16x")
assert _HEADER.size == 128 and _TENSOR.size == 96 and _OP.size == 176 and _OP_V2.size == 192 and _OP_V3.size == 224 and _OP_V4.size == 192
assert _BINDING.size == 128


def grouped_tc_span(cin: int, cout: int, groups: int, cin_phys: int, cout_phys: int) -> int:
    """K elements per filter tap in the weight row of a grouped fp16 convolution that runs on the tensor cores, or 0 when
    its geometry runs on the SIMT convolution.  Tensor-core geometries have Cin/g == Cout/g == cpg with cpg | 64 (a group
    lies inside one 64-channel block: span 64) or 64 | cpg (span cpg)."""
    if groups <= 1 or cin != cout or cin_phys != cout_phys or cin_phys % 64 or cout_phys % 32:
        return 0
    cpg = cin // groups
    if 64 % cpg and cpg % 64:
        return 0
    return max(cpg, 64)


def grouped_1byte_span(cin: int, cout: int, groups: int) -> int:
    """K bytes per filter tap in the weight row of a grouped INT8 / FP8 convolution, or 0 when the 1-byte kernels do not
    run its geometry.  They need Cin/g == Cout/g == cpg with cpg | 128 (a group lies inside one 128-channel row of the
    1-byte layout: span 128) or 128 | cpg (span cpg)."""
    if groups <= 1 or cin != cout or cin % groups:
        return 0
    cpg = cin // groups
    if 128 % cpg and cpg % 128:
        return 0
    return max(cpg, 128)


def expand_grouped_weights(W: np.ndarray, groups: int, span: int, cout_phys: int) -> np.ndarray:
    """Block-diagonal weight rows of a tensor-core grouped convolution: W [Cout, taps, cpg] -> [Cout_phys, taps, span].
    Row o is read against the `span` input channels starting at channel (o // span) * span, so its cpg real weights sit
    at columns g*cpg - (o // span)*span ... (g = o's group) and every other column is zero."""
    cout, taps, cpg = W.shape
    out = np.zeros((cout_phys, taps, span), dtype=W.dtype)
    o = np.arange(cout)
    col = (o // cpg) * cpg - (o // span) * span
    out[o[:, None, None], np.arange(taps)[None, :, None], (col[:, None] + np.arange(cpg)[None, :])[:, None, :]] = W
    return out


def _roundup(v: int, m: int) -> int:
    return (v + m - 1) // m * m


def _pad_vec(v: np.ndarray, n: int) -> np.ndarray:
    out = np.zeros(n, dtype=np.float32)
    out[:len(v)] = v
    return out


def phys_channels(c: int, precision: int) -> int:
    """Channel padding policy of activation tensors.  fp16/tcgen05: 8 (one 16-byte TMA element row,
    un-swizzled K-chunks) for thin inputs, otherwise a multiple of 64 (one 128-byte swizzle row)."""
    if precision == PREC_FP32:
        return c
    return 8 if c <= 8 else _roundup(c, 64)


def stem_s2d_transform(W: np.ndarray, k: int, pad: int, w_in: int):
    """Re-express a stride-2, thin-input (Cin <= 4) convolution on a horizontally space-to-depth packed input.

    The packed tensor holds pixel pairs: X2[n, h, w2, dw*4 + c] = X[n, c, h, 2*w2 + dw].  Column 2q - pad + s of
    the original becomes packed column q + a with a = floor((s - pad)/2), dw = (s - pad) mod 2, so the
    kxk / stride-2 conv turns into a k x kw2 conv with stride (2, 1) over 8 channels -- 4/7 of the im2col TMA
    loads and of the zero-padded K for the 7x7 stem.  Returns (W2 [cout, k, kw2, 8], kw2, pad_lo, pad_hi).
    """
    cout, kh, kw, cin = W.shape
    assert kh == kw == k and cin <= 4 and w_in % 2 == 0
    a_min = (0 - pad) // 2
    a_max = (k - 1 - pad) // 2
    kw2 = a_max - a_min + 1
    W2 = np.zeros((cout, kh, kw2, 8), dtype=W.dtype)
    for s_ in range(k):
        a = (s_ - pad) // 2
        dw = (s_ - pad) - 2 * a
        W2[:, :, a - a_min, dw * 4:dw * 4 + cin] = W[:, :, s_, :]
    q = (w_in + 2 * pad - k) // 2 + 1
    pad_lo = -a_min
    pad_hi = q - 1 + kw2 - w_in // 2 - pad_lo
    assert pad_hi >= 0
    return W2, kw2, pad_lo, pad_hi


def pack_weights_sw128(W: np.ndarray) -> np.ndarray:
    """[Cout_phys, K] fp16 (K % 64 == 0, Cout_phys % 32 == 0) -> blocks [K/64][Cout/32][32 rows][128 B] whose bytes are
    exactly what the kernel wants in shared memory for a 64-K weight sub-tile under the 128-byte swizzle (16-byte
    chunk j of row r sits at chunk j ^ (r % 8)).  The N tile of ANY width BN in {32, 64, 128} for k-block kb is then
    ONE contiguous run of BN*128 bytes = one `cp.async.bulk` instruction (instruction issue, ~200 cycles per TMA op
    from a single thread, is what paces the main loop)."""
    cout, K = W.shape
    assert cout % 32 == 0 and K % 64 == 0 and W.dtype == np.float16
    blk = W.reshape(cout // 32, 32, K // 64, 8, 8)            # [nb, r, kb, chunk, elem]
    blk = blk.transpose(2, 0, 1, 3, 4)                         # [kb, nb, r, chunk, elem]
    out = np.empty_like(blk)
    r = np.arange(32)
    for j in range(8):
        out[:, :, r, j ^ (r % 8), :] = blk[:, :, r, j, :]
    return np.ascontiguousarray(out).reshape(-1)


def pack_weights_sw128_i8(W: np.ndarray) -> np.ndarray:
    """INT8 twin of :func:`pack_weights_sw128`: [Cout_phys, K] int8 (K % 128 == 0) -> blocks [K/128][Cout/32][32 rows][128 B],
    16-byte chunk j of row r at chunk j ^ (r % 8): the shared-memory image of a 128-K weight sub-tile."""
    cout, K = W.shape
    assert cout % 32 == 0 and K % 128 == 0 and W.dtype == np.int8
    blk = W.reshape(cout // 32, 32, K // 128, 8, 16).transpose(2, 0, 1, 3, 4)   # [kb, nb, r, chunk, 16 bytes]
    out = np.empty_like(blk)
    r = np.arange(32)
    for j in range(8):
        out[:, :, r, j ^ (r % 8), :] = blk[:, :, r, j, :]
    return np.ascontiguousarray(out).reshape(-1)


def _name(s: str) -> bytes:
    b = s.encode()
    if len(b) > 63:
        b = b[:63]
    return b


def build_plan(lowered: dict, precision: int = PREC_FP16, max_batch: int = 8,
               outputs: Optional[Sequence[str]] = None, name: Optional[str] = None, stem_s2d: bool = True,
               pack_weights: bool = True, input_dtype: str = "f32") -> bytes:
    """Serialize ``lowered`` (from :func:`graph.lower` with weights) into a plan blob.

    ``input_dtype``: "f32" = the reference's binding contract (pybind casts inputs to float, infer.cc:435-441);
    "f16" (fp16 engines only) = the secondary mode of SURVEY.md §8(d): half the H2D bytes per request.

    ``outputs``: tensor names to expose as output bindings (default: the graph output).  4-D activation
    outputs get an ``OUTPUT_CAST`` to fp32 NCHW; vector outputs (fc / softmax) are written in place.
    """
    if precision not in (PREC_FP32, PREC_FP16, PREC_INT8, PREC_FP8):
        raise ValueError("precision must be PREC_FP32, PREC_FP16, PREC_INT8 or PREC_FP8")
    int8 = precision == PREC_INT8
    if int8 != bool(lowered.get("int8")):
        raise ValueError("PREC_INT8 takes a graph quantized by quantize.quantize_lowered (and only that precision does)")
    if (precision == PREC_FP8) != bool(lowered.get("fp8")):
        raise ValueError("PREC_FP8 takes a graph quantized by quantize.quantize_lowered(..., fmt='e4m3') (and only that "
                         "precision does)")
    tscale = lowered.get("tensor_scales", {})   # 1-byte (INT8 / FP8) tensors: name -> scale
    if precision in (PREC_INT8, PREC_FP8):  # the fp16 part of an INT8 / FP8 engine follows the fp16 engine's layout rules
        precision_fp = PREC_FP16
    else:
        precision_fp = precision
    wdtype = np.float16 if precision_fp == PREC_FP16 else np.float32
    outputs = list(outputs) if outputs else [lowered["output"]]
    concat = any("out_c0" in op for op in lowered["ops"])
    if (concat or any(op["type"] == G.OP_LRN for op in lowered["ops"])) and precision != PREC_FP16:
        raise ValueError("a graph with a Concat or LRN layer builds in fp16 only: channel concatenation and LRN have no fp32, "
                         "INT8 or FP8 kernels")
    shapes: Dict[str, tuple] = dict(lowered["tensors"])
    fcs = [op for op in lowered["ops"] if op["type"] == G.OP_FC]
    for op in fcs:
        if op.get("relu") and precision != PREC_FP16:
            raise ValueError(f"fc {op['name']}: an InnerProduct with a fused ReLU builds in fp16 only: hidden fully-connected "
                             "layers have no fp32, INT8 or FP8 kernels")
    # a plan with a hidden FC (or an FC with a fused ReLU) runs every FC on the streaming tensor-core kernel; hidden FC
    # outputs are fp16 activations
    fc_stream = precision == PREC_FP16 and any(op.get("hidden") or op.get("relu") for op in fcs)
    hidden = {op["output"] for op in fcs if fc_stream and op.get("hidden")}
    vec_tensors = {op["output"] for op in lowered["ops"] if op["type"] in (G.OP_FC, G.OP_SOFTMAX)} - hidden

    tensors: List[dict] = []
    tindex: Dict[str, int] = {}

    def add_tensor(tname: str) -> int:
        if tname in tindex:
            return tindex[tname]
        c, h, w = shapes[tname]
        if tname in vec_tensors:
            rec = dict(name=tname, kind=T_VEC, h=1, w=1, c=c * h * w, c_phys=c * h * w, binding=-1)
        elif tname in hidden:  # [1, 1, C]: the reader's K is c_phys, a multiple of 64
            rec = dict(name=tname, kind=T_ACT, h=1, w=1, c=c, c_phys=_roundup(c, 64), binding=-1)
        elif tname in tscale:  # 1-byte activations: one 128-byte swizzle row = 128 channels
            rec = dict(name=tname, kind=T_ACT, h=h, w=w, c=c, c_phys=_roundup(c, 128), binding=-1, scale=float(np.float32(tscale[tname])))
        else:
            rec = dict(name=tname, kind=T_ACT, h=h, w=w, c=c, c_phys=phys_channels(c, precision_fp), binding=-1)
        tindex[tname] = len(tensors)
        tensors.append(rec)
        return tindex[tname]

    bindings: List[dict] = []
    ops: List[dict] = []
    payload = bytearray()

    def add_payload(arr: np.ndarray):
        while len(payload) % 256:
            payload.append(0)
        off = len(payload)
        raw = np.ascontiguousarray(arr).tobytes()
        payload.extend(raw)
        return off, len(raw)

    # input binding + cast
    cin, hin, win = lowered["input_shape"]
    t_in = add_tensor(lowered["input"])
    if input_dtype not in ("f32", "f16") or (input_dtype == "f16" and precision_fp != PREC_FP16):
        raise ValueError("input_dtype is 'f32' (the reference's binding contract) or, for fp16 engines, 'f16'")
    bindings.append(dict(name=lowered["input"], is_input=1, dtype=1 if input_dtype == "f16" else 0, tensor=t_in,
                         dims=[cin, hin, win]))
    ops.append(dict(name="cast:" + lowered["input"], type=OP_INPUT_CAST, inp=-1, res=-1, out=t_in, binding=0))
    # fp16 stem: a stride-2 conv that is the only reader of a thin (<= 4 channel) even-width input runs on a
    # horizontally space-to-depth packed copy of the input (see stem_s2d_transform)
    readers = [o for o in lowered["ops"] if o["input"] == lowered["input"] or o.get("residual") == lowered["input"]]
    s2d_op = None
    if (precision_fp == PREC_FP16 and stem_s2d and len(readers) == 1 and readers[0]["type"] == G.OP_CONV
            and readers[0]["stride"] == 2 and cin <= 4 and win % 2 == 0 and lowered["input"] not in outputs
            and readers[0]["k"] >= 3 and readers[0].get("groups", 1) == 1):
        s2d_op = readers[0]
        _, _, s2d_lo, s2d_hi = stem_s2d_transform(s2d_op["W"], s2d_op["k"], s2d_op["pad"], win)
        # the horizontal padding is made PHYSICAL (zero pixels written by the cast), so the conv has pad_w = 0 and its
        # kw taps are contiguous in memory: the engine reads a whole filter row as one 64-byte TMA "pixel"
        tensors[t_in].update(w=win // 2 + s2d_lo + s2d_hi, c=8, c_phys=8)
        ops[0].update(k=2, pad=s2d_lo, stride=s2d_hi)

    # concatenated tensors: each input convolution writes [out_c0, out_c0 + width); the last one's width runs to c_phys, so
    # its zero weight rows rewrite the tail padding on every pass
    slice_width: Dict[str, int] = {}
    writers: Dict[str, List[dict]] = {}
    for op in lowered["ops"]:
        if "out_c0" in op:
            writers.setdefault(op["output"], []).append(op)
    for tname, ws in writers.items():
        c_phys = phys_channels(shapes[tname][0], PREC_FP16)
        ws = sorted(ws, key=lambda o: o["out_c0"])
        for k, op in enumerate(ws):
            if op["out_c0"] % 8:
                raise ValueError(f"Concat {tname}: input {op['name']} starts at channel {op['out_c0']}, not a multiple of 8 "
                                 "(the 16-byte alignment of the convolution's output store)")
            if op["type"] == G.OP_MAXPOOL and k + 1 < len(ws):  # a max pool writes its input's padded channels
                slice_width[op["name"]] = phys_channels(shapes[op["input"]][0], PREC_FP16)
            else:
                slice_width[op["name"]] = c_phys - op["out_c0"] if k + 1 == len(ws) else op["cout"]

    for op in lowered["ops"]:
        t = op["type"]
        ti = add_tensor(op["input"])
        to = add_tensor(op["output"])
        rec = dict(name=op["name"], inp=ti, res=-1, out=to, binding=-1)
        if t == "quantize":
            rec.update(type=OP_QUANTIZE)
        elif t == G.OP_CONV and (op.get("int8") or op.get("fp8")):
            cin_phys, cout_phys = tensors[ti]["c_phys"], tensors[to]["c_phys"]
            k = op["k"]
            taps = k * k
            groups = op.get("groups", 1)
            if groups > 1:  # block-diagonal rows [Cout_phys][taps][span], packed as a dense [Cout_phys, taps * span] matrix
                span = grouped_1byte_span(op["cin"], op["cout"], groups)
                if not span:
                    raise ValueError(f"conv {op['name']}: no 1-byte kernel for {op['cin']} -> {op['cout']} channels in {groups} groups")
                Wg = op["Wq"].view(np.int8).reshape(op["cout"], taps, op["cin"] // groups)
                Wx = expand_grouped_weights(Wg, groups, span, cout_phys)
                w_off, w_bytes = add_payload(pack_weights_sw128_i8(Wx.reshape(cout_phys, taps * span)))
                rec["groups"] = groups
            else:
                Wq = np.zeros((cout_phys, taps, cin_phys), dtype=np.int8)   # E4M3 codes travel as their bytes; 0x00 is +0
                Wq[:op["cout"], :, :op["cin"]] = op["Wq"].view(np.int8).reshape(op["cout"], taps, op["cin"])
                w_off, w_bytes = add_payload(pack_weights_sw128_i8(Wq.reshape(cout_phys, taps * cin_phys)))
            rq = np.zeros(2 * cout_phys + 4, dtype=np.float32)   # [m | b | r 0 0 0]; padded channels requantise to 0
            rq[:op["cout"]] = op["m"]
            rq[cout_phys:cout_phys + op["cout"]] = op["b"]
            rq[2 * cout_phys] = op["r"] if op["r"] is not None else 0.0
            b_off, b_bytes = add_payload(rq)
            rec.update(type=OP_CONV, k=k, stride=op["stride"], pad=op["pad"], relu=int(op["relu"]) | 2 | 4,
                       cin=op["cin"], cout=op["cout"], cin_phys=cin_phys, cout_phys=cout_phys, taps=taps, taps_phys=taps,
                       w_off=w_off, w_bytes=w_bytes, b_off=b_off, b_bytes=b_bytes)
            if op["residual"] is not None:
                rec["res"] = add_tensor(op["residual"])
        elif t == G.OP_CONV and op.get("groups", 1) > 1:
            if "W" not in op:
                raise ValueError(f"conv {op['name']}: lowered graph carries no weights")
            # tensor-core geometry: packed block-diagonal rows [Cout_phys][taps][span]; otherwise (SIMT, fp32 engines)
            # row-major [Cout_phys][taps][Cin/groups]
            groups = op["groups"]
            cin_phys, cout_phys = tensors[ti]["c_phys"], tensors[to]["c_phys"]
            k = op["k"]
            taps, cpg_in = k * k, op["cin"] // groups
            Wg = op["W"].reshape(op["cout"], taps, cpg_in)
            span = grouped_tc_span(op["cin"], op["cout"], groups, cin_phys, cout_phys)
            packed = precision_fp == PREC_FP16 and pack_weights and span > 0
            if packed:
                Wx = expand_grouped_weights(Wg.astype(np.float16), groups, span, cout_phys)
                w_off, w_bytes = add_payload(pack_weights_sw128(Wx.reshape(cout_phys, taps * span)))
            else:
                W = np.zeros((cout_phys, taps, cpg_in), dtype=np.float32)
                W[:op["cout"]] = Wg
                w_off, w_bytes = add_payload(W.astype(wdtype))
            bias = np.zeros(cout_phys, dtype=np.float32)
            bias[:op["cout"]] = op["bias"]
            b_off, b_bytes = add_payload(bias)
            rec.update(type=OP_CONV, k=k, stride=op["stride"], pad=op["pad"], relu=int(op["relu"]) | (2 if packed else 0),
                       cin=op["cin"], cout=op["cout"], cin_phys=cin_phys, cout_phys=cout_phys, taps=taps, taps_phys=taps,
                       w_off=w_off, w_bytes=w_bytes, b_off=b_off, b_bytes=b_bytes, groups=groups)
            if op["residual"] is not None:
                rec["res"] = add_tensor(op["residual"])
        elif t == G.OP_CONV:
            if "W" not in op:
                raise ValueError(f"conv {op['name']}: lowered graph carries no weights")
            cin_phys = tensors[ti]["c_phys"]
            if op["input"] in writers and op["cin"] < shapes[op["input"]][0]:  # input prefix: channels [0, cin) of a concatenation
                cin_phys = _roundup(op["cin"], 64)
            cout_phys = tensors[to]["c_phys"]
            k = op["k"]
            Wsrc, cin_eff, extra = op["W"], op["cin"], {}
            if op["name"] in slice_width:  # weight rows = the slice width rounded up to 64; rows past cout are zero
                cw = slice_width[op["name"]]
                cout_phys = _roundup(cw, 64)
                extra = dict(out_c0=op["out_c0"], out_cw=cw)
                if cin_phys % 64 or not pack_weights or op is s2d_op:
                    raise ValueError(f"conv {op['name']}: a concatenated convolution needs a multiple of 64 input channels "
                                     "and packed weights")
            taps = k * k
            if op is s2d_op:
                Wsrc, kw2, pad_lo, pad_hi = stem_s2d_transform(op["W"], k, op["pad"], win)
                cin_eff, taps = 8, k * kw2
                extra = dict(kw=kw2, stride_w=1, pad_w_lo=0, pad_w_hi=0, ceil_mode=op["cin"] * k * k)
            taps_phys = _roundup(taps, 2) if (precision_fp == PREC_FP16 and cin_phys == 8) else taps
            W = np.zeros((cout_phys, taps_phys, cin_phys), dtype=np.float32)
            W[:op["cout"], :taps, :cin_eff] = Wsrc.reshape(op["cout"], taps, cin_eff)
            bias = np.zeros(cout_phys, dtype=np.float32)
            bias[:op["cout"]] = op["bias"]
            packed = precision_fp == PREC_FP16 and cin_phys % 64 == 0 and cout_phys % 32 == 0 and pack_weights
            if packed:
                w_off, w_bytes = add_payload(pack_weights_sw128(W.astype(np.float16).reshape(cout_phys, taps_phys * cin_phys)))
            else:
                w_off, w_bytes = add_payload(W.astype(wdtype))
            pre = 0
            if op.get("pre"):  # b = [bias cout_phys][scale cin_phys][shift cin_phys]
                if precision_fp != PREC_FP16 or not packed:
                    raise ValueError(f"conv {op['name']}: a BatchNorm + ReLU input prologue needs an fp16 plan with packed weights")
                bias = np.concatenate([bias, _pad_vec(op["pre_scale"], cin_phys), _pad_vec(op["pre_shift"], cin_phys)])
                pre = CONV_PREACT
            b_off, b_bytes = add_payload(bias)
            rec.update(type=OP_CONV, k=k, stride=op["stride"], pad=op["pad"], relu=int(op["relu"]) | (2 if packed else 0) | pre,
                       cin=cin_eff, cout=op["cout"], cin_phys=cin_phys, cout_phys=cout_phys,
                       taps=taps, taps_phys=taps_phys, w_off=w_off, w_bytes=w_bytes, b_off=b_off, b_bytes=b_bytes)
            rec.update(extra)
            if op["residual"] is not None:
                rec["res"] = add_tensor(op["residual"])
        elif t == G.OP_MAXPOOL:
            rec.update(type=OP_MAXPOOL, k=op["k"], stride=op["stride"], pad=op["pad"], ceil_mode=int(op["ceil_mode"]))
            if op["name"] in slice_width:
                if precision_fp != PREC_FP16:
                    raise ValueError(f"maxpool {op['name']}: a concatenated max pool needs an fp16 plan")
                rec.update(out_c0=op["out_c0"], out_cw=slice_width[op["name"]])
        elif t == G.OP_AVGPOOL and op.get("pre"):  # b = [scale c_phys][shift c_phys]
            if precision_fp != PREC_FP16:
                raise ValueError(f"avgpool {op['name']}: a BatchNorm + ReLU input prologue needs an fp16 plan")
            c_phys = tensors[ti]["c_phys"]
            b_off, b_bytes = add_payload(np.concatenate([_pad_vec(op["pre_scale"], c_phys), _pad_vec(op["pre_shift"], c_phys)]))
            rec.update(type=OP_AVGPOOL, k=op["k"], stride=op["k"], relu=CONV_PREACT, b_off=b_off, b_bytes=b_bytes)
        elif t == G.OP_AVGPOOL:
            if tensors[to]["h"] != 1 or tensors[to]["w"] != 1:
                raise ValueError(f"avgpool {op['name']}: a windowed average pool runs only with a BatchNorm + ReLU input prologue")
            rec.update(type=OP_AVGPOOL, k=op["k"], stride=op["stride"])
        elif t == G.OP_FC and fc_stream:  # weights pack_weights_sw128 [cout_phys, K], bias [cout_phys]; plan_format.h kFcStream
            c, h, w = op["in_chw"]
            c_phys = tensors[ti]["c_phys"]
            if tensors[ti]["kind"] != T_ACT or (h * w * c_phys) % 64:
                raise ValueError(f"fc {op['name']}: a streaming FC layer reads an fp16 activation whose h * w * c_phys is a multiple of "
                                 f"64 (here {h} * {w} * {c_phys})")
            cout_phys = _roundup(op["cout"], 128)
            Wf = np.zeros((cout_phys, h * w, c_phys), dtype=np.float32)
            Wf[:op["cout"], :, :c] = op["W"].reshape(op["cout"], h * w, c)
            w_off, w_bytes = add_payload(pack_weights_sw128(Wf.astype(np.float16).reshape(cout_phys, h * w * c_phys)))
            b_off, b_bytes = add_payload(_pad_vec(op["bias"], cout_phys))
            rec.update(type=OP_FC, relu=int(bool(op.get("relu"))) | FC_STREAM, cin=op["cin"], cout=op["cout"], cin_phys=h * w * c_phys,
                       cout_phys=cout_phys, w_off=w_off, w_bytes=w_bytes, b_off=b_off, b_bytes=b_bytes)
        elif t == G.OP_FC:
            c, h, w = op["in_chw"]
            c_phys = tensors[ti]["c_phys"]
            Wf = np.zeros((op["cout"], h * w, c_phys), dtype=np.float32)
            Wf[:, :, :c] = op["W"].reshape(op["cout"], h * w, c)
            w_off, w_bytes = add_payload(Wf.astype(wdtype))
            b_off, b_bytes = add_payload(op["bias"].astype(np.float32))
            rec.update(type=OP_FC, cin=op["cin"], cout=op["cout"], cin_phys=h * w * c_phys, cout_phys=op["cout"],
                       w_off=w_off, w_bytes=w_bytes, b_off=b_off, b_bytes=b_bytes)
        elif t == G.OP_SOFTMAX:
            rec.update(type=OP_SOFTMAX)
        elif t == G.OP_LRN:
            b_off, b_bytes = add_payload(np.array([op["alpha"], op["beta"], op["k"]], dtype=np.float32))
            rec.update(type=OP_LRN, k=op["local_size"], b_off=b_off, b_bytes=b_bytes)
        else:
            raise ValueError(f"unsupported lowered op {t}")
        ops.append(rec)

    for oname in outputs:
        if oname not in tindex:
            raise ValueError(f"output tensor {oname!r} is not produced by the graph")
        ti = tindex[oname]
        trec = tensors[ti]
        bidx = len(bindings)
        if trec["kind"] == T_VEC:
            if trec["binding"] >= 0:
                raise ValueError(f"tensor {oname} bound twice")
            trec["binding"] = bidx
            bindings.append(dict(name=oname, is_input=0, dtype=0, tensor=ti, dims=[trec["c"]]))
        else:
            bindings.append(dict(name=oname, is_input=0, dtype=0, tensor=ti, dims=[trec["c"], trec["h"], trec["w"]]))
            ops.append(dict(name="cast:" + oname, type=OP_OUTPUT_CAST, inp=ti, res=-1, out=-1, binding=bidx))

    return _serialize(tensors, ops, bindings, payload, precision, max_batch, name or lowered["name"])


def _serialize(tensors: List[dict], ops: List[dict], bindings: List[dict], payload: bytearray, precision: int, max_batch: int,
               name: str) -> bytes:
    # version 1 unless a convolution is grouped (2) or the plan has transformer ops / GELU (3): every plan without them
    # stays byte-identical to what older builders wrote
    # version 4 when a convolution writes a channel slice or an op is an LRN
    # (and when an FC streams: kFcStream)
    concat = any(o["type"] == OP_LRN or "out_cw" in o or (o["type"] == OP_FC and o.get("relu", 0) & FC_STREAM) for o in ops)
    transformer = any(OP_EMBED_LN <= o["type"] <= OP_CLS_HEAD or (o["type"] == OP_CONV and o.get("relu", 0) & CONV_GELU) for o in ops)
    if concat and transformer:
        raise ValueError("a plan holds channel slices / LRN or transformer ops, not both")
    grouped = any(o.get("groups", 1) > 1 for o in ops)
    op_struct = _OP_V4 if concat else _OP_V3 if transformer else _OP_V2 if grouped else _OP
    version = VERSION_CONCAT if concat else VERSION_TRANSFORMER if transformer else VERSION_GROUPED if grouped else VERSION
    tables = _HEADER.size + len(tensors) * _TENSOR.size + len(ops) * op_struct.size + len(bindings) * _BINDING.size
    payload_offset = _roundup(tables, 256)
    blob = bytearray()
    blob += _HEADER.pack(MAGIC, version, precision, max_batch, len(tensors), len(ops),
                         len(bindings), payload_offset, len(payload), _name(name))
    for t in tensors:
        blob += _TENSOR.pack(_name(t["name"]), t["kind"], t["h"], t["w"], t["c"], t["c_phys"], t["binding"], t.get("scale", 0.0))
    for o in ops:
        fields = (_name(o["name"]), o["type"], o["inp"], o["res"], o["out"], o["binding"],
                  o.get("k", 0), o.get("stride", 0), o.get("pad", 0), o.get("relu", 0), o.get("ceil_mode", 0),
                  o.get("cin", 0), o.get("cout", 0), o.get("cin_phys", 0), o.get("cout_phys", 0),
                  o.get("taps", 0), o.get("taps_phys", 0),
                  o.get("w_off", 0), o.get("w_bytes", 0), o.get("b_off", 0), o.get("b_bytes", 0),
                  o.get("kw", 0), o.get("stride_w", 0), o.get("pad_w_lo", 0), o.get("pad_w_hi", 0))
        if transformer:
            blob += op_struct.pack(*fields, o.get("groups", 1), o.get("heads", 0), o.get("vocab", 0), o.get("positions", 0),
                                   o.get("types", 0), o.get("binding2", -1), o.get("binding3", -1), o.get("out2", -1),
                                   o.get("eps", 0.0), o.get("flags", 0))
        elif concat:
            blob += op_struct.pack(*fields, o.get("groups", 1), o.get("out_c0", 0), o.get("out_cw", 0))
        else:
            blob += op_struct.pack(*fields, o.get("groups", 1)) if grouped else op_struct.pack(*fields)
    for b in bindings:
        dims = list(b["dims"]) + [0] * (8 - len(b["dims"]))
        blob += _BINDING.pack(_name(b["name"]), b["is_input"], b["dtype"], b["tensor"], len(b["dims"]), *dims)
    blob += b"\0" * (payload_offset - len(blob))
    blob += payload
    return bytes(blob)


def build_bert_plan(cfg=None, weights=None, max_batch: int = 16, seed: int = 0, precision: int = PREC_FP16,
                    name: Optional[str] = None, taps: Sequence[str] = (), remove_padding: bool = False) -> bytes:
    """BERT encoder + pooler (``bert.BertConfig``; default BERT-base at S = 128; S = 64, 128, 256, 384 or 512) -> fp16
    plan (version 3).

    ``weights``: a dict or ``.npz`` path in Hugging Face ``BertModel`` names (``bert.load_weights``); default: seeded
    ``bert.random_weights(cfg, seed)``.  Activations are ``T_ACT`` tensors [N, 1, S, C], so every GEMM is a 1x1
    convolution on the tensor cores: Q, K and V fused into one layer of 3H output channels, ordered (part, head, d) --
    channel part * H + 64 * head + d with part 0 = Q, 1 = K, 2 = V; the attention output projection and the second FFN
    GEMM with the layer input as fused residual; the first FFN GEMM with GELU.  Bindings: int32 ``input_ids``,
    ``segment_ids``, ``input_mask`` ([S] per item, mask 1 = attend); fp32 ``last_hidden_state`` ([S, H], token-major) and
    ``pooled_output`` ([H]).  ``taps``: names of intermediate activation tensors (``embeddings``, ``l{i}.qkv``,
    ``l{i}.context``, ``l{i}.attn_sum``, ``l{i}.attn_ln``, ``l{i}.ffn``, ``l{i}.ffn_sum``, ``l{i}.out``) to expose as
    extra fp32 [S, C] output bindings of the same names.

    ``remove_padding``: a packed plan.  Same bindings, but only the tokens with ``input_mask != 0`` are computed: the
    embedding packs each batch's valid tokens into consecutive rows (in item and position order, each with its original
    position embedding), every GEMM and LayerNorm stops at the live row count, and attention runs per item over its own
    tokens.  ``last_hidden_state`` and the taps hold the encoder output at valid positions and exactly 0 at masked ones;
    ``pooled_output`` pools position 0, which is a zero row -- giving tanh(bias) -- when position 0 is masked.  For
    right-padded masks the valid rows are bit-identical to the padded plan's; any mask pattern is accepted."""
    from . import bert as Bm
    cfg = cfg or Bm.BERT_BASE
    if precision == PREC_FP32:
        raise ValueError("BERT plans are fp16 only: the attention, LayerNorm and embedding kernels exist for fp16 activations")
    if precision == PREC_INT8:
        raise ValueError("BERT plans are fp16 only: INT8 BERT (quantised GEMMs and attention) is not implemented")
    if precision == PREC_FP8:
        raise ValueError("BERT plans are fp16 only: FP8 BERT (quantised GEMMs and attention) is not implemented")
    if precision != PREC_FP16:
        raise ValueError("precision must be PREC_FP16")
    S, H, F = cfg.seq, cfg.hidden, cfg.ffn
    if S not in (64, 128, 256, 384, 512):
        raise ValueError(f"sequence length {S}: a plan is built for S a multiple of 64 up to 128, or a multiple of 128 up to 512")
    if cfg.heads * 64 != H:
        raise ValueError(f"heads * 64 must equal the hidden size ({cfg.heads} * 64 != {H})")
    if F % 64 or H > 1024 or S > cfg.positions:
        raise ValueError("the FFN width must be a multiple of 64, the hidden size at most 1024, and S at most the positions")
    W = Bm.load_weights(weights if weights is not None else Bm.random_weights(cfg, seed), cfg)

    tensors: List[dict] = []
    ops: List[dict] = []
    payload = bytearray()

    def add_payload(arr: np.ndarray):
        while len(payload) % 256:
            payload.append(0)
        off = len(payload)
        raw = np.ascontiguousarray(arr).tobytes()
        payload.extend(raw)
        return off, len(raw)

    def act(tname: str, c: int) -> int:
        tensors.append(dict(name=tname, kind=T_ACT, h=1, w=S, c=c, c_phys=c, binding=-1))
        return len(tensors) - 1

    def vec(tname: str, c: int, binding: int = -1) -> int:
        tensors.append(dict(name=tname, kind=T_VEC, h=1, w=1, c=c, c_phys=c, binding=binding))
        return len(tensors) - 1

    def gemm(oname: str, ti: int, to: int, Wm: np.ndarray, b: np.ndarray, res: int = -1, gelu: bool = False) -> dict:
        cout, cin = Wm.shape
        w_off, w_bytes = add_payload(pack_weights_sw128(Wm.astype(np.float16)))
        b_off, b_bytes = add_payload(b.astype(np.float32))
        return dict(name=oname, type=OP_CONV, inp=ti, res=res, out=to, binding=-1, k=1, stride=1, pad=0,
                    relu=CONV_PACKED | (CONV_GELU if gelu else 0), cin=cin, cout=cout, cin_phys=cin, cout_phys=cout, taps=1,
                    taps_phys=1, w_off=w_off, w_bytes=w_bytes, b_off=b_off, b_bytes=b_bytes, flags=pk)

    def gamma_beta(prefix: str):
        return add_payload(np.concatenate([W[prefix + ".weight"], W[prefix + ".bias"]]).astype(np.float32))

    # bindings 0..2: int32 inputs, 3: last_hidden_state, 4: pooled_output
    pk = FLAG_PACKED if remove_padding else 0
    x = act("embeddings", H)
    # padded: the additive attention mask [S]; packed: the packing index (pos_map and seq_off, S + 2 int32 words per item)
    mask = vec("packing_index", S + 2) if remove_padding else vec("attention_mask_add", S)
    tables = np.concatenate([W["embeddings.word_embeddings.weight"], W["embeddings.position_embeddings.weight"],
                             W["embeddings.token_type_embeddings.weight"]]).astype(np.float16)
    w_off, w_bytes = add_payload(tables)
    b_off, b_bytes = gamma_beta("embeddings.LayerNorm")
    ops.append(dict(name="embeddings", type=OP_EMBED_LN, inp=-1, res=-1, out=x, binding=0, binding2=1, binding3=2, out2=mask,
                    cin=H, cout=H, cin_phys=H, cout_phys=H, vocab=cfg.vocab, positions=cfg.positions, types=cfg.types,
                    eps=cfg.eps, w_off=w_off, w_bytes=w_bytes, b_off=b_off, b_bytes=b_bytes, flags=pk))
    for i in range(cfg.layers):
        p = f"encoder.layer.{i}."
        qkv, ctx, att, h1 = act(f"l{i}.qkv", 3 * H), act(f"l{i}.context", H), act(f"l{i}.attn_sum", H), act(f"l{i}.attn_ln", H)
        ffn, fsum, h2 = act(f"l{i}.ffn", F), act(f"l{i}.ffn_sum", H), act(f"l{i}.out", H)
        Wqkv = np.concatenate([W[p + f"attention.self.{m}.weight"] for m in ("query", "key", "value")])
        bqkv = np.concatenate([W[p + f"attention.self.{m}.bias"] for m in ("query", "key", "value")])
        ops.append(gemm(f"l{i}.qkv", x, qkv, Wqkv, bqkv))
        ops.append(dict(name=f"l{i}.attention", type=OP_ATTENTION, inp=qkv, res=mask, out=ctx, binding=-1, heads=cfg.heads, flags=pk))
        ops.append(gemm(f"l{i}.attn_out", ctx, att, W[p + "attention.output.dense.weight"], W[p + "attention.output.dense.bias"], res=x))
        b_off, b_bytes = gamma_beta(p + "attention.output.LayerNorm")
        ops.append(dict(name=f"l{i}.attn_ln", type=OP_LAYERNORM, inp=att, res=-1, out=h1, binding=-1, eps=cfg.eps, b_off=b_off, b_bytes=b_bytes,
                        flags=pk))
        ops.append(gemm(f"l{i}.ffn1", h1, ffn, W[p + "intermediate.dense.weight"], W[p + "intermediate.dense.bias"], gelu=True))
        ops.append(gemm(f"l{i}.ffn2", ffn, fsum, W[p + "output.dense.weight"], W[p + "output.dense.bias"], res=h1))
        b_off, b_bytes = gamma_beta(p + "output.LayerNorm")
        ops.append(dict(name=f"l{i}.out_ln", type=OP_LAYERNORM, inp=fsum, res=-1, out=h2, binding=-1, eps=cfg.eps, b_off=b_off, b_bytes=b_bytes,
                        flags=pk))
        x = h2
    pooled = vec("pooled_output", H, binding=4)
    w_off, w_bytes = add_payload(W["pooler.dense.weight"].astype(np.float16))
    b_off, b_bytes = add_payload(W["pooler.dense.bias"].astype(np.float32))
    ops.append(dict(name="pooler", type=OP_POOLER, inp=x, res=-1, out=pooled, binding=-1, cin=H, cout=H, cin_phys=H, cout_phys=H,
                    w_off=w_off, w_bytes=w_bytes, b_off=b_off, b_bytes=b_bytes, flags=pk))
    ops.append(dict(name="cast:last_hidden_state", type=OP_OUTPUT_CAST, inp=x, res=-1, out=-1, binding=3, flags=FLAG_ROWS_OUT | pk))
    bindings = [dict(name=n, is_input=1, dtype=3, tensor=0, dims=[S]) for n in ("input_ids", "segment_ids", "input_mask")]
    bindings.append(dict(name="last_hidden_state", is_input=0, dtype=0, tensor=x, dims=[S, H]))
    bindings.append(dict(name="pooled_output", is_input=0, dtype=0, tensor=pooled, dims=[H]))
    for tap in taps:
        ti = next((k for k, t in enumerate(tensors) if t["name"] == tap and t["kind"] == T_ACT), None)
        if ti is None:
            raise ValueError(f"tap {tap!r}: no such activation tensor")
        bindings.append(dict(name=tap, is_input=0, dtype=0, tensor=ti, dims=[S, tensors[ti]["c"]]))
        ops.append(dict(name="cast:" + tap, type=OP_OUTPUT_CAST, inp=ti, res=-1, out=-1, binding=len(bindings) - 1, flags=FLAG_ROWS_OUT | pk))
    default_name = f"bert_l{cfg.layers}_h{H}_s{S}" + ("_packed" if remove_padding else "")
    return _serialize(tensors, ops, bindings, payload, PREC_FP16, max_batch, name or default_name)


def build_vit_plan(cfg=None, weights=None, max_batch: int = 8, seed: int = 0, precision: int = PREC_FP16,
                   name: Optional[str] = None, taps: Sequence[str] = ()) -> bytes:
    """Vision Transformer classifier (``vit.VitConfig``; default ViT-B/16 at 224 x 224, 1000 classes) -> fp16 plan
    (version 3).

    ``weights``: a dict or ``.npz`` path in Hugging Face ``ViTForImageClassification`` names (``vit.load_weights``);
    default: seeded ``vit.random_weights(cfg, seed)``.  Bindings: fp32 ``data`` [3, image, width] (input, as ResNet's),
    fp32 ``prob`` [classes] and ``logits`` [classes] (outputs).  Ops: ``OP_PATCHIFY`` (the image as fp16 patch rows
    [P, 3 p^2], column c p^2 + dy p + dx), the patch projection as a 1x1 GEMM with the [H, 3 p^2] reshape of the
    convolution weight, ``OP_TOKENS`` (class token and position embeddings, and the packing index), then per pre-LN layer
    ln1 = LN(x), qkv = GEMM(ln1) (Q, K, V fused as in ``build_bert_plan``), ctx = attention(qkv), x1 = GEMM(ctx) + x,
    ln2 = LN(x1), f = GELU(GEMM(ln2)), x2 = GEMM(f) + x1; then ``OP_CLS_HEAD`` (final LayerNorm of the class token and the
    classifier) and the softmax.  Every item has L = P + 1 tokens, so the plan is a packed plan whose index says so:
    every encoder op runs on packed rows and attention on the variable-length kernels.

    ``taps``: activation tensors (``patches``, ``patch_embed``, ``tokens``, ``l{i}.ln1``, ``l{i}.qkv``, ``l{i}.context``,
    ``l{i}.attn_sum``, ``l{i}.ln2``, ``l{i}.ffn``, ``l{i}.out``, ``final_ln``) to expose as extra fp32 [rows, C] output
    bindings of the same names.  ``final_ln`` is the final LayerNorm of every token, computed by an extra LayerNorm op
    only when it is tapped; the head computes the class token's row with the same arithmetic.

    Geometry: image divisible by p, L <= 512, H = 64 heads <= 1024, FFN a multiple of 64, 3 p^2 a multiple of 64."""
    from . import vit as Vm
    cfg = cfg or Vm.VIT_B16
    for prec, what in ((PREC_FP32, "fp32"), (PREC_INT8, "INT8"), (PREC_FP8, "FP8")):
        if precision == prec:
            raise ValueError(f"ViT plans are fp16 only: {what} ViT is not implemented")
    if precision != PREC_FP16:
        raise ValueError("precision must be PREC_FP16")
    H, F, p, L, P = cfg.hidden, cfg.ffn, cfg.patch, cfg.tokens, cfg.patches
    if cfg.image % p or cfg.width % p:
        raise ValueError(f"the image size ({cfg.image} x {cfg.width}) must be divisible by the patch size ({p})")
    if (3 * p * p) % 64:
        raise ValueError(f"3 p^2 must be a multiple of 64 (p = {p}: 3 p^2 = {3 * p * p}), the K block of the patch GEMM")
    if L > 512:
        raise ValueError(f"{L} tokens: a plan takes at most 512 (patches + the class token)")
    if cfg.heads * 64 != H or H > 1024:
        raise ValueError(f"the hidden size must be heads * 64 and at most 1024 ({cfg.heads} * 64, H = {H})")
    if F % 64:
        raise ValueError(f"the FFN width must be a multiple of 64 (F = {F})")
    W = Vm.load_weights(weights if weights is not None else Vm.random_weights(cfg, seed), cfg)

    tensors: List[dict] = []
    ops: List[dict] = []
    payload = bytearray()

    def add_payload(arr: np.ndarray):
        while len(payload) % 256:
            payload.append(0)
        off = len(payload)
        raw = np.ascontiguousarray(arr).tobytes()
        payload.extend(raw)
        return off, len(raw)

    def act(tname: str, c: int, rows: int = L) -> int:
        tensors.append(dict(name=tname, kind=T_ACT, h=1, w=rows, c=c, c_phys=c, binding=-1))
        return len(tensors) - 1

    def vec(tname: str, c: int, binding: int = -1) -> int:
        tensors.append(dict(name=tname, kind=T_VEC, h=1, w=1, c=c, c_phys=c, binding=binding))
        return len(tensors) - 1

    def gemm(oname: str, ti: int, to: int, Wm: np.ndarray, b: np.ndarray, res: int = -1, gelu: bool = False, flags: int = FLAG_PACKED):
        cout, cin = Wm.shape
        w_off, w_bytes = add_payload(pack_weights_sw128(Wm.astype(np.float16)))
        b_off, b_bytes = add_payload(b.astype(np.float32))
        return dict(name=oname, type=OP_CONV, inp=ti, res=res, out=to, binding=-1, k=1, stride=1, pad=0,
                    relu=CONV_PACKED | (CONV_GELU if gelu else 0), cin=cin, cout=cout, cin_phys=cin, cout_phys=cout, taps=1,
                    taps_phys=1, w_off=w_off, w_bytes=w_bytes, b_off=b_off, b_bytes=b_bytes, flags=flags)

    def layernorm(oname: str, ti: int, to: int, prefix: str) -> dict:
        b_off, b_bytes = add_payload(np.concatenate([W[prefix + ".weight"], W[prefix + ".bias"]]).astype(np.float32))
        return dict(name=oname, type=OP_LAYERNORM, inp=ti, res=-1, out=to, binding=-1, eps=cfg.eps, b_off=b_off, b_bytes=b_bytes,
                    flags=FLAG_PACKED)

    # bindings: 0 data, 1 prob, 2 logits, then the taps
    patches, pe = act("patches", 3 * p * p, P), act("patch_embed", H, P)
    ops.append(dict(name="patchify", type=OP_PATCHIFY, inp=-1, res=-1, out=patches, binding=0, k=p))
    ops.append(gemm("patch_embed", patches, pe, W["embeddings.patch_embeddings.projection.weight"].reshape(H, 3 * p * p),
                    W["embeddings.patch_embeddings.projection.bias"], flags=0))
    x = act("tokens", H)
    index = vec("packing_index", L + 2)
    table = np.concatenate([W["embeddings.cls_token"].reshape(1, H), W["embeddings.position_embeddings"].reshape(L, H)])
    w_off, w_bytes = add_payload(table.astype(np.float16))
    ops.append(dict(name="tokens", type=OP_TOKENS, inp=pe, res=-1, out=x, out2=index, binding=-1, cin=H, cout=H, cin_phys=H,
                    cout_phys=H, w_off=w_off, w_bytes=w_bytes, flags=FLAG_PACKED))
    for i in range(cfg.layers):
        q = f"encoder.layer.{i}."
        ln1, qkv, ctx, x1 = act(f"l{i}.ln1", H), act(f"l{i}.qkv", 3 * H), act(f"l{i}.context", H), act(f"l{i}.attn_sum", H)
        ln2, f, x2 = act(f"l{i}.ln2", H), act(f"l{i}.ffn", F), act(f"l{i}.out", H)
        Wqkv = np.concatenate([W[q + f"attention.attention.{m}.weight"] for m in ("query", "key", "value")])
        bqkv = np.concatenate([W[q + f"attention.attention.{m}.bias"] for m in ("query", "key", "value")])
        ops.append(layernorm(f"l{i}.ln1", x, ln1, q + "layernorm_before"))
        ops.append(gemm(f"l{i}.qkv", ln1, qkv, Wqkv, bqkv))
        ops.append(dict(name=f"l{i}.attention", type=OP_ATTENTION, inp=qkv, res=index, out=ctx, binding=-1, heads=cfg.heads,
                        flags=FLAG_PACKED))
        ops.append(gemm(f"l{i}.attn_out", ctx, x1, W[q + "attention.output.dense.weight"], W[q + "attention.output.dense.bias"], res=x))
        ops.append(layernorm(f"l{i}.ln2", x1, ln2, q + "layernorm_after"))
        ops.append(gemm(f"l{i}.ffn1", ln2, f, W[q + "intermediate.dense.weight"], W[q + "intermediate.dense.bias"], gelu=True))
        ops.append(gemm(f"l{i}.ffn2", f, x2, W[q + "output.dense.weight"], W[q + "output.dense.bias"], res=x1))
        x = x2
    if "final_ln" in taps:
        ops.append(layernorm("final_ln", x, act("final_ln", H), "layernorm"))
    prob, logits = vec("prob", cfg.classes, binding=1), vec("logits", cfg.classes, binding=2)
    w_off, w_bytes = add_payload(W["classifier.weight"].astype(np.float16))
    b_off, b_bytes = add_payload(np.concatenate([W["layernorm.weight"], W["layernorm.bias"], W["classifier.bias"]]).astype(np.float32))
    ops.append(dict(name="cls_head", type=OP_CLS_HEAD, inp=x, res=-1, out=logits, binding=-1, cin=H, cout=cfg.classes, cin_phys=H,
                    cout_phys=cfg.classes, eps=cfg.eps, w_off=w_off, w_bytes=w_bytes, b_off=b_off, b_bytes=b_bytes, flags=FLAG_PACKED))
    ops.append(dict(name="softmax", type=OP_SOFTMAX, inp=logits, res=-1, out=prob, binding=-1))
    bindings = [dict(name="data", is_input=1, dtype=0, tensor=patches, dims=[3, cfg.image, cfg.width]),
                dict(name="prob", is_input=0, dtype=0, tensor=prob, dims=[cfg.classes]),
                dict(name="logits", is_input=0, dtype=0, tensor=logits, dims=[cfg.classes])]
    for tap in taps:
        ti = next((k for k, t in enumerate(tensors) if t["name"] == tap and t["kind"] == T_ACT), None)
        if ti is None:
            raise ValueError(f"tap {tap!r}: no such activation tensor")
        bindings.append(dict(name=tap, is_input=0, dtype=0, tensor=ti, dims=[tensors[ti]["w"], tensors[ti]["c"]]))
        front = ti in (patches, pe)  # made before the tokens op: plain rows, not packed ones
        ops.append(dict(name="cast:" + tap, type=OP_OUTPUT_CAST, inp=ti, res=-1, out=-1, binding=len(bindings) - 1,
                        flags=FLAG_ROWS_OUT | (0 if front else FLAG_PACKED)))
    default_name = f"vit_l{cfg.layers}_h{H}_p{p}_i{cfg.image}" + (f"x{cfg.width}" if cfg.width != cfg.image else "")
    return _serialize(tensors, ops, bindings, payload, PREC_FP16, max_batch, name or default_name)


def build_resnext_plan(depth: int = 50, precision: int = PREC_FP16, max_batch: int = 8, seed: int = 0,
                       input_dtype: str = "f32", groups: int = 32, width_per_group: int = 4, calib_batch: int = 8) -> bytes:
    """Convenience: generated ResNeXt (:func:`graph.resnext_caffe`) + deterministic weights -> plan.  PREC_INT8 / PREC_FP8:
    post-training quantization with the grouped convolutions included, calibrated like :func:`build_resnet_plan`."""
    from . import weights as Wt
    net = G.resnext_caffe(depth, groups, width_per_group)
    low = G.lower(net, Wt.random_weights(net, seed))
    if precision in (PREC_INT8, PREC_FP8):
        from . import quantize
        low = quantize.quantize_lowered(low, Wt.synthetic_input(calib_batch, seed=4321),
                                        fmt="e4m3" if precision == PREC_FP8 else "int8", grouped=True)
    return build_plan(low, precision, max_batch, input_dtype=input_dtype)


def build_googlenet_plan(precision: int = PREC_FP16, max_batch: int = 8, seed: int = 0, input_dtype: str = "f32",
                         weights: Optional[dict] = None) -> bytes:
    """Convenience: generated BVLC GoogLeNet (:func:`graph.googlenet_caffe`) + deterministic (or given, BVLC-named) weights
    -> fp16 plan.  Each inception module's four branch convolutions write their channel slices of the module's output
    directly; the two LRN layers run lrn_h8_kernel.  fp16 only."""
    if precision != PREC_FP16:
        raise ValueError("GoogLeNet builds in fp16 only: channel concatenation and LRN have no fp32, INT8 or FP8 kernels")
    from . import weights as Wt
    net = G.googlenet_caffe()
    low = G.lower(net, weights if weights is not None else Wt.random_weights(net, seed))
    return build_plan(low, precision, max_batch, input_dtype=input_dtype)


def build_densenet_plan(depth: int = 121, max_batch: int = 8, seed: int = 0, weights: Optional[dict] = None,
                        precision: int = PREC_FP16, input_dtype: str = "f32") -> bytes:
    """Convenience: generated DenseNet-{121,169,201} (:func:`graph.densenet_caffe`) + deterministic (or given, Caffe-named:
    ``weights.random_weights``, ``caffemodel``, ``densenet.load_weights``) weights -> fp16 plan.  Each dense block is one
    tensor: the stem's max pool or the transition convolution writes its first channels and every 3x3 its 32, and every
    1x1 reads the channel prefix written so far through a BatchNorm + ReLU input prologue.  fp16 only."""
    if precision != PREC_FP16:
        raise ValueError("DenseNet builds in fp16 only: the BatchNorm + ReLU prologue and channel concatenation have no fp32, "
                         "INT8 or FP8 kernels")
    from . import weights as Wt
    net = G.densenet_caffe(depth)
    low = G.lower(net, weights if weights is not None else Wt.random_weights(net, seed))
    return build_plan(low, precision, max_batch, input_dtype=input_dtype)


def build_vgg_plan(depth: int = 16, max_batch: int = 8, seed: int = 0, weights: Optional[dict] = None,
                   input_dtype: str = "f32") -> bytes:
    """Convenience: generated VGG-{16,19} (:func:`graph.vgg_caffe`) + deterministic (or given, Caffe-named:
    ``weights.random_weights``, ``caffemodel``, ``vgg.load_weights``) weights -> fp16 plan (version 4).  fc6 and fc7 fuse
    their ReLUs and write fp16 activations; fc6, fc7 and fc8 run on the streaming tensor-core FC kernel."""
    from . import weights as Wt
    net = G.vgg_caffe(depth)
    low = G.lower(net, weights if weights is not None else Wt.random_weights(net, seed))
    return build_plan(low, PREC_FP16, max_batch, input_dtype=input_dtype)


def build_resnet_plan(depth: int = 50, precision: int = PREC_FP16, max_batch: int = 8, seed: int = 0,
                      input_dtype: str = "f32", calib_batch: int = 8) -> bytes:
    """Convenience: generated Caffe-v1 ResNet + deterministic weights -> plan.  PREC_INT8 / PREC_FP8: post-training
    quantization calibrated (max-abs) on ``calib_batch`` synthetic images (seed 4321), see quantize.py."""
    from . import weights as Wt
    net = G.resnet_caffe(depth)
    low = G.lower(net, Wt.random_weights(net, seed))
    if precision in (PREC_INT8, PREC_FP8):
        from . import quantize
        low = quantize.quantize_lowered(low, Wt.synthetic_input(calib_batch, seed=4321),
                                        fmt="e4m3" if precision == PREC_FP8 else "int8")
    return build_plan(low, precision, max_batch, input_dtype=input_dtype)


def single_conv_net(cin: int, h: int, w: int, cout: int, k: int, stride: int, pad: int, relu: bool = True,
                    residual: bool = False, bias: bool = True, group: int = 1) -> dict:
    """Raw layer list of a one-convolution network (kernel-level parity tests go through the public ABI).
    With ``residual`` the net is  y = relu(conv_b(x) + conv_a(x))  so the fused add path is exercised; ``group`` applies
    to conv_b (the fused one) only."""
    L = []
    if residual:
        L.append(dict(name="short", type="Convolution", bottoms=["data"], tops=["short"], num_output=cout,
                      kernel_size=k, pad=pad, stride=stride, bias_term=bias))
    L.append(dict(name="conv", type="Convolution", bottoms=["data"], tops=["conv"], num_output=cout,
                  kernel_size=k, pad=pad, stride=stride, bias_term=bias))
    if group != 1:
        L[-1]["group"] = group
    top = "conv"
    if residual:
        L.append(dict(name="sum", type="Eltwise", bottoms=["short", "conv"], tops=["sum"], operation="SUM"))
        top = "sum"
    if relu:
        L.append(dict(name="relu", type="ReLU", bottoms=[top], tops=[top]))
    gtag = f"g{group}" if group != 1 else ""
    return {"name": f"conv{k}x{k}s{stride}{gtag}_{cin}x{h}x{w}_{cout}", "input": "data", "input_dims": [1, cin, h, w],
            "layers": L}


def attach_tactics(blob: bytes, tactics: np.ndarray) -> bytes:
    """Append a tactic table (``capi.Engine.tactics()`` after ``Engine.tune()``: [n, 10] uint32 records
    {op, batch, bn, stages, splits, sps, ws, cn, halo, 0}) to a plan blob -- the role of the tactics a TensorRT plan file
    carries (reference models/setup.py:53-55: trtexec tunes offline).  An engine deserialized from the result never tunes."""
    tactics = np.ascontiguousarray(tactics, dtype=np.uint32).reshape(-1, 10)
    hdr = list(_HEADER.unpack_from(blob, 0))
    base = blob
    old_n, _, old_off = struct.unpack_from("<IIQ", blob, _HEADER.size - 16)
    if old_n:  # replace an existing table
        base = blob[:old_off]
    off = (len(base) + 63) // 64 * 64
    out = bytearray(base) + bytes(off - len(base)) + tactics.tobytes()
    struct.pack_into("<IIQ", out, _HEADER.size - 16, tactics.shape[0], 0, off)
    del hdr
    return bytes(out)
