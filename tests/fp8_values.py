"""Crafted FP8 (E4M3) convolutions whose device results are checkable bit for bit -- test infrastructure (like
bert_values.py), shared by tests/test_fp8_values_cpu.py (which proves each set discriminates) and
tests/test_gpu_fp8_values.py (which runs them).

The tensor core's FP8 accumulation cannot be reproduced on the CPU, so random data only bounds a convolution's codes by
an interval (tests/test_gpu_fp8.py).  These cases make the accumulator exact instead: every output channel has a ONE-HOT
weight row (the code of 1.0 at one (tap, input channel), zeros elsewhere), so its accumulator is one exact product plus
exact zeros -- the same in any accumulator width and order.  The GPU's codes must then equal ``requant(A)`` exactly.
With the quantize scale s = 1 and fp16 inputs that are E4M3 values, the input codes are the inputs themselves.

Each output channel is a PROBE (input class, m, b): it reads an input channel of one class, whose pixels are
+-magnitude (random signs, some zeros), and its epilogue is t = fma(A, m, b).  The probes put t on E4M3 ties in the
normal and subnormal binades and one fp32 ulp either side, where fma and a multiply-then-add round differently, on
448 <= t < 464 and t >= 464, and (at the padded border taps, A = 0) on t = b.  Output channel c reads its probe's class
at input channel class + NCLASS * j with j stepping through every 128-channel K block (the partial last one too), at
tap c mod k*k, so a lost K block or a wrong im2col tap changes an exact value.

Two traps for a crafted graph:
  * the engine does not read ``op["inv_scale"]``: it derives the quantize multiplier from the stored tensor scale,
    ``float(1.0 / double(scale))`` (engine.cu, L_QUANTIZE_F8).  ``set_scale`` changes both together, or the oracle and
    the engine would disagree for reasons that have nothing to do with the kernel;
  * ``fmaxf(-0, +0)`` may return either zero: compare values, not codes, wherever a zero can come out of the ReLU.
"""
from __future__ import annotations

import numpy as np

from oracle import fp8_forward as O8
from oracle.int8_forward import fma32
from tensorrt_laboratory_b200 import builder, graph, quantize, weights

f32 = np.float32
ONE = 0x38                      # E4M3 code of 1.0
R_RES = f32(0.70710677)         # the residual multiplier r of the residual cases: q_res * r is inexact for most codes

# input classes: the magnitude of an input channel's pixels (all E4M3 values, so fp16 values too)
MAGS = np.array([1.0, 0.125, 4.0, 1.875, 1.625, 3 * 2.0 ** -9, 7 * 2.0 ** -9, 2.0 ** -6], f32)
NCLASS = len(MAGS)
SUBNORMAL_CLASSES = (5, 6)


def _tie_probes():
    """(class, m, b, kind): t = +-m exactly on a tie, and one fp32 ulp either side."""
    p = []
    for g in (-2, 0, 3):                                      # normal binades: (1 + o/16) * 2^g is a midpoint for odd o
        for o in range(1, 16, 2):
            p.append((0, f32((16 + o) / 16 * 2.0 ** g), f32(0), "tie"))
    for o in (1, 11, 13):                                     # the top binade: 272, 432 (-> 448), 464 (the saturation tie)
        p.append((0, f32((16 + o) / 16 * 256), f32(0), "tie" if o != 13 else "sat"))
    for o in range(1, 16, 2):
        m = f32((16 + o) / 16)
        p += [(0, np.nextafter(m, f32(np.inf)), f32(0), "near"), (0, np.nextafter(m, f32(0)), f32(0), "near")]
    for k in range(8):                                        # subnormal binade: (2k + 1) * 2^-10 between k and k + 1 units
        p.append((0, f32((2 * k + 1) * 2.0 ** -10), f32(0), "tie"))
    for k in (0, 3, 7):
        m = f32((2 * k + 1) * 2.0 ** -10)
        p += [(0, np.nextafter(m, f32(np.inf)), f32(0), "near"), (0, np.nextafter(m, f32(0)), f32(0), "near")]
    return p


def _fma_probes(n, cls, seed):
    """(class, m, b, "fma"): t = fma(+-mag, m, b) lands next to a tie, on the other side from fl(fl(mag * m) + b) for at
    least one sign -- found by a seeded search."""
    rng = np.random.default_rng(seed)
    v = np.array([MAGS[cls], -MAGS[cls]], f32)
    out = []
    while len(out) < n:
        m = f32(rng.uniform(0.5, 4.0))
        tie = f32(rng.choice(TIES[(TIES > 0.5) & (TIES < 12)]))
        b = f32(np.float64(tie) - np.float64(v[0]) * np.float64(m))
        fused = O8.e4m3(fma32(v, np.full(2, m), np.full(2, b)))
        split = O8.e4m3((v * m).astype(f32) + b)
        if (fused != split).any():
            out.append((cls, m, b, "fma"))
    return out


def _e4m3_ties():
    vals = O8.E4M3_VALUES[np.isfinite(O8.E4M3_VALUES)]
    pos = np.unique(vals[vals >= 0]).astype(np.float64)
    return ((pos[:-1] + pos[1:]) / 2).astype(f32)           # exact in fp32


TIES = _e4m3_ties()


def _probes():
    p = _tie_probes()
    p += _fma_probes(6, 3, 1) + _fma_probes(4, 4, 2)
    for t in (448.0, 455.99, 456.0, 463.99997, 464.0, 470.0, 480.0, 1e4, 3e38):   # saturation, both signs (ReLU off)
        p.append((0, f32(t), f32(0), "sat"))
    for b in (1.0625, -1.1875, 3 * 2.0 ** -10, -5 * 2.0 ** -10, 464.0, -1000.0):  # bias-heavy: t = b at the border
        p.append((1, f32(1), f32(b), "bias"))
    for cls in SUBNORMAL_CLASSES:                            # subnormal operands: kept, the product exact
        p += [(cls, f32(256), f32(0), "subnormal"), (cls, f32(1), f32(0), "subnormal")]
    p += [(2, f32(1), f32(0), "plain"), (7, f32(1), f32(0), "plain")]
    return p


PROBES = _probes()


def _res_probes(n, seed):
    """(main class, m, b, shortcut class): t = fma(value(q_res), r, fma(+-mag, m, b)) next to an E4M3 tie, on the other
    side from a separate multiply and add of the residual for at least one pair of signs."""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        cls, scls = int(rng.choice([0, 3, 4])), int(rng.choice([3, 4]))
        v = np.array([MAGS[cls], -MAGS[cls], MAGS[cls], -MAGS[cls]], f32)
        q = np.array([MAGS[scls], MAGS[scls], -MAGS[scls], -MAGS[scls]], f32)
        m = f32(rng.uniform(0.25, 2.0))
        tie = f32(rng.choice(TIES[(TIES > 0.25) & (TIES < 8)]))
        b = f32(np.float64(tie) - np.float64(v[0]) * np.float64(m) - np.float64(q[0]) * np.float64(R_RES))
        t1 = fma32(v, np.full(4, m), np.full(4, b))
        fused = O8.e4m3(fma32(q, np.full(4, R_RES), t1))
        split = O8.e4m3(((q * R_RES).astype(f32) + t1).astype(f32))
        if (fused != split).any():
            out.append((cls, m, b, scls))
    return out


RES_PROBES = _res_probes(24, 3)


def set_scale(lq: dict, name: str, s: float) -> None:
    """Store tensor scale s for ``name`` (and, for a quantize output, the multiplier the engine derives from it)."""
    s = float(f32(s))
    lq["tensor_scales"][name] = s
    for op in lq["ops"]:
        if op["type"] == "quantize" and op["output"] == name:
            op["scale"] = s
            op["inv_scale"] = f32(1.0 / s)                  # engine.cu: float(1.0 / double(scale))


def base_plan(cin, h, w, cout, k, stride, pad, relu=False, residual=False, seed=0):
    """quantize_lowered(..., fmt="e4m3") of builder.single_conv_net, calibrated on random data, every scale then 1."""
    net = builder.single_conv_net(cin, h, w, cout, k, stride, pad, relu=relu, residual=residual)
    low = graph.lower(net, weights.random_weights(net, seed))
    x = np.random.default_rng(seed).standard_normal((1, cin, h, w)).astype(np.float16).astype(f32)
    lq = quantize.quantize_lowered(low, x, fmt="e4m3")
    for name in list(lq["tensor_scales"]):
        set_scale(lq, name, 1.0)
    for op in lq["ops"]:
        if op.get("fp8") and op["residual"] is not None:
            op["r"] = f32(1.0)
    return lq


def one_hot(cout, k, cin, picks):
    """picks [(tap, ci)] per output channel -> Wq [cout, k, k, cin] with code 1.0 there, 0 elsewhere."""
    Wq = np.zeros((cout, k, k, cin), np.uint8)
    for c, (tap, ci) in enumerate(picks):
        Wq[c, tap // k, tap % k, ci] = ONE
    return Wq


def _channel(cls, j, cin):
    """Input channel of class ``cls``, the j-th of them counted through every 128-channel block in turn."""
    per = cin // NCLASS
    nblk = (cin + 127) // 128
    blk = j % nblk
    lo, hi = blk * 128 // NCLASS, min((blk + 1) * 128, cin) // NCLASS
    idx = lo + (j // nblk) % max(hi - lo, 1)
    return cls + NCLASS * min(idx, per - 1)


def crafted_input(batch, cin, h, w, seed, zero_share=0.1):
    """fp32 [batch, cin, h, w]: channel ci holds +-MAGS[ci % NCLASS] with random signs and about ``zero_share`` zeros."""
    rng = np.random.default_rng(seed)
    mag = MAGS[np.arange(cin) % NCLASS].reshape(1, cin, 1, 1)
    sign = rng.choice(np.array([-1.0, 1.0], f32), size=(batch, cin, h, w))
    x = (sign * mag * (rng.random((batch, cin, h, w)) >= zero_share)).astype(f32)
    assert np.array_equal(x.astype(np.float16).astype(f32), x)
    return x


def crafted(geom, relu=False, residual=False, batch=3, seed=0):
    """-> (lq, x): a single-convolution FP8 plan at geom = (cin, h, w, cout, k, stride, pad) with one-hot weights and the
    probes' epilogues, and its input.  With ``residual``, the shortcut convolution is one-hot too (m = 1, b = 0: its codes
    are +-magnitudes and zeros), and the fused convolution runs RES_PROBES with r = R_RES."""
    cin, h, w, cout, k, stride, pad = geom
    lq = base_plan(cin, h, w, cout, k, stride, pad, relu=relu, residual=residual, seed=seed)
    taps = k * k
    convs = [op for op in lq["ops"] if op.get("fp8")]
    main = convs[-1]
    probes = RES_PROBES if residual else PROBES
    picks, m, b = [], np.zeros(cout, f32), np.zeros(cout, f32)
    short_picks = []
    for c in range(cout):
        pr = probes[c % len(probes)]
        j = c // len(probes) + c
        picks.append((c % taps, _channel(pr[0], j, cin)))
        m[c], b[c] = pr[1], pr[2]
        if residual:
            short_picks.append(((c + 1) % taps, _channel(pr[3], j + 1, cin)))
    main["Wq"] = one_hot(cout, k, cin, picks)
    main["m"], main["b"] = m, b
    main["picks"] = picks
    if residual:
        short = convs[0]
        short["Wq"] = one_hot(cout, k, cin, short_picks)
        short["m"], short["b"] = np.ones(cout, f32), np.zeros(cout, f32)
        short["picks"] = short_picks
        main["r"] = R_RES
    return lq, crafted_input(batch, cin, h, w, seed + 1)


def expected(lq, x, keep=None):
    """The FP8 oracle's codes of every FP8 tensor (exact: the accumulators are)."""
    _, snap = O8.fp8_forward(lq, x, keep=keep or list(lq["tensor_scales"]))
    return snap


def epilogue_inputs(lq, x):
    """-> {conv output: (A, res codes or None, op)} from the oracle: the exact accumulators and residual codes."""
    snap = expected(lq, x)
    out = {}
    for op in lq["ops"]:
        if op.get("fp8"):
            A, _ = O8.conv_fp8(snap[op["input"]], op, with_p=False)
            out[op["output"]] = (A, snap[op["residual"]] if op["residual"] is not None else None, op)
    return out


def t_values(A, op, res):
    """The pre-conversion epilogue value t per output (fp32), as the contract computes it (before ReLU)."""
    mm = np.broadcast_to(op["m"].reshape(1, -1, 1, 1), A.shape)
    bb = np.broadcast_to(op["b"].reshape(1, -1, 1, 1), A.shape)
    t = fma32(A.astype(f32), mm, bb)
    if res is not None:
        t = fma32(O8.value(res), np.broadcast_to(f32(op["r"]), A.shape), t)
    return t


# ------------------------------------------------------------------------------------------------------------------
# pool and quantize inputs
# ------------------------------------------------------------------------------------------------------------------
def quantize_values():
    """fp16 values for the quantize kernel: every E4M3 tie (all are fp16 values) and one fp16 ulp either side, the whole
    fp16 range below 2^-5 (the E4M3 subnormals and the lowest normal binades), +-0, values past 448 up to 65504 -- both
    signs."""
    ties = TIES.astype(np.float16)
    assert np.array_equal(ties.astype(f32), TIES)
    near = np.concatenate([np.nextafter(ties, np.float16(0)), np.nextafter(ties, np.float16(np.inf))])
    small = np.arange(0, int(np.float16(2.0 ** -5).view(np.uint16)) + 1, dtype=np.uint16).view(np.float16)
    big = np.array([448, 449, 456, 460, 463, 464, 465, 480, 500, 1000, 4096, 30000, 65504], np.float16)
    v = np.concatenate([ties, near, small, big, O8.E4M3_VALUES[np.isfinite(O8.E4M3_VALUES)].astype(np.float16)])
    v = np.concatenate([v, -v])
    return v.astype(f32)


def quantize_input(vals, s, shape, seed):
    """vals scaled by s (then rounded to fp16: near-ties of the product h * fl(1/s) when 1/s is not a power of two), and
    for s != 1 the three fp16 neighbours either side of each scaled tie, spread over ``shape``, every value at least
    once."""
    v = (vals.astype(np.float64) * s).astype(np.float16)
    if s != 1:
        around = [(TIES.astype(np.float64) * s).astype(np.float16)]
        for d in (np.float16(0), np.float16(np.inf)):
            h = around[0]
            for _ in range(3):
                h = np.nextafter(h, d)
                around.append(h)
        around = np.concatenate(around)
        v = np.concatenate([v, around, -around])
    v = v.astype(f32)
    n = int(np.prod(shape))
    assert len(v) <= n, (len(v), n)
    x = v[np.random.default_rng(seed).integers(0, len(v), n)]
    x[:len(v)] = v
    return x.reshape(shape)


def _pool_orders(v):
    """[..., HW] values -> the fp32 sums in pixel order, in reverse order, and pairwise (a tree), each [...]."""
    fwd = np.zeros(v.shape[:-1], f32)
    rev = np.zeros(v.shape[:-1], f32)
    for i in range(v.shape[-1]):
        fwd = (fwd + v[..., i]).astype(f32)
        rev = (rev + v[..., v.shape[-1] - 1 - i]).astype(f32)
    pair = v.astype(f32)
    while pair.shape[-1] > 1:
        if pair.shape[-1] % 2:
            pair = np.concatenate([pair, np.zeros(pair.shape[:-1] + (1,), f32)], axis=-1)
        pair = (pair[..., 0::2] + pair[..., 1::2]).astype(f32)
    return fwd, rev, pair[..., 0]


def pool_finish(sums, k):
    """h = fp16(fl(sum * k)) as float64."""
    return (np.asarray(sums, f32) * f32(k)).astype(f32).astype(np.float16).astype(np.float64)


def pool_input_values(batch, c, hw, seed, crafted_channels=8):
    """E4M3 codes [batch, c, hw, hw] for the average pool: random values, and for HW >= 74 the first
    ``crafted_channels`` channels of image 0 made order-sensitive: 74 values of 448 take the running fp32 sum past 2^15
    (ulp 2^-8), where a following multiple of 2^-9 rounds, and the last two values are searched so that the mean lands
    next to an fp16 tie -- the pixel-order sum then gives other fp16 bits than the reversed or the pairwise sum."""
    rng = np.random.default_rng(seed)
    vals = O8.E4M3_VALUES[np.isfinite(O8.E4M3_VALUES)]
    q = O8.e4m3(rng.choice(vals[np.abs(vals) <= 64], (batch, c, hw * hw)).astype(f32))
    n = hw * hw
    if n >= 74:
        k = f32(1.0 / n)
        small = vals[(vals > 0) & (vals <= 8)]
        cand_a = np.arange(1, 8, dtype=f32) * f32(2.0 ** -9)
        cand_b = vals[(vals >= 0) & (vals <= 64)]
        A, B = [x.ravel() for x in np.meshgrid(cand_a, cand_b)]
        found = 0
        while found < crafted_channels:
            tail = rng.choice(small, n - 76).astype(f32)
            seq = np.concatenate([np.full(74, 448.0, f32), tail])
            v = np.concatenate([np.broadcast_to(seq, (len(A), n - 2)), A[:, None], B[:, None]], axis=1)
            fwd, rev, pair = (pool_finish(s, k) for s in _pool_orders(v))
            ok = np.flatnonzero((fwd != rev) & (fwd != pair))
            if len(ok):
                q[0, found] = O8.e4m3(v[ok[0]])
                found += 1
    return q.reshape(batch, c, hw, hw)


def pool_plan(c, hw, cout, seed=0):
    """conv 1x1 (c -> cout, no ReLU, one-hot: cout channel i reads input channel i mod c, m = 1, b = 0) -> global AVE, every
    scale 1 except the pool's k = fl(1 / HW); with pool_input_values as the input, the conv passes the codes through."""
    net = builder.single_conv_net(c, hw, hw, cout, 1, 1, 0, relu=False)
    net["layers"].append(dict(name="pool", type="Pooling", bottoms=["conv"], tops=["pool"], pool="AVE", kernel_size=hw, stride=1,
                              pad=0))
    low = graph.lower(net, weights.random_weights(net, seed))
    x = np.random.default_rng(seed).standard_normal((1, c, hw, hw)).astype(np.float16).astype(f32)
    lq = quantize.quantize_lowered(low, x, fmt="e4m3")
    for name in list(lq["tensor_scales"]):
        set_scale(lq, name, 1.0)
    conv = next(op for op in lq["ops"] if op.get("fp8"))
    conv["Wq"] = one_hot(cout, 1, c, [(0, i % c) for i in range(cout)])
    conv["m"], conv["b"] = np.ones(cout, f32), np.zeros(cout, f32)
    pool = next(op for op in lq["ops"] if op["type"] == "avgpool")
    pool["in_scale"] = 1.0
    pool["k_scale"] = f32(1.0 / (hw * hw))
    return lq
