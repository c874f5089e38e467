"""Per-layer rooflines of a lowered graph's convolutions (pure arithmetic on shapes; no GPU).

For each convolution at a given batch: the tensor-core floor (2*M*N*K over the sustained fp16/bf16 peak) and the memory
floor for L2-resident activations -- algorithmic bytes (activations in + weights + residual read, output written, fp16)
over the bandwidth the memory system gives UNIQUE streaming data, which differs for reads and writes (measure it with
tools/micro/l2_stream.cu on the GPU in question).  A layer's floor is the larger of the two; the sum over layers is what a
forward pass costs if every kernel sat on its own roof.  Used by tools/roofline_saturated.py."""
from __future__ import annotations

from typing import Dict, List

def conv_floors(lowered: dict, batch: int, peak_tflops: float, l2_read_bps: float, l2_write_bps: float,
                elt_bytes: int = 2) -> List[Dict]:
    T = lowered["tensors"]
    out = []
    for op in lowered["ops"]:
        if op["type"] != "conv":
            continue
        cin, hi, wi = T[op["input"]]
        cout, ho, wo = T[op["output"]]
        flops = 2.0 * batch * ho * wo * cout * cin * op["k"] ** 2
        rd = batch * hi * wi * max(cin, 8) * elt_bytes + cout * cin * op["k"] ** 2 * elt_bytes
        if op.get("residual"):
            rd += batch * ho * wo * cout * elt_bytes
        wr = batch * ho * wo * cout * elt_bytes
        t_tensor = flops / (peak_tflops * 1e12) * 1e6
        t_mem = (rd / l2_read_bps + wr / l2_write_bps) * 1e6
        out.append(dict(name=op["name"], flops=flops, read_bytes=rd, write_bytes=wr, tensor_floor_us=t_tensor, memory_floor_us=t_mem,
                        floor_us=max(t_tensor, t_mem), roof="tensor" if t_tensor >= t_mem else "memory"))
    return out
