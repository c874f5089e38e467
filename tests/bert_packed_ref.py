"""CPU reference of the packed (padding-free) BERT contract, ``builder.build_bert_plan(..., remove_padding=True)``, built on
the oracle's public forwards:

* item n is the sequence of its tokens with ``input_mask != 0``, kept in order, each at its ORIGINAL position -- run on
  its own as a sequence of that length (the position table is re-indexed so that compact column j reads the row of the
  token's original position);
* ``last_hidden_state`` rows of masked positions are exactly 0;
* ``pooled_output`` pools position 0, a zero row when position 0 is masked: tanh(bias).  An item with no valid token gives
  zeros and tanh(bias).
"""
from __future__ import annotations

import numpy as np

from oracle import bert_forward as O


def packed_forward(W, cfg, ids, segs, mask, fp16: bool = True):
    """-> (last_hidden_state [N, S, H], pooled_output [N, H]) under the packed contract (fp16 emulation or fp32)."""
    fwd = O.forward_fp16 if fp16 else O.forward_fp32
    ids, segs, mask = (np.asarray(a) for a in (ids, segs, mask))
    N, S = ids.shape
    hidden = np.zeros((N, S, cfg.hidden), np.float32)
    pooled = np.zeros((N, cfg.hidden), np.float32)
    bias = np.asarray(W["pooler.dense.bias"], np.float32)
    for n in range(N):
        sel = np.nonzero(mask[n] != 0)[0]
        pooled[n] = np.tanh(bias)
        if not len(sel):
            continue
        Wn = dict(W)
        pos = np.array(W["embeddings.position_embeddings.weight"], copy=True)
        pos[:len(sel)] = W["embeddings.position_embeddings.weight"][sel]
        Wn["embeddings.position_embeddings.weight"] = pos
        h, p = fwd(Wn, cfg, ids[n:n + 1, sel], segs[n:n + 1, sel], np.ones((1, len(sel)), np.int32))
        hidden[n, sel] = h[0]
        if sel[0] == 0:
            pooled[n] = p[0]
    return hidden, pooled


def right_padded(S: int, lengths) -> np.ndarray:
    """input_mask [len(lengths), S]: item n is lengths[n] ones followed by zeros"""
    mask = np.zeros((len(lengths), S), np.int32)
    for n, L in enumerate(lengths):
        mask[n, :L] = 1
    return mask
