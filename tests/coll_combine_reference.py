"""Order-exact reference of the expert combine (b200collAllToAllvCombine): per token, the slots' weighted expert rows summed in fp32 in
slot order, each product and each sum rounded on its own, then one multiply by the scale and one rounding to the output type."""
import numpy as np
import torch

from tests.coll_fp_reference import cast


def combine(lookup, index, weights, scale, out_dt):
    """index: [tokens, top_k] int numpy; weights: [tokens, top_k] float32 numpy or None (all ones); lookup(column) -> (valid [tokens]
    bool, rows [tokens, row_elems] float32) gives the expert row each index of one slot column names, valid False for a dropped slot.
    Returns round_once(scale * ((+0 + w0*y0) + w1*y1 + ...)) as a [tokens, row_elems] tensor of out_dt."""
    tokens, top_k = index.shape
    acc = None
    with np.errstate(invalid="ignore", over="ignore"):
        for j in range(top_k):
            valid, y = lookup(index[:, j])
            if acc is None:
                acc = np.zeros(y.shape, dtype=np.float32)
            w = np.float32(1.0) if weights is None else weights[:, j:j + 1].astype(np.float32)
            prod = (w * y.astype(np.float32)).astype(np.float32)
            acc = np.where(valid[:, None], (acc + prod).astype(np.float32), acc)
        out = (acc * np.float32(scale)).astype(np.float32)
    return cast(torch.from_numpy(out), out_dt)


def plan_lookup(expert_out, rows, send_row_off, recv_row_off_at_peer):
    """The lookup of one rank: dispatch row i in [send_row_off[p], + rows[p]) is row recv_row_off_at_peer[p] + i - send_row_off[p] of
    expert_out[p] (a [recv_rows, row_elems] float32 numpy array per rank); every other index is a dropped slot."""
    def f(col):
        col = np.asarray(col, dtype=np.int64)
        valid = np.zeros(col.shape, dtype=bool)
        y = np.zeros((col.size, expert_out[0].shape[1]), dtype=np.float32)
        for p, (r, so, ro) in enumerate(zip(rows, send_row_off, recv_row_off_at_peer)):
            m = (col >= so) & (col < so + r)
            valid |= m
            y[m] = expert_out[p][ro + col[m] - so]
        return valid, y
    return f
