"""Order-exact reference of b200collAllReduceRmsNormQuantized (coll/include/b200coll.h): steps 1-5 are
coll_rmsnorm_reference.rms_norm's, and step 6 quantises every row of its out, cut into blocks of `block` elements, with
coll_quant_reference.quantize, the one quantiser of the tests.

Not collected by pytest (no test_ prefix)."""
import torch

from tests import coll_quant_reference as Q
from tests import coll_rmsnorm_reference as R


def rms_norm_quantized(xs, residual, gamma, eps, dt, block, wire):
    """xs: the N ranks' [rows, row_len] tensors; residual [rows, row_len]; gamma [row_len]; all of dt (CPU). Returns (new residual of dt,
    q [rows, row_len] of wire, scales [rows, row_len // block] fp32)."""
    h, out = R.rms_norm(xs, residual, gamma, eps, dt)
    rows, row_len = out.shape
    q = torch.empty(rows, row_len, dtype=wire)
    s = torch.empty(rows, row_len // block, dtype=torch.float32)
    for i in range(rows):
        q[i], s[i], _ = Q.quantize(out[i], block, wire)
    return h, q, s
