"""CPU checks that the bounds of tests/test_gpu_stem_bf16x3.py separate the split-bf16 stem from its likely faults.

The three-term product (x = hi + lo with hi = bf16(x), lo = bf16(x - hi); A W ~ A_hi W_hi + A_lo W_hi + A_hi W_lo in fp32) is
restated in torch and measured as the GPU tests measure the kernels, max |got - ref| / (|A| @ |W|):
  * the forward product at layer 0's K = 9216 against TOL_LINEAR.  Over 9216 terms the roundings of a faulty scheme average
    out as 1 / sqrt(K) just as the correct scheme's do, so the margin here is what it is: plain bf16 operands and a dropped
    A_lo W_hi term exceed the bound by more than MARGIN_K times, not by orders of magnitude;
  * the weight gradient of a layer with M = 245 rows (contraction padded to 256) against TOL_CONV["dkernel"]: the same two
    faults, garbage in columns M..Mp-1 and a Philox index shifted by one quad each exceed it by more than MARGIN times."""
import numpy as np
import torch

from tests.test_gpu_stem_bf16x3 import TOL_CONV, TOL_LINEAR
from tests.test_gpu_wgmma import keep_mask
from tests.test_stem_tc_training import _patches
from tests.test_tc32_bounds import _split, bf16, tc3

MARGIN_K, MARGIN = 5, 30


def dropped_term(a, b):
    """the split product without A_lo W_hi (a segment of the K loop skipped)"""
    ah, _ = _split(a)
    bh, bl = _split(b)
    return ah @ bh + ah @ bl


def _ratio(got, a, b):
    a, b = a.double(), b.double()
    return float(((got.double() - a @ b).abs() / (a.abs() @ b.abs())).max())


def test_forward_bound_at_k_9216():
    g = torch.Generator().manual_seed(1)
    K = 9216
    A = torch.relu(torch.randn(64, K, generator=g))
    W = torch.randn(K, 128, generator=g) * K ** -0.5
    tol = TOL_LINEAR[K]
    r = {f.__name__: _ratio(f(A, W), A, W) for f in (tc3, bf16, dropped_term)}
    print("K = 9216, of TOL_LINEAR: %s" % {k: "%.2f" % (v / tol) for k, v in r.items()})
    assert r["tc3"] <= tol, r
    assert r["bf16"] > MARGIN_K * tol and r["dropped_term"] > MARGIN_K * tol, r


def _wgrad_case():
    """one layer's weight-gradient operands at B=5, 7x7, 128 -> 128, keep 0.82: fp32 dropout(x) patches [245, 1152] and dZ"""
    B, H, W, C, Cout, keep, seed, site, step = 5, 7, 7, 128, 128, 0.82, 4321, 33, 5
    g = torch.Generator().manual_seed(2)
    x = torch.relu(torch.randn(B, H, W, C, generator=g))
    dz = torch.randn(B * H * W, Cout, generator=g)
    sc = np.float32(1.0) / np.float32(keep)
    draws = keep_mask(seed, site, step, (B * H * W * C + 4,), keep, device="cpu")
    cols = lambda off: _patches((x * sc) * draws[off:off + x.numel()].view(x.shape))
    return cols(0), cols(4), dz


def _wgrad(mm, cols, dz, pad_fill=None):
    """dKernel = cols^T dZ contracted over Mp = M rounded up to 64, the padding rows zero or `pad_fill`"""
    M, Mp = cols.shape[0], (cols.shape[0] + 63) // 64 * 64
    pad = lambda t: torch.cat([t, pad_fill(Mp - M, t.shape[1]) if pad_fill else torch.zeros(Mp - M, t.shape[1])], 0)
    return mm(pad(cols).t().contiguous(), pad(dz))


def test_weight_gradient_bound_rejects_each_planted_fault():
    cols, cols_shifted, dz = _wgrad_case()
    tol = TOL_CONV["dkernel"]
    ratio = lambda got: _ratio(got, cols.t(), dz) / tol
    g = torch.Generator().manual_seed(3)
    r = {"tc3": ratio(_wgrad(tc3, cols, dz)),
         "plain bf16": ratio(_wgrad(bf16, cols, dz)),
         "dropped A_lo W_hi": ratio(_wgrad(dropped_term, cols, dz)),
         "garbage padding": ratio(_wgrad(tc3, cols, dz, pad_fill=lambda r_, k: torch.randn(r_, k, generator=g))),
         "Philox index + 4": ratio(_wgrad(tc3, cols_shifted, dz))}
    print("weight gradient, of TOL_CONV['dkernel']: %s" % {k: "%.1f" % v for k, v in r.items()})
    assert r.pop("tc3") <= 1.0
    assert all(v > MARGIN for v in r.values()), r
