"""CPU check of the bounds in tests/test_gpu_wgmma.py, with that file's own reference code: a product accumulated in fp32
passes them, and the same product with one k-block (64 consecutive k) or one split-K slice dropped is rejected by a wide
margin -- also at the headline contraction K = B*N = 12 544 of the weight gradients, where a k-block is 1/196 of the sum."""
import torch

from tests.test_gpu_wgmma import (TOL_SKINNY_SINGLE, TOL_SKINNY_SPLIT, TOL_TC, TOL_WGRAD, excess, split_hi_lo,
                                  bf16_round)


def _drop(x, k0, k1):
    x = x.clone()
    x[:, k0:k1] = 0
    return x


def test_skinny_bounds_reject_a_missing_k_block():
    g = torch.Generator().manual_seed(1)
    M, K, n = 64, 1024, 256
    X = torch.randn(M, K, generator=g)
    W = torch.randn(K, n, generator=g) * K ** -0.5
    xh, xl = split_hi_lo(X)
    wh, wl = split_hi_lo(W)
    absprod = X.double().abs() @ W.double().abs()
    exact = xh @ wh + xl @ wh + xh @ wl
    f32 = lambda a, b: a.float() @ b.float()
    ok = f32(xh, wh) + f32(xl, wh) + f32(xh, wl)
    assert excess(ok, exact, absprod) <= TOL_SKINNY_SPLIT
    for k0 in (0, K - 64):
        bad = f32(_drop(xh, k0, k0 + 64), wh) + f32(_drop(xl, k0, k0 + 64), wh) + f32(_drop(xh, k0, k0 + 64), wl)
        e = excess(bad, exact, absprod)
        print("skinny split, k-block at %d dropped: %.2e (bound %.0e)" % (k0, e, TOL_SKINNY_SPLIT))
        assert e > 100 * TOL_SKINNY_SPLIT
    single = xh @ wh
    assert excess(f32(xh, wh), single, xh.abs() @ wh.abs()) <= TOL_SKINNY_SINGLE
    assert excess(f32(_drop(xh, 512, 576), wh), single, xh.abs() @ wh.abs()) > 100 * TOL_SKINNY_SINGLE


def test_bf16_output_bound_rejects_a_missing_k_block():
    """bf16 outputs get one bf16 ulp on top of tol * |A| @ |B|; a dropped k-block at K = 512 is still far outside."""
    g = torch.Generator().manual_seed(2)
    A = bf16_round(torch.randn(147, 512, generator=g))
    Wt = bf16_round(torch.randn(512, 512, generator=g) * 512 ** -0.5)
    ref = A @ Wt
    absprod = A.abs() @ Wt.abs()
    assert excess(bf16_round(A.float() @ Wt.float()), ref, absprod, ulps=1) <= TOL_TC
    e = excess(bf16_round(_drop(A, 448, 512).float() @ Wt.float()), ref, absprod, ulps=1)
    print("bf16 output, last k-block dropped: %.2e (bound %.0e)" % (e, TOL_TC))
    assert e > 100 * TOL_TC


def test_splitk_bounds_reject_a_missing_k_block_or_slice():
    """dW0 + X^T G at K = 12 544 (196 k-blocks; S = 14 slices of 14 k-blocks at the 512 x 512 headline weight)."""
    g = torch.Generator().manual_seed(3)
    n, K, S = 128, 12544, 14
    X = bf16_round(torch.randn(n, K, generator=g))
    G = bf16_round(torch.randn(n, K, generator=g))
    dW0 = torch.randn(n, n, generator=g).double() * 3
    ref = dW0 + X @ G.t()
    absprod = X.abs() @ G.abs().t() + dW0.abs()
    ks = K // S
    ok = dW0.float() + sum((X[:, s * ks:(s + 1) * ks].float() @ G[:, s * ks:(s + 1) * ks].float().t() for s in range(S)))
    assert excess(ok, ref, absprod) <= TOL_WGRAD
    kblock = dW0.float() + _drop(X, 64 * 100, 64 * 101).float() @ G.float().t()
    slice_ = dW0.float() + _drop(X, 3 * ks, 4 * ks).float() @ G.float().t()
    e_k, e_s = excess(kblock, ref, absprod), excess(slice_, ref, absprod)
    print("wgrad K=12544: one k-block dropped %.2e, one slice dropped %.2e (bound %.0e)" % (e_k, e_s, TOL_WGRAD))
    assert e_k > 100 * TOL_WGRAD and e_s > 100 * TOL_WGRAD
