"""CPU checks of tests/test_gpu_backward_kernels.py with that file's own reference and bound code.

1. The fp64 references are the gradients: at a small shape they match torch.autograd of the forward they differentiate.
2. The bounds are tight enough: a computation done right in fp32 passes them, and each of these planted faults is rejected
   by a wide margin -- a dropped split-K slice at K = 12 544, a dropped 64-row block of the row-dot reduction, the batch
   row off by one at a batch boundary of the row-scaled concat, the naive softmax backward at peaked attention, and dby
   summed from a partially overwritten dy."""
import numpy as np
import torch

from tests.test_gpu_backward_kernels import (TOL_KB, TOL_LINEAR, TOL_READ, TOL_ROWDOT, control_bwd_reference,
                                             linear_bwd_reference, peaked_softmax, read_bwd_reference, read_masks, ratio)

MARGIN = 100


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _read_inputs(B, N, d, seed):
    g = _gen(seed)
    r = lambda *s, scale=1.0: torch.randn(*s, generator=g, dtype=torch.float64) * scale
    W = {"Wx": r(d, d, scale=d ** -0.5), "bx": r(d, scale=0.1), "Wy": r(d, d, scale=d ** -0.5), "by": r(d, scale=0.1),
         "Wm": r(2 * d, d, scale=(2 * d) ** -0.5), "bm": r(d, scale=0.1), "Wm2": r(d, d, scale=d ** -0.5),
         "bm2": r(d, scale=0.1), "wr": r(d, scale=4 * d ** -0.5)}
    return W, torch.nn.functional.elu(r(B, N, d)), r(B, d), r(B, d), r(B, d)


def _read_forward(kb, mem, c, W, masks, br=0.25):
    """the read unit of include/mac_b200.h in fp64 torch ops: (P, H, I1, y, att, info)"""
    B, N, d = kb.shape
    mkb, mmem, mint = masks
    y = (mem * mmem) @ W["Wy"] + W["by"]
    P = (kb.reshape(B * N, d) * mkb) @ W["Wx"] + W["bx"]
    yb = y.repeat_interleave(N, 0)
    H = torch.nn.functional.elu(torch.cat([P * yb, P], 1) @ W["Wm"] + W["bm"])
    I1 = H @ W["Wm2"] + W["bm2"]
    I2 = torch.nn.functional.elu(I1 * c.repeat_interleave(N, 0))
    att = torch.softmax(((I2 * mint) @ W["wr"] + br).view(B, N), 1)
    return P, H, I1, y, att, torch.einsum("bn,bnd->bd", att, kb)


def test_read_reference_is_the_gradient():
    B, N, d, keep, seed, step = 3, 5, 8, 0.85, 11, 2
    W, kb, mem, c, dinfo = _read_inputs(B, N, d, 1)
    masks = read_masks(keep, seed, step, B, N, d, "cpu")
    leaves = {"kb": kb, "mem": mem, "c": c, **W}
    for t in leaves.values():
        t.requires_grad_(True)
    P, H, I1, y, att, info = _read_forward(kb, mem, c, W, masks)
    (info * dinfo).sum().backward()
    with torch.no_grad():
        r = read_bwd_reference(kb, mem, c, W, att, P, H, I1, y, dinfo, keep, seed, step)
    want = {"dkb": kb.grad, "dmem_in": mem.grad, "dcontrol": c.grad, "dWx": W["Wx"].grad, "dbx_part": W["bx"].grad,
            "dWy": W["Wy"].grad, "dby": W["by"].grad, "dWm": W["Wm"].grad, "dbm_part": W["bm"].grad,
            "dWm2": W["Wm2"].grad, "dbm2_part": W["bm2"].grad, "dwr_part": W["wr"].grad}
    for k, v in want.items():
        got = r[k][0].sum(0) if k.endswith("_part") else r[k][0]     # per-sample partials, reduced over the batch
        assert torch.allclose(got, v, rtol=1e-10, atol=1e-12), k
        assert bool((r[k][1] >= r[k][0].abs() - 1e-12).all()), k      # the bound dominates the value
    assert abs(float(r["dbr_part"][0].sum())) < 1e-12                # d/dbr of a softmax is zero


def test_control_reference_is_the_gradient():
    T, B, S, d = 2, 3, 6, 8
    g = _gen(2)
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    cc, inw, outw, w, gout, dq0 = r(T, B, d), r(B, S, d), r(B, S, d), r(d), r(T, B, d), r(T, B, d)
    for t in (cc, inw, outw, w):
        t.requires_grad_(True)
    att = torch.softmax(torch.einsum("tbd,bsd->tbs", cc * w, inw), 2)
    (torch.einsum("tbs,bsd->tbd", att, outw) * gout).sum().backward()
    with torch.no_grad():
        ref, dq = control_bwd_reference(cc, inw, outw, w, att, gout, dq0, 1)
    assert torch.allclose(ref["din"][0], inw.grad, rtol=1e-10, atol=1e-12)
    assert torch.allclose(ref["dout"][0], outw.grad, rtol=1e-10, atol=1e-12)
    assert torch.allclose(ref["dw"][0].sum(0), w.grad, rtol=1e-10, atol=1e-12)
    assert torch.allclose(torch.stack([v for v, _ in dq]) - dq0, cc.grad, rtol=1e-10, atol=1e-12)
    assert float(ref["db"][0].abs().max()) < 1e-12


def _check(ok, bad, ref, absref, tol, what):
    e_ok, e_bad = ratio(ok, ref, absref), ratio(bad, ref, absref)
    print("%s: fp32 %.2e, fault %.2e (bound %.0e)" % (what, e_ok, e_bad, tol))
    assert e_ok <= tol, (what, e_ok)
    assert e_bad > MARGIN * tol, (what, e_bad)


def test_linear_bound_rejects_a_dropped_splitk_slice():
    """dW = X^T dy at K = M = 12 544 in S = 17 slices (the sgemm's split at 512 x 512 with 128-wide tiles)"""
    g = _gen(3)
    M, k, n, S = 12544, 64, 64, 17
    X, dy = torch.randn(M, k, generator=g), torch.randn(M, n, generator=g)
    Wt = torch.randn(n, k, generator=g)
    _, (ref, absref), _ = linear_bwd_reference([X], Wt, dy)
    per = -(-M // S)
    parts = [X[s * per:(s + 1) * per].t() @ dy[s * per:(s + 1) * per] for s in range(S)]
    ok = sum(parts[1:], parts[0])
    bad = sum(parts[:3] + parts[4:], torch.zeros(k, n))
    _check(ok, bad, ref, absref, TOL_LINEAR, "linear dW, one split-K slice dropped")


def test_rowdot_bound_rejects_a_dropped_row_block():
    g = _gen(4)
    R, K = 12544, 128
    X, gr = torch.randn(R, K, generator=g), torch.randn(R, generator=g)
    ref, absref = gr.double() @ X.double(), gr.double().abs() @ X.double().abs()
    parts = [gr[i:i + 64] @ X[i:i + 64] for i in range(0, R, 64)]
    ok = sum(parts[1:], parts[0])
    bad = sum(parts[:100] + parts[101:], torch.zeros(K))
    _check(ok, bad, ref, absref, TOL_ROWDOT, "rowdot dw, one 64-row block dropped")


def test_read_bound_rejects_a_batch_row_off_by_one():
    """dWm = [P*y, P]^T dZ where row k of P is scaled by y[k / N]; the fault takes y of the previous sample for the first
    row of every sample after the first"""
    B, N, d, keep, seed, step = 8, 49, 64, 0.85, 5, 1
    W, kb, mem, c, dinfo = _read_inputs(B, N, d, 6)
    P, H, I1, y, att, _ = _read_forward(kb, mem, c, W, read_masks(keep, seed, step, B, N, d, "cpu"))
    r = read_bwd_reference(kb, mem, c, W, att, P, H, I1, y, dinfo, keep, seed, step)
    ref, absref = r["dWm"]
    dZ = r["_dZ"][0].float()
    Pf, yf = P.float(), y.float()
    rows = torch.arange(B * N) // N
    ok = torch.cat([Pf * yf[rows], Pf], 1).t() @ dZ
    rows_bad = rows.clone()
    rows_bad[N::N] -= 1
    bad = torch.cat([Pf * yf[rows_bad], Pf], 1).t() @ dZ
    _check(ok, bad, ref, absref, TOL_READ["dWm"], "read dWm, batch row off by one")


def test_kb_bound_rejects_the_naive_softmax_backward():
    """at peaked attention ka[n] * (dka[n] - sum ka dka) loses the small result of the peak cell to the rounding of the
    two nearly equal terms; the kernel's sum of weighted differences does not"""
    B, N = 4, 196
    g = _gen(7)
    a = peaked_softmax(g, B, N)
    assert float(a.max(1).values.min()) > 1 - 1e-6
    dka = torch.randn(B, N, generator=g)
    ad, kd = a.double(), dka.double()
    ref = ad * (ad[:, None, :] * (kd[:, :, None] - kd[:, None, :])).sum(2)
    absref = ad * (ad[:, None, :] * (kd[:, :, None] - kd[:, None, :]).abs()).sum(2)
    ok = a * (a[:, None, :] * (dka[:, :, None] - dka[:, None, :])).sum(2)
    naive = a * (dka - (a * dka).sum(1, keepdim=True))
    _check(ok, naive, ref, absref, TOL_KB, "kb dkl, naive softmax backward at peaked attention")


def test_read_bound_rejects_dby_from_an_overwritten_dy():
    """dby = colsum_b(dy) with the first 2 048 floats of dy replaced by the values of another product (the split-K
    partials that overlapped dy at small N)"""
    B, N, d, keep, seed, step = 64, 3, 512, 1.0, 8, 0
    W, kb, mem, c, dinfo = _read_inputs(B, N, d, 9)
    P, H, I1, y, att, _ = _read_forward(kb, mem, c, W, read_masks(keep, seed, step, B, N, d, "cpu"))
    r = read_bwd_reference(kb, mem, c, W, att, P, H, I1, y, dinfo, keep, seed, step)
    ref, absref = r["dby"]
    dy = r["_dy"][0].float()
    ok = dy.sum(0)
    over = dy.clone().view(-1)
    over[:2048] = torch.from_numpy(np.random.default_rng(0).standard_normal(2048).astype(np.float32)) * float(dy.std())
    bad = over.view(B, d).sum(0)
    _check(ok, bad, ref, absref, TOL_READ["dby"], "read dby, dy partly overwritten")
