"""CPU checks of tests/test_gpu_forward_kernels.py with that file's own reference and bound code.

1. The fp64 references are the operations: at a small shape they match plain torch ops (and the numpy restatement of the
   optimizer step in mac_network_b200/dp.py).
2. The bounds are tight enough: a computation done right in fp32 passes them, and each of these planted faults is rejected
   by a wide margin -- one of the skinny kernel's 8 K-slices dropped, one split-K slice dropped, a segment read at the
   wrong k offset, the batch row off by one in the row-scaled concat, a logit part missing from the knowledge-base
   softmax, Adam with m not carried from the previous step, and the EMA taken from the pre-update parameters."""
import numpy as np
import torch

from mac_network_b200.dp import adam_reference as adam_numpy
from tests.test_backward_bounds import _read_forward, _read_inputs
from tests.test_gpu_backward_kernels import ratio, read_masks
from tests.test_gpu_forward_kernels import (ADAM_HYPER, TOL_ADAM, TOL_ATT, TOL_LINEAR, TOL_READ, adam_inputs,
                                            adam_reference, kb_attend_reference, linear_reference, read_forward_stages)

MARGIN = 100


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _check(ok, bad, ref, absref, tol, what, tiny=0.0):
    e_ok, e_bad = ratio(ok, ref, absref, tiny), ratio(bad, ref, absref, tiny)
    print("%s: fp32 %.2e, fault %.2e (bound %.0e)" % (what, e_ok, e_bad, tol))
    assert e_ok <= tol, (what, e_ok)
    assert e_bad > MARGIN * tol, (what, e_bad)


# ------------------------------------------------------------------------------------------------ 1. the references
def test_linear_reference_is_the_linear_layer():
    g = _gen(1)
    xs = [torch.randn(7, k, generator=g, dtype=torch.float64) for k in (4, 20, 8)]
    W, b = torch.randn(32, 5, generator=g, dtype=torch.float64), torch.randn(5, generator=g, dtype=torch.float64)
    z, az = linear_reference(xs, W, b, 0.25)
    want = torch.nn.functional.linear(torch.cat(xs, 1), W.t(), b) + 0.25
    assert torch.allclose(z, want, rtol=1e-12, atol=1e-12)
    assert bool((az >= z.abs() - 1e-12).all())


def test_kb_attend_reference_is_softmax_and_weighted_sum():
    g = _gen(2)
    parts, kb = torch.randn(3, 11, 8, generator=g), torch.randn(3, 11, 6, generator=g)
    att, aatt, info, ainfo = kb_attend_reference(parts, 0.3, kb)
    a = torch.softmax(parts.double().sum(-1) + 0.3, 1)
    assert torch.allclose(att, a, rtol=1e-12, atol=0)
    assert torch.allclose(info, torch.einsum("bn,bnd->bd", a, kb.double()), rtol=1e-12, atol=1e-14)
    assert bool((aatt >= att).all()) and bool((ainfo >= info.abs() - 1e-12).all())


def test_read_stages_are_the_read_unit():
    """from the fp64 forward's own P, y, H, every stage reference reproduces the next stage"""
    B, N, d, keep, seed, step = 3, 5, 8, 0.85, 11, 2
    W, kb, mem, c, _ = _read_inputs(B, N, d, 1)
    masks = read_masks(keep, seed, step, B, N, d, "cpu")
    P, H, I1, y, _, _ = _read_forward(kb, mem, c, W, masks)
    r = read_forward_stages(kb, mem, W, masks, P, y, H)
    for name, want in (("y", y), ("P", P), ("H", H), ("I1", I1)):
        assert torch.allclose(r[name][0], want, rtol=1e-12, atol=1e-12), name
        assert bool((r[name][1] >= r[name][0].abs() - 1e-12).all()), name


def test_adam_reference_is_the_optimizer_step():
    """against dp.adam_reference with hyperparameters that are exact in fp32 (so both use the same values)"""
    g = _gen(3)
    n = 1000
    p, grads, m, v, ema = (t.double() for t in adam_inputs(g, n, "cpu"))
    h = dict(lr=2.0 ** -10, b1=0.875, b2=1 - 2.0 ** -10, eps=2.0 ** -20, decay=1 - 2.0 ** -10)
    for step in (1, 2, 1000):
        norm = float(grads.norm())
        clip = 0.5 * norm
        p1, m1, v1, e1, _ = adam_numpy(p.numpy(), grads.numpy(), m.numpy(), v.numpy(), ema.numpy(), step, lr=h["lr"],
                                       clip=clip, b1=h["b1"], b2=h["b2"], eps=h["eps"], ema_decay=h["decay"])
        t = lambda a: torch.from_numpy(a)
        r = adam_reference(p, grads, m, v, ema, clip / norm, 1.0, h["lr"], h["b1"], h["b2"], h["eps"], step, h["decay"],
                           t(m1), t(v1), t(p1))
        for k, want in (("m", m1), ("v", v1), ("p", p1), ("ema", e1)):
            assert np.allclose(r[k][0].numpy(), want, rtol=1e-12, atol=1e-15), (k, step)


# ------------------------------------------------------------------------------------------------ 2. planted faults
def test_linear_bound_rejects_a_dropped_skinny_slice():
    """M = 64, K = 512: the cluster kernel's 8 CTAs each own a 64-wide K-slice; drop slice 5"""
    g = _gen(4)
    M, K, n = 64, 512, 64
    X, W, b = torch.randn(M, K, generator=g), torch.randn(K, n, generator=g) * K ** -0.5, torch.randn(n, generator=g)
    ref, absref = linear_reference([X], W, b, 0.0)
    parts = [X[:, s * 64:(s + 1) * 64] @ W[s * 64:(s + 1) * 64] for s in range(8)]
    ok = sum(parts[1:], parts[0]) + b
    bad = sum(parts[:5] + parts[6:], torch.zeros(M, n)) + b
    _check(ok, bad, ref, absref, TOL_LINEAR, "linear y, one of 8 skinny K-slices dropped")


def test_linear_bound_rejects_a_dropped_splitk_slice():
    """M = 700, K = 2048 in 11 split-K slices (the sgemm's split of a 24-tile product); drop slice 7"""
    g = _gen(5)
    M, K, n, S = 700, 2048, 64, 11
    X, W = torch.randn(M, K, generator=g), torch.randn(K, n, generator=g) * K ** -0.5
    ref, absref = linear_reference([X], W, None, 0.0)
    per = -(-K // S)
    parts = [X[:, s * per:(s + 1) * per] @ W[s * per:(s + 1) * per] for s in range(S)]
    ok = sum(parts[1:], parts[0])
    bad = sum(parts[:7] + parts[8:], torch.zeros(M, n))
    _check(ok, bad, ref, absref, TOL_LINEAR, "linear y, one split-K slice dropped")


def test_linear_bound_rejects_a_segment_at_the_wrong_offset():
    """segments of width 4, 20, 488 as column blocks of wider buffers; the fault reads the 20-wide segment 4 columns late
    (from its buffer's padding)"""
    g = _gen(6)
    M, n = 37, 20
    bufs = [torch.randn(M, k + pad, generator=g) for k, pad in ((4, 4), (20, 12), (488, 0))]
    xs = [bufs[0][:, :4], bufs[1][:, :20], bufs[2]]
    W = torch.randn(512, n, generator=g) * 512 ** -0.5
    ref, absref = linear_reference(xs, W, None, 0.0)
    ok = torch.cat(xs, 1) @ W
    bad = torch.cat([xs[0], bufs[1][:, 4:24], xs[2]], 1) @ W
    _check(ok, bad, ref, absref, TOL_LINEAR, "linear y, segment read at k offset + 4")


def test_read_bound_rejects_a_batch_row_off_by_one():
    """H = ELU([P*y, P] @ Wm + bm) where row k of P is scaled by y[k / N]; the fault takes y of the previous sample for
    the first row of every sample after the first"""
    B, N, d, keep, seed, step = 8, 49, 64, 0.85, 5, 1
    W, kb, mem, c, _ = _read_inputs(B, N, d, 7)
    masks = read_masks(keep, seed, step, B, N, d, "cpu")
    P, H, _, y, _, _ = _read_forward(kb, mem, c, W, masks)
    Pf, yf = P.float(), y.float()
    r = read_forward_stages(kb, mem, W, masks, Pf, yf, H)
    ref, absref = r["H"]
    Wm, bm = W["Wm"].float(), W["bm"].float()
    rows = torch.arange(B * N) // N
    ok = torch.nn.functional.elu(torch.cat([Pf * yf[rows], Pf], 1) @ Wm + bm)
    rows_bad = rows.clone()
    rows_bad[N::N] -= 1
    bad = torch.nn.functional.elu(torch.cat([Pf * yf[rows_bad], Pf], 1) @ Wm + bm)
    _check(ok, bad, ref, absref, TOL_READ, "read H, batch row off by one")


def test_kb_bound_rejects_a_missing_logit_part():
    """8 partial logits per row (64-wide column tiles at d = 512); the fault sums 7 of them"""
    g = _gen(8)
    B, N, d, P = 3, 196, 64, 8
    parts, kb = torch.randn(B, N, P, generator=g), torch.randn(B, N, d, generator=g)
    att, aatt, info, ainfo = kb_attend_reference(parts, 0.3, kb)

    def fp32(pp):
        a = torch.softmax(pp.sum(-1) + 0.3, 1)
        return a, torch.einsum("bn,bnd->bd", a, kb)

    ok_a, ok_i = fp32(parts)
    bad_a, bad_i = fp32(torch.cat([parts[..., :3], parts[..., 4:]], -1))
    _check(ok_a, bad_a, att, aatt, TOL_ATT, "kb att, one logit part missing")
    _check(ok_i, bad_i, info, ainfo, TOL_ATT, "kb info, one logit part missing")


def _adam_fp32(p, grads, m, v, ema, clip, step, carry_m=True, ema_of_new=True):
    """the kernel's arithmetic in fp32 torch ops, with the two faults as switches"""
    h = ADAM_HYPER
    f = lambda x: torch.tensor(x, dtype=torch.float32)
    b1, b2, lr, eps, dec = f(h["b1"]), f(h["b2"]), f(h["lr"]), f(h["eps"]), f(h["decay"])
    gi = grads * f(clip)
    mi = (b1 * m if carry_m else 0.0) + (1 - b1) * gi
    vi = b2 * v + (1 - b2) * gi * gi
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    pn = p - lr * torch.sqrt(bc2) / bc1 * mi / (torch.sqrt(vi) + eps)
    en = dec * ema + (1 - dec) * (pn if ema_of_new else p)
    return pn, mi, vi, en


def test_adam_bound_rejects_m_not_carried():
    g = _gen(9)
    p, grads, m, v, ema = adam_inputs(g, 4099, "cpu")
    h = ADAM_HYPER
    pn, mi, vi, _ = _adam_fp32(p, grads, m, v, ema, 0.5, 2)
    _, mb, _, _ = _adam_fp32(p, grads, m, v, ema, 0.5, 2, carry_m=False)
    r = adam_reference(p, grads, m, v, ema, 0.5, 1.0, h["lr"], h["b1"], h["b2"], h["eps"], 2, h["decay"], mi, vi, pn)
    _check(mi, mb, r["m"][0], r["m"][1], TOL_ADAM, "adam m, not carried from the previous step")


def test_ema_bound_rejects_the_pre_update_parameters():
    g = _gen(10)
    p, grads, m, v, ema = adam_inputs(g, 4099, "cpu")
    h = ADAM_HYPER
    pn, mi, vi, en = _adam_fp32(p, grads, m, v, ema, 1.0, 1)
    _, _, _, eb = _adam_fp32(p, grads, m, v, ema, 1.0, 1, ema_of_new=False)
    r = adam_reference(p, grads, m, v, ema, 1.0, 1.0, h["lr"], h["b1"], h["b2"], h["eps"], 1, h["decay"], mi, vi, pn)
    ref, absref, tiny = r["p"]
    assert ratio(pn, ref, absref, tiny) <= TOL_ADAM
    _check(en, eb, r["ema"][0], r["ema"][1], TOL_ADAM, "ema, taken from the pre-update parameters")
