"""The fused read step (read_step_kernel, csrc/read_step.cuh, then kb_attend) row by row against fp64, its tiling
invariance bit for bit (and that of the e4m3 step, csrc/read_step_fp8.cuh), and the read unit's forward at batches past
gridDim.y's 65535.

1. Per-row logits.  The kernel leaves its logits (I2 . wr, without br) in `inv` (read_inv_layout(MAC_PREC_BF16)'s logits).
   Each row is checked against an fp64 reference fed with the kernel's own operands, within a bound derived from them
   (step_reference):
     P*y   PY = bf16_rn(fp32(P16 * y_b)), the kernel's operand exactly (it never leaves shared memory).
     H     H* = ELU(PY @ Wm16[0:d] + Q16).  The kernel rounds v = elu_fast(acc + Q) to bf16, with |v - H*| <= e =
           TOL_TC * (|PY| @ |Wm16[0:d]| + |Q|) + EPS_ELU (ELU is 1-Lipschitz).  Rounding is monotone, so the kernel's H
           lies in [bf16(fp32(H* - e)), bf16(fp32(H* + e))]: the reference is H~ = bf16(fp32(H*)) and dH the distance to
           the far end of that interval -- 0 except where a bf16 rounding midpoint lies within e of H*.  (Half a bf16 ulp
           of |H*| on every element would be sound too, but it adds up to about one logit unit, wider than a missing
           k-block or a wrong sample would move a logit.)
     I1    I1* = H~ @ Wm2_16 + bm2,  |dI1| <= dH @ |Wm2_16| + TOL_TC * ((|H~| + dH) @ |Wm2_16| + |bm2|).
     I2    I2* = ELU(I1* c_b),  |dI2| <= |c_b| |dI1| + 2^-24 |c_b| (|I1*| + |dI1|) + EPS_ELU.
     logit logit* = sum I2* wr,  bound = sum |wr| |dI2| + GAMMA * sum (|I2*| + |dI2|) |wr|: each half of the row is 64
           fmaf per thread, two shuffle adds and half0 + half1, 67 roundings deep.
   EPS_ELU is the absolute error of elu_fast's negative branch, ex2.approx.ftz(x * log2e) - 1 (csrc/tc_gemm.cuh): the PTX
   ISA gives ex2.approx.f32 at most 2 ulp of error, below 2^-22 of 2^x <= 1; the rounded argument x * fp32(log2e) moves
   2^x by at most e^x |x| 2^-23 < 2^-24; the subtraction of 1 rounds by at most 2^-25.  The sum is below 2^-21.  Near 0-
   the subtraction cancels, so the error is absolute, not relative to the result.
   att and info are then checked through test_gpu_wgmma.softmax_bound_check fed with these logits and bounds.  Each case
   also checks canaries: att and info NaN-filled before and finite after; every `inv` byte past the M logits keeps its fill
   pattern (rows past M in the last tile are not stored); P, Q, the knowledge base, y and control bit-unchanged.
   tests/test_read_step_bounds.py shows on the CPU, with this file's reference, that an emulation of the kernel's
   arithmetic passes the bound and that planted faults fail it by a wide margin.
2. Tiling invariance.  Every output element takes the same operations in the same order wherever its row sits in a tile,
   so copies of one sample placed at every start offset of a tile (N odd, B = 128: sample b starts at row b*N mod 128)
   must give bit-identical P and Q rows (mac_read_invariant: no split-K, no atomics), logits, att and info rows.  And a
   sample's results must not depend on its neighbours: with every third sample held fixed and the others redrawn, the
   fixed samples' outputs stay bit-identical.
3. Large batches.  kb_attend runs B * d / 128 CTAs on a 1-D grid, so the fused step, and mac_read_fwd_inv in bf16, e4m3 and
   fp32, work at B = 65535, 65536 and 200 003 with N = 1 (tests/test_read_limits_refusals.py has the refusals past the
   GEMMs' row limits)."""
import ctypes

import pytest
import torch

from mac_network_b200 import _lib as L_
from tests.test_gpu_wgmma import (TOL_TC, align1k, bf16_slab, elu, lib, nanfill, randn, read_setup,
                                  softmax_bound_check)

pytestmark = pytest.mark.gpu

D = 512
FP32, BF16, FP8 = 0, 1, 3
EPS_ELU = 2.0 ** -21
U32 = 2.0 ** -24
GAMMA = 67 * U32 / (1 - 67 * U32)
FILL = 0xA5                          # byte pattern of `inv` before mac_read_invariant


# ------------------------------------------------------------------------------------------------ the reference and its bound
def step_reference(P16, Q16, yb, cb, W1, W2, bm2, wr):
    """fp64 reference of the fused step's logits and their bound, one per row (see the module docstring).  P16, Q16 [R, d]
    bf16; yb, cb [R, d] fp32, each row's sample's y and control; W1 = the bf16 pack of Wm[0:d] and W2 that of Wm2, both
    [out, in]; bm2, wr [d] fp32.  Returns (logit*, bound) as float64 [R]."""
    PY = (P16.float() * yb.float()).to(torch.bfloat16).double()
    W1d, W2d, Qd = W1.double().t(), W2.double().t(), Q16.double()
    Hs = elu(PY @ W1d + Qd)
    e = TOL_TC * (PY.abs() @ W1d.abs() + Qd.abs()) + EPS_ELU
    bf = lambda t: t.float().to(torch.bfloat16).double()
    Ht = bf(Hs)
    dH = torch.maximum(bf(Hs + e) - Ht, Ht - bf(Hs - e))
    bm2d, wrd, cd = bm2.double(), wr.double(), cb.double()
    I1 = Ht @ W2d + bm2d
    dI1 = dH @ W2d.abs() + TOL_TC * ((Ht.abs() + dH) @ W2d.abs() + bm2d.abs())
    I2 = elu(I1 * cd)
    dI2 = cd.abs() * dI1 + U32 * cd.abs() * (I1.abs() + dI1) + EPS_ELU
    return I2 @ wrd, dI2 @ wrd.abs() + GAMMA * ((I2.abs() + dI2) @ wrd.abs())


def rows_over(got, ref, bound, N, limit=8):
    """the rows whose error exceeds the bound: (row, sample, row % 128, got, ref, bound)"""
    r = (got.double() - ref).abs() / bound
    bad = torch.nonzero(~(r <= 1)).flatten()[:limit].tolist()
    return [(k, k // N, k % 128, float(got[k]), float(ref[k]), float(bound[k])) for k in bad]


# ------------------------------------------------------------------------------------------------ plumbing
def add_fp8_packs(W, rw):
    """e4m3 packs of Wm[0:d] and Wm2 with their column scales into rw; returns them (the caller keeps them alive)"""
    from tests.test_gpu_read_step_fp8 import _pack8
    W1, s1 = _pack8(L_, lib(), W["Wm"][:D])
    W2, s2 = _pack8(L_, lib(), W["Wm2"])
    rw.Wm_fp8, rw.Wm_fp8_scale, rw.Wm2_fp8, rw.Wm2_fp8_scale = W1.data_ptr(), s1.data_ptr(), W2.data_ptr(), s2.data_ptr()
    return W1, s1, W2, s2


def inv_views(inv, prec, B, N, d=D):
    """P and Q (bf16 [M, d]) and the logits (fp32 [M]) of `inv`, and the byte offset just past the logits"""
    M = B * N
    al = lambda b: (b + 1023) & ~1023
    io, b16 = align1k(inv), al(M * d * 2)
    if prec == BF16:
        o_P, o_Q, o_lg = io, io + b16, io + 2 * b16
    else:                                             # [P8 | sP | Q | logits | P]
        o_Q = io + al(M * d) + al(M * 4)
        o_lg = o_Q + b16
        o_P = o_lg + al(M * 4)
    return (bf16_slab(inv, o_P, M, d), bf16_slab(inv, o_Q, M, d), inv[o_lg:o_lg + 4 * M].view(torch.float32),
            o_lg + 4 * M)


def run_read(prec, rw, kb16, y, c, B, N):
    """mac_read_invariant, then the read step: mac_read_step_fused (bf16) or mac_read_fwd_inv with y_pre (fp8).  `inv` is
    FILL-filled first, att and info NaN-filled.  Returns inv, P, Q, logits, att, info and the offset past the logits."""
    lb = lib()
    nb = lb.mac_read_invariant_bytes(B, N, D, prec)
    inv = torch.full((nb,), FILL, dtype=torch.uint8, device="cuda")
    L_.check(lb.mac_read_invariant(None, L_.ptr(kb16), ctypes.byref(rw), prec, L_.ptr(inv), nb, B, N, D, L_.stream_ptr()),
             "mac_read_invariant")
    info, att = nanfill(B, D), nanfill(B, N)
    if prec == BF16:
        L_.check(lb.mac_read_step_fused(L_.ptr(inv), L_.ptr(kb16), L_.ptr(y), L_.ptr(c), ctypes.byref(rw), L_.ptr(info),
                                        L_.ptr(att), B, N, D, L_.stream_ptr()), "mac_read_step_fused")
    else:
        wsb = lb.mac_read_workspace_bytes(B, N, D, prec)
        ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
        L_.check(lb.mac_read_fwd_inv(None, L_.ptr(kb16), L_.ptr(inv), L_.ptr(y), L_.ptr(y), L_.ptr(c), ctypes.byref(rw),
                                     prec, L_.ptr(info), L_.ptr(att), L_.ptr(ws), wsb, B, N, D, L_.stream_ptr()),
                 "mac_read_fwd_inv")
    torch.cuda.synchronize()
    P, Q, lg, end = inv_views(inv, prec, B, N)
    return dict(inv=inv, P=P, Q=Q, logits=lg, att=att, info=info, end=end)


def bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


# ================================================================================================ 1. row by row against fp64
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


SHAPES = [(1, 1), (5, 1), (300, 1),                  # one-row samples, 128 per tile; the last tile partial at 300
          (64, 2), (200, 3),                          # 64 and about 43 samples per tile
          (1, 128), (1, 129), (1, 255), (1, 256),     # one tile exactly, one row over, one short, two full
          (3, 43), (1, 193), (5, 51),                 # last tile: 1 row (across samples), 65 rows (one in warpgroup 1), 127
          (64, 49), (64, 196), (384, 196),            # GQA, headline, batched request
          ("2sms+1", 128)]                            # a tile count one above a multiple of the SM count


@pytest.mark.parametrize("B,N", SHAPES)
def test_fused_read_step_logits_match_fp64_row_by_row(B, N):
    if B == "2sms+1":
        B = 2 * _sms() + 1
    lb = lib()
    assert lb.mac_read_step_fused_supported(B, N, D) == 1
    g, W, Pk, _, rw = read_setup(D, 7 * B + N)
    M = B * N
    kb16 = elu(randn(g, B, N, D)).to(torch.bfloat16)
    y, c = randn(g, B, D), randn(g, B, D)
    # the inputs as they are before the step (P and Q: after mac_read_invariant, read back below)
    kb0, y0, c0 = kb16.clone(), y.clone(), c.clone()
    nb = lb.mac_read_invariant_bytes(B, N, D, BF16)
    inv = torch.full((nb,), FILL, dtype=torch.uint8, device="cuda")
    L_.check(lb.mac_read_invariant(None, L_.ptr(kb16), ctypes.byref(rw), BF16, L_.ptr(inv), nb, B, N, D, L_.stream_ptr()))
    P, Q, lg, end = inv_views(inv, BF16, B, N)
    torch.cuda.synchronize()
    P0, Q0 = P.clone(), Q.clone()
    assert bool((inv[end:] == FILL).all()), "mac_read_invariant wrote past the logit scratch"
    info, att = nanfill(B, D), nanfill(B, N)
    L_.check(lb.mac_read_step_fused(L_.ptr(inv), L_.ptr(kb16), L_.ptr(y), L_.ptr(c), ctypes.byref(rw), L_.ptr(info),
                                    L_.ptr(att), B, N, D, L_.stream_ptr()), "mac_read_step_fused")
    torch.cuda.synchronize()
    for name, now, was in (("P", P, P0), ("Q", Q, Q0), ("kb", kb16, kb0), ("y", y, y0), ("control", c, c0)):
        assert torch.equal(bits(now), bits(was)), "%s changed by the step" % name
    assert bool((inv[end:] == FILL).all()), "bytes past the M logits written (rows past M of the last tile stored?)"
    assert bool(torch.isfinite(lg).all()), "non-finite logit"
    ref, bound = step_reference(P, Q, y.repeat_interleave(N, 0), c.repeat_interleave(N, 0), Pk["Wm"][:, :D], Pk["Wm2"],
                                W["bm2"], W["wr"])
    r = float(((lg.double() - ref).abs() / bound).max())
    ra, ri = softmax_bound_check(att, info, ref + 0.25, bound + 1e-6 * ((ref + 0.25).abs() + 1), kb16, B, N)
    print("fused read step B=%d N=%d: logits use %.3f of their bound (median bound %.2e), att %.3f, info %.3f"
          % (B, N, r, float(bound.median()), ra, ri))
    assert r <= 1, rows_over(lg, ref, bound, N)
    assert ra <= 1 and ri <= 1, (ra, ri)


# ================================================================================================ 2. tiling invariance
def _setup(prec, seed):
    g, W, Pk, _, rw = read_setup(D, seed)
    keep = add_fp8_packs(W, rw) if prec == FP8 else ()
    return g, W, (Pk, keep), rw


def _sample_inputs(g, n, N):
    return elu(randn(g, n, N, D)).to(torch.bfloat16), randn(g, n, D), randn(g, n, D)


def _first_diff(t, B):
    """the copies b whose rows differ from copy 0's"""
    v = bits(t).view(B, -1)
    return [b for b in range(B) if not torch.equal(v[b], v[0])]


COPIES = [pytest.param(prec, N, B, id="%s-N%d-B%d" % (name, N, B))
          for prec, name, Ns in ((BF16, "bf16", (1, 3, 49, 127, 129, 255)), (FP8, "fp8", (1, 3, 49, 65, 127, 129, 255)))
          for N, B in [(n, 128) for n in Ns] + [(1, 257)]]


@pytest.mark.parametrize("prec,N,B", COPIES)
def test_read_step_copies_of_one_sample_are_bit_identical(prec, N, B):
    """B copies of one sample (rows distinct within it): with N odd the copies start at every row offset of a tile, in
    both warpgroups and every swizzle phase, and at B = 257, N = 1 one copy sits alone in a partial third tile."""
    g, _, keep, rw = _setup(prec, 1000 + N)
    kb1, y1, c1 = _sample_inputs(g, 1, N)
    kb16, y, c = kb1.repeat(B, 1, 1).contiguous(), y1.repeat(B, 1).contiguous(), c1.repeat(B, 1).contiguous()
    o = run_read(prec, rw, kb16, y, c, B, N)
    off = lambda bs: [(b, b * N % 128) for b in bs[:8]]
    # mac_read_invariant first: its GEMMs have no split-K and no atomics on this path
    for name in ("P", "Q"):
        bad = _first_diff(o[name].view(B, N, D), B)
        assert not bad, ("mac_read_invariant %s rows differ between copies (copy, start row in tile)" % name, off(bad))
    for name in ("logits", "att", "info"):
        assert bool(torch.isfinite(o[name]).all()), name
        bad = _first_diff(o[name].view(B, -1), B)
        assert not bad, ("%s differs between copies (copy, start row in tile)" % name, off(bad))


@pytest.mark.parametrize("prec", [pytest.param(BF16, id="bf16"), pytest.param(FP8, id="fp8")])
@pytest.mark.parametrize("B,N", [(128, 49), (300, 1), (20, 17)])
def test_read_step_sample_does_not_depend_on_its_neighbours(prec, B, N):
    """Two runs in which every third sample keeps its knowledge base, y and control and the others are redrawn: the fixed
    samples' logits, att and info rows are bit-identical.  A row reading a neighbour's y or control fails this."""
    g, _, keep, rw = _setup(prec, 2000 + B + N)
    kb16, y, c = _sample_inputs(g, B, N)
    fixed = torch.arange(0, B, 3, device="cuda")
    outs = []
    for run in range(2):
        if run:
            kb2, y2, c2 = _sample_inputs(g, B, N)
            kb2[fixed], y2[fixed], c2[fixed] = kb16[fixed], y[fixed], c[fixed]
            kb16, y, c = kb2, y2, c2
        o = run_read(prec, rw, kb16, y, c, B, N)
        outs.append({k: o[k].view(B, -1)[fixed].clone() for k in ("logits", "att", "info")})
    for k in ("logits", "att", "info"):
        assert bool(torch.isfinite(outs[1][k]).all()), k
        same = (bits(outs[0][k]) == bits(outs[1][k])).all(1)
        assert bool(same.all()), ("%s of fixed samples changed with their neighbours" % k,
                                  fixed[~same][:8].tolist())


# ================================================================================================ 3. large batches
def _sample_rows(M, seed, n=300):
    """n rows spread over [0, M), the first and the last included"""
    r = torch.randperm(M, generator=torch.Generator().manual_seed(seed))[:n - 2]
    return torch.cat([torch.tensor([0, M - 1]), r]).unique().cuda()


@pytest.mark.parametrize("B", [65535, 65536, 200003])
def test_read_forward_at_large_batch(B):
    """N = 1: the fused step, mac_read_fwd_inv at bf16 and e4m3 (d = 512) and at fp32 (d = 128).  With one row per sample
    att is exactly 1 and info exactly the knowledge-base row, so both are checked for every sample (NaN before the call);
    the logits of a few hundred rows (the last included) against the part 1 bound, and the fp32 form's P, Q and H against
    test_gpu_forward_kernels' references."""
    lb = lib()
    N = 1
    rows = _sample_rows(B, B)
    g, W, Pk, _, rw = read_setup(D, 31 + B)
    keep = add_fp8_packs(W, rw)
    kb16, y, c = _sample_inputs(g, B, N)
    # the fused step, then the same step through mac_read_fwd_inv: bit for bit the same outputs
    o = run_read(BF16, rw, kb16, y, c, B, N)
    assert bool((o["att"] == 1).all()) and torch.equal(o["info"], kb16.float().view(B, D)), "att / info (fused step)"
    ref, bound = step_reference(o["P"][rows], o["Q"][rows], y[rows], c[rows], Pk["Wm"][:, :D], Pk["Wm2"], W["bm2"], W["wr"])
    lg = o["logits"][rows]
    r = float(((lg.double() - ref).abs() / bound).max())
    assert r <= 1, rows_over(lg, ref, bound, N)
    logits0 = o["logits"].clone()
    wsb = lb.mac_read_workspace_bytes(B, N, D, BF16)
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    info, att = nanfill(B, D), nanfill(B, N)
    L_.check(lb.mac_read_fwd_inv(None, L_.ptr(kb16), L_.ptr(o["inv"]), L_.ptr(y), L_.ptr(y), L_.ptr(c), ctypes.byref(rw),
                                 BF16, L_.ptr(info), L_.ptr(att), L_.ptr(ws), wsb, B, N, D, L_.stream_ptr()), "mac_read_fwd_inv")
    torch.cuda.synchronize()
    assert torch.equal(bits(o["logits"]), bits(logits0)) and torch.equal(att, o["att"]) and torch.equal(info, o["info"])
    del o, ws, info, att
    torch.cuda.empty_cache()
    # e4m3: P and Q as the bf16 form computes them; att and info exact
    o8 = run_read(FP8, rw, kb16, y, c, B, N)
    assert bool((o8["att"] == 1).all()) and torch.equal(o8["info"], kb16.float().view(B, D)), "att / info (e4m3 step)"
    assert bool(torch.isfinite(o8["logits"]).all())
    del o8
    torch.cuda.empty_cache()
    # fp32 at d = 128 (the four-launch chain, then kb_attend on the fp32 knowledge base)
    from tests.test_gpu_forward_kernels import TOL_READ, read_ws_offsets, ws_floats
    d = 128
    _, W, _, _, rw = read_setup(d, 37 + B)
    kb = elu(randn(g, B * N, d))
    y = randn(g, B, d)
    nb = lb.mac_read_invariant_bytes(B, N, d, FP32)
    inv = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    L_.check(lb.mac_read_invariant(L_.ptr(kb), None, ctypes.byref(rw), FP32, L_.ptr(inv), nb, B, N, d, L_.stream_ptr()))
    wsb = lb.mac_read_workspace_bytes(B, N, d, FP32)
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    info, att = nanfill(B, d), nanfill(B, N)
    L_.check(lb.mac_read_fwd_inv(L_.ptr(kb), None, L_.ptr(inv), L_.ptr(y), L_.ptr(y), L_.ptr(y), ctypes.byref(rw), FP32,
                                 L_.ptr(info), L_.ptr(att), L_.ptr(ws), wsb, B, N, d, L_.stream_ptr()), "mac_read_fwd_inv fp32")
    torch.cuda.synchronize()
    assert bool((att == 1).all()) and torch.equal(info, kb.view(B, d)), "att / info (fp32)"
    M = B * N
    P, Q = ws_floats(inv, 0, M, d)[rows].double(), ws_floats(inv, M * d * 4, M, d)[rows].double()
    H = ws_floats(ws, read_ws_offsets(B, N, d)["H"], M, d)[rows].double()
    Wx, Wm = W["Wx"].double(), W["Wm"].double()
    kbr = kb[rows].double()
    PY = P * y[rows].double()
    worst = 0.0
    for got, want, scale in ((P, kbr @ Wx + W["bx"].double(), kbr.abs() @ Wx.abs() + W["bx"].double().abs()),
                             (Q, P @ Wm[d:] + W["bm"].double(), P.abs() @ Wm[d:].abs() + W["bm"].double().abs()),
                             (H, elu(PY @ Wm[:d] + Q), PY.abs() @ Wm[:d].abs() + Q.abs())):
        worst = max(worst, float(((got - want).abs() / scale).max()))
    print("read forward at B=%d: bf16 step logits use %.3f of their bound; fp32 P, Q, H %.2e (bound %.1e)"
          % (B, r, worst, TOL_READ))
    assert worst <= TOL_READ, worst
