"""The backward kernels (csrc/backward.cu) against fp64 references of their OWN operation, called through the C ABI.

Each reference is computed on exactly the operands the kernel sees (for the read unit: the forward's own saved P, H, I1, y
and attention), so forward rounding does not enter.  Every reference is evaluated a second time on absolute values --
each operand replaced by |.|, each ELU' or softmax factor by its absolute value, the softmax backward in the kernel's
cancellation-free form ka[n] * sum_m ka[m] * |dka[n] - dka[m]| -- and the bound is element-wise:

    |got - ref| <= tol * absref + tiny

A gradient that is large only through cancellation gets a large absref and passes; a dropped split-K slice, tile, row
block or batch row does not (tests/test_backward_bounds.py shows that on the CPU with this file's reference code).

Every case also checks the header's contracts: "+=" outputs are prefilled with random values and only the increment may
change them; "=" outputs are NaN-filled, so an unwritten element fails; two runs from the same state are bit-identical
(the reductions have a fixed order); the split-K counters (the first 4 096 bytes of a workspace) are zero afterwards.

Each `tol` is a few times the worst value measured on an H100 80GB HBM3 (SXM, 132 SMs) at a 400 W power limit, written
beside it.  The ratios are a property of the arithmetic, not of the clock: with fixed seeds and fixed-order reductions
every run gives the same bits.  The absolute-value chain through three or four products is loose by ~sqrt(K) per
product, so the measured ratios of the deep gradients (dy, dby, dmem_in) are small; their tols are set from measurement,
which keeps them as sharp as the shallow ones."""
import ctypes
import math

import numpy as np
import pytest
import torch

from mac_network_b200 import _lib as L_
from tests.test_gpu_wgmma import excess, keep_mask

pytestmark = pytest.mark.gpu

MAC_OK, ERR_INVALID, ERR_UNSUPPORTED = 0, -1, -3
SITE_READ_KB, SITE_READ_MEM, SITE_READ_INTER = L_.SITE_READ_KB, L_.SITE_READ_MEM, L_.SITE_READ_INTER
COUNTER_BYTES = 4096

# ---- bounds (fraction of absref); measured worst value on the H100 beside each
# mac_read_bwd, per output (fp32 throughout)                                  measured
TOL_READ = {"dkb": 5e-7,                                                      # 1.2e-7
            "dmem_in": 1e-8,                                                  # 1.0e-9
            "dcontrol": 4e-6,                                                 # 9.2e-7
            "dWx": 2e-7, "dbx_part": 2e-7,                                    # 4.6e-8, 5.8e-8
            "dWy": 2e-7, "dby": 2e-7,                                         # 5.1e-8, 3.9e-8
            "dWm": 2e-7, "dbm_part": 3e-7,                                    # 4.7e-8, 7.2e-8
            "dWm2": 2e-7, "dbm2_part": 2e-6,                                  # 5.9e-8, 4.9e-7
            "dwr_part": 3e-6, "dbr_part": 3e-8}                               # 7.0e-7, 6.2e-9
# mac_read_bwd_tc, per output: bf16 operands in the six [B*N, .] products; the logits backward stays fp32
TOL_READ_TC = {"dkb": 1.2e-5,                                                 # 3.1e-6
               "dmem_in": 5e-6,                                               # 1.3e-6
               "dcontrol": 3e-7,                                              # 5.6e-8
               "dWx": 2.5e-5, "dbx_part": 1.5e-5,                             # 6.4e-6, 3.7e-6
               "dWy": 3e-5, "dby": 1.2e-5,                                    # 7.5e-6, 3.0e-6
               "dWm": 5e-4, "dbm_part": 1.5e-4,                               # 1.2e-4, 3.4e-5
               "dWm2": 8e-4, "dbm2_part": 3e-7,                               # 2.1e-4, 5.8e-8
               "dwr_part": 3e-7, "dbr_part": 3e-8}                            # 5.7e-8, 6.2e-9
TOL_LINEAR = 1.5e-6      # mac_linear_bwd dx, dW, db                                            measured 4.1e-7
TOL_KB = 1.2e-6          # mac_kb_attend_bwd dka, dkl, dkb, dbr                                 measured 3.0e-7
TOL_CTRL = 6e-7          # mac_control_attend_bwd                                               measured 1.7e-7
TOL_ROWDOT = 4e-7        # mac_rowdot_bwd                                                       measured 8.4e-8
TOL_BCAST = 4e-7         # mac_bcast_op_bwd                                                     measured 1.1e-7
TOL_BN = 3e-6            # mac_batchnorm_fwd / _bwd                                             measured 7.7e-7
TOL_COLSUM = 3e-7        # mac_colsum                                                           measured 7.6e-8
TOL_ELEM = 6e-7          # mac_gate_bwd, mac_activation_bwd, mac_axpy (a few fp32 roundings)    measured 2.0e-7


# ------------------------------------------------------------------------------------------------ helpers
def gen(seed, device="cuda"):
    return torch.Generator(device=device).manual_seed(seed)


def randn(g, *shape, scale=1.0):
    return (torch.randn(*shape, device=g.device, generator=g) * scale).contiguous()


def ratio(got, ref, absref, tiny=0.0):
    """the worst (|got - ref| - tiny) / absref over the elements; inf when the kernel left a non-finite value"""
    if not bool(torch.isfinite(got).all()):
        return float("inf")
    return excess(got, ref, absref, tiny=tiny)


class Report:
    """Collects the ratio of every output of one case, prints them all, then asserts: one GPU run shows every margin."""

    def __init__(self, name):
        self.name, self.rows = name, []

    def add(self, what, got, ref, absref, tol, tiny=0.0):
        self.rows.append((what, ratio(got, ref, absref, tiny), tol))

    def add_inc(self, what, got, pre, inc, absinc, tol):
        """a "+=" output: got must be pre + inc"""
        pre = pre.double()
        self.add(what, got, pre + inc, absinc + pre.abs(), tol)

    def check(self, cond, what):
        self.rows.append((what, 0.0 if cond else float("inf"), 0.0))

    def done(self):
        print("%s: %s" % (self.name, ", ".join("%s %.2e" % (w, e) for w, e, _ in self.rows)))
        bad = [(w, e, t) for w, e, t in self.rows if not e <= t]
        assert not bad, (self.name, bad)


def prefill(g, absref):
    """random start values for a "+=" output, of the size of its increment"""
    return randn(g, *absref.shape, scale=float(absref.mean()) + 1e-3).float()


def same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def ptrs(ts, T=ctypes.c_void_p):
    return (T * len(ts))(*[(t.data_ptr() if t is not None else None) for t in ts])


def ints(v):
    return (ctypes.c_int * len(v))(*v)


def lib():
    return L_.load()


def run_twice(call, outs):
    """call() twice from the same starting values of `outs` (dict name -> tensor); returns the first run's results and
    whether the second run reproduced them bit for bit"""
    start = {k: v.clone() for k, v in outs.items() if v is not None}
    call()
    first = {k: v.clone() for k, v in outs.items() if v is not None}
    for k, v in start.items():
        outs[k].copy_(v)
    call()
    torch.cuda.synchronize()
    same = all(same_bits(first[k], outs[k]) for k in first)
    return first, same


# ================================================================================================ 1. read unit
def read_masks(keep, seed, step, B, N, d, device):
    """the forward's dropout of the knowledge base, of memory_in and of I2, as fp64 multipliers (mask * 1/keep)"""
    M = B * N
    if keep >= 1.0:
        one = lambda *s: torch.ones(*s, dtype=torch.float64, device=device)
        return one(M, d), one(B, d), one(M, d)
    sc = float(np.float32(1.0) / np.float32(keep))
    m = lambda site, shape: keep_mask(seed, site, step, shape, keep, device=device).double() * sc
    return m(SITE_READ_KB, (M, d)), m(SITE_READ_MEM, (B, d)), m(SITE_READ_INTER, (M, d))


def softmax_bwd_reference(a, dka, adka):
    """dkl[n] = ka[n] * sum_m ka[m] * (dka[n] - dka[m]) and its bound: |dka[n] - dka[m]| for the rounding of the kernel's
    form, plus adka[n] + adka[m] for the error of dka itself (the m = n term is exactly zero in the kernel's form)"""
    N = a.shape[1]
    dkl = a * (dka - (a * dka).sum(1, keepdim=True))
    diff = (dka[:, :, None] - dka[:, None, :]).abs()
    pair = (adka[:, :, None] + adka[:, None, :]).masked_fill(torch.eye(N, dtype=torch.bool, device=a.device), 0.0)
    adkl = a * (a[:, None, :] * (diff + pair)).sum(2)
    # dbr: sum_n ka[n] * (dka[n] - sum_m ka[m] dka[m]), the kernel's direct form (zero up to rounding)
    adot = (a * adka).sum(1, keepdim=True)
    return dkl, adkl, dkl.sum(1), (a * (adka + adot)).sum(1)


def read_bwd_reference(kb, mem, c, W, att, P, H, I1, y, dinfo, keep, seed, step):
    """fp64 gradients of the read unit (mac_b200.h) from the forward's saved P, H, I1, y and att, and their absolute-value
    counterparts: name -> (ref, absref).  Per-sample partials ([B, d] / [B]) as the kernel leaves them."""
    B, N, d = kb.shape
    M = B * N
    dev = kb.device
    D = lambda t: t.double()
    mkb, mmem, mint = read_masks(keep, seed, step, B, N, d, dev)
    kbv, di, a = D(kb).view(M, d), D(dinfo), D(att)
    P, H, I1, y = D(P), D(H), D(I1), D(y)
    Wx, Wy, Wm, Wm2, wr = D(W["Wx"]), D(W["Wy"]), D(W["Wm"]), D(W["Wm2"]), D(W["wr"])
    cb, yb = D(c).repeat_interleave(N, 0), y.repeat_interleave(N, 0)
    bsum = lambda t: t.view(B, N, -1).sum(1)
    r = {}
    # (1) softmax over the knowledge base and info = sum_n att * KB
    dka = torch.einsum("bnd,bd->bn", kbv.view(B, N, d), di)
    adka = torch.einsum("bnd,bd->bn", kbv.view(B, N, d).abs(), di.abs())
    dkl, adkl, dbr, adbr = softmax_bwd_reference(a, dka, adka)
    r["dbr_part"] = (dbr, adbr)
    # (2) logits: T = I1*c, I2 = ELU(T), kl = dropout(I2) . wr + br
    t = I1 * cb
    i2 = torch.where(t > 0, t, torch.expm1(t))
    e_t = torch.where(t > 0, torch.ones_like(t), torch.exp(t))          # ELU'(T) > 0
    g, ag = dkl.reshape(M, 1), adkl.reshape(M, 1)
    dT, adT = g * wr * mint * e_t, ag * wr.abs() * mint * e_t
    dI1, adI1 = dT * cb, adT * cb.abs()
    r["dcontrol"] = (bsum(dT * I1), bsum(adT * I1.abs()))
    r["dwr_part"] = (bsum(g * i2 * mint), bsum(ag * i2.abs() * mint))
    r["dbm2_part"] = (bsum(dI1), bsum(adI1))
    # (3) I1 = H @ Wm2 + bm2, H = ELU(Z): ELU'(Z) through the saved output, H > 0 ? 1 : H + 1
    r["dWm2"] = (H.t() @ dI1, H.abs().t() @ adI1)
    eH = torch.where(H > 0, torch.ones_like(H), H + 1).abs()
    dZ, adZ = (dI1 @ Wm2.t()) * eH, (adI1 @ Wm2.abs().t()) * eH
    r["dbm_part"] = (bsum(dZ), bsum(adZ))
    # (4) Z = [P*y, P] @ Wm + bm
    I0 = torch.cat([P * yb, P], 1)
    r["dWm"] = (I0.t() @ dZ, I0.abs().t() @ adZ)
    dI0, adI0 = dZ @ Wm.t(), adZ @ Wm.abs().t()
    # (5) dP, dy, dbx
    dP = dI0[:, :d] * yb + dI0[:, d:]
    adP = adI0[:, :d] * yb.abs() + adI0[:, d:]
    dy, ady = bsum(dI0[:, :d] * P), bsum(adI0[:, :d] * P.abs())
    r["dbx_part"] = (bsum(dP), bsum(adP))
    # (6) P = dropout(KB) @ Wx + bx;  dKB also gets att (x) dinfo from (1)
    kbd = kbv * mkb
    r["dWx"] = (kbd.t() @ dP, kbd.abs().t() @ adP)
    r["dkb"] = (((dP @ Wx.t()) * mkb).view(B, N, d) + a[:, :, None] * di[:, None, :],
                ((adP @ Wx.abs().t()) * mkb).view(B, N, d) + a[:, :, None] * di.abs()[:, None, :])
    # (7) y = dropout(memory_in) @ Wy + by
    md = D(mem) * mmem
    r["dWy"] = (md.t() @ dy, md.abs().t() @ ady)
    r["dby"] = (dy.sum(0), ady.sum(0))
    r["dmem_in"] = ((dy @ Wy.t()) * mmem, (ady @ Wy.abs().t()) * mmem)
    r["_I0"], r["_dZ"], r["_dy"] = (I0, I0.abs()), (dZ, adZ), (dy, ady)         # intermediates, for the CPU bound checks
    return r


READ_GRADS = ["dkb", "dmem_in", "dcontrol", "dWx", "dbx_part", "dWy", "dby", "dWm", "dbm_part", "dWm2", "dbm2_part",
              "dwr_part", "dbr_part"]


def read_case(B, N, d, keep, seed):
    """weights, inputs and the fp32 forward with `save`: what both backward entry points start from"""
    lb = lib()
    g = gen(seed)
    W = {"Wx": randn(g, d, d, scale=d ** -0.5), "bx": randn(g, d, scale=0.1), "Wy": randn(g, d, d, scale=d ** -0.5),
         "by": randn(g, d, scale=0.1), "Wm": randn(g, 2 * d, d, scale=(2 * d) ** -0.5), "bm": randn(g, d, scale=0.1),
         "Wm2": randn(g, d, d, scale=d ** -0.5), "bm2": randn(g, d, scale=0.1), "wr": randn(g, d, scale=4 * d ** -0.5)}
    v = lambda t: t.data_ptr()
    rw = L_.ReadWeights(v(W["Wx"]), v(W["bx"]), v(W["Wy"]), v(W["by"]), v(W["Wm"]), v(W["bm"]), v(W["Wm2"]), v(W["bm2"]),
                        v(W["wr"]), 0.25, None, None, None, None, None, None, None)
    kb = torch.nn.functional.elu(randn(g, B, N, d))
    mem, c = randn(g, B, d), randn(g, B, d)
    step = 3
    M = B * N
    wsb = lb.mac_read_workspace_bytes(B, N, d, 0)
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    save = torch.full((3 * M * d + B * d,), float("nan"), device="cuda")
    info, att = torch.empty(B, d, device="cuda"), torch.empty(B, N, device="cuda")
    L_.check(lb.mac_read_fwd(L_.ptr(kb), None, L_.ptr(mem), L_.ptr(c), ctypes.byref(rw), keep, seed, step, 0, L_.ptr(info),
                             L_.ptr(att), L_.ptr(save), L_.ptr(ws), wsb, B, N, d, L_.stream_ptr()), "mac_read_fwd")
    torch.cuda.synchronize()
    P, H, I1 = (save[i * M * d:(i + 1) * M * d].view(M, d) for i in range(3))
    y = save[3 * M * d:].view(B, d)
    dinfo = randn(g, B, d)
    ref = read_bwd_reference(kb, mem, c, W, att, P, H, I1, y, dinfo, keep, seed, step)
    return g, W, rw, kb, mem, c, att, save, dinfo, step, ref


def run_read_bwd(tc, B, N, d, keep, seed, with_dkb=True):
    lb = lib()
    g, W, rw, kb, mem, c, att, save, dinfo, step, ref = read_case(B, N, d, keep, seed)
    outs = {}
    for k in READ_GRADS:
        if k == "dmem_in":
            outs[k] = torch.full((B, d), float("nan"), device="cuda")
        elif k == "dkb" and not with_dkb:
            outs[k] = None
        else:
            outs[k] = prefill(g, ref[k][1])
    pre = {k: v.clone() for k, v in outs.items() if v is not None}
    wsb = (lb.mac_read_bwd_tc_workspace_bytes if tc else lb.mac_read_bwd_workspace_bytes)(B, N, d)
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    Wt = {k: W[k].t().contiguous() for k in ("Wx", "Wy", "Wm", "Wm2")}
    o = [L_.ptr(outs[k]) for k in READ_GRADS]

    def call():
        if tc:
            st = lb.mac_read_bwd_tc(L_.ptr(kb), L_.ptr(mem), L_.ptr(c), ctypes.byref(rw), L_.ptr(Wt["Wy"]), L_.ptr(att),
                                    L_.ptr(save), L_.ptr(dinfo), keep, seed, step, *o, L_.ptr(ws), wsb, B, N, d,
                                    L_.stream_ptr())
        else:
            st = lb.mac_read_bwd(L_.ptr(kb), L_.ptr(mem), L_.ptr(c), ctypes.byref(rw), L_.ptr(Wt["Wx"]), L_.ptr(Wt["Wy"]),
                                 L_.ptr(Wt["Wm"]), L_.ptr(Wt["Wm2"]), L_.ptr(att), L_.ptr(save), L_.ptr(dinfo), keep, seed,
                                 step, *o, L_.ptr(ws), wsb, B, N, d, L_.stream_ptr())
        L_.check(st, "mac_read_bwd_tc" if tc else "mac_read_bwd")

    got, same = run_twice(call, outs)
    rep = Report("%s %s keep %.2f%s" % ("mac_read_bwd_tc" if tc else "mac_read_bwd", (B, N, d), keep,
                                        "" if with_dkb else " dkb NULL"))
    tols = TOL_READ_TC if tc else TOL_READ
    for k in READ_GRADS:
        if k not in got:
            continue
        r, a = ref[k]
        if k == "dmem_in":
            rep.add(k, got[k], r, a, tols[k])
        else:
            rep.add_inc(k, got[k], pre[k].view(r.shape), r, a, tols[k])
    rep.check(same, "bit-identical rerun")
    rep.check(not bool(ws[:COUNTER_BYTES].any()), "split-K counters zero")
    rep.done()


# (B, N, d, keep): the training shape; N = 1 and 3 at B = 64, where a split-K projY weight gradient would write its partials
# over dy (at N = 1 the softmax passes no gradient to the logits, so dy is zero: only N = 3 shows a corrupted dy); B = 65,
# where the projY dx product leaves the M <= 64 skinny kernel; d not a multiple of 128 (a partial last column block); one
# sample
READ_CASES = [
    (64, 196, 512, 0.85),
    (64, 1, 512, 1.0),
    (64, 3, 512, 0.85),
    (65, 2, 512, 1.0),
    (3, 49, 64, 0.85),
    (5, 33, 192, 1.0),
    (1, 1, 64, 0.85),
]


@pytest.mark.parametrize("B,N,d,keep", READ_CASES)
def test_read_bwd_matches_fp64(B, N, d, keep):
    run_read_bwd(False, B, N, d, keep, seed=B * 1000 + N * 10 + d)


def test_read_bwd_without_dkb():
    run_read_bwd(False, 64, 3, 512, 0.85, seed=17, with_dkb=False)


@pytest.mark.parametrize("B,N,d,keep", [(64, 196, 512, 0.85), (4, 16, 128, 0.85), (2, 32, 256, 1.0)])
def test_read_bwd_tc_matches_fp64(B, N, d, keep):
    """bf16 operands on the six [B*N, .] products: each rounding moves a product by at most 2^-8 of its absolute value,
    and the deepest gradient (dKB) passes through three of them after the fp32 logits backward."""
    run_read_bwd(True, B, N, d, keep, seed=B * 1000 + N * 10 + d + 1)


def test_read_bwd_tc_refuses_unsupported_shapes():
    lb = lib()
    t = torch.zeros(1 << 20, device="cuda")
    rw = L_.ReadWeights(*([t.data_ptr()] * 9), 0.0, *([None] * 7))
    p = L_.ptr(t)
    for B, N, d in ((1, 64, 192), (5, 13, 128)):
        st = lb.mac_read_bwd_tc(p, p, p, ctypes.byref(rw), p, p, p, p, 1.0, 0, 0, *([p] * 13), p,
                                lb.mac_read_bwd_tc_workspace_bytes(B, N, d), B, N, d, L_.stream_ptr())
        assert st == ERR_UNSUPPORTED, (B, N, d, st)
    torch.cuda.synchronize()


# ================================================================================================ 2. mac_linear_bwd
def linear_bwd_reference(xs, Wt, dy):
    """dx_s = dy @ W_s^T, dW = concat(x)^T @ dy, db = colsum(dy), with their absolute-value counterparts"""
    X = torch.cat([x.double() for x in xs], 1)
    Wd, dyd = Wt.double(), dy.double()
    dx, koff = [], 0
    for x in xs:
        k = x.shape[1]
        dx.append((dyd @ Wd[:, koff:koff + k], dyd.abs() @ Wd[:, koff:koff + k].abs()))
        koff += k
    return dx, (X.t() @ dyd, X.abs().t() @ dyd.abs()), (dyd.sum(0), dyd.abs().sum(0))


def strided(g, M, k, pad):
    """[M, k] view of a [M, k + pad] tensor (leading dimension > k when pad > 0)"""
    return randn(g, M, k + pad)[:, :k] if pad else randn(g, M, k)


def base(t):
    """the whole [M, ld] buffer behind a strided() view"""
    return t.as_strided((t.shape[0], t.stride(0)), (t.stride(0), 1))


# (M, segments, n_out, per-segment (ldx pad, ld_dx pad, has dx, accumulate), ldy pad, dW, db, workspace)
# workspace: "full", "fit1" / "fit2" (room for exactly 1 / 2 split-K slices of the widest weight gradient), None
LINEAR_CASES = [
    (1, (64,), 32, [(0, 0, True, 0)], 0, True, True, "full"),
    (64, (512, 16), 512, [(4, 0, True, 1), (0, 4, True, 0)], 0, True, True, "full"),
    (65, (128, 64, 16, 32), 96, [(0, 0, True, 0), (8, 8, False, 0), (0, 0, True, 1), (0, 4, True, 1)], 0, True, True,
     "full"),
    (700, (512, 512), 512, [(0, 0, True, 0), (0, 0, True, 1)], 0, True, True, "full"),
    (700, (256, 16), 128, [(4, 4, True, 1), (0, 0, True, 0)], 8, True, False, "fit2"),
    (12544, (512,), 512, [(0, 0, True, 0)], 0, True, True, "full"),
    (12544, (1024, 16), 512, [(0, 0, False, 0), (0, 0, True, 1)], 0, True, True, "fit1"),
    (12544, (512, 512), 256, [(0, 0, True, 1), (0, 0, True, 0)], 0, True, True, None),
    (64, (512,), 512, [(0, 0, True, 0)], 0, False, False, "full"),
    (4096, (64, 64, 64), 64, [(0, 0, True, 0), (0, 0, False, 0), (0, 0, True, 0)], 0, False, True, "fit2"),
]


@pytest.mark.parametrize("M,segs,n_out,seg_opts,ldy_pad,with_dW,with_db,wsmode", LINEAR_CASES)
def test_linear_bwd_matches_fp64(M, segs, n_out, seg_opts, ldy_pad, with_dW, with_db, wsmode):
    """skinny (M <= 64) vs FMA-pipe sgemm, split vs unsplit and 64- vs 128-wide tiles for the dx products; the weight
    gradients K = M with every split-K factor the workspace allows (fit = 1, 2, the full 32, or no workspace)"""
    lb = lib()
    g = gen(M * 31 + n_out + len(segs))
    xs = [strided(g, M, k, o[0]) for k, o in zip(segs, seg_opts)]
    K = sum(segs)
    Wt = randn(g, n_out, K, scale=K ** -0.5)
    dy = strided(g, M, n_out, ldy_pad)
    dx_ref, dW_ref, db_ref = linear_bwd_reference(xs, Wt, dy)
    dxs = [strided(g, M, k, o[1]) if o[2] else None for k, o in zip(segs, seg_opts)]
    for dx, o in zip(dxs, seg_opts):
        if dx is not None and not o[3]:
            dx.fill_(float("nan"))
    dW = prefill(g, dW_ref[1]) if with_dW else None
    db = prefill(g, db_ref[1]) if with_db else None
    kmax = max(segs)
    if wsmode is None:
        ws, wsb = None, 0
    elif wsmode == "full":      # 32 slices of the widest weight gradient, and of the dx products where they split
        wsb = COUNTER_BYTES + 32 * kmax * (n_out + (M if M <= 4096 else 0)) * 4
        ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    else:                       # room for exactly 1 or 2 slices of the widest weight gradient
        wsb = COUNTER_BYTES + {"fit1": 1, "fit2": 2}[wsmode] * kmax * n_out * 4 + 64
        ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    # whole buffers (with their ld_dx padding) are compared, so padding written by the kernel fails too
    outs = {"dW": dW, "db": db}
    outs.update({"dx%d" % i: base(dx) for i, dx in enumerate(dxs) if dx is not None})
    pre = {k: v.clone() for k, v in outs.items() if v is not None}

    def call():
        st = lb.mac_linear_bwd(ptrs(xs), ints(list(segs)), ints([x.stride(0) for x in xs]), len(segs), L_.ptr(Wt),
                               L_.ptr(dy), dy.stride(0), ptrs(dxs), ints([dx.stride(0) if dx is not None else 0 for dx in dxs]),
                               ints([o[3] for o in seg_opts]), L_.ptr(dW), L_.ptr(db), M, n_out, L_.ptr(ws), wsb,
                               L_.stream_ptr())
        L_.check(st, "mac_linear_bwd")

    got, same = run_twice(call, outs)
    rep = Report("mac_linear_bwd M=%d segs=%s n_out=%d ws=%s" % (M, segs, n_out, wsmode))
    for i, (dx, o) in enumerate(zip(dxs, seg_opts)):
        if dx is None:
            continue
        k = dx.shape[1]
        r, a = dx_ref[i]
        p = pre["dx%d" % i].double()
        ref, ab = p.clone(), p.abs()
        if o[3]:
            ref[:, :k] += r
            ab[:, :k] += a
        else:
            ref[:, :k], ab[:, :k] = r, a
        rep.add("dx%d" % i, got["dx%d" % i], ref, ab, TOL_LINEAR)
    if with_dW:
        rep.add_inc("dW", got["dW"], pre["dW"], *dW_ref, TOL_LINEAR)
    if with_db:
        rep.add_inc("db", got["db"], pre["db"], *db_ref, TOL_LINEAR)
    rep.check(same, "bit-identical rerun")
    if ws is not None:
        rep.check(not bool(ws[:COUNTER_BYTES].any()), "split-K counters zero")
    rep.done()


def test_linear_bwd_db_needs_dense_dy():
    lb = lib()
    g = gen(3)
    M, k, n_out = 8, 64, 64
    x = randn(g, M, k)
    dy = randn(g, M, n_out + 4)[:, :n_out]
    Wt = randn(g, n_out, k)
    db = torch.zeros(n_out, device="cuda")
    st = lb.mac_linear_bwd(ptrs([x]), ints([k]), ints([k]), 1, L_.ptr(Wt), L_.ptr(dy), dy.stride(0), None, None, None, None,
                           L_.ptr(db), M, n_out, None, 0, L_.stream_ptr())
    torch.cuda.synchronize()
    assert st == ERR_UNSUPPORTED


# ================================================================================================ 3. mac_kb_attend_bwd
def peaked_softmax(g, B, N):
    """softmax rows with one cell above 1 - 1e-6 (fp32), the rest ~1e-9 each"""
    logits = randn(g, B, N).double()
    idx = torch.randint(0, N, (B,), device=g.device, generator=g)
    logits[torch.arange(B, device=g.device), idx] += 20.0 + math.log(N)
    return torch.softmax(logits, 1).float()


@pytest.mark.parametrize("N", [1, 31, 32, 33, 196, 257, 1500])
@pytest.mark.parametrize("d,peaked", [(4, False), (64, True), (512, False)])
def test_kb_attend_bwd_matches_fp64(N, d, peaked):
    """dka = KB . dinfo (read back from the scratch), the softmax backward from the kernel's own dka -- in the
    cancellation-free form the bound is tight even where one cell holds all the attention -- dKB += att (x) dinfo, and
    dbr_part += sum_n dkl"""
    lb = lib()
    B = 3
    g = gen(N * 10 + d + peaked)
    kb = randn(g, B, N, d)
    att = peaked_softmax(g, B, N) if peaked else torch.softmax(randn(g, B, N), 1)
    if peaked and N > 1:
        assert float(att.max(1).values.min()) > 1 - 1e-6
    dinfo = randn(g, B, d)
    a, di = att.double(), dinfo.double()
    dka_ref = torch.einsum("bnd,bd->bn", kb.double(), di)
    adka = torch.einsum("bnd,bd->bn", kb.double().abs(), di.abs())
    dkb_ref, adkb = a[:, :, None] * di[:, None, :], a[:, :, None] * di.abs()[:, None, :]
    dka = torch.full((B, N), float("nan"), device="cuda")
    dkl = torch.full((B, N), float("nan"), device="cuda")
    dkb = prefill(g, adkb)
    dbr = randn(g, B)
    pre_dkb, pre_dbr = dkb.clone(), dbr.clone()
    outs = {"dka": dka, "dkl": dkl, "dkb": dkb, "dbr": dbr}

    def call():
        L_.check(lb.mac_kb_attend_bwd(L_.ptr(kb), L_.ptr(att), L_.ptr(dinfo), L_.ptr(dka), L_.ptr(dkl), L_.ptr(dkb),
                                      L_.ptr(dbr), B, N, d, L_.stream_ptr()), "mac_kb_attend_bwd")

    got, same = run_twice(call, outs)
    rep = Report("mac_kb_attend_bwd N=%d d=%d%s" % (N, d, " peaked" if peaked else ""))
    rep.add("dka", got["dka"], dka_ref, adka, TOL_KB)
    # the softmax backward on exactly the dka the kernel used: only the rounding of its own form is left
    k = got["dka"].double()
    dkl_ref = a * (a[:, None, :] * (k[:, :, None] - k[:, None, :])).sum(2)
    adkl = a * (a[:, None, :] * (k[:, :, None] - k[:, None, :]).abs()).sum(2)
    rep.add("dkl", got["dkl"], dkl_ref, adkl, TOL_KB)
    _, _, dbr_ref, adbr = softmax_bwd_reference(a, k, k.abs())
    rep.add_inc("dbr", got["dbr"], pre_dbr, dbr_ref, adbr, TOL_KB)
    rep.add_inc("dkb", got["dkb"], pre_dkb, dkb_ref, adkb, TOL_KB)
    rep.check(same, "bit-identical rerun")
    rep.done()
    # without dkb and dbr_part: dkl alone, the same bits
    dkl2 = torch.full((B, N), float("nan"), device="cuda")
    L_.check(lb.mac_kb_attend_bwd(L_.ptr(kb), L_.ptr(att), L_.ptr(dinfo), L_.ptr(dka), L_.ptr(dkl2), None, None, B, N, d,
                                  L_.stream_ptr()))
    torch.cuda.synchronize()
    assert same_bits(dkl2, got["dkl"])


# ================================================================================================ 4. mac_control_attend_bwd
def control_bwd_reference(cc, inw, outw, w, att, gout, dq_pre, dq_acc):
    """views: cc [T, B, d], inw / outw [B, S, d], att [T, B, S], gout [T, B, d] -> increments of d_in, d_out, dw_part,
    db_part and the values of dq [T, B, d], each with its absolute-value counterpart"""
    T = cc.shape[0]
    D = lambda t: t.double()
    inw, outw, w = D(inw), D(outw), D(w)
    r = {k: [0.0, 0.0] for k in ("din", "dout", "dw", "db")}
    dq = []
    for t in range(T):
        q, g, a = D(cc[t]), D(gout[t]), D(att[t])
        datt = torch.einsum("bsd,bd->bs", outw, g)
        adatt = torch.einsum("bsd,bd->bs", outw.abs(), g.abs())
        dot = (a * datt).sum(1, keepdim=True)
        adot = (a * adatt).sum(1, keepdim=True)
        dl, adl = a * (datt - dot), a * (adatt + adot)
        sx = torch.einsum("bs,bsd->bd", dl, inw)
        asx = torch.einsum("bs,bsd->bd", adl, inw.abs())
        for k, v, av in (("dout", a[:, :, None] * g[:, None, :], a[:, :, None] * g.abs()[:, None, :]),
                         ("din", dl[:, :, None] * (q * w)[:, None, :], adl[:, :, None] * (q * w).abs()[:, None, :]),
                         ("dw", q * sx, q.abs() * asx), ("db", dl.sum(1), adl.sum(1))):
            r[k][0] = r[k][0] + v
            r[k][1] = r[k][1] + av
        base = D(dq_pre[t]) if dq_acc else 0.0
        dq.append((base + w * sx, (D(dq_pre[t]).abs() if dq_acc else 0.0) + w.abs() * asx))
    return r, dq


# (layout, B, S, d, nsteps, masked, dq_accumulate)
#   "control": the control unit (cc [B, T*d] per step, words [B, S, d], d_in_words == d_out_words)
#   "alias":   in_words == out_words and d_in_words == d_out_words
#   "history": the write unit's self-attention over the step-major memory / control history (rstride = B*d)
CTRL_CASES = [
    ("control", 3, 1, 64, 1, False, 0),
    ("control", 4, 40, 100, 4, True, 1),
    ("control", 2, 300, 20, 2, True, 1),
    ("alias", 3, 40, 300, 1, False, 0),
    ("alias", 5, 33, 512, 3, True, 1),
    ("history", 4, 5, 512, 1, False, 0),
    ("history", 3, 12, 36, 1, True, 1),
]


@pytest.mark.parametrize("layout,B,S,d,T,masked,dq_acc", CTRL_CASES)
def test_control_attend_bwd_matches_fp64(layout, B, S, d, T, masked, dq_acc):
    lb = lib()
    g = gen(B * 100 + S * 7 + d + T)
    w = randn(g, d)
    logits = randn(g, T, B, S)
    lens = torch.randint(1, S + 1, (B,), device="cuda", generator=g) if masked else torch.full((B,), S, device="cuda")
    keep = torch.arange(S, device="cuda")[None, :] < lens[:, None]
    att = torch.softmax(logits.masked_fill(~keep[None], float("-inf")), 2).contiguous()
    gout = randn(g, T, B, d)
    if layout == "history":
        Sh = S + 2                                          # slots behind the attended ones are not read or written
        hc, hm = randn(g, Sh, B, d), randn(g, Sh, B, d)
        inw_buf, outw_buf = hc, hm
        in_b, in_r, out_b, out_r = d, B * d, d, B * d
        din_buf, dout_buf = randn(g, Sh, B, d), randn(g, Sh, B, d)
    else:
        in_b, in_r, out_b, out_r = S * d, d, S * d, d
        inw_buf = randn(g, B, S, d)
        outw_buf = inw_buf if layout == "alias" else randn(g, B, S, d)
        din_buf = randn(g, B, S, d)
        dout_buf = din_buf
    cc_buf = randn(g, B, T * d)                             # [B, T*d]: tstride d, bstride T*d
    dq_buf = randn(g, B, T * d) if dq_acc else torch.full((B, T * d), float("nan"), device="cuda")
    view = lambda t, bs, rs: t.as_strided((B, S, d), (bs, rs, 1))
    tview = lambda t: t.as_strided((T, B, d), (d, T * d, 1))
    inw, outw = view(inw_buf, in_b, in_r), view(outw_buf, out_b, out_r)
    r, dq_ref = control_bwd_reference(tview(cc_buf), inw, outw, w, att, gout, tview(dq_buf), dq_acc)
    dw, db = randn(g, B, d), randn(g, B)
    pre = {"din": din_buf.clone(), "dout": dout_buf.clone(), "dq": dq_buf.clone(), "dw": dw.clone(), "db": db.clone()}
    outs = {"din": din_buf, "dout": dout_buf, "dq": dq_buf, "dw": dw, "db": db}

    def call():
        L_.check(lb.mac_control_attend_bwd(L_.ptr(cc_buf), d, T * d, L_.ptr(inw_buf), in_b, in_r, L_.ptr(outw_buf), out_b,
                                           out_r, L_.ptr(w), L_.ptr(att), L_.ptr(gout), B * d, d, L_.ptr(din_buf),
                                           L_.ptr(dout_buf), L_.ptr(dq_buf), d, T * d, dq_acc, L_.ptr(dw), L_.ptr(db), T, B,
                                           S, d, L_.stream_ptr()), "mac_control_attend_bwd")

    got, same = run_twice(call, outs)
    rep = Report("mac_control_attend_bwd %s B=%d S=%d d=%d T=%d%s acc=%d" % (layout, B, S, d, T, " masked" if masked else "",
                                                                          dq_acc))
    # word gradients: compare the whole buffers (slots outside the view must keep their start values)
    def expect(buf_pre, bs, rs, parts):
        ref, ab = buf_pre.double().clone(), buf_pre.double().abs()
        for k in parts:
            ref.as_strided((B, S, d), (bs, rs, 1)).add_(r[k][0])
            ab.as_strided((B, S, d), (bs, rs, 1)).add_(r[k][1])
        return ref, ab
    if din_buf is dout_buf:
        rep.add("d_words", got["din"], *expect(pre["din"], in_b, in_r, ("din", "dout")), TOL_CTRL)
    else:
        rep.add("d_in", got["din"], *expect(pre["din"], in_b, in_r, ("din",)), TOL_CTRL)
        rep.add("d_out", got["dout"], *expect(pre["dout"], out_b, out_r, ("dout",)), TOL_CTRL)
    dq_got = tview(got["dq"])
    for t in range(T):
        rep.add("dq[%d]" % t, dq_got[t], *dq_ref[t], TOL_CTRL)
    rep.add_inc("dw_part", got["dw"], pre["dw"], *r["dw"], TOL_CTRL)
    rep.add_inc("db_part", got["db"], pre["db"], *r["db"], TOL_CTRL)
    if masked:          # attention exactly zero: those word rows get exactly +0
        for name in {"din", "dout"}:
            bs, rs = (in_b, in_r) if name == "din" else (out_b, out_r)
            gv, pv = view(got[name], bs, rs), view(pre[name], bs, rs)
            rep.check(same_bits(gv[~keep], pv[~keep]), "%s masked rows unchanged" % name)
    rep.check(same, "bit-identical rerun")
    rep.done()


# ================================================================================================ 5. mac_rowdot_bwd
# (R, segments, (ldx pad, has dx, ld_dx pad) per segment, db)
ROWDOT_CASES = [
    (1, (64, 32, 31), [(4, True, 0), (0, False, 0), (8, True, 4)], True),
    (63, (64, 64), [(0, True, 0), (4, True, 0)], True),
    (64, (64, 32, 32), [(4, True, 4), (8, True, 0), (0, False, 0)], False),
    (65, (127,), [(1, True, 3)], True),
    (12544, (64, 32, 32), [(4, True, 0), (0, False, 0), (8, True, 8)], True),
    (12544, (100, 27), [(0, False, 0), (5, True, 0)], True),
]


@pytest.mark.parametrize("R,segs,seg_opts,with_db", ROWDOT_CASES)
def test_rowdot_bwd_matches_fp64(R, segs, seg_opts, with_db):
    """K_total = 127 / 128 put the bias column at the end of a 128-column block or alone in the next one; R around the
    64-row partial blocks, and R = 12 544 (196 blocks reduced in order)"""
    lb = lib()
    g = gen(R + sum(segs) * 3 + len(segs))
    xs = [strided(g, R, k, o[0]) for k, o in zip(segs, seg_opts)]
    Kt = sum(segs)
    w = randn(g, Kt)
    gr = randn(g, R)
    X = torch.cat([x.double() for x in xs], 1)
    gd = gr.double()
    dw_ref, adw = gd @ X, gd.abs() @ X.abs()
    db_ref, adb = gd.sum().view(1), gd.abs().sum().view(1)
    dxs = [strided(g, R, k, o[2]) if o[1] else None for k, o in zip(segs, seg_opts)]
    dw = prefill(g, adw)
    db = randn(g, 1) if with_db else None
    outs = {"dw": dw, "db": db}
    outs.update({"dx%d" % i: base(dx) for i, dx in enumerate(dxs) if dx is not None})
    pre = {k: v.clone() for k, v in outs.items() if v is not None}
    wsb = lb.mac_rowdot_bwd_workspace_bytes(R, Kt)
    ws = torch.full((wsb // 4,), float("nan"), device="cuda")

    def call():
        L_.check(lb.mac_rowdot_bwd(ptrs(xs), ints(list(segs)), ints([x.stride(0) for x in xs]), len(segs), L_.ptr(w),
                                   L_.ptr(gr), ptrs(dxs), ints([dx.stride(0) if dx is not None else 0 for dx in dxs]),
                                   L_.ptr(dw), L_.ptr(db), L_.ptr(ws), wsb, R, L_.stream_ptr()), "mac_rowdot_bwd")

    got, same = run_twice(call, outs)
    rep = Report("mac_rowdot_bwd R=%d segs=%s" % (R, segs))
    koff = 0
    for i, (k, dx) in enumerate(zip(segs, dxs)):
        if dx is not None:         # whole buffers: the ld_dx padding keeps its start values
            ws_ = w[koff:koff + k].double()
            ref = pre["dx%d" % i].double().clone()
            ab = ref.abs()
            ref[:, :k] += gd[:, None] * ws_[None, :]
            ab[:, :k] += gd.abs()[:, None] * ws_.abs()[None, :]
            rep.add("dx%d" % i, got["dx%d" % i], ref, ab, TOL_ROWDOT)
        koff += k
    rep.add_inc("dw", got["dw"], pre["dw"], dw_ref, adw, TOL_ROWDOT)
    if with_db:
        rep.add_inc("db", got["db"], pre["db"], db_ref, adb, TOL_ROWDOT)
    rep.check(same, "bit-identical rerun")
    rep.done()


# ================================================================================================ 6. mac_bcast_op_bwd
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("N,d", [(7, 20), (33, 130)])
@pytest.mark.parametrize("outs_given", [(True, True, True), (False, True, True), (True, False, False)])
def test_bcast_op_bwd_matches_fp64(mode, N, d, outs_given):
    lb = lib()
    B, mb = 3, 0.5
    g = gen(mode * 100 + N + d + sum(i << k for k, i in enumerate(outs_given)))
    x, v, gr = randn(g, B, N, d), randn(g, B, d), randn(g, B, N, d)
    out = torch.tanh(x + v[:, None, :])
    X, V, G, O = x.double(), v.double()[:, None, :], gr.double(), out.double()
    if mode == 0:
        gx, agx, gv, agv = G * (V + mb), G.abs() * (V.abs() + mb), G * (X + mb), G.abs() * (X.abs() + mb)
    elif mode == 1:
        gx, agx, gv, agv = G * V, G.abs() * V.abs(), G * X, G.abs() * X.abs()
    else:
        gx = gv = G * (1 - O * O)
        agx = agv = G.abs() * (1 + O * O)
    want_dx, want_dv, want_db = outs_given
    dx = randn(g, B, N, d) if want_dx else None
    dv = randn(g, B, d) if want_dv else None
    dbias = randn(g, B, d) if want_db else None
    pre = {k: t.clone() for k, t in (("dx", dx), ("dv", dv), ("dbias", dbias)) if t is not None}
    outs = {"dx": dx, "dv": dv, "dbias": dbias}

    def call():
        L_.check(lb.mac_bcast_op_bwd(L_.ptr(x), L_.ptr(v), L_.ptr(out), L_.ptr(gr), mode, mb, L_.ptr(dx), L_.ptr(dv),
                                     L_.ptr(dbias), B, N, d, L_.stream_ptr()), "mac_bcast_op_bwd")

    got, same = run_twice(call, outs)
    rep = Report("mac_bcast_op_bwd mode %d N=%d d=%d given %s" % (mode, N, d, outs_given))
    if want_dx:
        rep.add_inc("dx", got["dx"], pre["dx"], gx, agx, TOL_BCAST)
    if want_dv:
        rep.add_inc("dv", got["dv"], pre["dv"], gv.sum(1), agv.sum(1), TOL_BCAST)
    if want_db:
        if mode == 1:
            rep.add_inc("dbias", got["dbias"], pre["dbias"], G.sum(1), G.abs().sum(1), TOL_BCAST)
        else:
            rep.check(same_bits(got["dbias"], pre["dbias"]), "dbias untouched outside mode 1")
    rep.check(same, "bit-identical rerun")
    rep.done()


# ================================================================================================ 7. batch normalisation
@pytest.mark.parametrize("B", [1, 2, 64, 300])
@pytest.mark.parametrize("training", [1, 0])
@pytest.mark.parametrize("affine,alias,offset", [(True, False, 0.0), (False, True, 0.0), (True, True, 1000.0)])
def test_batchnorm_matches_fp64(B, training, affine, alias, offset):
    """forward (statistics, the in-place moving-average update with the Bessel factor B / max(B - 1, 1), y) and backward,
    with gamma / beta given or NULL, y aliasing x, and data on a large common offset (two-pass variance)"""
    lb = lib()
    d, decay, eps = 130, 0.99, 1e-3
    g = gen(B * 10 + training + (2 if affine else 0) + int(offset))
    x = (randn(g, B, d) * 2.0 + offset + randn(g, 1, d) * 0.1).contiguous()
    gamma = (randn(g, d) * 0.5 + 1.0) if affine else None
    beta = randn(g, d) if affine else None
    mm0, mv0 = randn(g, d) + offset, randn(g, d).abs() + 0.5
    mm, mv = mm0.clone(), mv0.clone()
    x0 = x.clone()
    y = x if alias else torch.full((B, d), float("nan"), device="cuda")
    smean, sinv = torch.full((d,), float("nan"), device="cuda"), torch.full((d,), float("nan"), device="cuda")
    L_.check(lb.mac_batchnorm_fwd(L_.ptr(x), L_.ptr(gamma), L_.ptr(beta), L_.ptr(mm), L_.ptr(mv), decay, eps, training,
                                  L_.ptr(y), L_.ptr(smean), L_.ptr(sinv), B, d, L_.stream_ptr()), "mac_batchnorm_fwd")
    torch.cuda.synchronize()
    X = x0.double()
    gm = gamma.double() if affine else torch.ones(d, dtype=torch.float64, device="cuda")
    bt = beta.double() if affine else torch.zeros(d, dtype=torch.float64, device="cuda")
    rep = Report("mac_batchnorm B=%d %s%s%s%s" % (B, "training" if training else "eval", "" if affine else " no gamma/beta",
                                                   " y=x" if alias else "", " offset %g" % offset if offset else ""))
    amean = X.abs().mean(0)
    if training:
        mean = X.mean(0)
        var = ((X - mean) ** 2).mean(0)
        unbiased = var * (B / max(B - 1, 1))
        rep.add("save_mean", smean, mean, amean, TOL_BN)
        mmr, mvr = mm0.double() - (mm0.double() - mean) * (1 - decay), mv0.double() - (mv0.double() - unbiased) * (1 - decay)
        rep.add("moving_mean", mm, mmr, mm0.double().abs() + (mm0.double().abs() + amean) * (1 - decay), TOL_BN)
        rep.add("moving_var", mv, mvr, mv0.double().abs() + (mv0.double().abs() + unbiased) * (1 - decay), TOL_BN,
                tiny=1e-12)
    else:
        mean, var = mm0.double(), mv0.double()
        rep.check(same_bits(mm, mm0) and same_bits(mv, mv0), "moving statistics unchanged in eval")
        rep.check(same_bits(smean, mm0), "save_mean = moving mean")
    inv = 1 / torch.sqrt(var + eps)
    rep.add("save_invstd", sinv, inv, inv, TOL_BN)
    # y: the mean's own rounding (of the size of eps * mean |x|) enters through x - mean
    rep.add("y", y, (X - mean) * inv * gm + bt, ((X - mean).abs() + (amean if training else 0)) * inv * gm.abs() + bt.abs(),
            TOL_BN)
    # backward from the kernel's own saved statistics
    sm, si = smean.double(), sinv.double()
    dy = randn(g, B, d)
    DY = dy.double()
    xh = (X - sm) * si
    axh = xh.abs()
    if training:
        m1, m2, am1, am2 = DY.mean(0), (DY * xh).mean(0), DY.abs().mean(0), (DY.abs() * axh).mean(0)
        dx_ref = gm * si * (DY - m1 - xh * m2)
        adx = gm.abs() * si * (DY.abs() + am1 + axh * am2)
    else:
        dx_ref, adx = gm * si * DY, gm.abs() * si * DY.abs()
    dx, dgam, dbet = prefill(g, adx), randn(g, d), randn(g, d)
    pre = {"dx": dx.clone(), "dg": dgam.clone(), "db": dbet.clone()}
    outs = {"dx": dx, "dg": dgam if affine else None, "db": dbet}

    def call():
        L_.check(lb.mac_batchnorm_bwd(L_.ptr(x0), L_.ptr(gamma), L_.ptr(smean), L_.ptr(sinv), L_.ptr(dy), training,
                                      L_.ptr(dx), L_.ptr(dgam) if affine else None, L_.ptr(dbet), B, d, L_.stream_ptr()),
                 "mac_batchnorm_bwd")

    got, same = run_twice(call, outs)
    rep.add_inc("dx", got["dx"], pre["dx"], dx_ref, adx, TOL_BN)
    if affine:
        rep.add_inc("dgamma", got["dg"], pre["dg"], (DY * xh).sum(0), (DY.abs() * axh).sum(0), TOL_BN)
    rep.add_inc("dbeta", got["db"], pre["db"], DY.sum(0), DY.abs().sum(0), TOL_BN)
    rep.check(same, "bit-identical rerun")
    rep.done()


# ================================================================================================ 8. small kernels
@pytest.mark.parametrize("d,misalign", [(512, False), (130, False), (3, False), (128, True)])
@pytest.mark.parametrize("accumulate", [0, 1])
def test_colsum_matches_fp64(d, misalign, accumulate):
    """the float4 path (d % 4 == 0, x 16-byte aligned) and the scalar path (d % 4 != 0, or x one float off alignment)"""
    lb = lib()
    B, N = 3, 37
    g = gen(d * 2 + misalign + accumulate)
    base = randn(g, B * N * d + 1)
    x = base[1:] if misalign else base[:-1]
    X = x.double().view(B, N, d)
    out = randn(g, B, d) if accumulate else torch.full((B, d), float("nan"), device="cuda")
    pre = out.clone()
    outs = {"out": out}
    got, same = run_twice(lambda: L_.check(lb.mac_colsum(L_.ptr(x), L_.ptr(out), B, N, d, accumulate, L_.stream_ptr())),
                          outs)
    rep = Report("mac_colsum d=%d%s accumulate=%d" % (d, " misaligned" if misalign else "", accumulate))
    if accumulate:
        rep.add_inc("out", got["out"], pre, X.sum(1), X.abs().sum(1), TOL_COLSUM)
    else:
        rep.add("out", got["out"], X.sum(1), X.abs().sum(1), TOL_COLSUM)
    rep.check(same, "bit-identical rerun")
    rep.done()


N_ELEM = 256 * 37 + 13          # not a multiple of the 256-thread block


def test_gate_bwd_matches_fp64():
    lb = lib()
    g = gen(21)
    n = N_ELEM
    gr, mnew, mprev = randn(g, n), randn(g, n), randn(g, n)
    z = torch.sigmoid(randn(g, n))
    dmnew, dpre = torch.full((n,), float("nan"), device="cuda"), torch.full((n,), float("nan"), device="cuda")
    dmprev = randn(g, n)
    pre = dmprev.clone()
    L_.check(lb.mac_gate_bwd(L_.ptr(gr), L_.ptr(z), L_.ptr(mnew), L_.ptr(mprev), L_.ptr(dmnew), L_.ptr(dmprev), L_.ptr(dpre),
                             n, L_.stream_ptr()))
    torch.cuda.synchronize()
    G, Z, Mn, Mp = gr.double(), z.double(), mnew.double(), mprev.double()
    rep = Report("mac_gate_bwd n=%d" % n)
    rep.add("dmnew", dmnew, G * Z, (G * Z).abs(), TOL_ELEM)
    rep.add_inc("dmprev", dmprev, pre, G * (1 - Z), G.abs() * (1 - Z).abs(), TOL_ELEM)
    rep.add("dpre", dpre, G * (Mn - Mp) * Z * (1 - Z), G.abs() * (Mn.abs() + Mp.abs()) * Z * (1 - Z), TOL_ELEM)
    rep.done()


@pytest.mark.parametrize("act", ["NON", "TANH", "SIGMOID", "ELU", "RELU_STD"])
def test_activation_bwd_matches_fp64(act):
    """dx = dy * act'(.) through the saved output y"""
    lb = lib()
    g = gen(L_.ACT[act] + 40)
    n = N_ELEM
    pre_act = randn(g, n) * 2
    y = {"NON": lambda t: t, "TANH": torch.tanh, "SIGMOID": torch.sigmoid, "ELU": torch.nn.functional.elu,
         "RELU_STD": torch.relu}[act](pre_act).contiguous()
    dy = randn(g, n)
    dx = torch.full((n,), float("nan"), device="cuda")
    L_.check(lb.mac_activation_bwd(L_.ptr(y), L_.ptr(dy), L_.ACT[act], L_.ptr(dx), n, L_.stream_ptr()))
    torch.cuda.synchronize()
    Y, DY = y.double(), dy.double()
    fac = {"NON": torch.ones_like(Y), "TANH": 1 - Y * Y, "SIGMOID": Y * (1 - Y), "ELU": torch.where(Y > 0, 1.0, Y + 1),
           "RELU_STD": (Y > 0).double()}[act]
    # bounds of the fp32 factor: 1 - y^2, y (1 - y) and y + 1 round relative to 1 + y^2, |y| (1 + |y|) and |y| + 1
    afac = {"TANH": 1 + Y * Y, "SIGMOID": Y.abs() * (1 + Y.abs()),
            "ELU": torch.where(Y > 0, 1.0, Y.abs() + 1)}.get(act, fac.abs())
    rep = Report("mac_activation_bwd %s" % act)
    rep.add("dx", dx, DY * fac, DY.abs() * afac, TOL_ELEM)
    rep.done()


def test_axpy_matches_fp64():
    lb = lib()
    g = gen(55)
    n, alpha = N_ELEM, -0.37
    dst, src = randn(g, n), randn(g, n)
    pre = dst.clone()
    L_.check(lb.mac_axpy(L_.ptr(dst), L_.ptr(src), alpha, n, L_.stream_ptr()))
    torch.cuda.synchronize()
    a = float(np.float32(alpha))
    rep = Report("mac_axpy n=%d" % n)
    rep.add_inc("dst", dst, pre, a * src.double(), abs(a) * src.double().abs(), TOL_ELEM)
    rep.done()
