"""The Hopper tensor-core kernels (csrc/tc_gemm.cuh, csrc/skinny_tc.cuh, csrc/read_step.cuh) against fp64 references of
their OWN operation, called through the C ABI.

Every reference is computed on exactly the operands the kernel sees: bf16-rounded inputs and packed weights, or the split
hi = bf16_rn(x), lo = bf16_rn(x - hi), with bf16 roundings at the kernel's intermediate points (intermediates are read back
from the kernel's own slabs where it keeps them).  The only legitimate difference left is the order of fp32 accumulation,
so the bounds are element-wise and scaled by the absolute product:

    |got - ref| <= tol * (|A| @ |B|) + (one bf16 ulp of ref for bf16 outputs) + (fp32 evaluation error of the epilogue)

With random data, one missing k-block at K = 12 544 moves a result by ~1e-3 of |A| @ |B| (more at smaller K); the bounds
below sit at 1.5e-7 .. 1e-5.  Each `tol` is a few times the worst value measured on an H100 80GB HBM3 (SXM, 700 W power
limit, 132 SMs), written beside it.  tests/test_wgmma_bounds.py shows on the CPU, with the reference code of this file,
that a dropped k-block or split-K slice is rejected."""
import ctypes
import math

import numpy as np
import pytest
import torch

from mac_network_b200 import _lib as L_
from oracle.philox import philox_uniform

pytestmark = pytest.mark.gpu

MAC_OK, ERR_INVALID, ERR_ALIGN, ERR_UNSUPPORTED = 0, -1, -2, -3
SITE_READ_KB, SITE_READ_MEM, SITE_READ_INTER = L_.SITE_READ_KB, L_.SITE_READ_MEM, L_.SITE_READ_INTER

# ---- bounds (fraction of |A| @ |B|); measured worst value on the H100 beside each
TOL_SKINNY_SPLIT = 3e-6        # split product vs the exact-split fp64 reference             measured 8.4e-7
TOL_SKINNY_TRUE = 6e-6         # split product vs fp64 of the fp32 inputs (header: ~1e-5)     measured 2.1e-6
TOL_SKINNY_SINGLE = 3e-7       # single bf16 pass vs fp64 of the bf16 operands                measured 7.2e-8
TOL_WGRAD = 1.5e-6             # split-K dW and every slice partial vs fp64                   measured 4.5e-7
TOL_TC = 2e-7                  # tc_gemm bf16 epilogues (P, P*y, Q, H, I1), beyond 1 bf16 ulp measured 4.1e-8
TOL_TC32 = 1e-5                # split-bf16 (tc32) P, Q, H vs fp64 of the fp32 inputs         measured 2.8e-6


# ------------------------------------------------------------------------------------------------ reference helpers
def bf16_round(x):
    """fp32 -> bf16 (round to nearest even) -> float64: the kernels' rounding of an fp32 value."""
    return x.float().to(torch.bfloat16).double()


def split_hi_lo(x):
    """hi = bf16_rn(x), lo = bf16_rn(x - hi) (x - hi exact in fp32), as float64."""
    x = x.float()
    hi = x.to(torch.bfloat16)
    lo = (x - hi.float()).to(torch.bfloat16)
    return hi.double(), lo.double()


def bf16_ulp(v):
    """one bf16 ulp of |v| (normal range): 2^(floor(log2|v|) - 7)."""
    _, e = torch.frexp(v.double().abs().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(v, dtype=torch.float64), e - 8)


def excess(got, ref, absprod, ulps=0, tiny=0.0):
    """max over elements of (|got - ref| - ulps * bf16_ulp(ref) - tiny) / absprod, floored at 0: the part of the error that
    fp32 accumulation has to account for, in units of |A| @ |B|.  Non-finite results fail."""
    got = got.double()
    assert bool(torch.isfinite(got).all()), "non-finite kernel output"
    err = (got - ref.double()).abs() - tiny
    if ulps:
        err = err - ulps * bf16_ulp(ref)
    return float((err.clamp_min(0) / absprod.double().clamp_min(1e-30)).max())


def elu(x):
    return torch.where(x > 0, x, torch.expm1(x))


def act_ref(name, x):
    return {"NON": lambda t: t, "TANH": torch.tanh, "SIGMOID": torch.sigmoid, "ELU": elu,
            "RELU_STD": lambda t: t.clamp_min(0)}[name](x)


def keep_threshold(keep):
    """the kernels' integer dropout threshold: keep element iff (philox word >> 8) >= threshold"""
    return math.ceil((1.0 - float(np.float32(keep))) * 16777216.0)


def keep_mask(seed, site, step, shape, keep, device="cuda"):
    n = int(np.prod(shape))
    u = philox_uniform(seed, site, step, n) * 16777216.0          # the 24-bit integer of each draw
    return torch.from_numpy(u >= keep_threshold(keep)).view(*shape).to(device)


def attention_bound_check(att, info, I1_ref, absI1, c, wr, br, kbv, B, N, tol, ms=None):
    """att = softmax_n(sum_k ELU(I1 * c_b) * ms * wr + br), info = sum_n att * kb, with I1 known to tol * absI1 (the
    accumulation bound of its product): the logit error is bounded through |d ELU(I1 c)/d I1| <= |c|, the softmax moves by
    at most att * expm1(2 max|dlogit|), and fp32 evaluation adds a few 1e-6 relative.  Returns the worst fraction of the
    bound used by att and by info."""
    cb = c.double().repeat_interleave(N, 0)
    t = elu(I1_ref * cb)
    f = wr.double()[None, :] * (1.0 if ms is None else ms)
    logits = (t * f).sum(1) + br
    dL = (f.abs() * cb.abs() * tol * absI1).sum(1) + (f.abs() * (1e-7 + 1e-6 * t.abs())).sum(1) + 1e-6 * (logits.abs() + 1)
    dL = dL.view(B, N).amax(1, keepdim=True)
    att_ref = torch.softmax(logits.view(B, N), 1)
    att_bnd = att_ref * (torch.expm1(2 * dL) + 4e-6) + 1e-12
    kbv = kbv.double().view(B, N, -1)
    info_ref = torch.einsum("bn,bnd->bd", att_ref, kbv)
    info_bnd = torch.einsum("bn,bnd->bd", att_bnd, kbv.abs()) + 4e-6 * torch.einsum("bn,bnd->bd", att_ref, kbv.abs()) + 1e-12
    assert bool(torch.isfinite(att).all()) and bool(torch.isfinite(info).all())
    r_att = float(((att.double() - att_ref).abs() / att_bnd).max())
    r_info = float(((info.double() - info_ref).abs() / info_bnd).max())
    return r_att, r_info


# ------------------------------------------------------------------------------------------------ library plumbing
def lib():
    lb = L_.load()
    if not getattr(lb, "_wgmma_internal_bound", False):
        # internal exports of units.cu (used by backward.cu; not part of the ABI header, hence not in PROTOTYPES)
        c_fp, c_int = ctypes.c_void_p, ctypes.c_int
        lb.mac_tc_wgrad_splitk_.restype = c_int
        lb.mac_tc_wgrad_splitk_.argtypes = [c_fp, c_fp, c_fp, c_fp, c_int, c_int, c_int, c_fp]
        lb.mac_tc_wgrad_partial_bytes_.restype = ctypes.c_size_t
        lb.mac_tc_wgrad_partial_bytes_.argtypes = [c_int, c_int]
        lb.mac_pack_t_bf16_.restype = c_int
        lb.mac_pack_t_bf16_.argtypes = [c_int, c_fp, c_fp, c_fp, c_int, c_int, c_fp, c_int, ctypes.c_uint32, ctypes.c_float,
                                        ctypes.c_uint64, c_int, c_int, c_fp]
        lb._wgmma_internal_bound = True
    return lb


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def randn(g, *shape, scale=1.0):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).contiguous()


def align1k(t, off=0):
    """byte offset inside uint8 tensor t of the first 1 KB-aligned address at or after t + off (the kernels' slab base)"""
    base = t.data_ptr()
    return ((base + off + 1023) & ~1023) - base


def bf16_slab(buf, off, rows, cols):
    return buf[off:off + rows * cols * 2].view(torch.bfloat16).view(rows, cols)


def pack16(W):
    """fp32 [in, out] -> bf16 [out, in] (mac_pack_weight_bf16), checked bit-exact against torch's rounding"""
    o = torch.empty((W.shape[1], W.shape[0]), dtype=torch.bfloat16, device="cuda")
    L_.check(lib().mac_pack_weight_bf16(L_.ptr(W), L_.ptr(o), W.shape[0], W.shape[1], L_.stream_ptr()))
    torch.cuda.synchronize()
    assert torch.equal(o.view(torch.int16), W.t().contiguous().to(torch.bfloat16).view(torch.int16))
    return o


def pack3(W):
    """fp32 [in, out] -> bf16 [out, 3 in] = [hi | hi | lo] (mac_pack_weight_split3), checked bit-exact"""
    K, n = W.shape
    o = torch.empty((n, 3 * K), dtype=torch.bfloat16, device="cuda")
    L_.check(lib().mac_pack_weight_split3(L_.ptr(W), L_.ptr(o), K, n, L_.stream_ptr()))
    torch.cuda.synchronize()
    hi = W.t().contiguous().to(torch.bfloat16)
    lo = (W.t().contiguous() - hi.float()).to(torch.bfloat16)
    assert torch.equal(o.view(torch.int16), torch.cat([hi, hi, lo], 1).view(torch.int16))
    return o


# ================================================================================================ 1. skinny split-bf16
def run_skinny(xs, hi, lo, b, bias_const, act, y, ldy, M, n_out, y2=None, n_split=0, gate=(None, None, None)):
    n = len(xs)
    arr_p = (ctypes.c_void_p * n)(*[x.data_ptr() for x in xs])
    arr_k = (ctypes.c_int * n)(*[x.shape[1] for x in xs])
    arr_ld = (ctypes.c_int * n)(*[x.stride(0) for x in xs])
    gn, go, gz = gate
    return lib().mac_linear_tc_small_fwd(arr_p, arr_k, arr_ld, n, L_.ptr(hi), L_.ptr(lo), L_.ptr(b), float(bias_const),
                                         L_.ACT[act], L_.ptr(y), ldy, L_.ptr(y2), int(n_split), L_.ptr(gn), L_.ptr(go),
                                         L_.ptr(gz), M, n_out, L_.stream_ptr())


def pack_split(W):
    """mac_pack_weight_bf16_split, checked bit-exact: hi = bf16(W^T), lo = bf16(W^T - hi)"""
    K, n = W.shape
    hi = torch.empty((n, K), dtype=torch.bfloat16, device="cuda")
    lo = torch.empty_like(hi)
    L_.check(lib().mac_pack_weight_bf16_split(L_.ptr(W), L_.ptr(hi), L_.ptr(lo), K, n, L_.stream_ptr()))
    torch.cuda.synchronize()
    rh = W.t().contiguous().to(torch.bfloat16)
    rl = (W.t().contiguous() - rh.float()).to(torch.bfloat16)
    assert torch.equal(hi.view(torch.int16), rh.view(torch.int16)) and torch.equal(lo.view(torch.int16), rl.view(torch.int16))
    return hi, lo


def make_segments(g, M, segs, wide):
    """fp32 activation segments; segment `wide` is the column block [64, 64 + k) of a [M, k + 128] tensor (ldx > k)"""
    xs = []
    for i, k in enumerate(segs):
        if i == wide:
            xs.append(randn(g, M, k + 128)[:, 64:64 + k])
        else:
            xs.append(randn(g, M, k))
    return xs


def skinny_refs(X, W, hi, lo, bias_vec, bias_const):
    """(exact-split reference, single-pass reference, true fp64 product, |X| @ |W| + |bias|) -- pre-activation"""
    xh, xl = split_hi_lo(X)
    wh, wl = hi.double().t(), lo.double().t()
    bias = bias_const + (bias_vec.double() if bias_vec is not None else 0.0)
    exact = xh @ wh + xl @ wh + xh @ wl + bias
    single = xh @ wh + bias
    true = X.double() @ W.double() + bias
    absprod = X.double().abs() @ W.double().abs() + (abs(bias_const) + (bias_vec.double().abs() if bias_vec is not None else 0.0))
    return exact, single, true, absprod


# (M, segments, n_out, split, bias, act, ldy - n_out, index of the ldx > k segment): every M of interest (warpgroup 1 empty,
# one row of it, full), 1 / 2 / 4 / 5 / 7 / 16 k-blocks (all remainders of the three-buffer rotation), BN = 32 and 64
SKINNY_CASES = [
    (1, (64,), 32, True, "vec", "NON", 0, None),
    (37, (64, 64), 96, True, "const", "TANH", 32, 0),
    (64, (512, 512), 1024, True, "vec", "NON", 0, 1),
    (65, (128, 64, 192, 64), 512, True, "none", "ELU", 64, 2),
    (100, (128, 128), 2048, False, "vec", "SIGMOID", 0, None),
    (128, (128, 64, 192, 64), 1024, False, "const", "RELU_STD", 32, 0),
    (128, (512, 512), 96, True, "vec", "ELU", 0, None),
    (100, (256, 64), 512, True, "vec", "RELU_STD", 0, 1),
    (65, (512,), 2048, True, "none", "SIGMOID", 0, 0),
]


@pytest.mark.parametrize("M,segs,n_out,split,bias,act,pad,wide", SKINNY_CASES)
def test_skinny_tc_matches_fp64(M, segs, n_out, split, bias, act, pad, wide):
    """mac_linear_tc_small_fwd (skinny_tc_kernel) against the fp64 product of exactly its operands, every epilogue option;
    the output is NaN-filled over all 128 rows and the ldy padding, and only [0, M) x [0, n_out) may be written."""
    g = gen(M * 7919 + n_out + len(segs))
    K = sum(segs)
    xs = make_segments(g, M, segs, wide)
    W = randn(g, K, n_out, scale=K ** -0.5)
    hi, lo = pack_split(W)
    b = randn(g, n_out, scale=0.5) if bias == "vec" else None
    bias_const = {"vec": -0.2, "const": 0.3, "none": 0.0}[bias]
    ldy = n_out + pad
    y = torch.full((128, ldy), float("nan"), device="cuda")
    L_.check(run_skinny(xs, hi, lo if split else None, b, bias_const, act, y, ldy, M, n_out), "mac_linear_tc_small_fwd")
    torch.cuda.synchronize()
    X = torch.cat([x.contiguous() for x in xs], 1)
    exact, single, true, absprod = skinny_refs(X, W, hi, lo, b, bias_const)
    got = y[:M, :n_out]
    ref = act_ref(act, exact if split else single)
    tiny = 0.0 if act == "NON" else 1e-6 * ref.abs() + 1e-7      # fp32 tanhf / expf / expm1f in the epilogue
    e = excess(got, ref, absprod, tiny=tiny)
    msg = (M, segs, n_out, split, act)
    if split:
        e_true = excess(got, act_ref(act, true), absprod, tiny=tiny)
        print("skinny split %s: vs exact split %.2e, vs fp64 of the fp32 inputs %.2e" % (msg, e, e_true))
        assert e <= TOL_SKINNY_SPLIT, (msg, e)
        assert e_true <= TOL_SKINNY_TRUE, (msg, e_true)
    else:
        print("skinny single pass %s: %.2e" % (msg, e))
        assert e <= TOL_SKINNY_SINGLE, (msg, e)
    assert bool(torch.isnan(y[M:]).all()), "rows >= M written"
    assert bool(torch.isnan(y[:, n_out:]).all()), "ldy padding written"


def test_skinny_tc_column_split_y2():
    """y2 / n_split (the folded write unit): columns >= n_split land in y2[m, n - n_split] with the same ldy, nothing else."""
    g = gen(4242)
    M, K, n_out, n_split, ldy = 100, 1024, 1024, 512, 544
    xs = make_segments(g, M, (512, 512), 0)
    W = randn(g, K, n_out, scale=K ** -0.5)
    hi, lo = pack_split(W)
    b = randn(g, n_out, scale=0.5)
    y = torch.full((128, ldy), float("nan"), device="cuda")
    y2 = torch.full((128, ldy), float("nan"), device="cuda")
    L_.check(run_skinny(xs, hi, lo, b, 0.0, "NON", y, ldy, M, n_out, y2=y2, n_split=n_split))
    torch.cuda.synchronize()
    exact, _, true, absprod = skinny_refs(torch.cat([x.contiguous() for x in xs], 1), W, hi, lo, b, 0.0)
    e1 = excess(y[:M, :n_split], exact[:, :n_split], absprod[:, :n_split])
    e2 = excess(y2[:M, :n_out - n_split], exact[:, n_split:], absprod[:, n_split:])
    print("skinny y2 split: %.2e / %.2e" % (e1, e2))
    assert max(e1, e2) <= TOL_SKINNY_SPLIT
    assert bool(torch.isnan(y[M:]).all()) and bool(torch.isnan(y[:, n_split:]).all())
    assert bool(torch.isnan(y2[M:]).all()) and bool(torch.isnan(y2[:, n_out - n_split:]).all())


@pytest.mark.parametrize("M", [37, 65, 128])
def test_skinny_tc_write_gate(M):
    """Gate epilogue (mac_cell.py:358-367): z = sigmoid(acc + b + bias_const), y = new*z + old*(1-z), z to gate_z; gate
    operands and outputs share ldy > n_out."""
    g = gen(M + 31)
    K, n_out, ldy = 512, 512, 544
    xs = make_segments(g, M, (K,), None)
    W = randn(g, K, n_out, scale=K ** -0.5)
    hi, lo = pack_split(W)
    b = randn(g, n_out, scale=0.5)
    gnew, gold = randn(g, 128, ldy), randn(g, 128, ldy)
    y = torch.full((128, ldy), float("nan"), device="cuda")
    z = torch.full((128, ldy), float("nan"), device="cuda")
    L_.check(run_skinny(xs, hi, lo, b, 1.0, "NON", y, ldy, M, n_out, gate=(gnew, gold, z)))
    torch.cuda.synchronize()
    exact, _, _, absprod = skinny_refs(xs[0], W, hi, lo, b, 1.0)
    z_ref = torch.sigmoid(exact)
    gn, go = gnew[:M, :n_out].double(), gold[:M, :n_out].double()
    y_ref = gn * z_ref + go * (1 - z_ref)
    ez = excess(z[:M, :n_out], z_ref, 0.25 * absprod, tiny=3e-7)
    ey = excess(y[:M, :n_out], y_ref, 0.25 * absprod * (gn - go).abs(),
                tiny=3e-7 * (gn - go).abs() + 4e-7 * (gn.abs() + go.abs()))
    print("skinny gate M=%d: z %.2e, y %.2e" % (M, ez, ey))
    assert ez <= TOL_SKINNY_SPLIT and ey <= TOL_SKINNY_SPLIT, (ez, ey)
    for t in (y, z):
        assert bool(torch.isnan(t[M:]).all()) and bool(torch.isnan(t[:, n_out:]).all())


def test_skinny_tc_status_codes():
    """Refused shapes return their status before any launch."""
    g = gen(5)
    W = randn(g, 64, 64, scale=0.125)
    hi, lo = pack_split(W)
    y = torch.zeros(129, 64, device="cuda")
    x = randn(g, 129, 64)
    assert run_skinny([x], hi, lo, None, 0.0, "NON", y, 64, 129, 64) == ERR_INVALID                 # M > 128
    assert run_skinny([x[:8]], hi, lo, None, 0.0, "NON", y, 64, 8, 48) == ERR_UNSUPPORTED           # n_out % 32
    x96 = randn(g, 8, 96)
    assert run_skinny([x96], hi, lo, None, 0.0, "NON", y, 64, 8, 64) == ERR_UNSUPPORTED             # 96-wide segment
    assert run_skinny([x[:8]], hi, lo, None, 0.0, "NON", y, 64, 8, 64, gate=(y, None, None)) == ERR_INVALID
    xm = randn(g, 8, 128)[:, 1:65]                                                                    # 4-byte offset
    assert run_skinny([xm], hi, lo, None, 0.0, "NON", y, 64, 8, 64) == ERR_ALIGN
    torch.cuda.synchronize()


# ================================================================================================ 2. split-K weight gradient
def pick_ksplit(K, out_tiles, sms):
    """restatement of tc_pick_ksplit: the largest S <= 28 dividing K/64 with >= 2 k-blocks per slice and <= 2 CTAs per SM"""
    kb, best = K // 64, 1
    for S in range(2, 29):
        if kb % S == 0 and kb // S >= 2 and out_tiles * S <= 2 * sms:
            best = S
    return best


@pytest.mark.parametrize("in_dim,out_dim", [(128, 128), (512, 512), (1024, 512)])
@pytest.mark.parametrize("kblocks", [8, 13, 196])
def test_splitk_weight_gradient(in_dim, out_dim, kblocks):
    """tc_wgrad_splitk: dW += xT @ gT^T over K = 64 * kblocks.  Every slice partial is checked against its own K range (the
    slice after the last must stay untouched, which pins S), dW against dW0 + the full fp64 product, and a second run from
    the same dW0 must be bit-identical (fixed slice order)."""
    lb = lib()
    K = 64 * kblocks
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    S = pick_ksplit(K, (in_dim // 128) * (out_dim // 128), sms)
    if kblocks == 8:
        assert S == 4
    elif kblocks == 13:
        assert S == 1
    else:
        assert S == {(128, 128): 28, (512, 512): 14, (1024, 512): 7}[(in_dim, out_dim)]
    g = gen(in_dim + out_dim + kblocks)
    xT = randn(g, in_dim, K).to(torch.bfloat16)
    gT = randn(g, out_dim, K).to(torch.bfloat16)
    dW0 = randn(g, in_dim, out_dim, scale=3.0)
    nbytes = lb.mac_tc_wgrad_partial_bytes_(in_dim, out_dim)
    assert nbytes == 28 * in_dim * out_dim * 4
    partial = torch.full((28, in_dim, out_dim), float("nan"), device="cuda")
    outs = []
    for _ in range(2):
        dW = dW0.clone()
        L_.check(lb.mac_tc_wgrad_splitk_(L_.ptr(xT), L_.ptr(gT), L_.ptr(dW), L_.ptr(partial), in_dim, out_dim, K,
                                         L_.stream_ptr()), "mac_tc_wgrad_splitk_")
        outs.append(dW)
    torch.cuda.synchronize()
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32)), "split-K result not deterministic"
    X, G = xT.double(), gT.double()
    ks = K // S
    worst_slice = 0.0
    for s in range(S):
        xs_, gs_ = X[:, s * ks:(s + 1) * ks], G[:, s * ks:(s + 1) * ks]
        worst_slice = max(worst_slice, excess(partial[s], xs_ @ gs_.t(), xs_.abs() @ gs_.abs().t()))
    if S < 28:
        assert bool(torch.isnan(partial[S]).all()), "more than S = %d slices written" % S
    ref = dW0.double() + X @ G.t()
    e = excess(outs[0], ref, X.abs() @ G.abs().t() + dW0.double().abs())
    print("wgrad %dx%d K=%d S=%d: slices %.2e, dW %.2e" % (in_dim, out_dim, K, S, worst_slice, e))
    assert worst_slice <= TOL_WGRAD and e <= TOL_WGRAD, (worst_slice, e)


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_pack_t_bf16_bit_exact(mode):
    """pack_t_bf16_kernel: X [K, N] fp32 -> bf16 X^T [N, K] and the row-major bf16 copy, with mode 1 = x * rowvec[k / rpb]
    and mode 2 = the forward's dropout (Philox, element index k * N + n), bit-exact against torch's round-to-nearest.
    K = 150 rows and N = 200 columns leave partial 64 x 64 tiles in both directions."""
    lb = lib()
    K, N, rpb = 150, 200, 50
    seed, site, step, keep = 1234, SITE_READ_KB, 3, 0.85
    g = gen(mode + 11)
    X = randn(g, K, N)
    rowvec = randn(g, K // rpb, N)
    thr = keep_threshold(keep)
    scale = np.float32(1.0) / np.float32(keep)
    Xt = torch.full((N, K), float("nan"), device="cuda").to(torch.bfloat16)
    Xrm = torch.full((K, N), float("nan"), device="cuda").to(torch.bfloat16)
    L_.check(lb.mac_pack_t_bf16_(mode, L_.ptr(X), L_.ptr(Xt), L_.ptr(Xrm), K, N, L_.ptr(rowvec) if mode == 1 else None, rpb,
                                 thr if mode == 2 else 0, float(scale), seed, site, step, L_.stream_ptr()), "mac_pack_t_bf16_")
    torch.cuda.synchronize()
    if mode == 0:
        v = X
    elif mode == 1:
        v = X * rowvec.repeat_interleave(rpb, 0)
    else:
        m = keep_mask(seed, site, step, (K, N), keep)
        v = torch.where(m, X * torch.tensor(scale, device="cuda"), torch.zeros_like(X))
        assert 0.1 < 1 - float(m.float().mean()) < 0.2
    ref = v.to(torch.bfloat16)
    assert torch.equal(Xrm.view(torch.int16), ref.view(torch.int16))
    assert torch.equal(Xt.view(torch.int16), ref.t().contiguous().view(torch.int16))


# ================================================================================================ 3. read-chain epilogues
def read_setup(d, seed, tc32=False):
    g = gen(seed)
    W = {"Wx": randn(g, d, d, scale=d ** -0.5), "bx": randn(g, d, scale=0.1), "Wy": randn(g, d, d, scale=d ** -0.5),
         "by": randn(g, d, scale=0.1), "Wm": randn(g, 2 * d, d, scale=(2 * d) ** -0.5), "bm": randn(g, d, scale=0.1),
         "Wm2": randn(g, d, d, scale=d ** -0.5), "bm2": randn(g, d, scale=0.1), "wr": randn(g, d, scale=4 * d ** -0.5)}
    randn(g, 2 * d, d), randn(g, d)     # unused draws: they keep the inputs each test draws next from g as measured
    P = {"Wx": pack16(W["Wx"]), "Wm": pack16(W["Wm"]), "Wm2": pack16(W["Wm2"])}
    s3 = {}
    if tc32:
        s3 = {"Wx": pack3(W["Wx"]), "Wma": pack3(W["Wm"][:d]), "Wmb": pack3(W["Wm"][d:]), "Wm2": pack3(W["Wm2"])}
    v = lambda t: t.data_ptr() if t is not None else None
    rw = L_.ReadWeights(v(W["Wx"]), v(W["bx"]), v(W["Wy"]), v(W["by"]), v(W["Wm"]), v(W["bm"]), v(W["Wm2"]), v(W["bm2"]),
                        v(W["wr"]), 0.25, v(P["Wx"]), v(P["Wm"]), v(P["Wm2"]),
                        v(s3.get("Wx")), v(s3.get("Wma")), v(s3.get("Wmb")), v(s3.get("Wm2")))
    return g, W, P, s3, rw


def nanfill(*shape):
    return torch.full(shape, float("nan"), device="cuda")


@pytest.mark.parametrize("B,N,d", [(3, 49, 512), (5, 30, 128)])
def test_bf16_training_read_chain_matches_fp64(B, N, d):
    """mac_read_fwd(prec = bf16, keep_read < 1) -- tc_read_chain: the dropout(KB) cast, TC_EPI_P (bf16 P and P*y), the
    two-segment [P*y, P] product with TC_EPI_ACT, TC_EPI_LOGITS with the READ_INTER mask and the I1 save.  Each slab the
    chain leaves in the workspace is checked against fp64 of the slabs before it; B*N is not a multiple of 128, so tiles
    straddle samples."""
    lb = lib()
    keep, seed, step = 0.85, 77, 2
    g, W, Pk, _, rw = read_setup(d, B * 100 + N)
    M = B * N
    kb = elu(randn(g, B, N, d))
    kb16 = kb.to(torch.bfloat16)
    mem, c = randn(g, B, d), randn(g, B, d)
    wsb = lb.mac_read_workspace_bytes(B, N, d, 1)
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    save = nanfill(3 * M * d + B * d)
    info, att = nanfill(B, d), nanfill(B, N)
    L_.check(lb.mac_read_fwd(L_.ptr(kb), L_.ptr(kb16), L_.ptr(mem), L_.ptr(c), ctypes.byref(rw), keep, seed, step, 1,
                             L_.ptr(info), L_.ptr(att), L_.ptr(save), L_.ptr(ws), wsb, B, N, d, L_.stream_ptr()), "mac_read_fwd")
    torch.cuda.synchronize()
    off = align1k(ws, lb.mac_read_workspace_bytes(B, N, d, 0))
    slab = (M * d * 2 + 1023) & ~1023
    P16, PY16, H16, I116 = (bf16_slab(ws, off + i * slab, M, d).double() for i in range(4))
    # `save` = [P | H | I1 | y] in fp32: the library widens its bf16 slabs, bit for bit
    for k, s16 in enumerate((P16, H16, I116)):
        assert torch.equal(save[k * M * d:(k + 1) * M * d].view(M, d), s16.float()), "save slab %d" % k
    y = save[3 * M * d:].view(B, d)
    scale = np.float32(1.0) / np.float32(keep)
    # y = dropout(memory) @ Wy + by (fp32 path)
    md = torch.where(keep_mask(seed, SITE_READ_MEM, step, (B, d), keep), mem * float(scale), torch.zeros_like(mem)).double()
    ey = excess(y, md @ W["Wy"].double() + W["by"].double(), md.abs() @ W["Wy"].double().abs() + W["by"].double().abs())
    # P = bf16(dropout(KB)) @ bf16(Wx) + bx  -> bf16 P, bf16 P*y
    kbd = bf16_round(torch.where(keep_mask(seed, SITE_READ_KB, step, (B, N, d), keep), kb * torch.tensor(scale, device="cuda"),
                                 torch.zeros_like(kb)).view(M, d))
    Wx = Pk["Wx"].double().t()
    P_ref = kbd @ Wx + W["bx"].double()
    absP = kbd.abs() @ Wx.abs() + W["bx"].double().abs()
    yb = y.double().repeat_interleave(N, 0)
    eP = excess(P16, P_ref, absP, ulps=1)
    ePY = excess(PY16, P_ref * yb, absP * yb.abs(), ulps=1)
    # H = ELU([P*y, P] @ bf16(Wm) + bm)
    Wm = Pk["Wm"].double().t()
    H_ref = elu(PY16 @ Wm[:d] + P16 @ Wm[d:] + W["bm"].double())
    absH = PY16.abs() @ Wm[:d].abs() + P16.abs() @ Wm[d:].abs() + W["bm"].double().abs()
    eH = excess(H16, H_ref, absH, ulps=1, tiny=1e-7)
    # I1 = H @ bf16(Wm2) + bm2 (saved as bf16); logits with the READ_INTER mask
    Wm2 = Pk["Wm2"].double().t()
    I1_ref = H16 @ Wm2 + W["bm2"].double()
    absI1 = H16.abs() @ Wm2.abs() + W["bm2"].double().abs()
    eI1 = excess(I116, I1_ref, absI1, ulps=1)
    ms = keep_mask(seed, SITE_READ_INTER, step, (M, d), keep).double() * float(scale)
    ra, ri = attention_bound_check(att, info, I1_ref, absI1, c, W["wr"], 0.25, kb16, B, N, TOL_TC, ms=ms)
    print("bf16 training read chain %s: y %.2e P %.2e P*y %.2e H %.2e I1 %.2e; att / info use %.2f / %.2f of their bound"
          % ((B, N, d), ey, eP, ePY, eH, eI1, ra, ri))
    assert ey <= 1e-5, ey
    assert max(eP, ePY, eH, eI1) <= TOL_TC, (eP, ePY, eH, eI1)
    assert ra <= 1 and ri <= 1, (ra, ri)


@pytest.mark.parametrize("B,N,d", [(2, 300, 512), (3, 49, 128), (3, 49, 256)])
def test_bf16_inference_read_chain_unfused_matches_fp64(B, N, d):
    """mac_read_invariant + mac_read_fwd_inv at bf16 on shapes the fused read step refuses, so the four-launch chain runs:
    P and Q (the ldw = 2d product) read back from inv, scale_rows_bf16_kernel's P*y bit-exact, TC_EPI_ADDACT's H, then the
    attention and retrieved information."""
    lb = lib()
    assert lb.mac_read_step_fused_supported(B, N, d) == 0
    g, W, Pk, _, rw = read_setup(d, B * 100 + N + d)
    M = B * N
    kb16 = elu(randn(g, B, N, d)).to(torch.bfloat16)
    y, mem, c = randn(g, B, d), randn(g, B, d), randn(g, B, d)
    nb = lb.mac_read_invariant_bytes(B, N, d, 1)
    inv = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    L_.check(lb.mac_read_invariant(None, L_.ptr(kb16), ctypes.byref(rw), 1, L_.ptr(inv), nb, B, N, d, L_.stream_ptr()))
    wsb = lb.mac_read_workspace_bytes(B, N, d, 1)
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    info, att = nanfill(B, d), nanfill(B, N)
    L_.check(lb.mac_read_fwd_inv(None, L_.ptr(kb16), L_.ptr(inv), L_.ptr(y), L_.ptr(mem), L_.ptr(c), ctypes.byref(rw), 1,
                                 L_.ptr(info), L_.ptr(att), L_.ptr(ws), wsb, B, N, d, L_.stream_ptr()), "mac_read_fwd_inv")
    torch.cuda.synchronize()
    slab = (M * d * 2 + 1023) & ~1023
    io = align1k(inv)
    P16, Q16 = bf16_slab(inv, io, M, d), bf16_slab(inv, io + slab, M, d)
    wo = align1k(ws, lb.mac_read_workspace_bytes(B, N, d, 0))
    PY16, H16 = bf16_slab(ws, wo + slab, M, d), bf16_slab(ws, wo + 2 * slab, M, d)
    kbv, Wx, Wm, Wm2 = kb16.double().view(M, d), Pk["Wx"].double().t(), Pk["Wm"].double().t(), Pk["Wm2"].double().t()
    eP = excess(P16, kbv @ Wx + W["bx"].double(), kbv.abs() @ Wx.abs() + W["bx"].double().abs(), ulps=1)
    Pd = P16.double()
    eQ = excess(Q16, Pd @ Wm[d:] + W["bm"].double(), Pd.abs() @ Wm[d:].abs() + W["bm"].double().abs(), ulps=1)
    PY_ref = (P16.float() * y.repeat_interleave(N, 0)).to(torch.bfloat16)
    assert torch.equal(PY16.view(torch.int16), PY_ref.view(torch.int16)), "P*y not bf16(P * y)"
    PYd, Qd = PY16.double(), Q16.double()
    eH = excess(H16, elu(PYd @ Wm[:d] + Qd), PYd.abs() @ Wm[:d].abs() + Qd.abs(), ulps=1, tiny=1e-7)
    Hd = H16.double()
    I1_ref = Hd @ Wm2 + W["bm2"].double()
    absI1 = Hd.abs() @ Wm2.abs() + W["bm2"].double().abs()
    ra, ri = attention_bound_check(att, info, I1_ref, absI1, c, W["wr"], 0.25, kb16, B, N, TOL_TC)
    print("bf16 inference chain %s: P %.2e Q %.2e H %.2e; att / info use %.2f / %.2f of their bound"
          % ((B, N, d), eP, eQ, eH, ra, ri))
    assert max(eP, eQ, eH) <= TOL_TC, (eP, eQ, eH)
    assert ra <= 1 and ri <= 1, (ra, ri)


@pytest.mark.parametrize("B,N,d", [(3, 49, 512), (2, 75, 128)])
def test_tc32_read_chain_matches_fp64(B, N, d):
    """prec = tc32: mac_read_invariant (P, Q as two-segment split-bf16 products, lda = 2K / ldw = 3K, TC_EPI_F32) and
    mac_read_fwd_inv (TC_EPI_ACT_SPLIT's H as hi | lo, then the logits) against the fp64 product of the fp32 inputs, with
    an M tail (B*N = 147, 150); the end result also against the all-fp64 chain at the 1e-4 bar."""
    lb = lib()
    g, W, _, _, rw = read_setup(d, B * 10 + N + d, tc32=True)
    M = B * N
    kb = elu(randn(g, B, N, d))
    y, mem, c = randn(g, B, d), randn(g, B, d), randn(g, B, d)
    nb = lb.mac_read_invariant_bytes(B, N, d, 2)
    inv = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    L_.check(lb.mac_read_invariant(L_.ptr(kb), None, ctypes.byref(rw), 2, L_.ptr(inv), nb, B, N, d, L_.stream_ptr()))
    wsb = lb.mac_read_workspace_bytes(B, N, d, 2)
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    info, att = nanfill(B, d), nanfill(B, N)
    L_.check(lb.mac_read_fwd_inv(L_.ptr(kb), None, L_.ptr(inv), L_.ptr(y), L_.ptr(mem), L_.ptr(c), ctypes.byref(rw), 2,
                                 L_.ptr(info), L_.ptr(att), L_.ptr(ws), wsb, B, N, d, L_.stream_ptr()), "mac_read_fwd_inv")
    torch.cuda.synchronize()
    Pk = inv[:M * d * 4].view(torch.float32).view(M, d)
    Qk = inv[M * d * 4:2 * M * d * 4].view(torch.float32).view(M, d)
    wo = align1k(ws, lb.mac_read_workspace_bytes(B, N, d, 0))
    Hs = bf16_slab(ws, wo + ((M * 2 * d * 2 + 1023) & ~1023), M, 2 * d).double()
    Hk = Hs[:, :d] + Hs[:, d:]
    kbv = kb.double().view(M, d)
    Wx, Wm, Wm2 = W["Wx"].double(), W["Wm"].double(), W["Wm2"].double()
    bx, bm, bm2 = W["bx"].double(), W["bm"].double(), W["bm2"].double()
    eP = excess(Pk, kbv @ Wx + bx, kbv.abs() @ Wx.abs() + bx.abs())
    Pd = Pk.double()
    eQ = excess(Qk, Pd @ Wm[d:] + bm, Pd.abs() @ Wm[d:].abs() + bm.abs())
    PY = Pd * y.double().repeat_interleave(N, 0)
    Qd = Qk.double()
    H_ref = elu(PY @ Wm[:d] + Qd)
    eH = excess(Hk, H_ref, PY.abs() @ Wm[:d].abs() + Qd.abs(), tiny=2.0 ** -17 * H_ref.abs() + 1e-7)
    I1_ref = Hk @ Wm2 + bm2
    absI1 = Hk.abs() @ Wm2.abs() + bm2.abs()
    ra, ri = attention_bound_check(att, info, I1_ref, absI1, c, W["wr"], 0.25, kb, B, N, TOL_TC32)
    # the whole chain in fp64 from the fp32 inputs
    P0 = kbv @ Wx + bx
    H0 = elu((P0 * y.double().repeat_interleave(N, 0)) @ Wm[:d] + P0 @ Wm[d:] + bm)
    I2 = elu((H0 @ Wm2 + bm2) * c.double().repeat_interleave(N, 0))
    att0 = torch.softmax(((I2 @ W["wr"].double()) + 0.25).view(B, N), 1)
    info0 = torch.einsum("bn,bnd->bd", att0, kb.double())
    e_att = float((att.double() - att0).abs().max() / att0.abs().max())
    e_info = float((info.double() - info0).abs().max() / info0.abs().max())
    print("tc32 chain %s: P %.2e Q %.2e H %.2e; att / info use %.2f / %.2f of their bound; vs all-fp64 chain att %.2e info %.2e"
          % ((B, N, d), eP, eQ, eH, ra, ri, e_att, e_info))
    assert max(eP, eQ, eH) <= TOL_TC32, (eP, eQ, eH)
    assert ra <= 1 and ri <= 1, (ra, ri)
    assert e_att < 1e-4 and e_info < 1e-4, (e_att, e_info)


# ================================================================================================ 4. read-step shape limits
def test_read_step_fused_shape_boundaries():
    """The supported-shape predicate at its edges, and the status an unsupported shape returns (before any launch)."""
    lb = lib()
    d = 512
    for B in (1, 64):
        assert lb.mac_read_step_fused_supported(B, 1, d) == 1 and lb.mac_read_step_fused_supported(B, 256, d) == 1
        assert lb.mac_read_step_fused_supported(B, 257, d) == 0 and lb.mac_read_step_fused_supported(B, 200, 256) == 0
    # the kernel indexes y [B, d] with 32-bit offsets
    assert lb.mac_read_step_fused_supported((1 << 22) - 1, 1, d) == 1 and lb.mac_read_step_fused_supported(1 << 22, 1, d) == 0
    g, _, _, _, rw = read_setup(d, 9)
    B = 2
    t = torch.zeros(16 << 20, dtype=torch.uint8, device="cuda")
    v = randn(g, B, d)
    st = lb.mac_read_step_fused(L_.ptr(t), L_.ptr(t), L_.ptr(v), L_.ptr(v), ctypes.byref(rw), L_.ptr(v), L_.ptr(t), B, 257, d,
                                L_.stream_ptr())
    assert st == ERR_UNSUPPORTED
    torch.cuda.synchronize()
