"""The e4m3 serving kernels element by element against fp64 of their own operands.

1. The accumulator.  Hopper's e4m3 wgmma (m64nNk32) adds its 32 products into the fp32 accumulator with fewer mantissa
   bits than fp32 keeps.  mac_linear_fp8_fwd with sa = sw = 1, no bias and NON returns its accumulator as it is, and e4m3
   products and their sums are exact in fp64 (every product is a multiple of 2^-18 below 2^18, so any sum of fewer than
   2^17 of them fits in 53 bits), so the loss is measured directly.  The model: each k32 instruction errs by at most
       TOL_E4M3 * (|exact running sum entering it| + sum of |its 32 products|)
   and the errors add along a chain of instructions into one accumulator (acc_terms).  The stem's kernel runs a chain of 4
   per 128-wide k-block and adds each k-block into an fp32 master accumulator (one more rounding of 2^-24 of the running
   sum per add); the read step's GEMMs are one chain of 16 over K = 512 (acc_bound).  test_e4m3_accumulator_error_model
   measures the worst ratio to the model over adversarial operands: exponents over the whole e4m3 range inside one
   32-group, one 448 among small values, cancelling pairs, subnormals only, and a steep exponent ramp along K.  The worst
   case is one 448 among small products at K = 128 (4.2e-4: the small ones lose their low bits against the large one);
   over 9 and 72 k-blocks the worst ratio falls to 1.5e-4 and 4.1e-5.
   The model is linear in |A| @ |B|, so it has to admit that worst case for every operand.  On the stem's operands the
   bound is used to 1-75 %.  The read step's chains of 16 instructions are measured through its logits: the smallest
   constant under which every row of (4) holds lies between 1e-5 and 3e-5 on the H100 (64 x 49, 64 x 196 and 265 x 64
   need more than 1e-5), below the chains of 4's worst case, so TOL_E4M3 covers them with room.
2. mac_linear_fp8_fwd, every output.  ref = act(fp64(A8 @ W8) * sa * sw + b) with the bound of (1) scaled by sa * sw,
   the fp32 epilogue (two multiplies and the bias add, 2^-24 each) and EPS_ELU for elu_fast (test_gpu_read_step_bounds), at
   NON, ELU and RELU with a bias and with NULL; rows scaled by 2^U(-20, 20), an all-zero row (sa = 0) and an all-zero
   weight column (sw = 0); y NaN-filled with a NaN guard behind M * N that must survive; a rerun gives the same bits.
3. Stem(prec="fp8") layer by layer: each layer's patch bytes and scales and its weight pack bit for bit against the fp32
   restatements, its output against (2), and the stem's own output bit for bit the same.
4. The read step's logits row by row on random operands (fp8_step_reference, the e4m3 counterpart of
   test_gpu_read_step_bounds.step_reference): A8 from the fp32 restatement exactly; H* = ELU(acc1 * fp32(sP * ay) * sW1
   + Q) within e from (1), the epilogue and EPS_ELU; the kernel's row amax lies in [max(|H*| - e), max(|H*| + e)], so its
   fp32(448 / am) and fp32(am / 448) lie in intervals, and e4m3 rounding is monotone: each H8 element lies between the
   roundings at the two ends of its product interval, which gives dH8; dH8, (1) and sh's interval carry through I1, I2
   and the logit.  The bound is sound but catches no realistic fault: the random-sign sums cancel to about 1/20 of
   |A| @ |B|, so (1) admits several percent of H, H8's intervals span an e4m3 step on most elements, and the bound is
   near 30 logit units (the logits use 0.1-2 % of it).  No sound bound can be much tighter here: on these operands the
   kernel's own accumulator differences flip H8 roundings and move logits by up to 0.4 % of |I2| . |wr|, within a
   factor of 4-30 of what a wrong row scale or a dropped k32 instruction moves them.  What this test adds is the
   canaries -- every `inv` byte but the M logits unchanged by the step (the padding behind the logits keeps its fill),
   the inputs unchanged, att and info NaN before and finite after -- the bit-exact P8 / sP, and the special samples.
5. The read step's logits row by row on operands that make every accumulator exact (exact_operands): the logits are
   then known to the fp32 order of their sum, and a wrong row scale, sample, column-scale half, amax half or k32
   instruction moves them 1000 times further.  This is the per-row check that bites; att and info go through
   test_gpu_wgmma.softmax_bound_check with its bound, one sample's knowledge base scaled by 1e-3.
tests/test_fp8_bounds.py shows on the CPU, with this file's references, that emulations of mac_linear_fp8_fwd under the
model of (1) and of the read step in the exact regime pass (2)'s and (5)'s bounds, and that planted faults fail them by
at least 100x.
Each bar is about three times the worst value measured on an H100 80GB HBM3 (700 W power limit), written beside it."""
import ctypes

import pytest
import torch

from mac_network_b200 import _lib as L_
from oracle import fp8_read_oracle as F8
from oracle import fp8_stem_oracle as F8S
from tests.test_gpu_read_step_bounds import EPS_ELU, FILL, GAMMA, U32, add_fp8_packs, bits, inv_views, rows_over
from tests.test_gpu_wgmma import align1k, elu, gen, lib, nanfill, randn, read_setup, softmax_bound_check

pytestmark = pytest.mark.gpu

D = 512
FP8 = 3
ACT = {"NON": 0, "ELU": 3, "RELU": 4}        # MAC_ACT_NON, MAC_ACT_ELU, MAC_ACT_RELU (Stem(relu="RELU") launches 4)
# per k32 instruction, of |running sum entering it| + sum of |its 32 products| (see (1))             measured
TOL_E4M3 = 1.25e-3                                                     # 4.2e-4 (K = 128, one 448 among small values)
E4M3_CHAIN_STEM = 4                          # instructions per accumulator chain: one 128-wide k-block (tc_gemm_fp8.cuh)
E4M3_CHAIN_READ = 16                         # the read step: one chain over K = 512 (read_step_fp8.cuh)


# ------------------------------------------------------------------------------------------------ the model and references
def acc_terms(A, B, chain):
    """The model's two parts for e4m3 values A [M, K], B [N, K] (fp64), chains of `chain` k32 instructions along K:
    (T, F) with |acc - A @ B.T| <= TOL_E4M3 * T + F.  T = sum over instructions of (|exact running sum entering it| +
    sum of |its 32 products|) = |A| @ |B| + the chain's |running sums| at every instruction boundary inside it; F = 2^-24
    of |master accumulator| after each chain's fp32 add past the first (the stem's two-level sum; 0 for a single chain)."""
    T = A.abs() @ B.abs().T
    F = torch.zeros_like(T)
    S, master = torch.zeros_like(T), torch.zeros_like(T)
    for i in range(A.shape[1] // 32):
        S = S + A[:, 32 * i:32 * i + 32] @ B[:, 32 * i:32 * i + 32].T
        if (i + 1) % chain:
            T = T + S.abs()
        else:
            master = master + S
            if i + 1 > chain:
                F = F + U32 * master.abs()
            S = torch.zeros_like(T)
    return T, F


def acc_bound(A, B, chain, tol=None):
    """Bound on |acc - A @ B.T| (acc_terms)"""
    T, F = acc_terms(A, B, chain)
    return (TOL_E4M3 if tol is None else tol) * T + F


def act_ref(act, x):
    return elu(x) if act == "ELU" else torch.relu(x) if act == "RELU" else x


def linear_reference(A8, sa, W8, sw, b, act, tol=None):
    """mac_linear_fp8_fwd's reference and bound per element: A8 [M, K], W8 [N, K] e4m3 values (fp64), fp32 sa [M],
    sw [N], b [N] or None.  Returns (act(A8 @ W8.T * sa * sw + b), bound), fp64 [M, N]."""
    acc = A8 @ W8.T
    E = acc_bound(A8, W8, E4M3_CHAIN_STEM, tol)
    sc = sa.double()[:, None] * sw.double()[None, :]
    x = acc * sc
    if b is not None:
        x = x + b.double()[None, :]
    lin = sc * (E + 2.001 * U32 * (acc.abs() + E))                  # the accumulator, then acc * sa * sw in fp32
    e = lin + 1.001 * U32 * (x.abs() + lin) + 2.0 ** -140            # the bias add (or the product's last rounding)
    if act == "ELU":
        e = e + EPS_ELU                                               # elu_fast; ELU and ReLU are 1-Lipschitz
    return act_ref(act, x), e


def step_operands(P8, sP, y, N):
    """(A8, rf) as the e4m3 read step forms them, in fp32 on the CPU: A8 = e4m3(P8 * fp32(y_b * fp32(1 / ay_b))) (fp64
    values) and rf = fp32(sP_r * ay_b), GEMM 1's row scale."""
    P8, sP, y = P8.double().cpu(), sP.float().cpu(), y.float().cpu()
    A8 = F8.a8_f32(P8, y, N)
    ay = y.abs().amax(1).repeat_interleave(N)
    return A8, (sP * ay).double()


def fp8_step_reference(A8, rf, Q16, cb, W1, s1, W2, s2, bm2, wr, tol=None):
    """The e4m3 read step's logits (I2 . wr, without br) and their bound, one per row (see (4) of the module docstring).
    A8 [R, d] e4m3 values and rf [R] from step_operands; Q16 [R, d] bf16; cb [R, d] each row's control; W1, W2 [out, in]
    e4m3 values (fp64) of the packs of Wm[0:d] and Wm2 with their fp32 column scales s1, s2 [d]; bm2, wr [d] fp32.
    Everything on W1's device.  Returns (logit*, bound, |I2*| . |wr|), fp64 [R]."""
    tol = TOL_E4M3 if tol is None else tol
    dev = W1.device
    A8, rf, Qd, cd = A8.to(dev), rf.to(dev)[:, None], Q16.double().to(dev), cb.double().to(dev)
    # GEMM 1 and its epilogue
    acc1 = A8 @ W1.T
    E1 = acc_bound(A8, W1, E4M3_CHAIN_READ, tol)
    sc1 = rf * s1.double()[None, :]
    x = acc1 * sc1 + Qd
    Hs = elu(x)
    lin = sc1 * (E1 + 2.001 * U32 * (acc1.abs() + E1))
    e = lin + 1.001 * U32 * (x.abs() + lin) + EPS_ELU
    # the row amax, 448 / am and am / 448 as intervals; H8 between the roundings of its product interval's ends
    am = Hs.abs().amax(1, keepdim=True)
    am_lo = (Hs.abs() - e).amax(1, keepdim=True).clamp_min(0)
    am_hi = (Hs.abs() + e).amax(1, keepdim=True)
    big = torch.full_like(am, 1e30)
    i_lo = torch.where(am_lo > 0, 448.0 / am_hi * (1 - 2.0 ** -23), torch.zeros_like(am))
    i_hi = torch.where(am_lo > 0, 448.0 / am_lo.clamp_min(1e-300) * (1 + 2.0 ** -23), big)
    H8 = F8.e4m3(Hs * torch.where(am > 0, 448.0 / am.clamp_min(1e-300), torch.zeros_like(am)))
    corners = torch.stack([(Hs - e) * i_lo, (Hs - e) * i_hi, (Hs + e) * i_lo, (Hs + e) * i_hi])
    lo, hi = F8.e4m3(corners.amin(0)).to(dev), F8.e4m3(corners.amax(0)).to(dev)
    H8 = H8.to(dev)
    dH8 = torch.maximum(hi - H8, H8 - lo)
    sh = am / 448.0
    dsh = torch.maximum(am_hi / 448.0 * (1 + 2.0 ** -23) - sh, sh - am_lo / 448.0 * (1 - 2.0 ** -23))
    # GEMM 2 and its epilogue
    acc2 = H8 @ W2.T
    # the kernel's H8 moves each running sum of the chain by at most dH8 @ |W2|
    D2 = (1 + E4M3_CHAIN_READ * tol) * (dH8 @ W2.abs().T) + acc_bound(H8, W2, E4M3_CHAIN_READ, tol)
    s2d = s2.double()[None, :]
    I1 = acc2 * sh * s2d + bm2.double()[None, :]
    dI1 = s2d * ((sh + dsh) * D2 + dsh * acc2.abs())
    dI1 = dI1 + 2.001 * U32 * s2d * (sh + dsh) * (acc2.abs() + D2)
    dI1 = dI1 + 1.001 * U32 * (I1.abs() + dI1)
    I2 = elu(I1 * cd)
    dI2 = cd.abs() * dI1 + U32 * cd.abs() * (I1.abs() + dI1) + EPS_ELU
    wrd = wr.double()
    return I2 @ wrd, dI2 @ wrd.abs() + GAMMA * ((I2.abs() + dI2) @ wrd.abs()), I2.abs() @ wrd.abs()


# ------------------------------------------------------------------------------------------------ plumbing
def _e4m3(u8):
    return u8.view(torch.float8_e4m3fn).double()


def _bytes(v):
    """e4m3 values (fp64) -> their bytes"""
    return v.float().to(torch.float8_e4m3fn).view(torch.uint8)


def _pack8(W):
    o = torch.empty((W.shape[1], W.shape[0]), dtype=torch.uint8, device="cuda")
    s = torch.empty(W.shape[1], dtype=torch.float32, device="cuda")
    L_.check(lib().mac_pack_weight_fp8(L_.ptr(W), L_.ptr(o), L_.ptr(s), W.shape[0], W.shape[1], L_.stream_ptr()), "pack8")
    return o, s


GUARD = 1024


def linear8(cols, sa, W8, sw, b, act):
    """mac_linear_fp8_fwd into a NaN-filled buffer with GUARD NaNs behind its M * N outputs: (y [M, N], the guard)"""
    M, K = cols.shape
    N = W8.shape[0]
    buf = torch.full((M * N + GUARD,), float("nan"), device="cuda")
    L_.check(lib().mac_linear_fp8_fwd(L_.ptr(cols), L_.ptr(sa), L_.ptr(W8), L_.ptr(sw), L_.ptr(b), ACT[act], L_.ptr(buf), M,
                                      K, N, L_.stream_ptr()), "mac_linear_fp8_fwd")
    return buf[:M * N].view(M, N), buf[M * N:]


def _ratio(got, ref, bound):
    """max |got - ref| / bound (an exact match where the bound is 0 counts 0)"""
    err = (got.double() - ref).abs()
    return float(torch.where(err == 0, torch.zeros_like(err), err / bound).max())


# ================================================================================================ 1. the accumulator
def _codes(g, shape, lo, hi):
    """random e4m3 bytes with magnitude codes in [lo, hi] (0x01-0x07 subnormal, 0x38 = 1, 0x7E = 448) and random signs"""
    c = torch.randint(lo, hi + 1, shape, device="cuda", generator=g, dtype=torch.int32)
    s = torch.randint(0, 2, shape, device="cuda", generator=g, dtype=torch.int32) * 0x80
    return (c | s).to(torch.uint8)


def adversarial_operands(K, seed):
    """A [640, K] in five 128-row patterns and W [256, K] in three column patterns (e4m3 bytes):
    A: the whole finite range; small values with one +-448 per 32-group; cancelling pairs (k, k+1) = (v, -v) of large v
       between small values; subnormals only; each 32-group a ramp from 2^8 down into the subnormals.
    W: +1 everywhere; one random power of two per pair (k, k+1) (pairs stay cancelling); the whole finite range."""
    g = gen(seed)
    full = _codes(g, (128, K), 0x00, 0x7E)
    one_big = _codes(g, (128, K), 0x08, 0x30).view(128, K // 32, 32)
    pos = torch.randint(0, 32, (128, K // 32, 1), device="cuda", generator=g)
    one_big.scatter_(2, pos, _codes(g, (128, K // 32, 1), 0x7E, 0x7E))
    cancel = _codes(g, (128, K), 0x01, 0x30).view(128, K // 32, 32)
    big = _codes(g, (128, K // 32, 8), 0x60, 0x7E)
    cancel[:, :, 0:16:2], cancel[:, :, 1:16:2] = big, big ^ 0x80
    sub = _codes(g, (128, K), 0x01, 0x07)
    j = torch.arange(32, device="cuda", dtype=torch.int32)
    ramp_code = (0x78 - 4 * j).clamp_min(0x01)                     # 2^8 down by half a binade per element
    ramp = (ramp_code.repeat(K // 32)[None, :] ^ (_codes(g, (128, K), 0, 0).to(torch.int32) & 0x80)).to(torch.uint8)
    A = torch.cat([full, one_big.view(128, K), cancel.view(128, K), sub, ramp]).contiguous()
    ones = torch.full((64, K), 0x38, dtype=torch.uint8, device="cuda")
    pw = _codes(g, (64, K // 2), 0x08, 0x70) & 0xF8                  # +-powers of two, 2^-6 .. 2^7
    pw = pw.repeat_interleave(2, 1)
    W = torch.cat([ones, pw, _codes(g, (128, K), 0x00, 0x7E)]).contiguous()
    return A, W


ACC_K = [128, 1152, 9216]
PATTERNS = ["full range", "one 448 per group", "cancelling", "subnormal", "ramp"]


@pytest.mark.parametrize("K", ACC_K)
def test_e4m3_accumulator_error_model(K):
    """The raw accumulator of mac_linear_fp8_fwd (sa = sw = 1, no bias, NON) against fp64 of its e4m3 operands, within the
    model of (1).  K = 128 is one chain of four instructions into a zero accumulator; longer K adds the fp32 master adds."""
    A, W = adversarial_operands(K, 9000 + K)
    Ad, Wd = _e4m3(A), _e4m3(W)
    M, N = A.shape[0], W.shape[0]
    ones_m, ones_n = torch.ones(M, device="cuda"), torch.ones(N, device="cuda")
    y, guard = linear8(A, ones_m, W, ones_n, None, "NON")
    torch.cuda.synchronize()
    assert bool(torch.isnan(guard).all()) and bool(torch.isfinite(y).all())
    ref = Ad @ Wd.T
    S, add = acc_terms(Ad, Wd, E4M3_CHAIN_STEM)
    err = ((y.double() - ref).abs() - add).clamp_min(0)
    assert bool((err[S == 0] == 0).all())
    r = torch.where(S > 0, err / S.clamp_min(1e-300), torch.zeros_like(S))
    worst = {p: float(r[128 * i:128 * (i + 1)].max()) for i, p in enumerate(PATTERNS)}
    print("e4m3 accumulator K=%d: worst error / the model's sum (acc_terms) by pattern %s; TOL_E4M3 = %.3e"
          % (K, {p: "%.3e" % v for p, v in worst.items()}, TOL_E4M3))
    assert max(worst.values()) <= TOL_E4M3, worst


# ================================================================================================ 2. mac_linear_fp8_fwd
# (M, K / 128, N, act, bias): M at tile edges and the stem's 7x7 / 14x14 batch-64 counts; k-block counts around the
# 6-stage ring, K = 9216 (1024 channels) and 18432 (GQA's 2048-channel layer 0); every act with and without a bias
LINEAR = [(1, 1, 128, "NON", False), (63, 2, 256, "ELU", True), (64, 5, 128, "RELU", True), (65, 6, 512, "NON", True),
          (127, 7, 128, "ELU", False), (128, 12, 256, "RELU", False), (129, 13, 128, "NON", True),
          (3136, 72, 128, "ELU", True), (12544, 72, 512, "NON", False), (12545, 144, 128, "RELU", True),
          (65, 144, 256, "ELU", False), (12545, 1, 256, "RELU", False)]


@pytest.mark.parametrize("M,KB,N,act,bias", LINEAR)
def test_linear_fp8_every_output_against_fp64(M, KB, N, act, bias):
    K = 128 * KB
    g = gen(M * 7 + KB * 131 + N)
    X = randn(g, M, K) * torch.exp2(torch.rand(M, 1, device="cuda", generator=g) * 40 - 20)
    if M > 1:
        X[M // 2] = 0                                               # sa = 0: y = act(b)
    A8, sa = F8.quant_rows_f32(X)
    cols = _bytes(A8).contiguous()
    Wf = randn(g, K, N, scale=K ** -0.5)
    Wf[:, 5] = 0                                                    # sw = 0
    Wf[:, 9] *= 2.0 ** -20
    W8, sw = _pack8(Wf)
    b = randn(g, N, scale=0.5) if bias else None
    y, guard = linear8(cols, sa, W8, sw, b, act)
    y2, _ = linear8(cols, sa, W8, sw, b, act)
    torch.cuda.synchronize()
    assert bool(torch.isnan(guard).all()), "written past M * N (rows past M of the last tile stored?)"
    assert bool(torch.isfinite(y).all()), "an output left unwritten or non-finite"
    assert torch.equal(bits(y), bits(y2)), "a rerun gave different bits"
    assert float(sw[5]) == 0.0 and (M == 1 or float(sa[M // 2]) == 0.0)
    ref, bound = linear_reference(A8, sa, _e4m3(W8), sw, b, act)
    r = _ratio(y, ref, bound)
    print("mac_linear_fp8_fwd M=%d K=%d N=%d %s bias=%s: worst |y - ref| / bound %.3f" % (M, K, N, act, bias, r))
    assert r <= 1, r


# ================================================================================================ 3. Stem(prec="fp8")
@pytest.mark.parametrize("relu", ["RELU", "ELU"])
@pytest.mark.parametrize("B,C,out", [(2, 128, 128), (64, 2048, 512)])
def test_stem_fp8_layer_by_layer(B, C, out, relu):
    """7x7 grids: C = 128 and GQA's 2048 channels, 2 layers.  Each layer: mac_im2col3x3_fp8's bytes and scales, the weight
    pack and its scales bit for bit against the fp32 restatements; the GEMM's every output within (2); the Stem's output
    bit for bit the layer chain's."""
    from mac_network_b200.stem import Stem, init_stem_params, stem_specs
    from tests.test_gpu_stem_fp8 import _im2col8
    p = {k: torch.from_numpy(v).cuda() for k, v in init_stem_params(stem_specs(C, out), seed=C + len(relu)).items()}
    st = Stem(p, relu=relu, prec="fp8")
    g = gen(C + 3)
    x = elu(randn(g, B, 7, 7, C))
    kb = st.forward(x)
    act = {MAC: name for name, MAC in ACT.items()}[st._act()]
    worst = []
    for i in range(st.nlayers):
        Wf, (W8, sw) = st._weights(i)
        cols, sa = _im2col8(x)
        torch.cuda.synchronize()
        cols_ref, sa_ref = F8S.quant_patches(x.cpu())
        assert torch.equal(cols.cpu(), _bytes(cols_ref)) and torch.equal(bits(sa.cpu()), bits(sa_ref)), ("patches", i)
        W8_ref, sw_ref = F8.pack_weight_f32(Wf.cpu())
        assert torch.equal(W8.cpu(), _bytes(W8_ref.T.contiguous())) and torch.equal(bits(sw.cpu()), bits(sw_ref)), ("pack", i)
        y, guard = linear8(cols, sa, W8, sw, st._bias(i), act)
        torch.cuda.synchronize()
        assert bool(torch.isnan(guard).all()) and bool(torch.isfinite(y).all())
        ref, bound = linear_reference(_e4m3(cols), sa, _e4m3(W8), sw, st._bias(i), act)
        worst.append(_ratio(y, ref, bound))
        x = y.view(B, 7, 7, -1)
    print("Stem(prec='fp8', relu=%s) B=%d C=%d: worst |y - ref| / bound per layer %s" % (relu, B, C, worst))
    assert max(worst) <= 1, worst
    assert torch.equal(bits(kb.reshape(-1)), bits(x.reshape(-1))), "the Stem's output differs from its layer chain's"


# ================================================================================================ 4. the read step's logits
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# B*N at 64-row tile edges (1, 63, 64, 65, 127, 128, 129); N = 1, 2, 3 and 31, so tiles hold third and later samples whose
# y and control come from global memory; N = 49, 196, 255, 256; GQA 64 x 49, headline 64 x 196; 2 * SMs + 1 tiles
STEP_SHAPES = [(1, 1), (21, 3), (32, 2), (65, 1), (127, 1), (1, 128), (43, 3), (7, 31), (3, 255), (2, 256), (5, 49),
               (64, 49), (64, 196), ("2sms+1", 64)]
SPECIAL = {(43, 3), (7, 31), (64, 49)}


def special_samples(W, kb16, y, c):
    """In place: bx = 0; sample 2 (the third of tile 0 when N <= 31) y = 0; sample 3 one y element 1e4 times the rest;
    sample 4 control = 0; sample 5 knowledge base scaled by 1e-3; sample 6's first rows zero (P = 0, sP = 0)"""
    W["bx"].zero_()
    y[2] = 0
    y[3] *= 1e-4
    y[3, 17] = 1.0
    c[4] = 0
    kb16[5] = (kb16[5].float() * 1e-3).to(torch.bfloat16)
    kb16[6, :2] = 0


@pytest.mark.parametrize("B,N", STEP_SHAPES)
def test_fp8_read_step_logits_row_by_row(B, N):
    if B == "2sms+1":
        B = 2 * _sms() + 1
    lb = lib()
    M = B * N
    g, W, Pk, _, rw = read_setup(D, 11 * B + N)
    keep = add_fp8_packs(W, rw)
    W1b, s1, W2b, s2 = keep
    kb16 = elu(randn(g, B, N, D)).to(torch.bfloat16)
    y, c = randn(g, B, D), randn(g, B, D)
    if (B, N) in SPECIAL:
        special_samples(W, kb16, y, c)
    kb0, y0, c0 = kb16.clone(), y.clone(), c.clone()
    nb = lb.mac_read_invariant_bytes(B, N, D, FP8)
    inv = torch.full((nb,), FILL, dtype=torch.uint8, device="cuda")
    L_.check(lb.mac_read_invariant(None, L_.ptr(kb16), ctypes.byref(rw), FP8, L_.ptr(inv), nb, B, N, D, L_.stream_ptr()),
             "mac_read_invariant")
    P, Q, lg, end = inv_views(inv, FP8, B, N)
    io = align1k(inv)
    P8, sP = inv[io:io + M * D].view(M, D), inv[io + ((M * D + 1023) & ~1023):][:4 * M].view(torch.float32)
    torch.cuda.synchronize()
    inv0 = inv.clone()
    # the invariant's quantisation bit for bit
    P8_ref, sP_ref = F8.quant_rows_f32(P.float().cpu())
    assert torch.equal(P8.cpu(), _bytes(P8_ref)) and torch.equal(bits(sP.cpu()), bits(sP_ref)), "P8 / sP"
    wsb = lb.mac_read_workspace_bytes(B, N, D, FP8)
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    info, att = nanfill(B, D), nanfill(B, N)
    L_.check(lb.mac_read_fwd_inv(None, L_.ptr(kb16), L_.ptr(inv), L_.ptr(y), L_.ptr(y), L_.ptr(c), ctypes.byref(rw), FP8,
                                 L_.ptr(info), L_.ptr(att), L_.ptr(ws), wsb, B, N, D, L_.stream_ptr()), "mac_read_fwd_inv")
    torch.cuda.synchronize()
    # canaries: only the M logits of `inv` change; the inputs are unchanged
    o_lg = end - 4 * M
    changed = torch.nonzero(inv != inv0).flatten()
    assert bool(((changed >= o_lg) & (changed < end)).all()), "the step wrote `inv` outside its M logits"
    assert bool((inv[end:o_lg + ((4 * M + 1023) & ~1023)] == FILL).all()), "bytes behind the M logits written"
    for name, now, was in (("kb", kb16, kb0), ("y", y, y0), ("control", c, c0)):
        assert torch.equal(bits(now), bits(was)), "%s changed by the step" % name
    assert bool(torch.isfinite(lg).all()), "non-finite logit"
    A8, rf = step_operands(P8.view(torch.float8_e4m3fn), sP, y, N)
    ref, bound, _ = fp8_step_reference(A8, rf, Q, c.repeat_interleave(N, 0), _e4m3(W1b), s1, _e4m3(W2b), s2, W["bm2"],
                                       W["wr"])
    r = float(((lg.double() - ref).abs() / bound).max())
    ra, ri = softmax_bound_check(att, info, ref + 0.25, bound + 1e-6 * ((ref + 0.25).abs() + 1), kb16, B, N)
    print("e4m3 read step B=%d N=%d: logits use %.3f of their bound (median bound %.2e), att %.3f, info %.3f"
          % (B, N, r, float(bound.median()), ra, ri))
    assert r <= 1, rows_over(lg, ref, bound, N)
    assert ra <= 1 and ri <= 1, (ra, ri)


# ================================================================================================ 5. the read step, exact regime
# Operands on which every accumulator of the e4m3 read step is exact, so its logits are known to fp32 summation order:
# P8 in {0, +-1, +-2}, y_b = 2^k_b (so y_b / ay_b = 1 and A8 = P8), W1 and W2 in {0, +-1} (a quarter nonzero).  GEMM 1's
# products are integers and its sums stay below 2^9.  H = acc1 * rf * sW1 + Q, with power-of-two rf * sW1 <= 1/4 and Q in
# [64, 128), lies in (48, 144), so H8 = e4m3(H * 448 / am) lies in [128, 448] (multiples of 16) and GEMM 2's sums stay
# below 128 * 448 < 2^16: an accumulator that keeps 13 bits below its largest addend's leading bit holds them exactly
# (part 1 measures about that).  Every scale but sh is a power of two, so no product rounds and fused or separate
# multiply-adds give the same fp32 values.  Q and control are positive and bm2 just large enough for every I1 to be, so
# both ELUs take their exact x > 0 branch.  What is left is the order of the fp32 logit sum (GAMMA).  A wrong row scale,
# sample, column-scale half, amax half or k32 instruction moves a logit 1000 times further (tests/test_fp8_bounds.py).
def exact_operands(B, N, seed):
    """CPU operands of the exact regime: P8, W1, W2 e4m3 values (fp64; W [out, in]); sP, s1, s2, y, c, bm2, wr fp32; Q bf16"""
    g = torch.Generator().manual_seed(seed)
    M = B * N
    ri = lambda *s, lo, hi: torch.randint(lo, hi, s, generator=g)
    P8 = (ri(M, D, lo=-2, hi=3)).double()
    sparse = lambda: (ri(D, D, lo=-1, hi=2) * (ri(D, D, lo=0, hi=4) == 0)).double()
    pow2 = lambda n, lo, hi: torch.exp2(-ri(n, lo=lo, hi=hi).float())
    o = dict(P8=P8, sP=pow2(M, 3, 6), Q=(64 + 64 * torch.rand(M, D, generator=g)).to(torch.bfloat16),
             y=torch.exp2((torch.arange(B) % 3).float())[:, None].expand(B, D).contiguous(),
             c=0.5 + torch.rand(B, D, generator=g), W1=sparse(), s1=pow2(D, 1, 3), W2=sparse(), s2=pow2(D, 4, 6),
             bm2=torch.zeros(D), wr=torch.randn(D, generator=g) * 4 * D ** -0.5, B=B, N=N)
    # bm2 just large enough that every I1 is positive
    I1 = exact_step(dict(o, c=torch.ones(B, D)))
    o["bm2"] = (1 - I1.amin(0)).clamp_min(1).float()
    return o


def exact_step(o, fault=None):
    """The read step's fp32 arithmetic on exact-regime operands with exact accumulators: I2 [M, d] fp32, and with `fault`
    one of EXACT_FAULTS planted"""
    B, N = o["B"], o["N"]
    M = B * N
    rows = torch.arange(M)
    s = rows // N
    y = o["y"]
    ay = y.abs().amax(1)
    iay = torch.ones_like(ay) / ay
    sc = iay[s]
    if fault == "third sample scaled by the first's ay":
        s_lo = (rows // 64 * 64) // N
        sc = torch.where(s - s_lo >= 2, iay[s_lo], sc)
    A8 = F8.e4m3(o["P8"].float() * (y[s] * sc[:, None]))
    sP = o["sP"][(rows + 1).clamp_max(M - 1)] if fault == "sP of the next row" else o["sP"]
    s1 = torch.cat([o["s1"][256:], o["s1"][:256]]) if fault == "sW1 halves swapped" else o["s1"]
    if fault == "one k32 instruction dropped":
        A8 = A8.clone()
        A8[:, 32:64] = 0
    acc1 = (A8 @ o["W1"].T).float()
    H = (acc1 * (sP * ay[s])[:, None]) * s1[None, :] + o["Q"].float()
    am = (H[:, :256] if fault == "H8 scaled by one half's amax" else H).abs().amax(1, keepdim=True)
    H8 = F8.e4m3(H * (torch.full_like(am, 448.0) / am))
    acc2 = (H8 @ o["W2"].T).float()
    I1 = (acc2 * (am / torch.full_like(am, 448.0))) * o["s2"][None, :] + o["bm2"][None, :]
    return I1 * o["c"][s]


def exact_reference(I2, wr):
    """(logits, bound): the fp64 sum of the fp32 I2 * wr and GAMMA of the absolute sum (the kernel's fmaf chains, two
    shuffle adds and the halves' add)"""
    I2, wr = I2.double(), wr.double()
    return I2 @ wr, GAMMA * (I2.abs() @ wr.abs()) + 1e-30


@pytest.mark.parametrize("B,N", [(1, 1), (43, 3), (7, 31), (64, 49), (3, 255), ("2sms+1", 64)])
def test_fp8_read_step_exact_regime_logits(B, N):
    """The read step through mac_read_fwd_inv on exact-regime operands written straight into `inv` and the packs: every
    logit within GAMMA of exact_step's, att and info through softmax_bound_check with that bound (one sample's knowledge
    base scaled by 1e-3, so its info is checked at its own scale); the logits' `inv` padding keeps its fill."""
    if B == "2sms+1":
        B = 2 * _sms() + 1
    lb = lib()
    M = B * N
    o = exact_operands(B, N, 17 * B + N)
    I2 = exact_step(o)
    assert bool((I2 > 0).all())
    ref, bound = exact_reference(I2, o["wr"])
    g, W, Pk, _, rw = read_setup(D, 5 * B + N)
    W["bm2"].copy_(o["bm2"])
    W["wr"].copy_(o["wr"])
    packs = [_bytes(o["W1"]).cuda(), o["s1"].cuda(), _bytes(o["W2"]).cuda(), o["s2"].cuda()]
    rw.Wm_fp8, rw.Wm_fp8_scale, rw.Wm2_fp8, rw.Wm2_fp8_scale = [t.data_ptr() for t in packs]
    kb16 = elu(randn(g, B, N, D)).to(torch.bfloat16)
    kb16[B // 2] = (kb16[B // 2].float() * 1e-3).to(torch.bfloat16)
    nb = lb.mac_read_invariant_bytes(B, N, D, FP8)
    inv = torch.full((nb,), FILL, dtype=torch.uint8, device="cuda")
    io = align1k(inv)
    al = lambda n: (n + 1023) & ~1023
    inv[io:io + M * D].copy_(_bytes(o["P8"]).view(-1))
    inv[io + al(M * D):io + al(M * D) + 4 * M].copy_(o["sP"].view(torch.uint8))
    o_Q = io + al(M * D) + al(M * 4)
    inv[o_Q:o_Q + 2 * M * D].copy_(o["Q"].view(-1).view(torch.uint8))
    o_lg = o_Q + al(2 * M * D)
    y, c = o["y"].cuda(), o["c"].cuda()
    wsb = lb.mac_read_workspace_bytes(B, N, D, FP8)
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    info, att = nanfill(B, D), nanfill(B, N)
    L_.check(lb.mac_read_fwd_inv(None, L_.ptr(kb16), L_.ptr(inv), L_.ptr(y), L_.ptr(y), L_.ptr(c), ctypes.byref(rw), FP8,
                                 L_.ptr(info), L_.ptr(att), L_.ptr(ws), wsb, B, N, D, L_.stream_ptr()), "mac_read_fwd_inv")
    torch.cuda.synchronize()
    lg = inv[o_lg:o_lg + 4 * M].view(torch.float32).cpu()
    assert bool((inv[o_lg + 4 * M:o_lg + al(4 * M)] == FILL).all()), "bytes behind the M logits written"
    r = float(((lg.double() - ref).abs() / bound).max())
    ra, ri = softmax_bound_check(att, info, (ref + 0.25).cuda(), (bound + 1e-6 * ((ref + 0.25).abs() + 1)).cuda(), kb16,
                                 B, N)
    print("e4m3 read step, exact regime, B=%d N=%d: logits use %.3f of GAMMA's bound (median %.2e), att %.3f, info %.3f"
          % (B, N, r, float(bound.median()), ra, ri))
    assert r <= 1, rows_over(lg, ref, bound, N)
    assert ra <= 1 and ri <= 1, (ra, ri)
