"""CPU checks of tests/test_gpu_fp8_kernels.py's references and bounds, with that file's own code.

The stem GEMM: an emulation of linear_fp8_kernel's arithmetic in torch -- each k32 instruction off by a random error
inside the model of TOL_E4M3 (its running sum entering it plus the sum of its 32 |products|), a fresh chain per 128-wide
k-block added into an fp32 master accumulator, then acc * sa * sw + b in fp32 and the activation (elu_fast with ex2
carrying a +-2^-22 relative error) -- passes the element-wise bound, and each of these planted faults is rejected by at
least 100x: sa taken from the next row, a k-block dropped, a k-block read twice (the ring's phase off by one), the bias
added twice, RELU computed as ELU.

The read step on exact-regime operands (test_gpu_fp8_kernels part 5): the kernel's fp32 arithmetic with its own order of
the logit sum passes the bound, and each of these planted faults is rejected by at least 100x, with tiles that hold third
and later samples: sP taken from the next row, a third sample scaled by the first sample's ay, sW1's two warpgroup halves
swapped, H8 scaled by one half's amax, one k32 instruction dropped.  A row past M written is caught by the canary on the
bytes behind the logits.  And a sample scaled by 1e-3 whose info is wholly wrong passes the read step's max-norm check
over the batch (test_gpu_read_step_fp8) but not the softmax bound that the exact-regime check feeds."""
import pytest
import torch

from oracle import fp8_read_oracle as F8
from tests.test_gpu_fp8_kernels import (E4M3_CHAIN_STEM, TOL_E4M3, exact_operands, exact_reference, exact_step,
                                         linear_reference)
from tests.test_read_step_bounds import _elu_fast

MARGIN = 100


def _operands(M, K, N, seed):
    """e4m3 values A [M, K] with row scales 2^U(-20, 20), an all-zero row; W [N, K] packed from K^-1/2 normals with an
    all-zero column; a bias"""
    g = torch.Generator().manual_seed(seed)
    X = torch.randn(M, K, generator=g) * torch.exp2(torch.rand(M, 1, generator=g) * 40 - 20)
    X[M // 2] = 0
    A8, sa = F8.quant_rows_f32(X)
    Wf = torch.randn(K, N, generator=g) * K ** -0.5
    Wf[:, 3] = 0
    W8, sw = F8.pack_weight_f32(Wf)
    return A8, sa, W8.T.contiguous(), sw, torch.randn(N, generator=g) * 0.5, g


def emulate(A8, sa, W8, sw, b, act, g, fault=None):
    """linear_fp8_kernel's output in torch arithmetic with an optional planted fault"""
    M, K = A8.shape
    kblocks = K // 128
    blocks = list(range(kblocks))
    if fault == "kblock dropped":
        blocks.remove(1)
    elif fault == "kblock read twice":
        blocks[1] = 0
    master = torch.zeros(M, W8.shape[0], dtype=torch.float32)
    for kb in blocks:
        S = torch.zeros(M, W8.shape[0], dtype=torch.float64)
        for i in range(E4M3_CHAIN_STEM):
            k0 = kb * 128 + 32 * i
            a, w = A8[:, k0:k0 + 32], W8[:, k0:k0 + 32]
            size = S.abs() + a.abs() @ w.abs().T
            u = torch.rand(S.shape, generator=g, dtype=torch.float64) * 2 - 1
            S = (S + a @ w.T + 0.9 * TOL_E4M3 * size * u).float().double()
        master = master + S.float()
    sa_used = torch.roll(sa, -1) if fault == "sa of the next row" else sa
    x = master * sa_used[:, None] * sw[None, :]
    x = x + b[None, :]
    if fault == "bias twice":
        x = x + b[None, :]
    if act == "ELU" or fault == "RELU as ELU":
        return _elu_fast(x, g)
    return torch.relu(x) if act == "RELU" else x


def _ratio(got, ref, bound):
    err = (got.double() - ref).abs()
    return float(torch.where(err == 0, torch.zeros_like(err), err / bound).max())


@pytest.mark.parametrize("act", ["NON", "ELU", "RELU"])
def test_emulated_linear_passes_the_bound(act):
    A8, sa, W8, sw, b, g = _operands(96, 768, 128, 1)
    ref, bound = linear_reference(A8, sa, W8, sw, b, act)
    r = _ratio(emulate(A8, sa, W8, sw, b, act, g), ref, bound)
    assert r <= 1, r


@pytest.mark.parametrize("fault,act", [("sa of the next row", "NON"), ("kblock dropped", "NON"),
                                       ("kblock read twice", "ELU"), ("bias twice", "RELU"), ("RELU as ELU", "RELU")])
def test_bound_rejects_a_planted_fault(fault, act):
    A8, sa, W8, sw, b, g = _operands(256, 256, 256, 2)
    ref, bound = linear_reference(A8, sa, W8, sw, b, act)
    r = _ratio(emulate(A8, sa, W8, sw, b, act, g, fault), ref, bound)
    assert r >= MARGIN, (fault, r)


# ------------------------------------------------------------------------------------------------ the read step, exact regime
READ_FAULTS = ["sP of the next row", "third sample scaled by the first's ay", "sW1 halves swapped",
               "H8 scaled by one half's amax", "one k32 instruction dropped"]


def kernel_logit_sum(I2, wr):
    """read_step_fp8_kernel's fp32 logit sum: per row, each of the 8 threads (2 warpgroups x 4 lanes) runs 64 fmaf over
    columns 256 g + 8 j + 2 t + e, then two shuffle adds and half 0 + half 1"""
    I2, wr = I2.double(), wr.double()
    f32 = lambda x: x.float().double()
    halves = []
    for g_ in range(2):
        parts = []
        for t in range(4):
            part = torch.zeros(I2.shape[0], dtype=torch.float64)
            for j in range(32):
                for e in range(2):
                    n = 256 * g_ + 8 * j + 2 * t + e
                    part = f32(I2[:, n] * wr[n] + part)
            parts.append(part)
        halves.append(f32(f32(parts[0] + parts[1]) + f32(parts[2] + parts[3])))
    return f32(halves[0] + halves[1]).float()


def _read_case(B, N, seed):
    o = exact_operands(B, N, seed)
    ref, bound = exact_reference(exact_step(o), o["wr"])
    return o, ref, bound


@pytest.mark.parametrize("B,N", [(43, 3), (7, 31), (8, 49)])
def test_emulated_read_step_passes_the_exact_bound(B, N):
    o, ref, bound = _read_case(B, N, 17 * B + N)
    r = _ratio(kernel_logit_sum(exact_step(o), o["wr"]), ref, bound)
    assert r <= 1, r


@pytest.mark.parametrize("fault", READ_FAULTS)
@pytest.mark.parametrize("B,N", [(43, 3), (7, 31)])
def test_exact_bound_rejects_a_planted_read_fault(fault, B, N):
    """N = 3 and 31: 64-row tiles hold third and later samples, which the kernel scales from global memory"""
    o, ref, bound = _read_case(B, N, 17 * B + N)
    r = _ratio(kernel_logit_sum(exact_step(o, fault), o["wr"]), ref, bound)
    assert r >= MARGIN, (fault, r)


def test_canary_rejects_a_row_past_m():
    """The GPU tests fill the bytes behind the M logits and require them unchanged: a last tile that stores its rows past M
    (here row M, computed from the clamped row M - 1) fails that, a correct one does not."""
    B, N = 43, 3
    o, ref, _ = _read_case(B, N, 9)
    M = B * N
    lg = kernel_logit_sum(exact_step(o), o["wr"])
    for fault in (False, True):
        buf = torch.full((M + 64,), float("nan"))
        rows = M + 1 if fault else M
        buf[:rows] = lg[torch.arange(rows).clamp_max(M - 1)]
        assert bool(torch.isnan(buf[M:]).all()) != fault


def test_max_norm_check_is_blind_to_a_scaled_sample():
    """Exact-regime logits with one of 43 samples' knowledge base scaled by 1e-3 and its info replaced by zeros:
    max|err| / max|ref| over the batch stays far below test_gpu_read_step_fp8's bar (half the restatement's distance from
    fp64, 0.02-0.07), while softmax_bound_check with the exact regime's logit bound -- what
    test_gpu_fp8_kernels.test_fp8_read_step_exact_regime_logits feeds it -- rejects it about 55-fold: that bound lets
    each att move by expm1(2 dL), about 2 %."""
    from tests.test_gpu_wgmma import softmax_bound_check
    B, N, d = 43, 3, 512
    o, ref, bound = _read_case(B, N, 11)
    g = torch.Generator().manual_seed(3)
    kb = torch.nn.functional.elu(torch.randn(B, N, d, generator=g)).double()
    kb[5] *= 1e-3
    logits = kernel_logit_sum(exact_step(o), o["wr"]).double() + 0.25
    att = torch.softmax(logits.view(B, N), 1)
    info = torch.einsum("bn,bnd->bd", att, kb)
    bad = info.clone()
    bad[5] = 0
    max_norm = float((bad - info).abs().max() / info.abs().max())
    assert max_norm < 0.5 * 0.02 / 10, max_norm
    dL = bound + 1e-6 * ((ref + 0.25).abs() + 1)
    r_att, r_ok = softmax_bound_check(att, info, ref + 0.25, dL, kb, B, N)
    assert r_att <= 1 and r_ok <= 1, (r_att, r_ok)
    _, r_info = softmax_bound_check(att, bad, ref + 0.25, dL, kb, B, N)
    assert r_info >= 10, r_info
