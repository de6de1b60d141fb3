"""CPU checks of tests/test_gpu_read_step_bounds.py's per-row reference and bound, with that file's own code.

An emulation of read_step_kernel's arithmetic in torch -- bf16 P*y; GEMM 1 in fp32 over 64-wide k-blocks summed in
reverse order; elu_fast with ex2 carrying a +-2^-22 relative error; bf16 H; GEMM 2 in fp32; the epilogue's fmaf chain over
each thread's 64 terms, the two shuffle adds and half0 + half1 -- passes the bound at d = 512, and each of these planted
faults is rejected by a wide margin: warpgroup 1's rows taking the y of the previous sample, one of GEMM 1's eight k-blocks
dropped, the Q of columns [256, 512) taken from [0, 256), the control of the next sample in the epilogue, half 1's partial
sum dropped, and H taking ELU's negative branch for positive arguments."""
import pytest
import torch

from tests.test_gpu_read_step_bounds import D, step_reference

MARGIN = 100
LOG2E = torch.tensor(1.4426950408889634, dtype=torch.float32)


def _inputs(B, N, seed):
    """the operands the kernel sees, in the test's distributions: bf16 P, Q, packs of Wm[0:d] and Wm2 ([out, in])"""
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s, scale=1.0: torch.randn(*s, generator=g) * scale
    M = B * N
    P16 = (rn(M, D) * 0.8).to(torch.bfloat16)
    Q16 = (rn(M, D) * 0.6).to(torch.bfloat16)
    W1 = rn(D, D, scale=(2 * D) ** -0.5).to(torch.bfloat16)
    W2 = rn(D, D, scale=D ** -0.5).to(torch.bfloat16)
    return dict(P16=P16, Q16=Q16, W1=W1, W2=W2, y=rn(B, D), c=rn(B, D), bm2=rn(D, scale=0.1), wr=rn(D, scale=4 * D ** -0.5),
                g=g)


def _elu_fast(x, g, neg_always=False):
    """fp32 x > 0 ? x : ex2(x * log2e) - 1, the ex2 off by +-2^-22 relative (random sign per element)"""
    t = x * LOG2E
    sign = torch.randint(0, 2, x.shape, generator=g).double() * 2 - 1
    e = (torch.exp2(t.double()) * (1 + sign * 2.0 ** -22)).float() - 1
    return e if neg_always else torch.where(x > 0, x, e)


def emulate(inp, B, N, fault=None):
    """read_step_kernel's logits (without br) in fp32 torch arithmetic, with an optional planted fault"""
    M, g = B * N, inp["g"]
    rows = torch.arange(M)
    samp = rows // N
    ysamp = samp.clone()
    if fault == "wg1_prev_y":
        wg1 = (rows % 128) >= 64
        ysamp[wg1] = (samp[wg1] - 1).clamp_min(0)
    PY = (inp["P16"].float() * inp["y"][ysamp]).to(torch.bfloat16).float()
    W1 = inp["W1"].float().t()
    acc = torch.zeros(M, D)
    for kb in reversed(range(D // 64)):
        if fault == "drop_kblock" and kb == 5:
            continue
        acc = acc + PY[:, kb * 64:(kb + 1) * 64] @ W1[kb * 64:(kb + 1) * 64]
    Q = inp["Q16"].float()
    if fault == "q_half":
        Q = torch.cat([Q[:, :256], Q[:, :256]], 1)
    H = _elu_fast(acc + Q, g, neg_always=fault == "elu_neg").to(torch.bfloat16).float()
    I1 = H @ inp["W2"].float().t() + inp["bm2"]
    csamp = (samp + 1).clamp_max(B - 1) if fault == "next_control" else samp
    I2 = _elu_fast(I1 * inp["c"][csamp], g)
    # epilogue: thread q of a row's four lanes holds columns 256 h + 8 j + 2 q + e, j = 0..31, e = 0, 1, summed by fmaf
    t = I2.view(M, 2, 32, 4, 2).double()
    w = inp["wr"].view(2, 32, 4, 2).double()
    s = torch.zeros(M, 2, 4)
    for j in range(32):
        for e in range(2):
            s = (t[:, :, j, :, e] * w[:, j, :, e] + s.double()).float()
    half = (s[..., 0] + s[..., 1]) + (s[..., 2] + s[..., 3])
    return half[:, 0] if fault == "drop_half1" else half[:, 0] + half[:, 1]


def _ratio(got, ref, bound):
    return float(((got.double() - ref).abs() / bound).max())


def _reference(inp, N):
    return step_reference(inp["P16"], inp["Q16"], inp["y"].repeat_interleave(N, 0), inp["c"].repeat_interleave(N, 0),
                          inp["W1"], inp["W2"], inp["bm2"], inp["wr"])


def test_reference_is_the_read_step():
    """the reference is the read step's logit ELU((ELU(P*y @ W1 + Q) @ W2 + bm2) * c) . wr with H rounded to bf16 as the
    kernel rounds it, and its bound is far below the logits' own scale"""
    N = 5
    inp = _inputs(3, N, 1)
    ref, bound = _reference(inp, N)
    elu = torch.nn.functional.elu
    PY = (inp["P16"].float() * inp["y"].repeat_interleave(N, 0)).to(torch.bfloat16).double()
    H = elu(PY @ inp["W1"].double().t() + inp["Q16"].double()).float().to(torch.bfloat16).double()
    cb = inp["c"].double().repeat_interleave(N, 0)
    want = elu((H @ inp["W2"].double().t() + inp["bm2"].double()) * cb) @ inp["wr"].double()
    assert torch.allclose(ref, want, rtol=1e-12, atol=1e-12)
    assert bool((bound > 0).all()) and float(bound.median()) < 1e-2 * float(ref.abs().median())


@pytest.mark.parametrize("B,N", [(1, 1), (3, 43), (1, 193), (5, 51), (2, 49)])
def test_emulated_kernel_passes_the_bound(B, N):
    inp = _inputs(B, N, B * 100 + N)
    ref, bound = _reference(inp, N)
    r = _ratio(emulate(inp, B, N), ref, bound)
    print("emulated read step B=%d N=%d: %.3f of the bound (median bound %.2e)" % (B, N, r, float(bound.median())))
    assert r <= 1, r


@pytest.mark.parametrize("fault", ["wg1_prev_y", "drop_kblock", "q_half", "next_control", "drop_half1", "elu_neg"])
def test_bound_rejects_a_planted_fault(fault):
    B, N = 5, 51                                    # 255 rows: two tiles, warpgroup 1 of each holding rows of two samples
    inp = _inputs(B, N, 7)
    ref, bound = _reference(inp, N)
    ok = _ratio(emulate(inp, B, N), ref, bound)
    inp = _inputs(B, N, 7)                          # the same draws for the faulty run
    bad = _ratio(emulate(inp, B, N, fault), ref, bound)
    print("%s: emulation %.3f of the bound, fault %.3g" % (fault, ok, bad))
    assert ok <= 1, ok
    assert bad > MARGIN, (fault, bad)
