"""Parity gated at the shapes bench.py reports (VERDICT r1, "what's weak" #1): the headline configuration
B=64, S=40, N=196, d=512, netLength=12 (BASELINE.json configs[2]/[3]) and configs[1] (B=32, S=20, L=4, forward+backward)
against the fp64 oracle (`oracle/mac_oracle.py`, pinned to the reference by tests/golden) -- per-step tensors, both a
tensor-level max-norm bound (north_star's "1e-4 relative") and an element-wise relative bound with an absolute floor.

bf16 tensor-core path: bounds are a few times the error the path reaches (a much looser bound would let a 20x regression
pass)."""
import numpy as np
import pytest
import torch

from mac_network_b200.config import MACConfig
from mac_network_b200.params import init_params, perturb_biases
from mac_network_b200.synthetic import SHAPES, make_inputs
from tests._util import max_rel
from tests.test_gpu_parity import run_gpu, run_oracle

pytestmark = pytest.mark.gpu

_ORACLE_CACHE = {}


def elem_rel(got, ref, floor):
    """max over elements of |got - ref| / max(|ref|, floor * max|ref|): an element-wise relative error whose denominator
    is floored at `floor` x the tensor's scale (so exact zeros / tiny entries do not divide by ~0)."""
    got = np.asarray(got, np.float64)
    ref = np.asarray(ref, np.float64)
    den = np.maximum(np.abs(ref), floor * np.max(np.abs(ref)) + 1e-300)
    return float(np.max(np.abs(got - ref) / den))


def headline_case(variant="args", shape=None, seeds=(1234, 100, 101)):
    shape = SHAPES["headline"] if shape is None else shape
    key = (variant, shape, seeds)
    if key not in _ORACLE_CACHE:
        B, S, N, d, L = shape
        cfg = MACConfig.args(variant, netLength=L, memDim=d, ctrlDim=d, attDim=d)
        inputs = make_inputs(B, S, N, d, seed=seeds[0], dtype=np.float64)
        params = perturb_biases(init_params(cfg, L, seed=seeds[1], dtype=np.float64), seed=seeds[2])
        ref = run_oracle(cfg, params, inputs, L)
        _ORACLE_CACHE[key] = (cfg, inputs, params, ref)
    return _ORACLE_CACHE[key]


PER_STEP = ("control", "memory", "info", "att_question", "att_kb")


def test_fp32_headline_shape_matches_oracle_per_step():
    """fp32 projection path at B=64, S=40, N=196, d=512, L=12: EVERY per-step control / memory / info / attention map
    within 1e-4 of the fp64 oracle (max-norm) and within 1e-3 element-wise (denominator floored at 1e-2 of the scale)."""
    cfg, inputs, params, ref = headline_case()
    L = SHAPES["headline"][4]
    got, _ = run_gpu(cfg, params, inputs, L, prec="fp32")
    worst = {}
    for k in PER_STEP:
        for i in range(L):
            e = max_rel(got[k][i], ref[k][i])
            worst[k] = max(worst.get(k, 0.0), e)
            assert e < 1e-4, (k, i, e)
            assert elem_rel(got[k][i], ref[k][i], 1e-2) < 1e-3, (k, i)
    print("fp32 headline-shape worst per-step max-rel:", worst)


def test_bf16_headline_shape_error_is_bounded_tightly():
    """bf16 tensor-core path (the configuration bench.py's headline line measures, read step included) at the full headline
    shape: memory, info and att_kb are bounded a few times above the bf16 rounding error over the 12 steps.  The control
    chain stays fp32: 1e-4."""
    cfg, inputs, params, ref = headline_case()
    L = SHAPES["headline"][4]
    got, _ = run_gpu(cfg, params, inputs, L, prec="bf16")
    errs = {k: max(max_rel(got[k][i], ref[k][i]) for i in range(L)) for k in PER_STEP}
    print("bf16 headline-shape worst per-step max-rel:", errs)
    assert errs["control"] < 1e-4 and errs["att_question"] < 1e-4
    assert errs["memory"] < 1.5e-3, errs       # measured 4.7e-4
    assert errs["info"] < 4e-3, errs           # measured 1.1e-3
    assert errs["att_kb"] < 3e-3, errs         # measured 7.7e-4


def test_bf16_gqa_shape_error_is_bounded_tightly():
    """BASELINE configs[4] (7x7 grid, self-attention + gate, L=6) on the tensor-core path (N <= 128 form of the fused kernel)."""
    shape = SHAPES["gqa"] if "gqa" in SHAPES else (64, 30, 49, 512, 6)
    cfg, inputs, params, ref = headline_case("gqa", shape, seeds=(41, 42, 43))
    L = shape[4]
    got, _ = run_gpu(cfg, params, inputs, L, prec="bf16")
    errs = {k: max(max_rel(got[k][i], ref[k][i]) for i in range(L)) for k in PER_STEP}
    print("bf16 GQA-shape worst per-step max-rel:", errs)
    assert errs["control"] < 1e-4
    assert errs["memory"] < 1.5e-3 and errs["info"] < 4e-3 and errs["att_kb"] < 3e-3, errs    # measured 3.6e-4 / 1.3e-3 / 7.2e-4


def test_fused_read_step_equals_unfused_chain(monkeypatch):
    """The fused read step (csrc/read_step.cuh) against the four-launch chain it replaces, same inputs through the C ABI:
    attention and retrieved information agree to fp32 summation order (the bf16 roundings are identical)."""
    import ctypes
    from mac_network_b200 import _lib as L_
    lib = L_.load()
    d = 512
    # 64-row tiles packed across sample boundaries: a partial last tile (3 x 49, 4 x 17, 11 x 131), tiles spanning many
    # samples (N = 17, 49), samples spread over five tiles (N = 255) and a single-sample launch
    for (B, N) in ((64, 196), (3, 49), (5, 130), (2, 256), (7, 128), (4, 17), (9, 200), (1, 129), (3, 255), (11, 131)):
        g = torch.Generator(device="cuda").manual_seed(B * 1000 + N)

        def rn(*s, scale=1.0):
            return (torch.randn(*s, device="cuda", generator=g) * scale).contiguous()
        W = {"Wx": rn(d, d, scale=d ** -0.5), "bx": rn(d, scale=0.1), "Wy": rn(d, d, scale=d ** -0.5), "by": rn(d, scale=0.1),
             "Wm": rn(2 * d, d, scale=(2 * d) ** -0.5), "bm": rn(d, scale=0.1), "Wm2": rn(d, d, scale=d ** -0.5),
             "bm2": rn(d, scale=0.1), "wr": rn(d, scale=4 * d ** -0.5)}

        def pack(w):
            o = torch.empty((w.shape[1], w.shape[0]), dtype=torch.bfloat16, device="cuda")
            L_.check(lib.mac_pack_weight_bf16(L_.ptr(w), L_.ptr(o), w.shape[0], w.shape[1], L_.stream_ptr()))
            return o
        W16 = [pack(W["Wx"]), pack(W["Wm"]), pack(W["Wm2"])]
        rw = L_.ReadWeights(W["Wx"].data_ptr(), W["bx"].data_ptr(), W["Wy"].data_ptr(), W["by"].data_ptr(),
                            W["Wm"].data_ptr(), W["bm"].data_ptr(), W["Wm2"].data_ptr(), W["bm2"].data_ptr(),
                            W["wr"].data_ptr(), 0.25, W16[0].data_ptr(), W16[1].data_ptr(), W16[2].data_ptr())
        kb = torch.nn.functional.elu(rn(B, N, d)).to(torch.bfloat16).contiguous()
        y, c, mem = rn(B, d), rn(B, d), rn(B, d)
        nb = lib.mac_read_invariant_bytes(B, N, d, 1)
        inv = torch.empty(nb, dtype=torch.uint8, device="cuda")
        L_.check(lib.mac_read_invariant(None, L_.ptr(kb), ctypes.byref(rw), 1, L_.ptr(inv), nb, B, N, d, L_.stream_ptr()))
        assert lib.mac_read_step_fused_supported(B, N, d) == 1
        info1, att1 = torch.full((B, d), float("nan"), device="cuda"), torch.full((B, N), float("nan"), device="cuda")
        L_.check(lib.mac_read_step_fused(L_.ptr(inv), L_.ptr(kb), L_.ptr(y), L_.ptr(c), ctypes.byref(rw), L_.ptr(info1),
                                         L_.ptr(att1), B, N, d, L_.stream_ptr()), "mac_read_step_fused")
        # the unfused chain through the generic tensor-core entry points: PY = P*y; H = ELU(PY@Wm[0:d] + Q); logits; softmax
        M = B * N
        slab = (M * d * 2 + 1023) & ~1023
        base = (inv.data_ptr() + 1023) & ~1023
        off = base - inv.data_ptr()
        P = inv[off:off + M * d * 2].view(torch.bfloat16).view(M, d).float()
        Q = inv[off + slab:off + slab + M * d * 2].view(torch.bfloat16).view(M, d).float()
        PY = (P.view(B, N, d) * y[:, None, :]).to(torch.bfloat16).float().view(M, d)
        Wm1 = W16[1][:, :d].float()                                         # [out, in] bf16 values
        H = torch.nn.functional.elu(PY.double() @ Wm1.double().T + Q.double()).float().to(torch.bfloat16).float()
        I1 = H.double() @ W16[2].float().double().T + W["bm2"].double()
        I2 = torch.nn.functional.elu(I1.view(B, N, d) * c.double()[:, None, :])
        logits = (I2 * W["wr"].double()).sum(-1) + 0.25
        att0 = torch.softmax(logits, dim=-1)
        info0 = (att0[:, :, None] * kb.double()).sum(1)
        torch.cuda.synchronize()
        # H's bf16 rounding can flip on ties between fp32 (kernel) and fp64 (this check) accumulation: a few 1e-3 on H
        # elements, far less on the attention after the K = 512 contraction
        assert float((att1.double() - att0).abs().max()) < 2e-3 * float(att0.max()) + 1e-6, (B, N)
        assert float((info1.double() - info0).abs().max()) < 2e-3 * float(info0.abs().max()), (B, N)
        assert float((att1.sum(1) - 1).abs().max()) < 1e-5
    assert lib.mac_read_step_fused_supported(4, 300, 512) == 0 and lib.mac_read_step_fused_supported(4, 49, 256) == 0


@pytest.mark.parametrize("variant,shape,dp", [
    ("args", (32, 20, 196, 512, 4), (0.85, 0.85, 1.0)),       # BASELINE configs[1]: forward + backward at its full size
    ("args", (64, 40, 196, 512, 12), (0.85, 0.85, 1.0)),      # BASELINE configs[3]: the per-GPU training shape, netLength = 12
])
def test_backward_full_shape_matches_autograd(variant, shape, dp):
    """mac_backward (hand-written kernels) vs torch.autograd on the fp64 restatement at configs[1]'s full shape and at
    netLength = 12: every parameter / input gradient within 3e-3 of its tensor scale, forward state within 1e-4.
    At configs[1]'s shape with the training dropouts: most tensors <= 3e-4, the worst three are
    dWm2 (memKbProj_2) 1.7e-3, the logit vector 1.0e-3 and dKB 1.0e-3 -- an order of magnitude above the <= 2e-4 the same
    kernels reach at the small shapes of test_gpu_backward.py (fp32 products of B*N = 6272 rows against an fp64 oracle);
    at B=64, L=12 they reach 6.6e-3 / 5.8e-3 (dWm2, dbm2).  These are exactly the tensors downstream of the KB softmax,
    whose gradient sums to zero over the N cells of a sample: dbm2 = sum_rows dI1 and dWm2 = H^T dI1 are sums of ~1e5-1e6
    nearly cancelling terms, so fp32 round-off is amplified by sum|terms| / |sum| (the cancellation-free softmax backward in
    kb_attend_bwd_kernel did not change them; an fp32 TensorFlow graph is subject to the same conditioning).  The bounds
    (3e-3 at L=4, 1e-2 at L=12) are regression gates for what is measured, not a claim of 1e-4 (north_star states no
    gradient tolerance)."""
    from mac_network_b200.autograd import mac_backward
    from mac_network_b200.mac_cell import MACCell, MACParams, mac_network
    from oracle import mac_torch_autograd as TA
    B, S, N, d, L = shape
    cfg = MACConfig.args(variant, netLength=L, memDim=d, ctrlDim=d, attDim=d)
    inputs = make_inputs(B, S, N, d, seed=151, dtype=np.float64)
    pv = perturb_biases(init_params(cfg, L, seed=152, dtype=np.float64), seed=153)
    rng = np.random.RandomState(154)
    gc, gm = rng.standard_normal((B, d)), rng.standard_normal((B, d))
    params = MACParams(cfg, L, values={k: v.astype(np.float32) for k, v in pv.items()})
    x = {k: torch.from_numpy(np.ascontiguousarray(v if v.dtype == np.int32 else v.astype(np.float32))).cuda()
         for k, v in inputs.items()}
    cell = MACCell(x["vecQuestions"], x["questionWords"], x["questionCntxWords"], x["questionLengths"],
                   x["knowledgeBase"], dp[0], dp[1], dp[2], B, True, config=cfg, params=params, seed=4242,
                   save_for_backward=True)
    control, memory = mac_network(cell, L)
    grads = mac_backward(cell, torch.from_numpy(gc.astype(np.float32)).cuda(), torch.from_numpy(gm.astype(np.float32)).cuda())
    torch.cuda.synchronize()
    rc, rm, rg = TA.run(cfg, pv, inputs, L, dp, cell.dropout_uniforms(), gc, gm)
    assert max_rel(memory.cpu().numpy(), rm) < 1e-4 and max_rel(control.cpu().numpy(), rc) < 1e-4
    worst = {}
    for k, ref in rg.items():
        got = grads[k].cpu().numpy().reshape(ref.shape)
        scale = np.max(np.abs(ref))
        if scale < 1e-12:
            assert np.max(np.abs(got)) < 1e-4, k
            continue
        worst[k] = float(np.max(np.abs(got - ref)) / scale)
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:5]
    print("full-shape backward, five worst gradient max-rel:", [(k.split("MACCell/")[-1], round(v, 6)) for k, v in top])
    bad = {k: v for k, v in worst.items() if v > (3e-3 if L <= 4 else 1e-2)}
    assert not bad, bad


def test_whole_step_kernel_matches_separate_launches(monkeypatch):
    """mac_step_fused (write unit of the previous step + projY in the fused kernel's prologue, ONE launch per reasoning step)
    against the same cell with read / write / projY as separate launches (MAC_STEP_FUSED=0), headline shape.  The only
    arithmetic difference is bf16 instead of fp32 weights in the two batch-sized matrix-vector products."""
    cfg, inputs, params, ref = headline_case()
    L = SHAPES["headline"][4]
    from mac_network_b200 import _lib
    monkeypatch.setenv("MAC_STEP_FUSED", "1")        # opt-in form (slower and less accurate than the default: DESIGN.md)
    n0 = _lib.load().mac_b200_launch_count()
    fused, cell = run_gpu(cfg, params, inputs, L, prec="bf16")
    n_fused = _lib.load().mac_b200_launch_count() - n0
    assert cell._step_fused, "whole-step form not selected at the headline shape"
    monkeypatch.setenv("MAC_STEP_FUSED", "0")
    n0 = _lib.load().mac_b200_launch_count()
    sep, cell2 = run_gpu(cfg, params, inputs, L, prec="bf16")
    n_sep = _lib.load().mac_b200_launch_count() - n0
    assert not cell2._step_fused
    print("launches per 12-step pass: whole-step %d, separate %d" % (n_fused, n_sep))
    assert n_fused < n_sep
    for k in ("memory", "info", "att_kb"):
        e = max(max_rel(fused[k][i], sep[k][i]) for i in range(L))
        print("whole-step vs separate launches,", k, e)
        assert e < 8e-3, (k, e)        # bf16 weights on the state path: memory 3.8e-3 vs the oracle (measured)
    assert np.array_equal(fused["control"], sep["control"])


@pytest.mark.parametrize("variant", ["args", "gqa"])
def test_bf16_throughput_form_small_projections_on_tensor_cores(monkeypatch, variant):
    """The throughput form of the bf16 cell (MACCell(small_tc=True) / MAC_SMALL_TC=1: projY, write unit, gate and ctrlProj
    as three-pass split-bf16 wgmma products, write unit folded with the next projY) against the fp64 oracle at the
    headline and GQA shapes: same bounds as the default form (the split keeps these projections at fp32-class accuracy)."""
    monkeypatch.setenv("MAC_SMALL_TC", "1")
    if variant == "args":
        cfg, inputs, params, ref = headline_case()
        L = SHAPES["headline"][4]
    else:
        shape = SHAPES["gqa"]
        cfg, inputs, params, ref = headline_case("gqa", shape, seeds=(41, 42, 43))
        L = shape[4]
    got, cell = run_gpu(cfg, params, inputs, L, prec="bf16")
    assert cell._small_tc
    errs = {k: max(max_rel(got[k][i], ref[k][i]) for i in range(L)) for k in PER_STEP}
    print("bf16 throughput form (%s) worst per-step max-rel:" % variant, errs)
    assert errs["control"] < 1e-4
    assert errs["memory"] < 1.5e-3 and errs["info"] < 4e-3 and errs["att_kb"] < 3e-3, errs
    if variant == "gqa":
        g = max(max_rel(got["att_gate"][i], ref["att_gate"][i]) for i in range(L))
        assert g < 1.5e-3, g


@pytest.mark.parametrize("variant,shape", [("args", None), ("gqa", (64, 30, 49, 512, 6))])
def test_tc32_split_bf16_tensor_core_path_is_inside_1e4(variant, shape):
    """prec="tc32": the three [B*N, .] read projections as split-bf16 wgmma products (x = hi + lo, three partial products,
    fp32 accumulation; csrc/tc_gemm.cuh tc3_*) -- a TENSOR-CORE path inside north_star's 1e-4: every per-step control /
    memory / info / attention map at the headline shape (and the GQA shape) against the fp64 oracle."""
    if shape is None:
        cfg, inputs, params, ref = headline_case()
        L = SHAPES["headline"][4]
    else:
        cfg, inputs, params, ref = headline_case(variant, shape, seeds=(41, 42, 43))
        L = shape[4]
    got, _ = run_gpu(cfg, params, inputs, L, prec="tc32")
    worst = {}
    for k in PER_STEP:
        for i in range(L):
            e = max_rel(got[k][i], ref[k][i])
            worst[k] = max(worst.get(k, 0.0), e)
            assert e < 1e-4, (k, i, e)
            assert elem_rel(got[k][i], ref[k][i], 1e-2) < 2e-3, (k, i)
    print("tc32 (%s) worst per-step max-rel:" % variant, worst)
