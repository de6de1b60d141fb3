"""The e4m3 read step (MAC_PREC_FP8, csrc/read_step_fp8.cuh) on the GPU.

- The weight pack and the step-invariant P8 / sP bit for bit against the fp32 restatements of the quantisers
  (F8.pack_weight_f32, F8.quant_rows_f32: the kernels' own fp32 divisions), at the pack's K and N tails and with zero rows
  from both invariant forms.
- The kernel, called through the C ABI, against the fp64 restatement of the scheme (oracle/fp8_read_oracle.py) fed with
  the library's own quantised operands, at the edge shapes of
  tests/test_gpu_fullshape.py::test_fused_read_step_equals_unfused_chain.
- Full passes at the headline and GQA shapes against the fp64 oracle, bounded a few times above the error measured on an
  H100.
- serving.HostPipeline(prec="fp8") against a direct cell, bit for bit; unsupported uses raise before any launch.

Why the kernel check is not exact (tests/test_gpu_fp8_kernels.py checks the logits row by row): the kernel rounds fp32
values to e4m3 twice per step (A8 = e4m3(P8 * y / ay) and H8 = e4m3(H / sH)), and a value it rounds differs from the
fp64 value the restatement rounds.  Where that difference straddles a rounding midpoint, one e4m3 element lands one step
(6-12 %) away.  With fp32 arithmetic alone such flips would be
rare: 1e-7 relative noise on both accumulators moves att_kb and info by ~3e-5 in a CPU model of the restatement.  But the
e4m3 wgmma of Hopper adds its products into the fp32 accumulator with fewer mantissa bits than fp32 keeps, and 1e-4 relative
noise on the accumulators moves them by 4-6e-3 in the same model; on an H100 the kernel sits 3e-3 to 1e-2 (max-norm) from
the restatement, 0.03 to 0.25 of the restatement's own distance from fp64 over the shapes below.  The bound is half that
distance (ERR_FRACTION): a systematic error -- a wrong scale, sample, swizzle or tile -- moves the output by at least as much
as the quantisation itself and fails it."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import fp8_read_oracle as F8

pytestmark = pytest.mark.gpu

D = 512
FP8 = 3
# kernel-vs-restatement distance over restatement-vs-fp64 distance (att_kb and info, max-norm); see the module docstring
ERR_FRACTION = 0.5


def _lib():
    from mac_network_b200 import _lib as L_
    return L_, L_.load()


def _rn(g, *s, scale=1.0):
    return (torch.randn(*s, device="cuda", generator=g) * scale).contiguous()


def _pack8(L_, lib, W):
    o = torch.empty((W.shape[1], W.shape[0]), dtype=torch.uint8, device="cuda")
    s = torch.empty(W.shape[1], dtype=torch.float32, device="cuda")
    L_.check(lib.mac_pack_weight_fp8(L_.ptr(W), L_.ptr(o), L_.ptr(s), W.shape[0], W.shape[1], L_.stream_ptr()), "pack8")
    return o, s


def _e4m3(u8):
    return u8.view(torch.float8_e4m3fn).double()


def _bytes(v):
    """e4m3 values -> their bytes"""
    return v.float().to(torch.float8_e4m3fn).view(torch.uint8)


def _case(B, N, seed):
    """Random read weights (init_params-like scales), their bf16 and e4m3 packs, a knowledge base and y / control."""
    L_, lib = _lib()
    d = D
    g = torch.Generator(device="cuda").manual_seed(seed)
    W = {"Wx": _rn(g, d, d, scale=d ** -0.5), "bx": _rn(g, d, scale=0.1), "Wy": _rn(g, d, d, scale=d ** -0.5),
         "by": _rn(g, d, scale=0.1), "Wm": _rn(g, 2 * d, d, scale=(2 * d) ** -0.5), "bm": _rn(g, d, scale=0.1),
         "Wm2": _rn(g, d, d, scale=d ** -0.5), "bm2": _rn(g, d, scale=0.1), "wr": _rn(g, d, scale=4 * d ** -0.5)}

    def pack16(w):
        o = torch.empty((w.shape[1], w.shape[0]), dtype=torch.bfloat16, device="cuda")
        L_.check(lib.mac_pack_weight_bf16(L_.ptr(w), L_.ptr(o), w.shape[0], w.shape[1], L_.stream_ptr()))
        return o
    keep = [pack16(W["Wx"]), pack16(W["Wm"]), pack16(W["Wm2"])]
    W1, s1 = _pack8(L_, lib, W["Wm"][:d])
    W2, s2 = _pack8(L_, lib, W["Wm2"])
    keep += [W1, s1, W2, s2]
    rw = L_.ReadWeights(W["Wx"].data_ptr(), W["bx"].data_ptr(), W["Wy"].data_ptr(), W["by"].data_ptr(),
                        W["Wm"].data_ptr(), W["bm"].data_ptr(), W["Wm2"].data_ptr(), W["bm2"].data_ptr(),
                        W["wr"].data_ptr(), 0.25, keep[0].data_ptr(), keep[1].data_ptr(), keep[2].data_ptr(),
                        None, None, None, None, W1.data_ptr(), s1.data_ptr(), W2.data_ptr(), s2.data_ptr())
    kb = torch.nn.functional.elu(_rn(g, B, N, d))
    kb16 = kb.to(torch.bfloat16).contiguous()
    return dict(W=W, keep=keep, W1=W1, s1=s1, W2=W2, s2=s2, rw=rw, kb=kb, kb16=kb16, y=_rn(g, B, d), c=_rn(g, B, d))


def _inv_slabs(inv, B, N):
    """[P8 | sP | Q | logit scratch | P] of an fp8 `inv` (each slab 1 KB aligned behind a 1 KB aligned base)."""
    M, d = B * N, D
    al = lambda b: (b + 1023) & ~1023
    o = ((inv.data_ptr() + 1023) & ~1023) - inv.data_ptr()
    P8 = inv[o:o + M * d].view(M, d)
    o += al(M * d)
    sP = inv[o:o + M * 4].view(torch.float32)
    o += al(M * 4)
    Q = inv[o:o + M * d * 2].view(torch.bfloat16).view(M, d)
    o += al(M * d * 2) + al(M * 4)
    P = inv[o:o + M * d * 2].view(torch.bfloat16).view(M, d)
    return P8, sP, Q, P


def _run_step(case, B, N):
    L_, lib = _lib()
    nb = lib.mac_read_invariant_bytes(B, N, D, FP8)
    inv = torch.empty(nb, dtype=torch.uint8, device="cuda")
    L_.check(lib.mac_read_invariant(None, L_.ptr(case["kb16"]), ctypes.byref(case["rw"]), FP8, L_.ptr(inv), nb, B, N, D,
                                    L_.stream_ptr()), "mac_read_invariant")
    ws_bytes = lib.mac_read_workspace_bytes(B, N, D, FP8)
    ws = torch.zeros(ws_bytes, dtype=torch.uint8, device="cuda")
    info = torch.full((B, D), float("nan"), device="cuda")
    att = torch.full((B, N), float("nan"), device="cuda")
    L_.check(lib.mac_read_fwd_inv(None, L_.ptr(case["kb16"]), L_.ptr(inv), L_.ptr(case["y"]), L_.ptr(case["y"]),
                                  L_.ptr(case["c"]), ctypes.byref(case["rw"]), FP8, L_.ptr(info), L_.ptr(att), L_.ptr(ws),
                                  ws_bytes, B, N, D, L_.stream_ptr()), "mac_read_fwd_inv")
    torch.cuda.synchronize()
    return inv, att, info


def _mr(a, b):
    return float((a.double() - b).abs().max() / b.abs().max())


def test_pack_weight_fp8_matches_restatement():
    """mac_pack_weight_fp8: the column scales are max|W[:, c]| / 448 in fp32, and the e4m3 bytes are the fp32 restatement's
    (F8.pack_weight_f32: the kernel's own fp32 division) bit for bit.  An all-zero column packs to zeros with scale 0."""
    L_, lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(5)
    W = _rn(g, 512, 384, scale=512 ** -0.5)
    W[:, 7] = 0
    W[3, 9] = 1e4                                  # one outlier: the rest of its column lands in e4m3's subnormals
    Wt, s = _pack8(L_, lib, W)
    torch.cuda.synchronize()
    W8, s_ref = F8.pack_weight_f32(W.cpu())
    amax = W.abs().amax(0).cpu().numpy()
    assert np.array_equal(s.cpu().numpy(), amax / np.float32(448))      # IEEE fp32 division, as the kernel does
    assert torch.equal(s.cpu(), s_ref)
    assert torch.equal(Wt.cpu(), _bytes(W8.T.contiguous()))
    assert int(Wt[7].count_nonzero()) == 0 and float(s[7]) == 0.0


# (K, N): 1, 31, 33, 100, 512 and 9216 on both sides, so the 32 x 32 tiles' K and N tails run
PACK_SHAPES = [(1, 1), (1, 9216), (9216, 1), (31, 33), (33, 31), (100, 100), (31, 512), (512, 33), (9216, 33), (33, 9216),
               (100, 9216), (9216, 100)]


@pytest.mark.parametrize("K,N", PACK_SHAPES)
def test_pack_weight_fp8_bit_for_bit_at_edge_shapes(K, N):
    """mac_pack_weight_fp8 against F8.pack_weight_f32 bit for bit, with an all-zero column, an outlier column (the rest of
    it in the subnormals or flushed to zero), values that land exactly on +-448 (each column's max) and columns whose
    values sit on a 1/64 grid."""
    L_, lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(K * 7 + N)
    W = _rn(g, K, N, scale=K ** -0.5)
    W[:, 0] = 0
    if N > 1:
        W[K // 2, 1] = 3e4
    if N > 2:
        W[:, 2] = torch.round(W[:, 2] * 64) / 64
        W[0, 2] = 4.0
    Wt, s = _pack8(L_, lib, W)
    torch.cuda.synchronize()
    W8, s_ref = F8.pack_weight_f32(W.cpu())
    assert torch.equal(s.cpu(), s_ref)
    assert torch.equal(Wt.cpu(), _bytes(W8.T.contiguous()))
    am = W.abs().amax(0)
    top = (W.abs() == am[None, :]) & (am[None, :] > 0)
    assert bool((_e4m3(Wt.T.contiguous()).abs()[top.cpu()] == 448).all())     # each column's max lands on 448
    assert int(Wt[0].count_nonzero()) == 0 and float(s[0]) == 0.0


def test_invariant_quantisation_bit_for_bit_in_both_forms():
    """P8 and sP from mac_read_invariant (bf16 knowledge base in) and mac_read_invariant_cast (fp32 in) equal
    F8.quant_rows_f32 of the library's own bf16 P bit for bit: with test_gpu_read_invariant's wide-exponent knowledge base,
    and with bx = 0 and all-zero knowledge-base rows, so those P rows are zero (sP = 0, zero bytes)."""
    from tests.test_gpu_read_invariant import _case as inv_case
    L_, lib = _lib()
    B, N = 5, 49
    M = B * N
    W, keep, rw, kb = inv_case(B, N, 77)
    W["bx"].zero_()
    kb[3] = 0
    kb[100:103] = 0
    kb[M - 1] = 0
    kb16 = kb.to(torch.bfloat16).contiguous()
    nb = lib.mac_read_invariant_bytes(B, N, D, FP8)
    forms = []
    for cast in (False, True):
        inv = torch.full((nb,), 0xA5, dtype=torch.uint8, device="cuda")
        if cast:
            k16 = torch.full((M, D), float("nan"), dtype=torch.bfloat16, device="cuda")
            L_.check(lib.mac_read_invariant_cast(L_.ptr(kb), L_.ptr(k16), ctypes.byref(rw), FP8, L_.ptr(inv), nb, B, N, D,
                                                 L_.stream_ptr()), "mac_read_invariant_cast")
        else:
            L_.check(lib.mac_read_invariant(None, L_.ptr(kb16), ctypes.byref(rw), FP8, L_.ptr(inv), nb, B, N, D,
                                            L_.stream_ptr()), "mac_read_invariant")
        torch.cuda.synchronize()
        P8, sP, _, P = _inv_slabs(inv, B, N)
        P8_ref, sP_ref = F8.quant_rows_f32(P.float().cpu())
        assert torch.equal(P8.cpu(), _bytes(P8_ref)), ("P8", cast, int((P8.cpu() != _bytes(P8_ref)).sum()))
        assert torch.equal(sP.cpu(), sP_ref), ("sP", cast)
        zero = (P.float().abs().amax(1) == 0).cpu()
        assert bool(zero[[3, 100, 101, 102, M - 1]].all()) and bool((sP.cpu()[zero] == 0).all())
        assert int(P8.cpu()[zero].count_nonzero()) == 0
        forms.append((P8.clone(), sP.clone()))
    assert torch.equal(forms[0][0], forms[1][0]) and torch.equal(forms[0][1], forms[1][1])


@pytest.mark.parametrize("B,N", [(64, 196), (3, 49), (4, 17), (11, 131), (3, 255), (9, 200), (2, 256), (1, 129), (1, 1),
                                 (64, 1), (3, 2), (5, 64)])
def test_fp8_read_step_equals_restatement(B, N):
    """The kernel through mac_read_invariant + mac_read_fwd_inv(MAC_PREC_FP8) against the fp64 restatement fed with the
    library's P8, sP, Q and packed weights.  Shapes: N = 17, 49, 131, 196, 255 and 256; partial last tiles (3 x 49, 11 x 131,
    9 x 200); a single sample (1 x 129, 1 x 1); tiles holding 64 one-row samples (64 x 1) or 32 two-row ones (3 x 2)."""
    case = _case(B, N, B * 1000 + N)
    inv, att, info = _run_step(case, B, N)
    M, d = B * N, D
    P8, sP, Q, P = _inv_slabs(inv, B, N)
    # the invariant: P8 / sP are the restatement's per-row quantisation of the library's bf16 P
    P8_ref, sP_ref = F8.quant_rows_f32(P.float().cpu())
    assert torch.equal(sP.cpu(), sP_ref) and torch.equal(P8.cpu(), _bytes(P8_ref))
    W = case["W"]
    args = (_e4m3(P8.cpu()), sP.cpu(), Q.double().cpu(), case["y"].cpu(), case["c"].cpu(),
            _e4m3(case["W1"].cpu()).T, case["s1"].cpu(), _e4m3(case["W2"].cpu()).T, case["s2"].cpu(),
            W["bm2"].cpu(), W["wr"].cpu(), 0.25, case["kb16"].reshape(M, d).cpu(), N)
    att_r, info_r = F8.read_step(*args)
    # fp64 without any e4m3 rounding (the bf16 P, Q and knowledge base kept): the scale of the quantisation error
    yb = case["y"].double().cpu().repeat_interleave(N, 0)
    H = torch.nn.functional.elu((P.double().cpu() * yb) @ W["Wm"][:d].double().cpu() + Q.double().cpu())
    I1 = H @ W["Wm2"].double().cpu() + W["bm2"].double().cpu()
    lg = torch.nn.functional.elu(I1 * case["c"].double().cpu().repeat_interleave(N, 0)) @ W["wr"].double().cpu() + 0.25
    att_x = torch.softmax(lg.reshape(B, N), 1)
    info_x = torch.einsum("bn,bnd->bd", att_x, case["kb16"].double().cpu())
    e = {"att": _mr(att.cpu(), att_r), "info": _mr(info.cpu(), info_r)}
    q = {"att": _mr(att_r, att_x), "info": _mr(info_r, info_x)}
    print("fp8 read step B=%d N=%d: kernel vs restatement %s, restatement vs fp64 %s" % (B, N, e, q))
    assert bool(torch.isfinite(att).all()) and bool(torch.isfinite(info).all())
    assert float((att.sum(1) - 1).abs().max()) < 1e-5
    for k in e:
        assert e[k] <= ERR_FRACTION * q[k] + 1e-6, (k, e, q)


def test_fp8_pass_headline_shape_error_is_bounded():
    """prec="fp8" at the headline shape (B=64, N=196, d=512, 12 steps) against the fp64 oracle: the control chain stays fp32
    (< 1e-4); memory, info and att_kb are bounded a few times above the error measured on an H100."""
    from mac_network_b200.synthetic import SHAPES
    from tests._util import max_rel
    from tests.test_gpu_fullshape import PER_STEP, headline_case
    from tests.test_gpu_parity import run_gpu
    cfg, inputs, params, ref = headline_case()
    L = SHAPES["headline"][4]
    got, _ = run_gpu(cfg, params, inputs, L, prec="fp8")
    errs = {k: max(max_rel(got[k][i], ref[k][i]) for i in range(L)) for k in PER_STEP}
    print("fp8 headline-shape worst per-step max-rel:", errs)
    assert errs["control"] < 1e-4 and errs["att_question"] < 1e-4
    assert errs["memory"] < 2e-3, errs         # measured 6.6e-4 (bf16: 4.7e-4)
    assert errs["info"] < 8e-3, errs           # measured 2.0e-3 (bf16: 1.1e-3)
    assert errs["att_kb"] < 3e-2, errs         # measured 8.5e-3 (bf16: 7.7e-4)


def test_fp8_pass_gqa_shape_error_is_bounded():
    """BASELINE configs[4] (7x7 grid, self-attention + gate, 6 steps) with prec="fp8" against the fp64 oracle."""
    from mac_network_b200.synthetic import SHAPES
    from tests._util import max_rel
    from tests.test_gpu_fullshape import PER_STEP, headline_case
    from tests.test_gpu_parity import run_gpu
    shape = SHAPES["gqa"] if "gqa" in SHAPES else (64, 30, 49, 512, 6)
    cfg, inputs, params, ref = headline_case("gqa", shape, seeds=(41, 42, 43))
    got, _ = run_gpu(cfg, params, inputs, shape[4], prec="fp8")
    errs = {k: max(max_rel(got[k][i], ref[k][i]) for i in range(shape[4])) for k in PER_STEP}
    print("fp8 GQA-shape worst per-step max-rel:", errs)
    assert errs["control"] < 1e-4
    assert errs["memory"] < 2e-3 and errs["info"] < 8e-3 and errs["att_kb"] < 3e-2, errs    # measured 6.1e-4 / 3.0e-3 / 8.9e-3


def test_fp8_host_pipeline_matches_direct_cell():
    """serving.HostPipeline(prec="fp8"), host bf16 cast of the knowledge base included, returns bit for bit what a direct
    small_tc cell computes from device-resident inputs."""
    from mac_network_b200.config import MACConfig
    from mac_network_b200.mac_cell import MACParams
    from mac_network_b200.params import init_params, perturb_biases
    from mac_network_b200.serving import HostPipeline
    from mac_network_b200.synthetic import make_inputs
    from tests.test_gpu_parity import run_gpu
    B, S, N, d, L = 8, 6, 49, 512, 3
    cfg = MACConfig.args("args", netLength=L, memDim=d, ctrlDim=d, attDim=d)
    pv = perturb_biases(init_params(cfg, L, seed=82), seed=83)
    params = MACParams(cfg, L, values=pv)
    pipe = HostPipeline(cfg, params, (B, S, N, d, L), prec="fp8", slots=2, cast_threads=3, host_cast=True)
    assert pipe.host_kb_bf16
    batches = [make_inputs(B, S, N, d, seed=90 + i) for i in range(3)]
    host = [{k: torch.from_numpy(v).pin_memory() for k, v in b.items() if k != "questionWords"} for b in batches]
    got = []
    for i, hb in enumerate(host):
        t = pipe.submit(hb, next_batch=host[(i + 1) % len(host)])
        got.append({k: v.clone() for k, v in pipe.result(t).items()})
    for b, g in zip(batches, got):
        ref, _ = run_gpu(cfg, pv, b, L, prec="fp8", small_tc=True)
        assert np.array_equal(g["memory"].numpy(), ref["memory"][-1])
        assert np.array_equal(g["control"].numpy(), ref["control"][-1])
        assert np.array_equal(g["att_kb"].numpy(), ref["att_kb"])


def test_fp8_unsupported_uses_raise_before_any_launch():
    """MACCell(prec="fp8") outside the inference read step raises NotImplementedError, and the C ABI returns
    MAC_ERR_UNSUPPORTED, without launching anything."""
    from mac_network_b200.config import MACConfig
    from mac_network_b200.mac_cell import MACCell, MACParams
    from mac_network_b200.synthetic import make_inputs
    L_, lib = _lib()
    L = 2

    def cell(N=49, d=512, flags="args", keeps=(1.0, 1.0, 1.0), **kw):
        cfg = MACConfig.args(flags, netLength=L, memDim=d, ctrlDim=d, attDim=d)
        params = MACParams(cfg, L, seed=1)
        x = {k: torch.from_numpy(v).cuda() for k, v in make_inputs(2, 5, N, d, seed=2).items()}
        n0 = lib.mac_b200_launch_count()
        with pytest.raises(NotImplementedError):
            MACCell(x["vecQuestions"], x["questionWords"], x["questionCntxWords"], x["questionLengths"], x["knowledgeBase"],
                    keeps[0], keeps[1], keeps[2], 2, False, config=cfg, params=params, prec="fp8", **kw)
        assert lib.mac_b200_launch_count() == n0
    cell(save_for_backward=True)                 # training forward
    cell(keeps=(1.0, 0.85, 1.0))                 # read dropout
    cell(N=257)                                  # more cells than the kernel's tiles take
    cell(d=256)                                  # the kernel is built for d = 512
    # the C ABI: mac_read_fwd (not the inference form), and shapes outside mac_read_step_fused_supported
    case = _case(2, 49, 7)
    nb = lib.mac_read_invariant_bytes(2, 300, D, FP8)
    inv = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    ws = torch.zeros(lib.mac_read_workspace_bytes(2, 300, D, FP8), dtype=torch.uint8, device="cuda")
    out = torch.zeros(2 * 300 * D, device="cuda")
    n0 = lib.mac_b200_launch_count()
    rw = ctypes.byref(case["rw"])
    p = L_.ptr
    assert lib.mac_read_invariant(None, p(case["kb16"]), rw, FP8, p(inv), nb, 2, 300, D, None) == -3
    assert lib.mac_read_invariant(p(case["kb"]), None, rw, FP8, p(inv), nb, 2, 49, D, None) == -3
    assert lib.mac_read_fwd_inv(None, p(case["kb16"]), p(inv), None, p(case["y"]), p(case["c"]), rw, FP8, p(out), p(out),
                                p(ws), ws.numel(), 2, 300, D, None) == -3
    assert lib.mac_read_fwd_inv(p(case["kb"]), None, p(inv), None, p(case["y"]), p(case["c"]), rw, FP8, p(out), p(out),
                                p(ws), ws.numel(), 2, 49, D, None) == -3
    assert lib.mac_read_fwd(p(case["kb"]), p(case["kb16"]), p(case["y"]), p(case["c"]), rw, 1.0, 0, 0, FP8, p(out), p(out),
                            None, p(ws), ws.numel(), 2, 49, D, None) == -3
    torch.cuda.synchronize()
    assert lib.mac_b200_launch_count() == n0
