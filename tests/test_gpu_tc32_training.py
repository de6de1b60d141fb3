"""Split-bf16 ("tc32") TRAINING of the read unit (DESIGN.md section 9, item 5):

  * `mac_read_fwd(MAC_PREC_TC32, save)` stage by stage against fp64 of the fp32 operands the kernel saw (the element-wise
    `|got - ref| <= tol * absref` form of tests/test_gpu_forward_kernels.py);
  * `mac_read_bwd_tc32` against `read_bwd_reference` of tests/test_gpu_backward_kernels.py;
  * the cell (`MACCell(prec="tc32")` + `mac_backward(tc=True)`) against torch.autograd on the fp64 restatement, at the fp32
    path's bars;
  * `DPTrainer(prec="tc32", bwd_tc=True)` at the bench training shape against its fp32 twin.

Each tol is about three times the worst ratio measured on an H100 80GB HBM3 (700 W power limit), written beside it.  The
point is fp32-class accuracy: on every output of a split product the backward tol sits 30-600x below the bf16 backward's
TOL_READ_TC (tests/test_tc32_bounds.py shows on the CPU that plain bf16 products fail them by more than 100x)."""
import ctypes

import numpy as np
import pytest
import torch

from mac_network_b200 import _lib as L_
from mac_network_b200.config import MACConfig
from mac_network_b200.params import init_params, perturb_biases
from mac_network_b200.synthetic import make_inputs
from tests._util import max_rel
from tests.test_gpu_backward_kernels import READ_GRADS, Report, gen, lib, prefill, randn, read_case, read_masks, run_twice
from tests.test_gpu_forward_kernels import add_attention, counters_zero, nanfill, read_forward_stages, read_weights
from tests.test_gpu_wgmma import attention_bound_check, elu

pytestmark = pytest.mark.gpu

PREC_TC32 = 2
ERR_INVALID, ERR_UNSUPPORTED = -1, -3

# mac_read_fwd(MAC_PREC_TC32, save): P, H, I1 against fp64 of the kernel's own previous stage;  y is the fp32 projY
TOL_FWD = {"y": 2e-7,                                                   # 6.6e-8 (fp32 projY)
           "P": 1e-5, "H": 6e-6, "I1": 9e-6}                            # 3.1e-6, 1.9e-6, 2.8e-6
# mac_read_bwd_tc32, per output (split-bf16 operands in the six [B*N, .] products; the logits backward stays fp32), with the
# bf16 backward's TOL_READ_TC beside it:                              measured        TOL_READ_TC
TOL_BWD = {"dkb": 3.5e-7,                                           # 1.2e-7          1.2e-5
           "dmem_in": 9e-9,                                         # 3.0e-9          5e-6
           "dcontrol": 2e-7,                                        # 5.7e-8          3e-7
           "dWx": 5e-7, "dbx_part": 1.5e-7,                         # 1.7e-7, 4.5e-8  2.5e-5, 1.5e-5
           "dWy": 1.7e-7, "dby": 1.3e-7,                            # 5.5e-8, 4.1e-8  3e-5, 1.2e-5
           "dWm": 7.5e-7, "dbm_part": 3e-7,                         # 2.5e-7, 9.4e-8  5e-4, 1.5e-4
           "dWm2": 4e-6, "dbm2_part": 1.8e-7,                       # 1.2e-6, 5.8e-8  8e-4, 3e-7
           "dwr_part": 1.7e-7, "dbr_part": 2e-8}                    # 5.5e-8, 6.5e-9  3e-7, 3e-8


def tc32_weights(g, d):
    """the fp32 read weights plus the split3 packs the training form reads (Wx_s3, Wm_s3, Wm2_s3)"""
    lb = lib()
    W, rw = read_weights(g, d)
    packs = {}
    for name, src in (("Wx_s3", W["Wx"]), ("Wm_s3", W["Wm"]), ("Wm2_s3", W["Wm2"])):
        K, n = src.shape
        o = torch.empty(n, 3 * K, dtype=torch.bfloat16, device="cuda")
        L_.check(lb.mac_pack_weight_split3(L_.ptr(src), L_.ptr(o), K, n, L_.stream_ptr()), "pack3")
        packs[name] = o
        setattr(rw, name, o.data_ptr())
    return W, rw, packs


# ================================================================================================ 1. forward entry point
FWD_SHAPES = [(64, 196, 512), (5, 49, 128), (3, 33, 256), (1, 1, 128)]


@pytest.mark.parametrize("B,N,d", FWD_SHAPES)
@pytest.mark.parametrize("keep", [0.85, 1.0])
def test_read_fwd_tc32_matches_fp64(B, N, d, keep):
    """y, P, H, I1 from `save` (NaN-prefilled: every element written), each against fp64 of the kernel's previous stage with
    the Philox masks; then att and info through the attention bound; a rerun is bit-identical"""
    lb = lib()
    g = gen(B * 1000 + N * 10 + d + 7)
    W, rw, packs = tc32_weights(g, d)
    kb = elu(randn(g, B, N, d)).float()
    mem, c = randn(g, B, d), randn(g, B, d)
    seed, step, M = 4243, 6, B * N
    wsb = lb.mac_read_workspace_bytes(B, N, d, PREC_TC32)
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    save, info, att = nanfill(3 * M * d + B * d), nanfill(B, d), nanfill(B, N)

    def call():
        L_.check(lb.mac_read_fwd(L_.ptr(kb), None, L_.ptr(mem), L_.ptr(c), ctypes.byref(rw), keep, seed, step, PREC_TC32,
                                 L_.ptr(info), L_.ptr(att), L_.ptr(save), L_.ptr(ws), wsb, B, N, d, L_.stream_ptr()),
                 "mac_read_fwd")

    got, same = run_twice(call, {"save": save, "info": info, "att": att})
    sv = got["save"]
    P, H, I1 = (sv[i * M * d:(i + 1) * M * d].view(M, d) for i in range(3))
    y = sv[3 * M * d:].view(B, d)
    masks = read_masks(keep, seed, step, B, N, d, "cuda")
    r = read_forward_stages(kb, mem, W, masks, P, y, H)
    rep = Report("mac_read_fwd tc32 %s keep %.2f" % ((B, N, d), keep))
    for name, t in (("y", y), ("P", P), ("I1", I1)):
        rep.add(name, t, *r[name], TOL_FWD[name])
    # the epilogue's ELU uses the SFU exponential: a few 1e-7 absolute near 0
    rep.add("H", H, *r["H"], TOL_FWD["H"], tiny=2.0 ** -17 * r["H"][0].abs() + 1e-7)
    add_attention(rep, attention_bound_check(got["att"], got["info"], *r["I1"], c, W["wr"], 0.25, kb, B, N, TOL_FWD["I1"],
                                             ms=masks[2]))
    rep.check(bool(torch.isfinite(sv).all()), "save fully written")
    rep.check(same, "bit-identical rerun")
    rep.check(counters_zero(ws), "split-K counters zero")       # the fp32 projY product's split-K runs on these counters
    rep.done()


def test_read_fwd_tc32_refusals_launch_nothing():
    """d % 128 != 0 (MAC_ERR_UNSUPPORTED) and a missing Wm_s3 pack (MAC_ERR_INVALID): refused before any launch or write"""
    lb = lib()
    for B, N, d, drop_pack in ((2, 9, 192, False), (2, 9, 64, False), (2, 9, 128, True)):
        g = gen(B + N + d)
        W, rw, packs = tc32_weights(g, d)
        if drop_pack:
            rw.Wm_s3 = None
        kb, mem, c = randn(g, B, N, d), randn(g, B, d), randn(g, B, d)
        M = B * N
        wsb = lb.mac_read_workspace_bytes(B, N, d, PREC_TC32)
        ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
        save, info, att = nanfill(3 * M * d + B * d), nanfill(B, d), nanfill(B, N)
        torch.cuda.synchronize()
        before = lb.mac_b200_launch_count()
        st = lb.mac_read_fwd(L_.ptr(kb), None, L_.ptr(mem), L_.ptr(c), ctypes.byref(rw), 0.85, 1, 0, PREC_TC32, L_.ptr(info),
                             L_.ptr(att), L_.ptr(save), L_.ptr(ws), wsb, B, N, d, L_.stream_ptr())
        torch.cuda.synchronize()
        assert st == (ERR_INVALID if drop_pack else ERR_UNSUPPORTED), (B, N, d, st)
        assert lb.mac_b200_launch_count() == before
        assert bool(save.isnan().all()) and bool(info.isnan().all()) and bool(att.isnan().all())
        assert not bool(ws.any())


# ================================================================================================ 2. backward entry point
def run_read_bwd_tc32(B, N, d, keep, seed, with_dkb=True):
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
    wsb = lb.mac_read_bwd_tc32_workspace_bytes(B, N, d)
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    # NaN bytes under the split operands: their zero padding columns must be written by the call, not assumed
    ws[lb.mac_read_bwd_workspace_bytes(B, N, d):].fill_(0xFF)
    Wy_t = W["Wy"].t().contiguous()
    o = [L_.ptr(outs[k]) for k in READ_GRADS]

    def call():
        L_.check(lb.mac_read_bwd_tc32(L_.ptr(kb), L_.ptr(mem), L_.ptr(c), ctypes.byref(rw), L_.ptr(Wy_t), L_.ptr(att),
                                      L_.ptr(save), L_.ptr(dinfo), keep, seed, step, *o, L_.ptr(ws), wsb, B, N, d,
                                      L_.stream_ptr()), "mac_read_bwd_tc32")

    got, same = run_twice(call, outs)
    rep = Report("mac_read_bwd_tc32 %s keep %.2f%s" % ((B, N, d), keep, "" if with_dkb else " dkb NULL"))
    for k in READ_GRADS:
        if k not in got:
            continue
        r, a = ref[k]
        if k == "dmem_in":
            rep.add(k, got[k], r, a, TOL_BWD[k])
        else:
            rep.add_inc(k, got[k], pre[k].view(r.shape), r, a, TOL_BWD[k])
    rep.check(same, "bit-identical rerun")
    rep.done()


@pytest.mark.parametrize("B,N,d,keep", [(64, 196, 512, 0.85), (4, 16, 128, 0.85), (5, 49, 128, 1.0), (2, 32, 256, 1.0),
                                        (1, 1, 128, 0.85)])
def test_read_bwd_tc32_matches_fp64(B, N, d, keep):
    """split-bf16 operands on the six [B*N, .] products (B*N = 245 and 1: contractions padded to 64)"""
    run_read_bwd_tc32(B, N, d, keep, seed=B * 1000 + N * 10 + d + 3)


def test_read_bwd_tc32_without_dkb():
    run_read_bwd_tc32(5, 49, 128, 0.85, seed=29, with_dkb=False)


def test_read_bwd_tc32_refuses_d_not_a_multiple_of_128():
    lb = lib()
    t = torch.zeros(1 << 20, device="cuda")
    rw = L_.ReadWeights(*([t.data_ptr()] * 9), 0.0, *([None] * 7))
    p = L_.ptr(t)
    torch.cuda.synchronize()
    before = lb.mac_b200_launch_count()
    for B, N, d in ((1, 64, 192), (5, 13, 64)):
        st = lb.mac_read_bwd_tc32(p, p, p, ctypes.byref(rw), p, p, p, p, 1.0, 0, 0, *([p] * 13), p,
                                  lb.mac_read_bwd_tc32_workspace_bytes(B, N, d), B, N, d, L_.stream_ptr())
        assert st == ERR_UNSUPPORTED, (B, N, d, st)
    torch.cuda.synchronize()
    assert lb.mac_b200_launch_count() == before
    assert not bool(t.any())


# ================================================================================================ 3. the cell vs fp64 autograd
@pytest.mark.parametrize("variant,shape,dp", [
    ("args", (8, 12, 196, 512, 2), (0.85, 0.85, 1.0)),
    ("gqa", (5, 7, 49, 128, 4), (0.9, 0.8, 0.9)),                     # B*N = 245
    ("args1", (5, 7, 20, 128, 4), (0.85, 0.85, 1.0)),                 # recurrent control chain
    ("args3", (4, 6, 20, 128, 3), (0.85, 1.0, 1.0)),
    ("args4", (4, 6, 20, 128, 3), (1.0, 0.85, 1.0)),
    ("args", (32, 20, 196, 512, 4), (0.85, 0.85, 1.0)),               # BASELINE config (2) with the training dropouts
])
def test_tc32_backward_matches_autograd(variant, shape, dp):
    """MACCell(prec="tc32") + mac_backward(tc=True) at the fp32 path's bars: forward < 1e-4, every gradient <= 2e-4 of its
    tensor's max"""
    from mac_network_b200.autograd import mac_backward
    from mac_network_b200.mac_cell import MACCell, MACParams, mac_network
    from oracle import mac_torch_autograd as TA
    B, S, N, d, L = shape
    over = dict(netLength=L, memDim=d, ctrlDim=d, attDim=d)
    if dp[2] < 1.0:
        over["writeDropout"] = dp[2]
    cfg = MACConfig.args(variant, **over)
    inputs = make_inputs(B, S, N, d, seed=51, dtype=np.float64)
    pv = perturb_biases(init_params(cfg, L, seed=52, dtype=np.float64), seed=53)
    rng = np.random.RandomState(54)
    gc, gm = rng.standard_normal((B, d)), rng.standard_normal((B, d))
    params = MACParams(cfg, L, values={k: v.astype(np.float32) for k, v in pv.items()})
    x = {k: torch.from_numpy(np.ascontiguousarray(v if v.dtype == np.int32 else v.astype(np.float32))).cuda()
         for k, v in inputs.items()}
    cell = MACCell(x["vecQuestions"], x["questionWords"], x["questionCntxWords"], x["questionLengths"],
                   x["knowledgeBase"], dp[0], dp[1], dp[2], B, True, config=cfg, params=params, seed=4242, prec="tc32",
                   save_for_backward=True)
    control, memory = mac_network(cell, L)
    grads = mac_backward(cell, torch.from_numpy(gc.astype(np.float32)).cuda(), torch.from_numpy(gm.astype(np.float32)).cuda(),
                         tc=True)
    torch.cuda.synchronize()
    rc, rm, rg = TA.run(cfg, pv, inputs, L, dp, cell.dropout_uniforms(), gc, gm)
    fwd = max(max_rel(memory.cpu().numpy(), rm), max_rel(control.cpu().numpy(), rc))
    worst = {}
    for k, ref in rg.items():
        got = grads[k].cpu().numpy()
        assert got.size == ref.size, k
        got = got.reshape(ref.shape)
        scale = np.max(np.abs(ref))
        if scale < 1e-12:
            assert np.max(np.abs(got)) < 1e-4, k
            continue
        worst[k] = float(np.max(np.abs(got - ref)) / scale)
    print("tc32 cell %s %s: forward %.2e, worst gradients %s" % (variant, shape, fwd,
          {k: "%.2e" % v for k, v in sorted(worst.items(), key=lambda kv: -kv[1])[:5]}))
    assert fwd < 1e-4, fwd
    bad = {k: v for k, v in worst.items() if v > 2e-4}
    assert not bad, bad


# ================================================================================================ 4. full shape
NULL_GRADIENTS = "inter2logits/linearLayerlogits/biases/bias"


def test_tc32_trainer_matches_its_fp32_twin_at_the_bench_shape():
    """DPTrainer(prec="tc32", bwd_tc=True) at B = 64, S = 40, N = 196, d = 512, L = 12: the first step's loss and every
    tensor of the gradient bucket within 2e-4 (of that tensor's max) of the fp32 trainer's"""
    from mac_network_b200.dp import DPTrainer
    B, S, N, d, L, A = 64, 40, 196, 512, 12, 32
    cfg = MACConfig.args("args", netLength=L, memDim=d, ctrlDim=d, attDim=d)
    batch = {k: torch.from_numpy(v).cuda() for k, v in make_inputs(B, S, N, d, seed=81).items()}
    answers = torch.from_numpy(np.random.RandomState(82).randint(0, A, size=(B,)).astype(np.int32)).cuda()
    out = {}
    for prec in ("fp32", "tc32"):
        tr = DPTrainer(cfg, L, seed=9, classifier=(A, [512]), prec=prec, bwd_tc=prec == "tc32")
        _, losses = tr.train_step_answers(0, batch, answers, B)
        torch.cuda.synchronize()
        out[prec] = (float(losses.mean()), tr.bucket.clone(), tr)
    l32, g32, tr32 = out["fp32"]
    lt, gt, _ = out["tc32"]
    worst, null = {}, {}
    gmax = float(g32.abs().max())
    for name in tr32.params.specs:
        o, n = tr32.params.offsets[name], int(np.prod(tr32.params.specs[name][0]) or 1)
        ref, got = g32[o:o + n].double(), gt[o:o + n].double()
        if name.endswith(NULL_GRADIENTS):
            # a softmax logit bias: its true gradient is exactly 0 (softmax is shift invariant), both buckets hold round-off
            null[name] = max(float(ref.abs().max()), float(got.abs().max())) / gmax
            continue
        scale = float(ref.abs().max())
        if scale < 1e-12:
            continue
        worst[name] = float((got - ref).abs().max()) / scale
    print("tc32 vs fp32 trainer: loss %.6f vs %.6f; worst gradients %s" % (
        lt, l32, {k.split("/")[-3] + "/" + k.split("/")[-1]: "%.2e" % v
                  for k, v in sorted(worst.items(), key=lambda kv: -kv[1])[:5]}))
    print("null gradients (of the bucket's max): %s" % {k.split("/")[-5]: "%.1e" % v for k, v in null.items()})
    assert abs(lt - l32) <= 2e-4 * abs(l32), (lt, l32)
    bad = {k: v for k, v in worst.items() if v > 2e-4}
    assert not bad, bad
    assert null and all(v < 1e-3 for v in null.values()), null


def test_tc32_train_step_full_lowers_the_loss():
    """the whole model (encoder and stem at their fp32 defaults) with the tc32 cell and the training dropouts:
    train_step_full lowers the loss"""
    from mac_network_b200.dp import DPTrainer
    from tests.test_full_model import _make
    B, S, V, E, d, H, W, C, A, L = 16, 9, 20, 20, 128, 5, 5, 32, 8, 3
    cfg, data = _make(B, S, V, E, d, H, W, C, A, L, seed=21)
    tr = DPTrainer(cfg, L, seed=6, lr=3e-3, classifier=(A, [32]), encoder=(V, E), stem=(C, 2), prec="tc32", bwd_tc=True)
    dev = {k: torch.from_numpy(v).cuda() for k, v in data.items()}
    hist = []
    for _ in range(12):
        _, losses = tr.train_step_full("t", dev, global_batch=B)
        hist.append(float(losses.mean().item()))
    print("tc32 train_step_full losses", [round(v, 4) for v in hist])
    assert np.all(np.isfinite(hist)) and min(hist[-3:]) < hist[0], hist
