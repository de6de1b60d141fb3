"""Tensor-core training and inference for the flag sets outside the shipped flag files ("P2", SURVEY section 8(a)):
`MACCell(prec="bf16")` with the composed read unit on `mac_linear_tc_seg_fwd`, and `mac_backward(tc=True)` on the tape
(`mac_linear_bwd_tc` for the composed read unit's [B*N, .] products, `mac_read_bwd_tc` for the fused one).

  * forward: the bf16 cell (eval, and train with the fixtures' dropouts) against the fp64 oracle (`oracle/mac_oracle.py`);
  * gradients: the tc=True tape gradients of every parameter and input against the fp32 tape gradients of the same cell and
    seed, which tests/test_gpu_tape_backward.py pins to finite differences of the oracle;
  * d = 512 at N = 196 for one composed-read and one fused-read flag set;
  * the whole model: `DPTrainer.train_step_full` with prec="bf16", bwd_tc=True against its fp32 twin.
Each bound is about three times the worst value measured on an H100 80GB HBM3, written beside it (DESIGN.md section 9)."""
import numpy as np
import pytest
import torch

from mac_network_b200.config import MACConfig
from mac_network_b200.params import init_params, perturb_biases
from mac_network_b200.synthetic import make_inputs
from tests._util import load_golden, max_rel

pytestmark = pytest.mark.gpu

P2_CASES = ["p2_control", "p2_control_feed", "p2_ablations", "p2_wholeq", "p2_unshared", "p2_read_bl", "p2_read_add",
            "p2_read_plain", "p2_read_noproj", "p2_write_info", "p2_write_sum", "p2_write_mem", "p2_write_mul",
            "p2_read_add_train", "p2_read_plain_train", "p2_memory_bn", "p2_memory_bn_train"]

#                                                                                                   measured
TOL_FWD = 2.5e-2         # bf16 cell against the fp64 oracle, max-rel of control_L / memory_L      7.3e-3 (1.5e-3 without
                         #   memoryBN's batch statistics over B = 4; 1.8e-3 at d = 512)
TOL_GRAD = 6e-2          # tc=True tape gradients against the fp32 tape, per tensor (_grad_errs)   1.9e-2 (8.4e-3 at d = 512)
TOL_NULL = 5e-3          # exactly-zero gradients (see _grad_errs): max |bf16| / median maximum    1.4e-3
WORST = {}


def _setup(case, B, N, d, S=5, seed=61):
    meta, _ = load_golden(case)
    L = meta["shape"]["L"]
    cfg = MACConfig(**dict(meta["cell_flags"], memDim=d, ctrlDim=d, attDim=d)).validate()
    inputs = make_inputs(B, S, N, d, seed=seed)
    pv = perturb_biases(init_params(cfg, L, seed=seed + 1), seed=seed + 2)
    dm = meta["dropouts"]
    return cfg, L, inputs, pv, (dm["memory"], dm["read"], dm["write"]), bool(meta["train"])


def _run(cfg, L, inputs, pv, dp, prec, train, save, seed=4242):
    from mac_network_b200.mac_cell import MACCell, MACParams, mac_network
    B = inputs["knowledgeBase"].shape[0]
    params = MACParams(cfg, L, values={k: v.astype(np.float32) for k, v in pv.items()})
    x = {k: torch.from_numpy(np.ascontiguousarray(v if v.dtype == np.int32 else v.astype(np.float32))).cuda()
         for k, v in inputs.items()}
    cell = MACCell(x["vecQuestions"], x["questionWords"], x["questionCntxWords"], x["questionLengths"], x["knowledgeBase"],
                   dp[0], dp[1], dp[2], B, train, config=cfg, params=params, prec=prec, seed=seed, save_for_backward=save)
    control, memory = mac_network(cell, L)
    return cell, control, memory


def _oracle(cfg, L, inputs, pv, dp, uniforms, train):
    from oracle.mac_oracle import MACOracle
    orc = MACOracle(cfg, pv, dtype=np.float64)
    orc.train = train
    return orc.run(L, inputs["vecQuestions"], inputs["questionWords"], inputs["questionCntxWords"], inputs["questionLengths"],
                   inputs["knowledgeBase"], memoryDropout=dp[0], readDropout=dp[1], writeDropout=dp[2], uniforms=uniforms)


def _note(key, v):
    WORST[key] = max(WORST.get(key, 0.0), v)
    return v


def _grad_errs(got, ref):
    """Per tensor: max |got - ref| over max(max |ref|, 1e-2 x the median of those maxima).  A gradient that is exactly zero in
    exact arithmetic -- the softmax logit biases, and whatever only shifts the logits of one softmax (shift invariance) --
    comes out of the fp32 tape at round-off (below 1e-4 x the median maximum): those are reported as "null:<name>" with
    max |got| over the median maximum, the level at which bf16 leaves them."""
    scales = {k: float(r.abs().max()) for k, r in ref.items()}
    med = float(np.median([v for v in scales.values() if v > 0]))
    out = {}
    for k, r in ref.items():
        if scales[k] < 1e-4 * med:
            out["null:" + k] = float(got[k].abs().max()) / med
        else:
            out[k] = float((got[k] - r).abs().max()) / max(scales[k], 1e-2 * med)
    return out


def _bad(errs):
    return {k: v for k, v in errs.items() if not v < (TOL_NULL if k.startswith("null:") else TOL_GRAD)}


def _show(errs, n=3):
    top = sorted(((k, v) for k, v in errs.items() if not k.startswith("null:")), key=lambda kv: -kv[1])[:n]
    null = [(k, v) for k, v in errs.items() if k.startswith("null:")]
    return ", ".join("%s %.2e" % (k.replace("MACnetwork/MACCell/", ""), v) for k, v in top + null)


def _forward_check(case, B, N, d):
    cfg, L, inputs, pv, dp, train = _setup(case, B, N, d)
    errs = {}
    for mode in ("eval", "train"):
        t = mode == "train"
        dpm = dp if t else (1.0, 1.0, 1.0)
        cell, control, memory = _run(cfg, L, inputs, pv, dpm, "bf16", train=t and train, save=t)
        torch.cuda.synchronize()
        us = cell.dropout_uniforms() if (t and min(dpm) < 1.0) else None
        ref = _oracle(cfg, L, inputs, pv, dpm, us, t and train)
        errs[mode] = _note("fwd", max(max_rel(control.cpu().numpy(), ref.control), max_rel(memory.cpu().numpy(), ref.memory)))
    print("%s B=%d N=%d d=%d bf16 forward vs fp64: eval %.2e train %.2e" % (case, B, N, d, errs["eval"], errs["train"]))
    return errs


def _grad_check(case, B, N, d):
    from mac_network_b200.autograd import mac_backward
    cfg, L, inputs, pv, dp, train = _setup(case, B, N, d)
    rng = np.random.RandomState(7)
    gc = torch.from_numpy(rng.standard_normal((B, d)).astype(np.float32)).cuda()
    gm = torch.from_numpy(rng.standard_normal((B, d)).astype(np.float32)).cuda()
    grads = {}
    for prec, tc in (("fp32", False), ("bf16", True)):
        cell, _, _ = _run(cfg, L, inputs, pv, dp, prec, train=train, save=True)
        assert cell._tape is not None
        g = mac_backward(cell, gc, gm, tc=tc)
        torch.cuda.synchronize()
        grads[prec] = {k: v.double().cpu() for k, v in g.items()}
    errs = _grad_errs(grads["bf16"], grads["fp32"])
    _note("grad", max(v for k, v in errs.items() if not k.startswith("null:")))
    _note("null", max([v for k, v in errs.items() if k.startswith("null:")] + [0.0]))
    print("%s B=%d N=%d d=%d tc tape grads vs fp32 tape over %d tensors: %s" % (case, B, N, d, len(errs), _show(errs)))
    return errs


@pytest.mark.parametrize("case", P2_CASES)
def test_p2_bf16_forward_matches_the_oracle(case):
    errs = _forward_check(case, 4, 16, 128)
    assert max(errs.values()) < TOL_FWD, errs


@pytest.mark.parametrize("case", P2_CASES)
def test_p2_tc_tape_gradients_match_the_fp32_tape(case):
    errs = _grad_check(case, 4, 16, 128)
    bad = _bad(errs)
    assert not bad, bad


def test_composed_read_with_bn_not_a_multiple_of_64():
    """B*N = 147: the composed read unit's products need no 64-row multiple."""
    errs = _forward_check("p2_read_add_train", 3, 49, 128)
    assert max(errs.values()) < TOL_FWD, errs
    errs = _grad_check("p2_read_add_train", 3, 49, 128)
    bad = _bad(errs)
    assert not bad, bad


@pytest.mark.parametrize("case,B", [("p2_read_add_train", 2), ("p2_memory_bn_train", 16)])
def test_headline_width(case, B):
    """d = 512, N = 196 (the 14 x 14 grid): forward and gradients against the fp32 cell / fp32 tape of the same seed."""
    from mac_network_b200.autograd import mac_backward
    d, N = 512, 196
    cfg, L, inputs, pv, dp, train = _setup(case, B, N, d)
    rng = np.random.RandomState(9)
    gm = torch.from_numpy(rng.standard_normal((B, d)).astype(np.float32)).cuda()
    out = {}
    for prec, tc in (("fp32", False), ("bf16", True)):
        cell, control, memory = _run(cfg, L, inputs, pv, dp, prec, train=train, save=True)
        g = mac_backward(cell, None, gm, tc=tc)
        torch.cuda.synchronize()
        out[prec] = (memory.double().cpu(), {k: v.double().cpu() for k, v in g.items()})
    fwd = float((out["bf16"][0] - out["fp32"][0]).abs().max() / out["fp32"][0].abs().max())
    errs = _grad_errs(out["bf16"][1], out["fp32"][1])
    _note("fwd512", fwd)
    _note("grad512", max(v for k, v in errs.items() if not k.startswith("null:")))
    _note("null", max([v for k, v in errs.items() if k.startswith("null:")] + [0.0]))
    print("%s B=%d N=%d d=%d: memory %.2e, gradients %s" % (case, B, N, d, fwd, _show(errs)))
    assert fwd < TOL_FWD
    bad = _bad(errs)
    assert not bad, bad


TOL_TRAINER_LOSS = 2.5e-4   # relative, both steps                                                 7.6e-5
TOL_TRAINER_GRAD = 3e-2     # gradient bucket per tensor (_grad_errs)                              9.9e-3


def test_full_model_p2_bf16_matches_its_fp32_twin():
    """train_step_full on the p2_read_add flags (composed read unit): prec="bf16", bwd_tc=True against prec="fp32" from
    the same parameters and data, dropouts off; then one more step of each from its own updated parameters."""
    from mac_network_b200.dp import DPTrainer
    from tests.test_full_model import _make
    B, S, V, E, d, H, W, C, A, L = 16, 7, 13, 16, 128, 4, 4, 128, 8, 2
    _, data = _make(B, S, V, E, d, H, W, C, A, L, seed=41)
    meta, _ = load_golden("p2_read_add")
    cfg = MACConfig(**dict(meta["cell_flags"], memDim=d, ctrlDim=d, attDim=d, netLength=L)).validate()
    kw = dict(classifier=(A, [32]), encoder=(V, E), stem=(C, 2), dropouts=(1.0, 1.0, 1.0), output_dropout=1.0,
              enc_dropouts=(1.0, 1.0), stem_dropout=1.0)
    dev = {k: torch.from_numpy(v).cuda() for k, v in data.items()}
    res, ref_flat = {}, None
    for prec in ("fp32", "bf16"):
        tr = DPTrainer(cfg, L, seed=8, prec=prec, bwd_tc=prec == "bf16", **kw)
        if ref_flat is None:
            ref_flat = tr.params.flat.clone()
        tr.params.flat.copy_(ref_flat)
        tr.params.touch()
        _, losses = tr.full_forward_backward("t", dev, global_batch=B)
        torch.cuda.synchronize()
        bucket = tr.bucket.double().cpu()
        tr.apply()
        _, losses2 = tr.train_step_full("t", dev, global_batch=B)
        torch.cuda.synchronize()
        res[prec] = (float(losses.double().mean()), bucket, float(losses2.double().mean()))
    specs = tr.params.specs
    sl = lambda b, n: b[tr.params.offsets[n]:tr.params.offsets[n] + (int(np.prod(specs[n][0])) if specs[n][0] else 1)]
    errs = _grad_errs({n: sl(res["bf16"][1], n) for n in specs}, {n: sl(res["fp32"][1], n) for n in specs})
    worst = max(((k, v) for k, v in errs.items() if not k.startswith("null:")), key=lambda kv: kv[1])
    loss_err = abs(res["bf16"][0] - res["fp32"][0]) / abs(res["fp32"][0])
    loss2_err = abs(res["bf16"][2] - res["fp32"][2]) / abs(res["fp32"][2])
    _note("trainer_loss", max(loss_err, loss2_err))
    _note("trainer_grad", worst[1])
    print("train_step_full p2_read_add bf16 vs fp32: loss %.4f vs %.4f (%.2e), next step %.4f vs %.4f (%.2e); gradients %s"
          % (res["bf16"][0], res["fp32"][0], loss_err, res["bf16"][2], res["fp32"][2], loss2_err, _show(errs)))
    assert np.isfinite(res["bf16"][2]) and loss_err < TOL_TRAINER_LOSS and loss2_err < TOL_TRAINER_LOSS
    assert worst[1] < TOL_TRAINER_GRAD, worst
    assert all(v < TOL_NULL for k, v in errs.items() if k.startswith("null:")), errs


def test_zz_print_worst():
    print("worst measured:", {k: "%.2e" % v for k, v in sorted(WORST.items())})
