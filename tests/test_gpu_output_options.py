"""The output unit's layouts (--outQuestion off, --outQuestionMul, --outputBN) on the GPU:
- `OutputUnit` against fp64 autograd (`oracle/output_options.output_graph`) for every layout at B = 64, memDim = 512,
  in training (dropout 0.85, batch statistics) and at evaluation (stored statistics), with the fp32 path's bars: the logits
  within 1e-4 of their max-norm, each gradient within 2e-4 of its tensor's maximum, the stored statistics within 1e-4;
- the whole model's training step against the fp64 graph of tests/test_gpu_model_gradients.py with the layout's output unit
  (`oracle/output_options.output_graph_for`) in place of the shipped one, in fp32 and on the tensor-core paths, at each
  precision's bar (STEP_BARS);
- `runBatch(train=False, use_ema=True)` evaluates on the live stored statistics; `ModelPipeline` and `TrainPipeline` bit for
  bit against `runBatch`; `MACModel.from_trainer` bit for bit against `DPTrainer`; a training-state round trip."""
import numpy as np
import pytest
import torch

from oracle import model_torch_autograd as MA
from oracle import output_options as OO
from oracle.philox import philox_uniform
from tests.test_gpu_wgmma import keep_threshold

pytestmark = pytest.mark.gpu

LAYOUTS = {"q0": dict(question=False, mul=False), "q1": dict(question=True, mul=False), "qmul": dict(question=True, mul=True)}
WIDTHS = [(), (512,), (512, 256)]


def _rel(got, want):
    return float((got.double() - want).abs().max()) / max(float(want.abs().max()), 1e-300)


@pytest.mark.parametrize("layout,bn", [(l, bn) for l in LAYOUTS for bn in (False, True)])
@pytest.mark.parametrize("hidden", WIDTHS, ids=["h0", "h512", "h512_256"])
@pytest.mark.parametrize("train", [False, True], ids=["eval", "train"])
def test_output_unit_against_fp64(layout, bn, hidden, train):
    from mac_network_b200.output_unit import SITE_OUTPUT, OutputUnit, init_output_params, output_specs
    B, d, A, keep, step, seed, decay = 64, 512, 64, 0.85 if train else 1.0, 3, 11, 0.9
    opts = LAYOUTS[layout]
    values = init_output_params(output_specs(d, d, hidden, A, bn=bn, **opts), seed=5)
    p = {k: torch.from_numpy(v).cuda() for k, v in values.items()}
    rng = np.random.RandomState(6)
    mem = torch.from_numpy(rng.standard_normal((B, d)).astype(np.float32)).cuda()
    vq = torch.from_numpy(np.tanh(rng.standard_normal((B, d))).astype(np.float32)).cuda()
    answers = torch.from_numpy(rng.randint(0, A, size=(B,)).astype(np.int32)).cuda()
    out = OutputUnit(p, relu="ELU", keep=keep, seed=seed, bn=bn, bn_decay=decay, **opts)
    logits, _, _ = out.forward(mem, vq, answers, step=step, loss_scale=1.0 / B, train=train)
    grads = {k: torch.zeros_like(v) for k, v in p.items()}
    d_mem, d_vq = torch.zeros_like(mem), torch.zeros_like(vq)
    out.backward(grads, d_mem, d_vq)
    torch.cuda.synchronize()
    # the fp64 graph, fed the kernels' exact dropout masks (Philox at the unit's sites, [B, F] numbering)
    masks = []
    if keep < 1.0:
        for i in range(out.nfc):
            F = values["classifier/linearLayerfc_%d/weights/weight" % i].shape[0]
            r = philox_uniform(seed, SITE_OUTPUT + i, step, B * F).reshape(B, F)
            masks.append(MA.mask_uniforms(r * 16777216.0 >= keep_threshold(keep)))
    t = {k: torch.from_numpy(v).double().cuda().requires_grad_("/moving_" not in k) for k, v in values.items()}
    m64, q64 = mem.double().requires_grad_(True), vq.double().requires_grad_(True)
    moving = {}
    ref_logits, losses = OO.output_graph("ELU", t, m64, q64, answers.long(), keep, [m.cuda() for m in masks], bn=bn,
                                         train=train, decay=decay, moving=moving, **opts)
    (losses.sum() / B).backward()
    errs = {"logits": _rel(logits, ref_logits.detach()), "d_memory": _rel(d_mem, m64.grad)}
    if opts["question"]:
        errs["d_vecQuestions"] = _rel(d_vq, q64.grad)
    else:
        assert not bool(d_vq.any())                     # no gradient into vecQuestions without the question
    # the question's bias shifts whole columns of q', which the batch statistics remove again: without the product its
    # gradient is 0 in exact arithmetic, so it is measured against the unit's largest gradient
    null = "outputUnit/linearLayeroutQuestion/biases/bias" if (bn and train and not opts["mul"]) else None
    gmax = max(float(v.grad.abs().max()) for v in t.values() if v.requires_grad)
    for k, v in t.items():
        if k == null:
            errs[k] = float(grads[k].double().abs().max()) / gmax
        elif v.requires_grad:
            errs[k] = _rel(grads[k], v.grad)
        else:
            assert not bool(grads[k].any()), k          # the stored statistics get no gradient
    bars = {k: (1e-4 if k == "logits" else 2e-4) for k in errs}
    for k in (k for k in values if "/moving_" in k):
        want = moving[k] if train else torch.from_numpy(values[k]).double().cuda()
        errs[k] = _rel(p[k], want)
        bars[k] = 1e-4
        assert torch.equal(p[k].cpu(), torch.from_numpy(values[k])) == (not train), k
    print(layout, bn, hidden, train, "worst %.2e" % max(errs.values()))
    assert all(errs[k] < bars[k] for k in errs), {k: v for k, v in errs.items() if not v < bars[k]}
    # the label-free form: bit for bit the forward at keep 1 on the stored statistics
    if not train:
        assert torch.equal(out.logits(mem, vq), logits)


# ------------------------------------------------------------------------------------------------ the whole model
STEP_CASES = {
    "q0_fp32": (dict(question=False, mul=False, bn=False), dict(d=64, C=32, HW=(3, 5))),
    "qmul_bn_fp32": (dict(question=True, mul=True, bn=True), dict(d=64, C=32, HW=(3, 5))),
    "q0_tc32_bf16x3": (dict(question=False, mul=False, bn=False),
                       dict(d=128, C=128, HW=(4, 4), prec="tc32", bwd_tc=True, stem_prec="bf16x3")),
    "qmul_bn_tc32_bf16x3": (dict(question=True, mul=True, bn=True),
                            dict(d=128, C=128, HW=(4, 4), prec="tc32", bwd_tc=True, stem_prec="bf16x3")),
    "qmul_bn_bf16": (dict(question=True, mul=True, bn=True),
                     dict(d=128, C=128, HW=(4, 4), prec="bf16", bwd_tc=True, stem_prec="bf16")),
}


# The suite's bars for each precision: 2e-4 for fp32 and the split-bf16 paths, the bf16 cell backward's 5e-2 for the bf16
# ones; the null gradients against the model's largest.  Measured worst on an H100 80GB HBM3 (700 W power limit): fp32
# 2.0e-6, tc32 / bf16x3 3.2e-5, bf16 1.2e-2; null 1.6e-7; the stored statistics 8.0e-6 (fp32), 9.1e-6 (tc32) and 1.3e-3
# (bf16: the batch mean of features computed by the bf16 cell).  The batch norm over B = 8 rows divides by a small
# batch's deviation, which is why some exceed the shipped layout's measured bars in test_gpu_model_gradients.py while
# staying well inside the precision's own.
STEP_BARS = {"fp32": 2e-4, "tc32": 2e-4, "bf16": 5e-2}
STAT_BARS = {"fp32": 1e-4, "tc32": 1e-4, "bf16": 5e-2}
NULL_BAR = 1e-6


@pytest.mark.parametrize("name", list(STEP_CASES))
def test_trainer_step_with_output_options(name, monkeypatch):
    from mac_network_b200.dp import DPTrainer
    from tests import test_gpu_model_gradients as G
    from tests.test_model_autograd_oracle import dropout_plan, make_data, model_config, training_keeps
    opts, shape = STEP_CASES[name]
    c = G._case(dict(flags="args", **shape))
    cfg, cell_dp = model_config(c["flags"], c["d"], G.L)
    H, W = c["HW"]
    tr = DPTrainer(cfg, G.L, seed=G.BASE_SEED, lr=1e-3, dropouts=cell_dp, classifier=(G.A, G.HIDDEN, opts),
                   encoder=(G.V, G.E), stem=(c["C"], 2), prec=c["prec"], bwd_tc=c["bwd_tc"], stem_prec=c["stem_prec"],
                   enc_prec=c["enc_prec"])
    first = make_data(G.B, G.S, G.V, G.B, H, W, c["C"], G.A, seed=60)
    tr.train_step_full("step0", {k: torch.from_numpy(v).cuda() for k, v in first.items()}, global_batch=G.B)
    data = make_data(G.B, G.S, G.V, G.B, H, W, c["C"], G.A, seed=61)
    keeps = training_keeps(cell_dp)
    dev = G._device(data, "nhwc")
    values = tr.params.numpy()
    logits, losses = tr.full_forward_backward("t", dev, global_batch=G.B)
    torch.cuda.synchronize()
    plan = dropout_plan(cfg, G.L, values, keeps, G.B, G.S, G.B, H, W, step=tr.step_id)
    raw = G.draws(plan, G.philox_seed(G.BASE_SEED, tr.step_id, 0))
    moving = {}                 # the whole-model graph with this layout's output unit in place of the shipped one
    monkeypatch.setattr(MA, "output_graph", OO.output_graph_for(opts, cfg.bnDecay, moving))
    ref = MA.run(cfg, G.L, values, G._oracle_data(data, dev), keeps, G.kernel_masks(plan, raw, keeps), global_batch=G.B,
                 device="cuda")
    p = tr.params
    got = {n: tr.bucket[p.offsets[n]:p.offsets[n] + max(1, int(np.prod(p.specs[n][0])))] for n in p.specs}
    assert opts["question"] == any(n.startswith("outputUnit/") for n in p.specs)
    errs, null = G._compare(got, ref, logits, losses)
    stats = {k: _rel(p.t[k], v) for k, v in moving.items()}     # after the training forward
    assert bool(stats) == opts["bn"]
    kind = G._kind(c)
    print("%s [%s]: worst %.2e (%s), null %.2e, statistics %.2e" % (
        name, kind, max(errs.values()), max(errs, key=errs.get), max(null.values()) if null else 0.0,
        max(stats.values()) if stats else 0.0))
    bar = STEP_BARS[kind]
    bad = {k: v for k, v in errs.items() if not v < bar}
    bad.update({k: v for k, v in null.items() if not v < NULL_BAR})
    bad.update({k: v for k, v in stats.items() if not v < STAT_BARS[kind]})
    assert not bad, (name, bad)


# ------------------------------------------------------------------------------------------------ model, pipelines, modules
V, E, C, A, L = 90, 300, 128, 28, 3
OUT = dict(out_question=True, out_question_mul=True, output_bn=True)


def _net(seed=3, **kw):
    from mac_network_b200.config import MACConfig
    from mac_network_b200.model import MACnet
    cfg = MACConfig.args("args", netLength=L)
    return MACnet(cfg, L, V, A, wrd_emb_dim=E, image_in_dim=C, classifier_dims=(512,), seed=seed, lr=1e-3,
                  ema_decay=0.9, **dict(OUT, **kw))


def _batch(seed, B=8, S=12, HW=8):
    rng = np.random.RandomState(seed)
    lengths = rng.randint(1, S + 1, size=(B,)).astype(np.int32)
    lengths[0] = S
    q = rng.randint(1, V + 1, size=(B, S)).astype(np.int32)
    q[np.arange(S)[None, :] >= lengths[:, None]] = 0
    return {"questions": q, "questionLengths": lengths, "answers": rng.randint(0, A, size=(B,)).astype(np.int32),
            "images": np.maximum(rng.standard_normal((B, C, HW, HW)), 0).astype(np.float32)}


def _run(net, b, train, **kw):
    return net.runBatch(None, {k: b[k] for k in ("questions", "questionLengths", "answers")}, {"images": b["images"]},
                        train=train, **kw)


def _moving(net):
    t = net.trainer
    return {k: v.clone() for k, v in t.params.t.items() if "classifier/" in k and "/moving_" in k}


def test_eval_with_ema_uses_live_statistics():
    net = _net(prec="fp32")
    for s in range(2):
        _run(net, _batch(40 + s), True)
    t = net.trainer
    live = _moving(net)
    assert t.n_train < t.params.numel and not torch.equal(t.ema[:t.n_train], t.params.flat[:t.n_train])
    before = t.params.flat.clone()
    net.use_ema = True
    r_ema = _run(net, _batch(50), False)
    net.use_ema = False
    assert torch.equal(t.params.flat, before)
    ema_logits = net._out.last_logits.clone()
    # the same evaluation by hand: the EMA weights, the live statistics
    saved = t.params.flat.clone()
    t.params.flat[:t.n_train].copy_(t.ema[:t.n_train])
    t.params.touch()
    assert all(torch.equal(v, live[k]) for k, v in _moving(net).items())
    r_hand = _run(net, _batch(50), False)
    assert torch.equal(net._out.last_logits, ema_logits) and r_hand["loss"] == r_ema["loss"]
    t.params.flat.copy_(saved)
    t.params.touch()
    # and evaluation does not move the statistics
    assert all(torch.equal(v, live[k]) for k, v in _moving(net).items())


def test_model_pipeline_equals_run_batch():
    from mac_network_b200.serving import ModelPipeline
    net = _net(prec="fp32")
    _run(net, _batch(40), True)                     # statistics and weights off their initial values
    pipe = ModelPipeline(net, (8, 12, 8, 8), slots=2)
    for s in (51, 52):
        b = _batch(s)
        _run(net, b, False)
        want = net._out.last_logits.cpu()
        out = pipe.result(pipe.submit({k: b[k] for k in ("questions", "questionLengths", "images")}))
        assert torch.equal(out["logits"], want), s


def test_train_pipeline_equals_run_batch():
    from mac_network_b200.serving import TrainPipeline
    a, b = _net(prec="bf16"), _net(prec="bf16")
    batches = [_batch(60 + i) for i in range(2)]
    wants = [_run(a, x, True) for x in batches]
    pipe = TrainPipeline(b, (8, 12, 8, 8), depth=2)
    tickets = [pipe.submit(x) for x in batches]
    for tk, w in zip(tickets, wants):
        r = pipe.result(tk)
        assert r["loss"] == w["loss"] and r["gradNorm"] == w["gradNorm"] and r["correctNum"] == w["correctNum"]
    pipe.drain()
    ta, tb = a.trainer, b.trainer
    for x, y in ((ta.params.flat, tb.params.flat), (ta.adam_m, tb.adam_m), (ta.adam_v, tb.adam_v), (ta.ema, tb.ema)):
        assert torch.equal(x, y)
    assert all(torch.equal(v, _moving(b)[k]) for k, v in _moving(a).items())


@pytest.mark.parametrize("opts", [dict(question=False, mul=False, bn=False), dict(question=True, mul=True, bn=True)],
                         ids=["q0", "qmul_bn"])
def test_mac_model_equals_the_trainer_bit_for_bit(opts):
    from mac_network_b200.config import MACConfig
    from mac_network_b200.dp import DPTrainer
    from mac_network_b200.modules import MACModel, answer_loss
    cfg = MACConfig.args("args", netLength=L, memDim=128, ctrlDim=128, attDim=128)
    t = DPTrainer(cfg, L, seed=3, classifier=(A, [64], opts), encoder=(V, 64), stem=(64, 2))

    def data(seed):
        b = _batch(seed)
        dev = {k: torch.from_numpy(b[k]).cuda() for k in ("questions", "questionLengths", "answers")}
        dev["images_nchw"] = torch.from_numpy(b["images"][:, :64]).cuda().contiguous()
        return dev
    t.train_step_full((8, 12), data(1), global_batch=8)
    m = MACModel.from_trainer(t)
    assert sorted(n for n, _ in m.named_buffers()) == sorted(k for k in t.params.specs
                                                              if k.startswith("classifier/") and "/moving_" in k)
    d2 = data(2)
    logits, _ = m(d2["questions"], d2["questionLengths"], images_nchw=d2["images_nchw"])
    answer_loss(logits, d2["answers"]).backward()
    t_logits, _ = t.full_forward_backward((8, 12), d2, global_batch=8)
    torch.cuda.synchronize()
    assert torch.equal(logits.detach(), t_logits)
    bad = [n for n, p in m.named_parameters()
           if not torch.equal(p.grad.reshape(-1), t.bucket[t.params.offsets[n]:t.params.offsets[n] + p.numel()])]
    assert not bad, bad
    for n, buf in m.named_buffers():                                  # the training forward moved the same statistics
        assert torch.equal(buf, t.params.t[n]), n
    m.eval()
    with torch.no_grad():
        e1, _ = m(d2["questions"], d2["questionLengths"], images_nchw=d2["images_nchw"])
    assert all(torch.equal(buf, t.params.t[n]) for n, buf in m.named_buffers())     # eval reads them only


def test_training_state_round_trip(tmp_path):
    from mac_network_b200.checkpoint import load_training_state, save_training_state
    a, b = _net(prec="fp32"), _net(prec="fp32")              # the same seed: the same dropout streams from here on
    _run(a, _batch(40), True)
    b.trainer.params.flat.add_(0.5)
    b.trainer.params.touch()
    names = save_training_state(str(tmp_path / "s.npz"), a.trainer)
    assert not any("/moving_" in n and n.endswith(("/ExponentialMovingAverage", "/Adam", "/Adam_1")) for n in names)
    load_training_state(str(tmp_path / "s.npz"), b.trainer)
    for k, v in a.trainer.params.t.items():
        assert torch.equal(v, b.trainer.params.t[k]), k
    wa, wb = _run(a, _batch(41), True), _run(b, _batch(41), True)
    assert wa["loss"] == wb["loss"] and torch.equal(a.trainer.params.flat, b.trainer.params.flat)
