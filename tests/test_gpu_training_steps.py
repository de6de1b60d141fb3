"""Training across optimizer steps, and the state that lives from one step to the next: the weight-derived entries of
`MACParams.cache` (packs, transposes, `ReadWeights`, folded weights, the scalar biases read with `.item()`), the cached
training cells with their persistent inputs and split-K workspaces, the tape and the encoder's / stem's saved state, the
step counter in Adam's bias correction and in every dropout seed, memoryBN's moving statistics, the EMA swap of
evaluation, and the graphs `serving.HostPipeline` captures.

(a) A long-lived `DPTrainer` against a freshly built twin loaded with its pre-step state, bit for bit at every step (the
    kernels are deterministic: split-K combines in a fixed order and nothing accumulates with atomics).  The long-lived
    trainer's steps reuse cached cells, rebuild an evicted one and reuse that again; the twin builds every cell.  Each optimizer
    step element by element against `dp.adam_reference`, which a twin that shares a wrongly plumbed step counter or
    hyperparameter would not catch.
(b) The fp32 trainer at weights that have moved (biases no longer 0) against the fp64 oracle chain and the fp64 autograd graph,
    and its tc32 twin there.
(c) Resume from `save_training_state` equals the uninterrupted run bit for bit.
(d) `MACnet.runBatch` evaluation between training steps equals a fresh model's, and does not disturb the training run.
(e) `HostPipeline` after a weight update equals a direct cell on the new weights."""
import numpy as np
import pytest
import torch

from mac_network_b200.config import MACConfig
from tests._util import load_golden, max_rel
from tests.test_full_model import _make, _oracle_loss, check_bucket_against_fp64
from tests.test_gpu_backward_kernels import same_bits

pytestmark = pytest.mark.gpu

# (B, S) per step: five distinct cell keys through the trainer's 4-entry LRU.  Step 3 reuses step 2's cell (a cache hit:
# persistent inputs copied again, workspaces, tape and saved state of the previous step); step 6 evicts (8, 6), step 7
# builds it again and step 8 reuses that rebuilt cell.  N = H * W = 16 keeps B * N a multiple of 64 (the tensor-core read
# backward).
KEYS = [(8, 6), (12, 7), (12, 7), (16, 5), (4, 7), (8, 4), (8, 6), (8, 6)]
HITS = {2, 7}                           # the steps (0-based) that reuse a cached cell
H, W, V, E, A, L = 4, 4, 20, 16, 8, 3
HP = dict(lr=1e-3, clip=1.0, ema_decay=0.99, beta1=0.9, beta2=0.999, eps=1e-8)

# case -> shipped flag file or golden fixture (its cell flags and dropouts), widths, precisions
CASES = {
    "fp32_scheduled": dict(flags="args", d=64, C=32),
    "fp32_history": dict(flags="gqa", d=64, C=32),                     # self-attention over the history, write gate
    "tape_memory_bn": dict(golden="p2_memory_bn_train", C=16),           # its own d = 16
    "tape_tc": dict(golden="p2_read_add_train", d=128, C=32, prec="bf16", bwd_tc=True),     # composed read unit
    "bf16": dict(flags="args", d=128, C=128, prec="bf16", bwd_tc=True, stem_prec="bf16"),
    "tc32": dict(flags="args", d=128, C=128, prec="tc32", stem_prec="bf16x3"),
    "all_tc": dict(flags="args", d=512, C=128, prec="tc32", bwd_tc=True, stem_prec="bf16x3", enc_prec="bf16"),
}
STATE = ("flat", "adam_m", "adam_v", "ema")


def _config(case):
    c = CASES[case]
    if "golden" in c:
        meta, _ = load_golden(c["golden"])
        d = c.get("d", meta["shape"]["d"])
        cfg = MACConfig(**dict(meta["cell_flags"], memDim=d, ctrlDim=d, attDim=d, netLength=L)).validate()
        dm = meta["dropouts"]
        return cfg, (dm["memory"], dm["read"], dm["write"])
    return MACConfig.args(c["flags"], netLength=L, memDim=c["d"], ctrlDim=c["d"], attDim=c["d"]), None


def _trainer(case):
    """The reference's training dropouts (the flag file's, or the fixture's for the cell) throughout."""
    from mac_network_b200.dp import DPTrainer
    c = CASES[case]
    cfg, dropouts = _config(case)
    return DPTrainer(cfg, L, seed=7, dropouts=dropouts, classifier=(A, [32]), encoder=(V, E), stem=(c["C"], 2),
                     prec=c.get("prec", "fp32"), bwd_tc=c.get("bwd_tc", False), stem_prec=c.get("stem_prec", "fp32"),
                     enc_prec=c.get("enc_prec", "fp32"), **HP)


def _data(case, i):
    B, S = KEYS[i]
    _, data = _make(B, S, V, E, 64, H, W, CASES[case]["C"], A, L, seed=200 + i)       # (its config is not used)
    return {k: torch.from_numpy(v).cuda() for k, v in data.items()}


def _state(tr):
    return dict({k: getattr(tr, k).clone() for k in STATE[1:]}, flat=tr.params.flat.clone(), step_id=tr.step_id)


def _load(tr, st):
    for k in STATE[1:]:
        getattr(tr, k).copy_(st[k])
    tr.params.flat.copy_(st["flat"])
    tr.step_id = st["step_id"]
    tr.params.touch()


def _step(tr, i, dev):
    """`train_step_full` in its two halves, keeping what each leaves: logits, losses, the bucket before the optimizer step
    (and the weights it starts from: memoryBN's forward writes its moving statistics into them), then the state after it."""
    B, S = KEYS[i]
    logits, losses = tr.full_forward_backward((B, S), dev, global_batch=B)
    rec = {"logits": logits.clone(), "losses": losses.clone(), "bucket": tr.bucket.clone(),
           "pre_apply": tr.params.flat.clone()}
    tr.apply()
    rec["norm"] = tr.norm.clone()
    rec.update({k: v for k, v in _state(tr).items() if k != "step_id"})
    return rec


def _differ(got, want):
    return [k for k in want if not same_bits(got[k], want[k])]


def _check_adam(rec, pre, step):
    """The fused clip / Adam / EMA step against dp.adam_reference from the pre-step state, at the bars of
    tests/test_gpu_backward.py::test_dp_half_batches_sum_to_full_batch_and_optimizer_step."""
    from mac_network_b200.dp import adam_reference
    h = lambda t: t.cpu().numpy()
    p1, m1, v1, e1, norm = adam_reference(h(rec["pre_apply"]), h(rec["bucket"]), h(pre["adam_m"]), h(pre["adam_v"]),
                                          h(pre["ema"]), step=step, lr=HP["lr"], clip=HP["clip"], b1=HP["beta1"],
                                          b2=HP["beta2"], eps=HP["eps"], ema_decay=HP["ema_decay"])
    errs = {"norm": abs(float(rec["norm"][0]) - norm) / norm, "flat": float(np.max(np.abs(h(rec["flat"]) - p1))),
            "ema": float(np.max(np.abs(h(rec["ema"]) - e1))), "adam_m": max_rel(h(rec["adam_m"]), m1),
            "adam_v": max_rel(h(rec["adam_v"]), v1)}
    bars = {"norm": 1e-4, "flat": 1e-6, "ema": 1e-6, "adam_m": 2e-4, "adam_v": 2e-4}
    bad = {k: v for k, v in errs.items() if not v < bars[k]}
    assert not bad, (step, bad)


def _bn_slices(tr):
    p = tr.params
    return [slice(p.offsets[k], p.offsets[k] + p.specs[k][0][0]) for k in p.specs
            if k.endswith(("/moving_mean", "/moving_variance"))]


# ================================================================================================ (a) against a fresh twin
@pytest.mark.parametrize("case", list(CASES))
def test_long_lived_trainer_equals_a_fresh_twin_at_every_step(case):
    tr = _trainer(case)
    bn = _bn_slices(tr)
    assert bool(bn) == (case == "tape_memory_bn")
    bn_moved = set()
    hits = set()
    for i in range(len(KEYS)):
        dev = _data(case, i)
        pre = _state(tr)
        cached = tr._cells.get(KEYS[i], (None,))[0]
        got = _step(tr, i, dev)
        if cached is not None:
            assert tr._cells[KEYS[i]][0] is cached, i          # the step ran on the cell of an earlier step
            hits.add(i)
        twin = _trainer(case)
        _load(twin, pre)
        want = _step(twin, i, dev)
        del twin
        torch.cuda.synchronize()
        bad = _differ(got, want)
        assert not bad, (case, "step %d, key %s" % (i + 1, KEYS[i]), bad)
        _check_adam(got, pre, step=i + 1)
        assert tr.step_id == i + 1 and len(tr._cells) <= tr.MAX_CACHED_CELLS
        if i == 5:
            assert KEYS[0] not in tr._cells         # evicted: the next step builds its cell again
        for j, s in enumerate(bn):
            # zero gradient, Adam's m and v stay 0: the update of the moving statistics is exactly 0, and the forward moved them
            assert same_bits(got["flat"][s], got["pre_apply"][s]), (i, j)
            assert not bool(got["adam_m"][s].any()) and not bool(got["adam_v"][s].any()), (i, j)
            if not same_bits(got["pre_apply"][s], pre["flat"][s]):
                bn_moved.add(j)
    assert hits == HITS, hits
    assert len(bn_moved) == len(bn), bn_moved


# ================================================================================================ (b) fp64 at moved weights
def test_fp32_trainer_matches_fp64_at_moved_weights_and_so_does_its_tc32_twin():
    """fp32 `args`, every dropout 1.0, lr = 3e-3: logits and losses against the fp64 oracle chain at every step's weights;
    at step K every gradient tensor element by element against the fp64 graph, then a tc32 / bf16x3-stem twin's bucket and loss against the fp32 ones
    at the bars of test_gpu_tc32_training.py's bench-shape twin test (measured there at initialised weights only)."""
    from mac_network_b200.dp import DPTrainer
    from tests.test_gpu_tc32_training import NULL_GRADIENTS
    B, S, d, C, K = 8, 6, 128, 128, 4
    cfg, data = _make(B, S, V, E, d, H, W, C, A, L, seed=31)
    kw = dict(seed=9, lr=3e-3, classifier=(A, [32]), encoder=(V, E), stem=(C, 2), dropouts=(1.0, 1.0, 1.0),
              output_dropout=1.0, enc_dropouts=(1.0, 1.0), stem_dropout=1.0)
    tr = DPTrainer(cfg, L, **kw)
    dev = {k: torch.from_numpy(v).cuda() for k, v in data.items()}
    for k in range(K + 1):
        values = tr.params.numpy()
        logits, losses = tr.full_forward_backward("t", dev, global_batch=B)
        torch.cuda.synchronize()
        ref = _oracle_loss(cfg, L, values, data)
        errs = (max_rel(logits.cpu().numpy(), ref["logits"]), max_rel(losses.cpu().numpy(), ref["losses"]))
        print("step %d: loss %.6f, logits %.2e, losses %.2e against fp64" % (k, ref["loss"], errs[0], errs[1]))
        assert max(errs) < 1e-4, (k, errs)
        if k < K:
            tr.apply()
    still = [n for n, v in values.items() if n.endswith("bias") and v.size > 1 and not np.max(np.abs(v)) > 1e-3]
    assert not still, still             # every bias vector has moved off TF's zero initialisation
    check_bucket_against_fp64(cfg, L, values, data, tr, "step %d" % K)
    g32, l32 = tr.bucket.double(), float(losses.double().mean())
    tw = DPTrainer(cfg, L, prec="tc32", bwd_tc=True, stem_prec="bf16x3", **kw)
    tw.params.flat.copy_(tr.params.flat)
    tw.step_id = tr.step_id
    tw.params.touch()
    _, losses_t = tw.full_forward_backward("t", dev, global_batch=B)
    torch.cuda.synchronize()
    gt, lt = tw.bucket.double(), float(losses_t.double().mean())
    gmax = float(g32.abs().max())
    worst, null = {}, {}
    for name, (shape, _) in tr.params.specs.items():
        o, n = tr.params.offsets[name], int(np.prod(shape)) if shape else 1
        ref, got = g32[o:o + n], gt[o:o + n]
        if name.endswith(NULL_GRADIENTS):
            null[name] = max(float(ref.abs().max()), float(got.abs().max())) / gmax
            continue
        scale = float(ref.abs().max())
        if scale < 1e-12:
            continue
        worst[name] = float((got - ref).abs().max()) / scale
    print("tc32 twin at step %d: loss %.6f vs %.6f; worst gradients %s; null %s" % (
        K, lt, l32, {k: "%.2e" % v for k, v in sorted(worst.items(), key=lambda kv: -kv[1])[:4]},
        {k: "%.1e" % v for k, v in null.items()}))
    assert abs(lt - l32) <= 2e-4 * abs(l32), (lt, l32)
    bad = {k: v for k, v in worst.items() if v > 2e-4}
    assert not bad, bad
    assert null and all(v < 1e-3 for v in null.values()), null


# ================================================================================================ (c) resume
@pytest.mark.parametrize("case", ["fp32_scheduled", "all_tc"])
def test_resume_from_a_saved_training_state_equals_the_uninterrupted_run(case, tmp_path):
    from mac_network_b200.checkpoint import load_training_state, save_training_state
    path = str(tmp_path / "state")
    tr = _trainer(case)
    run = []
    for i in range(len(KEYS)):
        run.append(_step(tr, i, _data(case, i)))
        if i == 1:
            save_training_state(path, tr)
    fresh = _trainer(case)
    assert load_training_state(path, fresh) == 2
    for i in range(2, len(KEYS)):
        got = _step(fresh, i, _data(case, i))
        bad = _differ(got, run[i])
        assert not bad, (case, "step %d" % (i + 1), bad)


# ================================================================================================ (d) evaluation between steps
EVAL = {"fp32": dict(prec="fp32"), "bf16": dict(prec="bf16"),
        "fp8": dict(prec="fp8", eval_stem_prec="fp8", eval_enc_prec="bf16"),
        "bf16x3": dict(prec="fp32", eval_stem_prec="bf16x3")}


def _eval_net(model):
    """test_gpu_model_pipeline.py's model dimensions (d = 512: the e4m3 read step's width), trained in fp32."""
    from mac_network_b200.model import MACnet
    from tests.test_gpu_model_pipeline import A as A_, C as C_, E as E_, V as V_
    cfg = MACConfig.args("args", netLength=L)
    return MACnet(cfg, L, V_, A_, wrd_emb_dim=E_, image_in_dim=C_, classifier_dims=(512,), seed=3, **EVAL[model])


@pytest.mark.parametrize("model", list(EVAL))
def test_evaluation_between_training_steps_equals_a_fresh_model(model):
    """runBatch(train=True) with runBatch(train=False, getAtt=True) on the live weights and on the EMA shadows after every
    step: each evaluation equals a fresh model's loaded with those weights, and the training run equals one that never
    evaluates."""
    from tests.test_gpu_model_pipeline import _batches, _reference
    B, S, Hh = 8, 10, 7
    net, plain = _eval_net(model), _eval_net(model)
    train = _batches(3, B, S, Hh, Hh, seed=51, longest=S)
    ev = _batches(1, B, S, Hh, Hh, seed=52, longest=S - 3)[0]
    rng = np.random.RandomState(53)

    def same_state(i):
        for k in STATE:
            a, b2 = (net.trainer.params.flat, plain.trainer.params.flat) if k == "flat" else \
                (getattr(net.trainer, k), getattr(plain.trainer, k))
            assert same_bits(a, b2), (i, k)

    for i, b in enumerate(train):
        data = {"questions": b["questions"], "questionLengths": b["questionLengths"],
                "answers": rng.randint(0, 28, size=(B,)).astype(np.int32)}
        r1 = net.runBatch(None, data, {"images": b["images"]}, train=True)
        r2 = plain.runBatch(None, data, {"images": b["images"]}, train=True)
        assert (r1["loss"], r1["gradNorm"]) == (r2["loss"], r2["gradNorm"]), (i, r1["loss"], r2["loss"])
        assert [p["prediction"] for p in r1["preds"]] == [p["prediction"] for p in r2["preds"]]
        same_state(i)
        for use_ema in (False, True):
            net.use_ema = use_ema
            got = _reference(net, ev)
            net.use_ema = False
            fresh = _eval_net(model)
            fresh.trainer.params.flat.copy_(net.trainer.ema if use_ema else net.trainer.params.flat)
            fresh.trainer.params.touch()
            want = _reference(fresh, ev)
            del fresh
            assert set(got) == set(want)
            for k in want:
                if k == "self":
                    assert all(np.array_equal(x, y) for x, y in zip(got[k], want[k])), (i, use_ema, k)
                else:
                    assert np.array_equal(got[k], want[k]), (model, "step %d" % (i + 1), "ema" if use_ema else "live", k)
    same_state("after the last evaluation")         # the EMA swap put the live weights and the shadows back


# ================================================================================================ (e) HostPipeline
@pytest.mark.parametrize("prec,d", [("fp32", 128), ("bf16", 128), ("fp8", 512)])
def test_host_pipeline_follows_a_weight_update(prec, d):
    """A graph pipeline serves a batch, the weights move (`flat.mul_(1.03)`, `touch()`), and the next submits return bit
    for bit what a direct cell (the same small_tc form) computes on the new weights."""
    from mac_network_b200.mac_cell import MACParams
    from mac_network_b200.params import init_params, perturb_biases
    from mac_network_b200.serving import HostPipeline
    from mac_network_b200.synthetic import make_inputs
    from tests.test_gpu_parity import run_gpu
    B, S, N = 8, 6, 49
    cfg = MACConfig.args("args", netLength=L, memDim=d, ctrlDim=d, attDim=d)
    params = MACParams(cfg, L, values=perturb_biases(init_params(cfg, L, seed=82), seed=83))
    pipe = HostPipeline(cfg, params, (B, S, N, d, L), prec=prec, slots=2, use_graph=True, cast_threads=3)
    assert all(s.graph is not None for s in pipe.slots)
    batch = make_inputs(B, S, N, d, seed=95)
    host = {k: torch.from_numpy(v).pin_memory() for k, v in batch.items() if k != "questionWords"}
    before = {k: v.clone() for k, v in pipe.result(pipe.submit(host)).items()}
    params.flat.mul_(1.03)
    params.touch()
    after = [{k: v.clone() for k, v in pipe.result(pipe.submit(host)).items()} for _ in range(2)]   # both slots
    moved = {k: v.reshape(params.specs[k][0]) for k, v in params.numpy().items()}     # 0-d biases: (1,) views -> ()
    ref, _ = run_gpu(cfg, moved, batch, L, prec=prec, small_tc=True)
    for got in after:
        assert np.array_equal(got["memory"].numpy(), ref["memory"][-1]), prec
        assert np.array_equal(got["control"].numpy(), ref["control"][-1]), prec
        assert np.array_equal(got["att_kb"].numpy(), ref["att_kb"]), prec
    assert not np.array_equal(after[0]["memory"].numpy(), before["memory"].numpy())
