"""The fp64 graph of the whole training loss (`oracle/model_torch_autograd.py`), pinned on the CPU before
tests/test_gpu_model_gradients.py trusts it to check the trainer's gradients element by element:

- its forward against the chain of numpy oracles (each pinned to the reference's own code on the TF1 shim), with every
  dropout at the reference's training rate, at 1e-12;
- a forward over k < B images with `imageIndex` against the forward fed the duplicated images with the per-image masks
  gathered the same way, and its image gradient against the duplicated images' gradient summed per image;
- every parameter gradient and the image gradient against central differences of the graph itself, element by element:
  every entry of the small tensors and a sample of every other tensor.

`dropout_plan` restates the order, Philox sites, steps and shapes of the trainer's dropout draws; the GPU test fills it
from `oracle/philox.py`, these tests from a plain generator."""
import numpy as np
import pytest
import torch

from oracle import model_torch_autograd as MA
from tests._util import load_golden, max_rel

# the reference's training dropouts outside the cell (config.py:202-206): encoder input / question, stem, output unit
ENC_KEEP, STEM_KEEP, OUT_KEEP = (0.85, 0.92), 0.82, 0.85


def model_config(flags, d, L):
    """A shipped flag file, or a golden fixture's cell flags and dropouts (`p2_*`); returns (cfg, cell dropouts)."""
    from mac_network_b200.config import MACConfig
    if flags.startswith("p2_"):
        meta, _ = load_golden(flags)
        cfg = MACConfig(**dict(meta["cell_flags"], memDim=d, ctrlDim=d, attDim=d, netLength=L)).validate()
        dm = meta["dropouts"]
        return cfg, (dm["memory"], dm["read"], dm["write"])
    cfg = MACConfig.args(flags, netLength=L, memDim=d, ctrlDim=d, attDim=d)
    return cfg, (cfg.memoryDropout, cfg.readDropout, cfg.writeDropout)


def training_keeps(cell_dropouts):
    return {"encoder": ENC_KEEP, "stem": STEM_KEEP, "cell": tuple(cell_dropouts), "output": OUT_KEEP}


def dropout_plan(cfg, L, values, keeps, B, S, k, H, W, step):
    """{unit: [(Philox site, step, shape)]} of the trainer's dropout draws, in the reference's call order: the encoder's
    input sequence and question vector, the stem's input of each layer over the k images, the cell's (the step index is
    the MAC iteration), the output unit's input of each classifier layer.  A keep of 1 draws nothing."""
    from mac_network_b200 import _lib
    from mac_network_b200.encoder import SITE_ENC_INPUT, SITE_ENC_QUESTION
    from mac_network_b200.output_unit import SITE_OUTPUT
    from mac_network_b200.stem import SITE_STEM
    plan = {u: [] for u in MA.UNITS}
    E = values["qEmbeddings/emb"].shape[1]
    hq = 2 * (values["encoder/birnnLayer/bidirectional_rnn/fw/basic_lstm_cell/kernel"].shape[1] // 4)
    for keep, site, shape in ((keeps["encoder"][0], SITE_ENC_INPUT, (B, S, E)),
                              (keeps["encoder"][1], SITE_ENC_QUESTION, (B, hq))):
        if keep < 1.0:
            plan["encoder"].append((site, step, shape))
    i = 0
    while "stem/cnnLayercnn_%d/kernels/kernel" % i in values:
        if keeps["stem"] < 1.0:
            plan["stem"].append((SITE_STEM + i, step, (k, H, W, values["stem/cnnLayercnn_%d/kernels/kernel" % i].shape[2])))
        i += 1
    i = 0
    while "classifier/linearLayerfc_%d/weights/weight" % i in values:
        if keeps["output"] < 1.0:
            plan["output"].append((SITE_OUTPUT + i, step, (B, values["classifier/linearLayerfc_%d/weights/weight" % i].shape[0])))
        i += 1
    # the cell (mac_cell.py:420-480, ops.py:1054-1067): the variational memory mask once per forward, then per step the
    # plain memory dropout, the read unit's projection inputs (knowledge base, memory) and attention interactions, and the
    # write unit's info
    c, d, N = cfg, cfg.memDim, H * W
    km, kr, kw = keeps["cell"]
    if c.memoryVariationalDropout and km < 1.0:
        plan["cell"].append((_lib.SITE_MEM_VAR, 0, (B, d)))
    if c.is_fast_path:
        inter = d
    else:
        dim = c.attDim if c.readProjInputs else c.memDim
        inter = dim if c.readMemProj else dim + ((c.attDim if c.readMemConcatProj else c.memDim) if c.readMemConcatKB else 0)
        if c.readCtrl and c.readCtrlConcatKB:
            inter += c.attDim if c.readCtrlConcatProj else c.memDim
    for it in range(L):
        if not c.memoryVariationalDropout and km < 1.0:
            plan["cell"].append((_lib.SITE_MEM_PLAIN, it, (B, d)))
        if kr < 1.0:
            if c.readProjInputs:
                plan["cell"].append((_lib.SITE_READ_KB, it, (B, N, d)))
                plan["cell"].append((_lib.SITE_READ_MEM, it, (B, d)))
            plan["cell"].append((_lib.SITE_READ_INTER, it, (B, N, inter)))
        if c.writeDropout < 1.0 and kw < 1.0:
            plan["cell"].append((_lib.SITE_WRITE_INFO, it, (B, d)))
    return plan


def random_uniforms(plan, seed):
    rng = np.random.RandomState(seed)
    return {u: [rng.uniform(size=shape) for _, _, shape in draws] for u, draws in plan.items()}


def model_values(cfg, L, V, E, C, A, hidden, seed):
    """Every variable of the whole model (DPTrainer's initialisation) with every bias moved off TF's zero."""
    from mac_network_b200.dp import model_parameters
    cell, _, extra, _, _ = model_parameters(cfg, L, seed, (A, list(hidden)), (V, E), (C, 2))
    rng = np.random.RandomState(seed + 1)
    out = {}
    for k, v in list(cell.items()) + list(extra.items()):
        v = np.asarray(v, np.float64)
        out[k] = v + 0.1 * rng.standard_normal(v.shape) if k.endswith("bias") else v
    return out


def make_data(B, S, V, k, H, W, C, A, seed, index=None):
    """Questions with lengths 1 and S and padded positions, k NHWC images, answers; `index` adds imageIndex."""
    rng = np.random.RandomState(seed)
    lengths = rng.randint(1, S + 1, size=(B,)).astype(np.int32)
    lengths[0], lengths[-1] = S, 1
    q = rng.randint(1, V + 1, size=(B, S)).astype(np.int32)
    q[np.arange(S)[None, :] >= lengths[:, None]] = 0
    data = {"questions": q, "questionLengths": lengths, "answers": rng.randint(0, A, size=(B,)).astype(np.int32),
            "images": np.maximum(rng.standard_normal((k, H, W, C)), 0).astype(np.float32)}
    if index is not None:
        data["imageIndex"] = np.asarray(index, np.int32)
    return data


def numpy_chain(cfg, L, values, data, keeps, uniforms):
    """The chain of numpy oracles (tests/test_full_model.py::_oracle_loss) with each unit's uniforms."""
    from tests.test_full_model import _oracle_loss
    return _oracle_loss(cfg, L, values, data, keeps=keeps, uniforms=uniforms)


# small model: B questions of up to S words, k images of H x W x C, d wide, L steps
B, S, V, E, H, W, C, A, HIDDEN, L = 5, 6, 11, 8, 3, 2, 6, 7, [9], 2


@pytest.mark.parametrize("flags", ["args", "gqa", "args1", "p2_memory_bn_train"])
def test_forward_equals_the_numpy_chain_with_training_dropouts(flags):
    d = 16
    cfg, cell_dp = model_config(flags, d, L)
    values = model_values(cfg, L, V, E, C, A, HIDDEN, seed=3)
    keeps = training_keeps(cell_dp)
    data = make_data(B, S, V, B, H, W, C, A, seed=4)
    plan = dropout_plan(cfg, L, values, keeps, B, S, B, H, W, step=0)
    assert all(plan[u] for u in MA.UNITS), {u: len(v) for u, v in plan.items()}
    us = random_uniforms(plan, seed=5)
    ref = numpy_chain(cfg, L, values, data, keeps, us)
    got = MA.run(cfg, L, values, data, keeps, us, grad=False)
    errs = {k: max_rel(got[k].numpy(), ref[k]) for k in ("logits", "losses")}
    print(flags, errs)
    assert max(errs.values()) < 1e-12, errs
    # a uniform too many is refused
    with pytest.raises(AssertionError, match="left over"):
        MA.run(cfg, L, values, data, keeps, dict(us, output=us["output"] + [us["output"][-1]]), grad=False)


def test_output_graph_matches_the_reference_fixture():
    from mac_network_b200.output_unit import init_output_params, output_specs
    from tests.test_output_unit import _load
    meta, g = _load("output_train")
    params = init_output_params(output_specs(meta["d"], meta["d"], meta["hidden"], meta["A"]), seed=meta["param_seed"],
                                dtype=np.float64)
    us = [g["uniform_%03d" % i] for i in range(meta["n_uniform"])]
    t = lambda a: torch.as_tensor(a, dtype=torch.float64)
    logits, losses = MA.output_graph(meta["relu"], {k: t(v) for k, v in params.items()}, t(g["memory"]),
                                     t(g["vecQuestions"]), torch.as_tensor(g["answers"]).long(), meta["keep"], us)
    assert np.max(np.abs(logits.numpy() - g["logits"])) < 1e-12
    assert np.max(np.abs(losses.numpy() - g["losses"])) < 1e-12


def test_indexed_images_equal_the_duplicated_images_with_gathered_masks():
    """k = 3 images for 6 questions, image 1 unused: the forward equals the one over images[index] with each stem mask
    gathered by the index, the parameter gradients agree, and each image's gradient is the sum of its questions'."""
    cfg, cell_dp = model_config("gqa", 16, L)
    values = model_values(cfg, L, V, E, C, A, HIDDEN, seed=6)
    keeps = training_keeps(cell_dp)
    Bq, k, index = 6, 3, np.array([2, 0, 2, 2, 0, 0])
    data = make_data(Bq, S, V, k, H, W, C, A, seed=7, index=index)
    us = random_uniforms(dropout_plan(cfg, L, values, keeps, Bq, S, k, H, W, step=0), seed=8)
    got = MA.run(cfg, L, values, data, keeps, us, global_batch=2 * Bq)
    dup = {kk: v for kk, v in data.items() if kk != "imageIndex"}
    dup["images"] = data["images"][index]
    dup_us = dict(us, stem=[u[index] for u in us["stem"]])
    want = MA.run(cfg, L, values, dup, keeps, dup_us, global_batch=2 * Bq)
    for kk in ("logits", "losses"):
        assert max_rel(got[kk].numpy(), want[kk].numpy()) < 1e-12, kk
    bad = {n: max_rel(got["grads"][n].numpy(), want["grads"][n].numpy()) for n in values
           if float(want["grads"][n].abs().max()) > 0}
    assert bad and max(bad.values()) < 1e-10, sorted(bad.items(), key=lambda kv: -kv[1])[:3]
    summed = torch.zeros_like(got["d_images"]).index_add_(0, torch.as_tensor(index), want["d_images"])
    assert max_rel(got["d_images"].numpy(), summed.numpy()) < 1e-12
    assert float(got["d_images"][1].abs().max()) == 0.0 and float(got["d_images"][[0, 2]].abs().min(0)[0].max()) > 0


def _entries(n, rng, full=24, sample=10):
    return np.arange(n) if n <= full else np.sort(rng.choice(n, sample, replace=False))


@pytest.mark.parametrize("flags,nchw,indexed", [("gqa", True, True), ("p2_memory_bn_train", False, False)])
def test_gradient_against_central_differences(flags, nchw, indexed):
    """Every parameter's and the images' gradient of sum(losses) / global_batch against central differences of the graph
    (step 1e-5 on every entry of a tensor of <= 24 entries, on 10 sampled entries of the others), with the training
    dropouts, global_batch = 2B, and for `indexed` k = 3 images for B = 4 questions with one image unused."""
    cfg, cell_dp = model_config(flags, 8, L)
    values = model_values(cfg, L, 7, 4, 3, 5, [6], seed=9)
    keeps = training_keeps(cell_dp)
    Bq, Sq, Hq, Wq, Cq = 4, 3, 2, 2, 3
    index = np.array([2, 0, 0, 2]) if indexed else None
    k = 3 if indexed else Bq
    data = make_data(Bq, Sq, 7, k, Hq, Wq, Cq, 5, seed=10, index=index)
    if nchw:
        data["images_nchw"] = np.ascontiguousarray(data.pop("images").transpose(0, 3, 1, 2))
    us = random_uniforms(dropout_plan(cfg, L, values, keeps, Bq, Sq, k, Hq, Wq, step=0), seed=11)
    gb = 2 * Bq
    ref = MA.run(cfg, L, values, data, keeps, us, global_batch=gb)
    img_key = "images_nchw" if nchw else "images"
    loss = lambda vals, dat: float(MA.run(cfg, L, vals, dat, keeps, us, global_batch=gb, grad=False)["loss"])
    rng = np.random.RandomState(12)
    eps = 1e-5
    errs_of, gmax = {}, 0.0
    tensors = [(n, v, ref["grads"][n].numpy()) for n, v in values.items() if "/BatchNorm/moving_" not in n]
    tensors.append((img_key, data[img_key].astype(np.float64), ref["d_images"].numpy()))
    for name, v, g in tensors:
        v = np.asarray(v, np.float64)
        errs = []
        for e in _entries(v.size, rng):
            vals, dat = dict(values), dict(data)
            fd = []
            for s in (eps, -eps):
                w = v.copy().reshape(-1)
                w[e] += s
                w = w.reshape(v.shape)
                if name == img_key:
                    dat[img_key] = w
                else:
                    vals[name] = w
                fd.append(loss(vals, dat))
            errs.append(abs((fd[0] - fd[1]) / (2 * eps) - g.reshape(-1)[e]))
        errs_of[name] = (max(errs), float(np.abs(g).max()))
        gmax = max(gmax, errs_of[name][1])
    # of each tensor's largest gradient, floored at 1 % of the model's: a softmax logit bias has a true gradient of 0
    worst = {n: e / max(m, 1e-2 * gmax) for n, (e, m) in errs_of.items()}
    if indexed:
        assert float(np.abs(ref["d_images"].numpy()[1]).max()) == 0.0            # image 1 has no question
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:4]
    print("%s: %d tensors, worst %s" % (flags, len(worst), ["%s %.1e" % kv for kv in top]))
    bad = {n: e for n, e in worst.items() if not e < 1e-6}
    assert not bad, bad


@pytest.mark.parametrize("flags", ["gqa", "p2_memory_bn_train"])
def test_trace_changes_neither_the_forward_nor_the_gradients(flags):
    """`trace=` records each step's state and attention maps and returns the tensors the cell reads, and nothing it
    computes moves: the logits, losses, every gradient and the image gradient equal the untraced run's bit for bit, with
    the training dropouts and k < B images.  The traced attention maps are distributions, exactly 0 beyond each length."""
    cfg, cell_dp = model_config(flags, 8, L)
    values = model_values(cfg, L, V, E, C, A, HIDDEN, seed=13)
    keeps = training_keeps(cell_dp)
    index = np.array([1, 0, 2, 1, 1])
    data = make_data(B, S, V, 3, H, W, C, A, seed=14, index=index)
    us = random_uniforms(dropout_plan(cfg, L, values, keeps, B, S, 3, H, W, step=0), seed=15)
    want = MA.run(cfg, L, values, data, keeps, us)
    trace = []
    got = MA.run(cfg, L, values, data, keeps, us, trace=trace)
    for k in ("logits", "losses", "loss", "d_images"):
        assert torch.equal(got[k], want[k]), k
    assert set(got["grads"]) == set(want["grads"])
    for n, g in want["grads"].items():
        assert torch.equal(got["grads"][n], g), n
    assert set(want) == {"logits", "losses", "loss", "grads", "d_images"}
    assert tuple(got["knowledgeBase"].shape) == (3, H * W, 8) and tuple(got["vecQuestions"].shape) == (B, 8)
    assert tuple(got["questionWords"].shape) == tuple(got["questionCntxWords"].shape) == (B, S, 8)
    assert len(trace) == L
    for step in trace:
        assert set(step) == {"control", "memory", "info", "att_question", "att_kb"}
        assert step["att_question"].shape == (B, S) and step["att_kb"].shape == (B, H * W)
        assert np.abs(step["att_question"].sum(1) - 1).max() < 1e-12 and np.abs(step["att_kb"].sum(1) - 1).max() < 1e-12
        assert not step["att_question"][np.arange(S)[None, :] >= data["questionLengths"][:, None]].any()
