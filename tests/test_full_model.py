"""The reference's whole training graph (`MACnet.build`, model.py:774-821) on the GPU: question input unit -> image stem ->
netLength MAC steps -> output unit -> classifier -> mean softmax-CE, and its hand-written backward.

Forward: against the chain of fp64 numpy oracles (each pinned to the reference's own code on the TF1 shim).
Backward: the flat gradient bucket element by element against torch.autograd on the fp64 graph of the same loss
(oracle/model_torch_autograd.py, pinned to that oracle chain and to central differences in
tests/test_model_autograd_oracle.py)."""
import numpy as np
import pytest

from tests._util import max_rel


def _oracle_loss(cfg, L, values, data, keeps=None, uniforms=None):
    """The chain of numpy oracles on `data` (NHWC "images", optionally "imageIndex").  `keeps` and `uniforms` as
    `oracle.model_torch_autograd.run` takes them: every dropout with its uniforms, the cell in training mode; by default
    every dropout off."""
    from oracle.encoder_oracle import encoder_forward
    from oracle.stem_oracle import stem_forward
    from oracle.output_oracle import output_forward
    from oracle.mac_oracle import MACOracle
    keeps = keeps or {"encoder": (1.0, 1.0), "stem": 1.0, "cell": (1.0, 1.0, 1.0), "output": 1.0}
    us = uniforms or {}
    v = {k: np.asarray(a, np.float64) for k, a in values.items()}
    eo = encoder_forward(v, data["questions"], data["questionLengths"], keeps["encoder"][0], keeps["encoder"][1],
                         us.get("encoder"))
    kb = stem_forward(cfg.relu, {k: a for k, a in v.items() if k.startswith("stem/")}, data["images"].astype(np.float64),
                      keeps["stem"], us.get("stem"))
    if data.get("imageIndex") is not None:
        kb = kb[np.asarray(data["imageIndex"])]
    cell = MACOracle(cfg, v, dtype=np.float64)
    cell.train = uniforms is not None
    dm, dr, dw = keeps["cell"]
    ref = cell.run(L, eo["vecQuestions"], eo["questionWords"], eo["questionCntxWords"], data["questionLengths"], kb,
                   memoryDropout=dm, readDropout=dr, writeDropout=dw, uniforms=us.get("cell"))
    out = output_forward(cfg.relu, {k: a for k, a in v.items() if k.startswith(("outputUnit/", "classifier/"))},
                         ref.memory, eo["vecQuestions"], data["answers"], keep=keeps["output"], uniforms=us.get("output"))
    return out


def _make(B, S, V, E, d, H, W, C, A, L, seed):
    from mac_network_b200.config import MACConfig
    rng = np.random.RandomState(seed)
    lengths = rng.randint(max(1, S // 2), S + 1, size=(B,)).astype(np.int32)
    lengths[0] = S
    q = rng.randint(1, V + 1, size=(B, S)).astype(np.int32)
    q[np.arange(S)[None, :] >= lengths[:, None]] = 0
    data = {"questions": q, "questionLengths": lengths,
            "images": np.maximum(rng.standard_normal((B, H, W, C)), 0).astype(np.float32),
            "answers": rng.randint(0, A, size=(B,)).astype(np.int32)}
    cfg = MACConfig.args("args", netLength=L, memDim=d, ctrlDim=d, attDim=d)
    return cfg, data


@pytest.mark.gpu
@pytest.mark.parametrize("flags", ["args", "gqa"])
def test_full_model_forward_and_gradient(flags):
    import torch
    from mac_network_b200.config import MACConfig
    from mac_network_b200.dp import DPTrainer
    B, S, V, E, d, H, W, C, A, L = 6, 7, 13, 12, 64, 4, 3, 16, 12, 3      # A % 4 == 0 (mac_linear_fwd: n_out % 4)
    _, data = _make(B, S, V, E, d, H, W, C, A, L, seed=11)
    cfg = MACConfig.args(flags, netLength=L, memDim=d, ctrlDim=d, attDim=d)
    tr = DPTrainer(cfg, L, seed=5, dropouts=(1.0, 1.0, 1.0), classifier=(A, [32]), output_dropout=1.0, encoder=(V, E),
                   stem=(C, 2), enc_dropouts=(1.0, 1.0), stem_dropout=1.0)
    # TF initialises every bias to zero; perturb them so that the bias gradients are exercised
    rng = np.random.RandomState(12)
    with torch.no_grad():
        for name, t in tr.params.t.items():
            if name.endswith(("bias", "biases/bias")) and t.numel() > 1:
                t.copy_(torch.from_numpy((0.1 * rng.standard_normal(tuple(t.shape))).astype(np.float32)))
    tr.params.touch()
    values = tr.params.numpy()
    dev = {k: torch.from_numpy(v).cuda() for k, v in data.items()}
    logits, losses = tr.full_forward_backward("t", dev, global_batch=B)
    torch.cuda.synchronize()
    ref = _oracle_loss(cfg, L, values, data)
    assert max_rel(logits.cpu().numpy(), ref["logits"]) < 1e-4
    assert max_rel(losses.cpu().numpy(), ref["losses"]) < 1e-4
    check_bucket_against_fp64(cfg, L, values, data, tr, flags)


# fp32 trainer against the fp64 graph, every dropout off (H100 80GB HBM3, 700 W power limit):           measured worst
BAR_GRAD = 1e-5             # at the initial weights with perturbed biases, and at weights moved by four steps   2.8e-6
BAR_NULL = 1e-7             # a softmax logit bias, of the model's largest gradient                               2.5e-8


def check_bucket_against_fp64(cfg, L, values, data, tr, tag, bar=BAR_GRAD, null_bar=BAR_NULL):
    """The trainer's gradient bucket of the loss at `values` on `data` (every dropout off) against torch.autograd on the
    fp64 graph (oracle/model_torch_autograd.py), element by element: max |got - ref| / max |ref| of each tensor; a softmax
    logit bias (true gradient 0) against the model's largest gradient.  Returns the worst errors."""
    import torch
    from oracle import model_torch_autograd as MA
    from tests.test_gpu_tc32_training import NULL_GRADIENTS
    keeps = {"encoder": (1.0, 1.0), "stem": 1.0, "cell": (1.0, 1.0, 1.0), "output": 1.0}
    ref = MA.run(cfg, L, values, data, keeps, device="cuda")["grads"]
    p = tr.params
    gmax = max(float(g.abs().max()) for g in ref.values())
    errs, null = {}, {}
    for n, g in ref.items():
        got = tr.bucket[p.offsets[n]:p.offsets[n] + g.numel()].double()
        if n.endswith(NULL_GRADIENTS):
            null[n] = float(got.abs().max()) / gmax
        elif "/BatchNorm/moving_" not in n:
            errs[n] = float((got - g.reshape(-1)).abs().max()) / float(g.abs().max())
    top = sorted(errs.items(), key=lambda kv: -kv[1])[:3]
    print("%s gradients against fp64: worst %s; null %.1e" % (tag, ["%s %.2e" % kv for kv in top], max(null.values())))
    bad = {n: e for n, e in errs.items() if not e < bar}
    bad.update({n: e for n, e in null.items() if not e < null_bar})
    assert not bad, (tag, bad)
    return errs


@pytest.mark.gpu
def test_full_model_train_steps_reduce_loss():
    """A few DP steps (world 1) of the whole model with the reference's training dropouts: the loss on the batch goes down
    and every sub-model's variables move."""
    import torch
    from mac_network_b200.dp import DPTrainer
    B, S, V, E, d, H, W, C, A, L = 16, 9, 20, 20, 64, 5, 5, 32, 8, 3
    cfg, data = _make(B, S, V, E, d, H, W, C, A, L, seed=21)
    tr = DPTrainer(cfg, L, seed=6, lr=3e-3, classifier=(A, [32]), encoder=(V, E), stem=(C, 2))
    dev = {k: torch.from_numpy(v).cuda() for k, v in data.items()}
    before = {k: v.clone() for k, v in tr.params.t.items()}
    hist = []
    for it in range(12):
        _, losses = tr.train_step_full("t", dev, global_batch=B)
        hist.append(float(losses.mean().item()))
    assert np.all(np.isfinite(hist)) and min(hist[-3:]) < hist[0], hist
    for prefix in ("encoder/", "qEmbeddings/", "stem/", "MACnetwork/", "classifier/"):
        moved = [float((tr.params.t[k] - before[k]).abs().max().item()) for k in before if k.startswith(prefix)]
        assert moved and max(moved) > 0, prefix
