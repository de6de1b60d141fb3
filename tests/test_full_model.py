"""The reference's whole training graph (`MACnet.build`, model.py:774-821) on the GPU: question input unit -> image stem ->
netLength MAC steps -> output unit -> classifier -> mean softmax-CE, and its hand-written backward.

Forward: against the chain of fp64 numpy oracles (each pinned to the reference's own code on the TF1 shim).
Backward: the flat gradient bucket against central differences of that fp64 oracle chain along random directions
restricted to each sub-model's variables (a check that needs no autograd restatement of the chained model)."""
import numpy as np
import pytest

from tests._util import max_rel


def _oracle_loss(cfg, L, values, data):
    from oracle.encoder_oracle import encoder_forward
    from oracle.stem_oracle import stem_forward
    from oracle.output_oracle import output_forward
    from oracle.mac_oracle import MACOracle
    v = {k: np.asarray(a, np.float64) for k, a in values.items()}
    eo = encoder_forward(v, data["questions"], data["questionLengths"])
    kb = stem_forward(cfg.relu, {k: a for k, a in v.items() if k.startswith("stem/")}, data["images"].astype(np.float64))
    ref = MACOracle(cfg, v, dtype=np.float64).run(L, eo["vecQuestions"], eo["questionWords"], eo["questionCntxWords"],
                                                  data["questionLengths"], kb)
    out = output_forward(cfg.relu, {k: a for k, a in v.items() if k.startswith(("outputUnit/", "classifier/"))},
                         ref.memory, eo["vecQuestions"], data["answers"])
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
    check_directional_derivatives(cfg, L, values, data, tr, flags)


def check_directional_derivatives(cfg, L, values, data, tr, tag):
    """The trainer's gradient bucket (of the loss at `values` on `data`) along one random direction per sub-model's
    variables against central differences of the fp64 oracle chain."""
    bucket = tr.bucket.cpu().numpy().astype(np.float64)
    offs, specs = tr.params.offsets, tr.params.specs
    groups = {"encoder": ("encoder/", "qEmbeddings/"), "stem": ("stem/",), "cell": ("MACnetwork/",),
              "output": ("outputUnit/", "classifier/")}
    for gname, prefixes in groups.items():
        names = [n for n in specs if n.startswith(prefixes)]
        assert names, gname
        drng = np.random.RandomState(100 + sorted(groups).index(gname))
        direction = {n: drng.standard_normal(values[n].shape) for n in names}
        analytic = 0.0
        for n in names:
            k = max(1, int(np.prod(specs[n][0])) if specs[n][0] else 1)
            analytic += float(np.dot(bucket[offs[n]:offs[n] + k], direction[n].reshape(-1)))
        eps = 1e-5
        lo = dict(values)
        hi = dict(values)
        for n in names:
            hi[n] = values[n].astype(np.float64) + eps * direction[n]
            lo[n] = values[n].astype(np.float64) - eps * direction[n]
        numeric = (_oracle_loss(cfg, L, hi, data)["loss"] - _oracle_loss(cfg, L, lo, data)["loss"]) / (2 * eps)
        print("%s %-8s directional derivative: analytic %.6e numeric %.6e" % (tag, gname, analytic, numeric))
        assert abs(analytic - numeric) <= 2e-3 * max(abs(numeric), 1e-3), (gname, analytic, numeric)


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
