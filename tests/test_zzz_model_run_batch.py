"""`model.MACnet.runBatch` (the reference's per-batch call, model.py:732-760) on the GPU.  A composition of classes that each
have their own hardware-validated parity tests (encoder, stem, cell, output unit, trainer)."""
import numpy as np
import pytest

from tests._util import max_rel
from tests.test_full_model import _oracle_loss

pytestmark = pytest.mark.gpu


def _batch(B, S, V, C, H, W, A, seed):
    rng = np.random.RandomState(seed)
    lengths = rng.randint(2, S - 1, size=(B,)).astype(np.int32)            # the longest question is shorter than S
    q = rng.randint(1, V + 1, size=(B, S)).astype(np.int32)
    q[np.arange(S)[None, :] >= lengths[:, None]] = 0
    data = {"questions": q, "questionLengths": lengths, "answers": rng.randint(0, A, size=(B,)).astype(np.int32)}
    images = {"images": np.maximum(rng.standard_normal((B, C, H, W)), 0).astype(np.float32)}
    return data, images


def test_run_batch_eval_matches_oracle_chain_and_training_learns():
    from mac_network_b200.config import MACConfig
    from mac_network_b200.model import MACnet
    B, S, V, E, d, H, W, C, A, L = 8, 10, 15, 12, 64, 4, 4, 16, 8, 3
    cfg = MACConfig.args("args", netLength=L, memDim=d, ctrlDim=d, attDim=d)
    net = MACnet(cfg, L, V, A, wrd_emb_dim=E, image_in_dim=C, classifier_dims=(32,), prec="fp32", lr=3e-3, seed=4)
    data, images = _batch(B, S, V, C, H, W, A, seed=5)
    res = net.runBatch(None, data, images, train=False, getAtt=True)
    Smax = int(data["questionLengths"].max())
    odata = {"questions": data["questions"][:, :Smax], "questionLengths": data["questionLengths"], "answers": data["answers"],
             "images": np.transpose(images["images"], (0, 2, 3, 1))}
    ref = _oracle_loss(cfg, L, net.trainer.params.numpy(), odata)
    assert abs(res["loss"] - ref["loss"]) < 1e-4 * max(1.0, abs(ref["loss"]))
    assert res["correctNum"] == int((ref["preds"] == data["answers"]).sum())
    att = res["preds"][0]["attentions"]
    assert np.asarray(att["kb"][0]).shape == (H, W) and len(att["question"][0]) == Smax
    assert abs(sum(att["question"][0]) - 1.0) < 1e-5 and abs(np.sum(att["kb"][L - 1]) - 1.0) < 1e-5
    first = net.runBatch(None, data, images, train=True)
    for _ in range(10):
        last = net.runBatch(None, data, images, train=True)
    assert first["gradNorm"] > 0 and np.isfinite(last["loss"]) and last["loss"] < first["loss"]
    # evaluation on the EMA shadows runs and restores the live weights
    before = net.trainer.params.flat.clone()
    net.use_ema = True
    net.runBatch(None, data, images, train=False)
    import torch
    assert torch.equal(before, net.trainer.params.flat)
