"""Training-mode forward of the composed (P2) read unit on the GPU: the product draws its Philox masks, the oracle -- pinned
to the reference's own training run of these flag sets by `tests/golden/p2_read_*_train.npz` -- is fed the same uniforms.
"""
import numpy as np
import pytest

from tests._util import load_golden, rebuild

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", ["p2_read_add_train", "p2_read_plain_train"])
def test_general_path_training_forward_matches_oracle(case):
    from tests.test_gpu_parity import compare, run_gpu, run_oracle
    meta, _ = load_golden(case)
    cfg, inputs, params = rebuild(meta)
    dp = (meta["dropouts"]["memory"], meta["dropouts"]["read"], meta["dropouts"]["write"])
    L = meta["shape"]["L"]
    got, cell = run_gpu(cfg, params, inputs, L, dropouts=dp, train=True, seed=987)
    ref = run_oracle(cfg, params, inputs, L, dropouts=dp, uniforms=cell.dropout_uniforms())
    compare(got, ref, what=case)


def test_memory_batch_norm_training_forward_and_stored_statistics():
    """memoryBN in training (mac_cell.py:369-373): batch statistics normalise, and the stored moving mean / variance move once
    per reasoning step -- against the oracle pinned to the reference's run of this flag set (tests/golden/p2_memory_bn_train)."""
    import torch
    from tests.test_gpu_parity import compare, run_gpu, run_oracle
    meta, gold = load_golden("p2_memory_bn_train")
    cfg, inputs, params = rebuild(meta)
    dp = (meta["dropouts"]["memory"], meta["dropouts"]["read"], meta["dropouts"]["write"])
    L = meta["shape"]["L"]
    got, cell = run_gpu(cfg, params, inputs, L, dropouts=dp, train=True, seed=4321)
    keep = []
    ref = run_oracle(cfg, params, inputs, L, dropouts=dp, uniforms=cell.dropout_uniforms(), train=True, keep=keep)
    compare(got, ref, what="p2_memory_bn_train")
    torch.cuda.synchronize()
    for tail in ("moving_mean", "moving_variance"):
        name = [n for n in keep[0].p if n.endswith("/BatchNorm/" + tail)][0]
        dev = cell.params.t[name].cpu().numpy()
        want = keep[0].p[name]
        assert np.max(np.abs(dev - want)) < 1e-5 * (1 + np.max(np.abs(want))), tail
        assert np.max(np.abs(want - params[name])) > 1e-4, "the statistics must have moved"
