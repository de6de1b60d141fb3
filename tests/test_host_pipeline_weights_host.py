"""CPU side of `serving.HostPipeline` following weight updates: when `params.version` moves (optimizer step, checkpoint
restore) the next `submit` drains the pipeline and gives every slot a new cell, eager pass and capture, so that no graph
replays over the packs of an earlier version or with its scalar biases; a submit without a version change captures
nothing.  Over the dry-run library (tests/_mocklib.py) with the CUDA stream / event / graph objects replaced by counters
(tests/test_model_pipeline_host.py); the numerics are tests/test_gpu_training_steps.py's."""
import numpy as np
import pytest
import torch

from tests import _mocklib
from tests.test_model_pipeline_host import _fake_cuda

B, S, N, L = 4, 5, 9, 2
SCALAR = "MACCell/read/inter2att/inter2logits/linearLayerlogits/biases/bias"     # a bias the read kernels take by value


def _setup(monkeypatch, d):
    """The dry-run library, the counting CUDA objects and CPU parameters of the `args` cell at width d."""
    from mac_network_b200.config import MACConfig
    from mac_network_b200.mac_cell import MACParams
    mock = _mocklib.install(monkeypatch)
    n = _fake_cuda(monkeypatch)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True), raising=False)
    cfg = MACConfig.args("args", netLength=L, memDim=d, ctrlDim=d, attDim=d)
    return mock, n, MACParams(cfg, L, seed=3, device="cpu")


def _pipeline(params, prec, slots, use_graph=True):
    from mac_network_b200.serving import HostPipeline
    d = params.cfg.memDim
    return HostPipeline(params.cfg, params, (B, S, N, d, L), prec=prec, slots=slots, use_graph=use_graph, host_cast=False)


def _batch(d, seed):
    rng = np.random.RandomState(seed)
    f = lambda *shape: torch.from_numpy(rng.standard_normal(shape).astype(np.float32))
    return {"vecQuestions": f(B, d), "questionCntxWords": f(B, S, d),
            "questionLengths": torch.tensor([5, 3, 1, 4], dtype=torch.int32), "knowledgeBase": f(B, N, d)}


@pytest.mark.parametrize("prec,d", [("fp32", 64), ("bf16", 128), ("fp8", 512)])
def test_host_pipeline_captures_again_when_the_weights_move(monkeypatch, prec, d):
    mock, n, params = _setup(monkeypatch, d)
    pipe = _pipeline(params, prec, slots=2)
    assert n.captures == 2 and n.stream_waits == 2      # every slot's stream waited for the caller's before its eager pass
    pipe.submit(_batch(d, 0))
    assert n.captures == 2 and n.replays == 1
    cells = [s.cell for s in pipe.slots]
    outs = [s.outs_host for s in pipe.slots]
    assert params.scalar(SCALAR) == 0.0
    with torch.no_grad():
        params[SCALAR].fill_(0.5)
    params.touch()
    del mock.calls[:]
    syncs = n.event_syncs
    pipe.submit(_batch(d, 1))
    assert n.captures == 4 and n.event_syncs == syncs + 1               # drained the one busy slot, then both captured again
    assert n.stream_waits == 4          # ... each after waiting for the stream the weights were moved on
    assert n.replays == 2               # the batch ran on a new graph
    assert all(s.cell is not c for s, c in zip(pipe.slots, cells))
    assert all(s.outs_host is o for s, o in zip(pipe.slots, outs))        # same shapes: the pinned outputs stay
    assert mock.calls.count("mac_read_invariant") >= 4                     # each slot: an eager and a captured pass
    if prec != "fp32":                  # new packs, built in the eager pass (the batch-sized products of small_tc)
        assert mock.calls.count("mac_pack_weight_bf16_split") >= 1
    if prec == "fp8":
        assert mock.calls.count("mac_pack_weight_fp8") >= 1
    assert params.cache.get(("scalar", SCALAR), lambda: None) == 0.5     # the new captures read the new bias
    del mock.calls[:]
    for i in range(3):
        pipe.submit(_batch(d, 2 + i))
    assert n.captures == 4 and n.replays == 5 and mock.calls == []


def test_host_pipeline_without_graph_builds_new_cells_when_the_weights_move(monkeypatch):
    mock, n, params = _setup(monkeypatch, 64)
    pipe = _pipeline(params, "fp32", slots=1, use_graph=False)
    pipe.submit(_batch(64, 0))
    cell = pipe.slots[0].cell
    params.touch()
    pipe.submit(_batch(64, 1))
    assert n.captures == 0 and n.replays == 0 and pipe.slots[0].cell is not cell
    assert n.stream_waits == 2          # the new cell's eager pass also waited for the caller's stream
    cell = pipe.slots[0].cell
    pipe.submit(_batch(64, 2))
    assert pipe.slots[0].cell is cell
