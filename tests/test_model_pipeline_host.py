"""CPU side of whole-model serving (serving.ModelPipeline, csrc/ingest.cuh, mac_answer_topk): the new entry points'
declarations and their rejections (which return before any CUDA call), numpy restatements of the ingest layout and of the
top-k tie rule against the stem oracle and torch, and the pipeline's host logic -- slot rotation, the staging ring, the
host-cast decision, re-capture when the weights move, refusals -- over the dry-run library (tests/_mocklib.py) with the CUDA
stream / event / graph objects replaced by counters."""
import contextlib
import ctypes

import numpy as np
import pytest
import torch

from mac_network_b200 import _lib as L_
from oracle.stem_oracle import stem_forward
from tests import _mocklib

INVALID, ALIGN, UNSUPPORTED = -1, -2, -3


# ------------------------------------------------------------------------------------------------ the C boundary
def test_new_symbols_are_declared_bound_and_exported():
    from tests.test_abi import _declared
    lib = L_.load()
    for name in ("mac_ingest_nchw", "mac_answer_topk"):
        assert name in _declared() and name in L_.PROTOTYPES and hasattr(lib, name)
    assert lib.mac_b200_abi_version() == 1


def test_entry_points_refuse_before_any_cuda_call():
    lib = L_.load()
    buf = (ctypes.c_float * 4096)()
    p = (ctypes.addressof(buf) + 15) & ~15                  # 16-byte aligned fake "device" pointer, never dereferenced
    ing = lambda x, xb, o, mode, B, C, H, W: lib.mac_ingest_nchw(x, xb, o, mode, B, C, H, W, None)
    assert ing(None, 0, p, 0, 1, 64, 7, 7) == INVALID and ing(p, 0, None, 1, 1, 64, 7, 7) == INVALID
    assert ing(p, 0, p, 0, 0, 64, 7, 7) == INVALID and ing(p, 0, p, 0, 1, 0, 7, 7) == INVALID
    assert ing(p, 0, p, 0, 1, 64, 0, 7) == INVALID and ing(p, 1, p, 1, 1, 64, 7, -2) == INVALID
    assert ing(p + 8, 0, p, 0, 1, 64, 7, 7) == ALIGN and ing(p, 1, p + 2, 1, 1, 64, 7, 7) == ALIGN
    assert ing(p, 0, p, 0, 1, 32, 7, 7) == UNSUPPORTED and ing(p, 0, p, 1, 1, 1000, 14, 14) == UNSUPPORTED
    assert ing(p, 0, p, 2, 1, 64, 7, 7) == UNSUPPORTED and ing(p, 1, p, -1, 1, 64, 7, 7) == UNSUPPORTED
    assert ing(p, 0, p, 0, 1, 64, 21, 21) == UNSUPPORTED     # 441 pixels: one more than fp32 -> NHWC fits in an SM
    assert ing(p, 0, p, 1, 1, 64, 100, 100) == UNSUPPORTED
    # 581 pixels at 400 bytes each fit 227 KB only without the kernel's 128 bytes of static shared memory
    assert ing(p, 0, p, 1, 1, 64, 7, 83) == UNSUPPORTED and ing(p, 1, p, 0, 1, 64, 7, 83) == UNSUPPORTED
    assert ing(p, 1, p, 1, 1, 64, 9, 95) == UNSUPPORTED       # 855 pixels, bf16 -> patches
    topk = lambda z, B, A, k, i, pr: lib.mac_answer_topk(z, B, A, k, i, pr, None)
    assert topk(None, 2, 8, 1, p, p) == INVALID and topk(p, 2, 8, 1, None, p) == INVALID and topk(p, 2, 8, 1, p, None) == INVALID
    assert topk(p, 0, 8, 1, p, p) == INVALID and topk(p, 2, 0, 1, p, p) == INVALID
    assert topk(p, 2, 8, 0, p, p) == INVALID and topk(p, 2, 28, 9, p, p) == INVALID and topk(p, 2, 4, 5, p, p) == INVALID


# ------------------------------------------------------------------------------------------------ restatements
def ingest_restated(x_nchw, patch):
    """csrc/ingest.cuh in numpy, with its own index arithmetic: per (sample, 64-channel slab), the slab as it lies in
    NCHW, transposed to pixel-major, then written per (pixel, tap) into the patch matrix or per pixel into NHWC."""
    B, C, H, W = x_nchw.shape
    HW = H * W
    flat = x_nchw.reshape(-1)
    out = np.full((B * HW, 9 * C) if patch else (B, H, W, C), np.nan, dtype=x_nchw.dtype)
    for b in range(B):
        for c0 in range(0, C, 64):
            start = (b * C + c0) * HW
            tile = flat[start:start + 64 * HW].reshape(64, HW).T          # [HW, 64]
            if not patch:
                out.reshape(B * HW, C)[b * HW:(b + 1) * HW, c0:c0 + 64] = tile
                continue
            for pix in range(HW):
                h, w = divmod(pix, W)
                for tap in range(9):
                    hs, ws = h + tap // 3 - 1, w + tap % 3 - 1
                    inside = 0 <= hs < H and 0 <= ws < W
                    out[b * HW + pix, tap * C + c0:tap * C + c0 + 64] = tile[hs * W + ws] if inside else 0
    return out


@pytest.mark.parametrize("B,C,H,W", [(2, 64, 3, 5), (1, 128, 7, 7)])
def test_ingest_layout_equals_the_oracle_patches_of_the_transposed_image(B, C, H, W):
    x = np.maximum(np.random.RandomState(C + H).standard_normal((B, C, H, W)), 0)
    nhwc = np.ascontiguousarray(x.transpose(0, 2, 3, 1))
    assert np.array_equal(ingest_restated(x, patch=False), nhwc)
    # the oracle's patch matrix, read out through an identity kernel (non-negative features pass its RELU unchanged)
    eye = {"stem/cnnLayercnn_0/kernels/kernel": np.eye(9 * C).reshape(3, 3, C, 9 * C),
           "stem/cnnLayercnn_0/biases/bias": np.zeros(9 * C)}
    want = stem_forward("RELU", eye, nhwc).reshape(B * H * W, 9 * C)
    assert np.array_equal(ingest_restated(x, patch=True), want)


def topk_restated(z, k):
    """mac_answer_topk's selection: round r takes the largest logit that sorts after round r-1's pick in (logit descending,
    id ascending) order."""
    ids = np.zeros((z.shape[0], k), dtype=np.int32)
    for b, row in enumerate(z):
        pv, pi = np.inf, -1
        for r in range(k):
            cand = [(v, a) for a, v in enumerate(row) if v < pv or (v == pv and a > pi)]
            pv, pi = max(cand, key=lambda va: (va[0], -va[1]))
            ids[b, r] = pi
    return ids


def test_topk_tie_rule_is_argmax_order():
    rng = np.random.RandomState(0)
    z = np.round(2 * rng.standard_normal((16, 37))).astype(np.float32)       # few distinct values: many ties
    z[3, :] = 1.5
    ids = topk_restated(z, 8)
    assert np.array_equal(ids[:, 0], torch.argmax(torch.from_numpy(z), dim=-1).numpy())
    assert np.array_equal(ids[3], np.arange(8))
    want = np.lexsort((np.broadcast_to(np.arange(37), z.shape), -z), axis=1)[:, :8]
    assert np.array_equal(ids, want)


# ------------------------------------------------------------------------------------------------ pipeline host logic
class _Counters(object):
    def __init__(self):
        self.event_syncs = self.replays = self.captures = self.streams = self.stream_waits = 0


def _fake_cuda(monkeypatch):
    from mac_network_b200 import serving
    n = _Counters()

    class Event(object):
        def record(self, stream=None):
            pass

        def synchronize(self):
            n.event_syncs += 1

    class Stream(object):
        def __init__(self):
            n.streams += 1

        def synchronize(self):
            pass

        def wait_stream(self, other):
            assert other is current
            n.stream_waits += 1

    current = object()

    class Graph(object):
        def replay(self):
            n.replays += 1

    @contextlib.contextmanager
    def graph(g, stream=None):
        n.captures += 1
        yield

    monkeypatch.setattr(torch.cuda, "Event", Event)
    monkeypatch.setattr(torch.cuda, "Stream", Stream)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda: current)
    monkeypatch.setattr(torch.cuda, "CUDAGraph", Graph)
    monkeypatch.setattr(torch.cuda, "graph", graph)
    monkeypatch.setattr(torch.cuda, "stream", lambda s: contextlib.nullcontext())
    monkeypatch.setattr(serving, "_pinned", lambda numel, dtype: torch.empty(numel, dtype=dtype))
    return n


B, S, V, E, H, W, C, A, L = 4, 6, 9, 12, 3, 3, 128, 8, 2


def _model(monkeypatch, prec="bf16", d=128, C_=C, **kw):
    mock = _mocklib.install(monkeypatch)
    counters = _fake_cuda(monkeypatch)
    from mac_network_b200.config import MACConfig
    from mac_network_b200.model import MACnet
    cfg = MACConfig.args("args", netLength=L, memDim=d, ctrlDim=d, attDim=d)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True), raising=False)
    net = MACnet(cfg, L, V, A, wrd_emb_dim=E, image_in_dim=C_, classifier_dims=(16,), prec=prec, device="cpu", **kw)
    return mock, counters, net


def _batch(seed):
    rng = np.random.RandomState(seed)
    lengths = np.array([5, 6, 2, 4], dtype=np.int32)
    q = rng.randint(1, V + 1, size=(B, S)).astype(np.int32)
    q[np.arange(S)[None, :] >= lengths[:, None]] = 0
    return {"questions": q, "questionLengths": lengths, "images": rng.standard_normal((B, C, H, W)).astype(np.float32)}


def test_pipeline_forward_order_slots_and_graph(monkeypatch):
    from mac_network_b200.serving import ModelPipeline
    mock, n, net = _model(monkeypatch)
    del mock.calls[:]
    pipe = ModelPipeline(net, (B, S, H, W), slots=3, host_cast=False, topk=2)
    assert n.streams == 3 and n.captures == 3 and not pipe.host_cast
    assert n.stream_waits == 3          # every slot's stream waited for the caller's before its eager pass
    # per slot: one eager pass and one captured pass, each ingest -> stem -> encoder -> cell -> logits -> top-k
    assert mock.calls.count("mac_ingest_nchw") == 6 and mock.calls.count("mac_answer_topk") == 6
    assert "mac_softmax_xent" not in mock.calls and "mac_host_cast_bf16_begin" not in mock.calls
    one = mock.calls[mock.calls.index("mac_ingest_nchw"):mock.calls.index("mac_answer_topk") + 1]
    assert one.index("mac_linear_tc_fwd") < one.index("mac_read_invariant") < one.index("mac_answer_topk")
    assert mock.calls.count("mac_pack_weight_bf16") >= 2 * 3            # every slot packs its own stem weights, once
    packs = mock.calls.count("mac_pack_weight_bf16")
    del mock.calls[:]
    tickets = [pipe.submit(_batch(i)) for i in range(7)]
    assert tickets == list(range(7)) and n.replays == 7 and mock.calls == []      # replays only: no library call per batch
    assert [t % 3 for t in tickets] == [0, 1, 2, 0, 1, 2, 0]
    for t in (4, 5, 6):
        assert pipe.result(t) is pipe.slots[t % 3].outs_host
    for t in (3, 7, -1):
        with pytest.raises(ValueError):
            pipe.result(t)
    out = pipe.result(6)
    assert set(out) == {"answers", "probs", "logits", "memory", "att_kb", "att_question"}
    assert out["answers"].shape == (B, 2) and out["answers"].dtype == torch.int32 and out["logits"].shape == (B, A)
    assert out["att_kb"].shape == (L, B, H * W) and out["att_question"].shape == (L, B, S)
    assert pipe.h2d_bytes == B * C * H * W * 4 + B * S * 4 + B * 4
    assert len(pipe.predictions(out)) == B
    assert packs == mock.calls.count("mac_pack_weight_bf16") + packs


def test_pipeline_without_graph_runs_the_forward_per_submit(monkeypatch):
    from mac_network_b200.serving import ModelPipeline
    mock, n, net = _model(monkeypatch, prec="fp32")
    pipe = ModelPipeline(net, (B, S, H, W), slots=2, use_graph=False)
    assert n.captures == 0 and not pipe.host_cast               # the fp32 stem reads the fp32 features: never cast
    del mock.calls[:]
    pipe.submit(_batch(0))
    assert mock.calls.count("mac_ingest_nchw") == 1 and mock.calls.count("mac_answer_topk") == 1 and n.replays == 0
    assert "mac_im2col3x3" in mock.calls                        # NHWC ingest, then the fp32 stem's own patch passes


def test_pipeline_staging_ring_and_cast_ahead(monkeypatch):
    from mac_network_b200.serving import ModelPipeline
    mock, n, net = _model(monkeypatch)
    pipe = ModelPipeline(net, (B, S, H, W), slots=4, host_cast=True, stage_ring=3, cast_threads=2)
    assert pipe.host_cast and len(pipe._ring.stages) == 3 and pipe.slots[0].x["images"].dtype == torch.bfloat16
    assert pipe.h2d_bytes == B * C * H * W * 2 + B * S * 4 + B * 4
    batches = [_batch(i) for i in range(8)]
    del mock.calls[:]
    for i, b in enumerate(batches):
        before = n.event_syncs
        pipe.submit(b, next_batch=batches[i + 1] if i + 1 < len(batches) else None)
        # the cast of batch i+1 started under batch i; its staging buffer (ring of 3) is waited for from the 4th cast on
        assert n.event_syncs - before == (1 if 2 <= i < 7 else 0), i
    assert mock.calls.count("mac_host_cast_bf16_begin") == 8 and mock.calls.count("mac_host_cast_bf16_end") == 8
    assert pipe._ring.casts == 8 and pipe._ring.pending is None
    assert [pipe._ring.busy[i] is not None for i in range(3)] == [True, True, True]
    # a next_batch that turns out not to be next: its cast is discarded and its buffer taken again
    pipe.submit(batches[0], next_batch=batches[1])
    casts = pipe._ring.casts
    pipe.submit(batches[2])
    assert pipe._ring.casts == casts + 0 and mock.calls.count("mac_host_cast_bf16_begin") == 11


@pytest.mark.parametrize("cast_ms,on", [(0.0, True), (1e3, False)])
def test_pipeline_host_cast_decision(monkeypatch, cast_ms, on):
    from mac_network_b200 import serving
    mock, n, net = _model(monkeypatch)
    monkeypatch.setattr(serving, "_time_cast", lambda lib, numel, threads: cast_ms)
    pipe = serving.ModelPipeline(net, (B, S, H, W), slots=1)
    assert pipe.host_cast is on and pipe.cast_ms == cast_ms
    assert serving._cast_pays(0.79 * 2 * 1e6 / 25e9 * 1e3, 10 ** 6) and not serving._cast_pays(0.81 * 2 * 1e6 / 25e9 * 1e3, 10 ** 6)
    # an e4m3 stem reads the fp32 features: the cast is off whatever is asked
    mock, n, net8 = _model(monkeypatch, d=128, eval_stem_prec="fp8")
    assert not serving.ModelPipeline(net8, (B, S, H, W), slots=1, host_cast=True).host_cast


def test_pipeline_captures_again_when_the_weights_move(monkeypatch):
    from mac_network_b200.serving import ModelPipeline
    mock, n, net = _model(monkeypatch)
    pipe = ModelPipeline(net, (B, S, H, W), slots=2, host_cast=False)
    pipe.submit(_batch(0))
    assert n.captures == 2
    del mock.calls[:]
    net.trainer.params.touch()
    syncs = n.event_syncs
    pipe.submit(_batch(1))
    assert n.captures == 4 and n.event_syncs == syncs + 1               # drained the one busy slot, then both captured again
    assert n.stream_waits == 4          # ... each after waiting for the stream the weights were moved on
    assert mock.calls.count("mac_pack_weight_bf16") >= 4                # new packs, built in the eager pass of each slot
    del mock.calls[:]
    pipe.submit(_batch(2))
    assert n.captures == 4 and mock.calls == []


def test_pipeline_refusals_precede_any_library_call(monkeypatch):
    from mac_network_b200 import serving
    mock, n, net = _model(monkeypatch)
    del mock.calls[:]
    for kw in (dict(topk=0), dict(topk=9), dict(slots=0)):
        with pytest.raises(ValueError):
            serving.ModelPipeline(net, (B, S, H, W), **kw)
    with pytest.raises(ValueError):
        serving.ModelPipeline(net, (B, 0, H, W))
    mock96, _, net96 = _model(monkeypatch, prec="fp32", C_=96)
    del mock96.calls[:]
    with pytest.raises(ValueError):
        serving.ModelPipeline(net96, (B, S, H, W))
    assert mock.calls == [] and mock96.calls == [] and n.streams == 0
    # the cell's own refusal (e4m3 read step at d != 512) passes through
    mock8, _, net8 = _model(monkeypatch, prec="fp8", d=128)
    with pytest.raises(NotImplementedError):
        serving.ModelPipeline(net8, (B, S, H, W), slots=1)
    mock, n, net = _model(monkeypatch)
    pipe = serving.ModelPipeline(net, (B, S, H, W), slots=1, host_cast=True)
    del mock.calls[:]
    good = _batch(0)
    for bad in (dict(good, questions=good["questions"][:, :S - 1]), dict(good, questionLengths=good["questionLengths"][:2]),
                dict(good, images=good["images"][:, :64]), dict(good, images=good["images"].transpose(0, 2, 3, 1))):
        with pytest.raises(ValueError):
            pipe.submit(bad)
        with pytest.raises(ValueError):
            pipe.submit(good, next_batch=bad)
    assert mock.calls == [] and n.replays == 0 and pipe._next == 0
