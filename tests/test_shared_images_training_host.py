"""CPU side of several questions per image in training (DPTrainer with data["imageIndex"], serving.TrainPipeline(images=U),
mac_kb_gather_bwd): the new entry point's declaration and its refusals through the real library (each status comes back
before any CUDA call), the trainer's and the pipeline's refusals before any library call, the launch order of an indexed step
and the pipeline's buffer sizes and copies, over the dry-run library (tests/_mocklib.py) with the CUDA stream / event objects
replaced by a log."""
import ctypes

import numpy as np
import pytest
import torch

from mac_network_b200 import _lib as L_
from tests.test_stem_tc_training import _fake_ptr, _recorder
from tests.test_train_pipeline_host import A, B, C, E, H, L, S, V, W, _batch, _fake_cuda

INVALID, ALIGN, UNSUPPORTED = -1, -2, -3


# ------------------------------------------------------------------------------------------------ the C boundary
def test_prototype_is_declared_bound_and_exported():
    from tests.test_abi import _declared
    lib = L_.load()
    assert "mac_kb_gather_bwd" in _declared() and hasattr(lib, "mac_kb_gather_bwd")
    c = ctypes
    assert L_.PROTOTYPES["mac_kb_gather_bwd"] == (c.c_int, [c.c_void_p] * 3 + [c.c_int] * 4 + [c.c_void_p])
    assert lib.mac_b200_abi_version() == 1


def test_kb_gather_bwd_refuses_before_any_cuda_call():
    lib = L_.load()
    buf = (ctypes.c_float * 4096)()
    p = _fake_ptr(buf)

    def call(g=p, idx=p, out=p, B=3, U=2, N=4, d=8):
        return lib.mac_kb_gather_bwd(g, idx, out, B, U, N, d, None)
    before = lib.mac_b200_launch_count()
    assert call(g=None) == INVALID and call(idx=None) == INVALID and call(out=None) == INVALID
    for kw in (dict(B=0), dict(U=0), dict(N=0), dict(d=0), dict(B=-1), dict(U=-3)):
        assert call(**kw) == INVALID, kw
    assert call(d=4) == UNSUPPORTED and call(d=12) == UNSUPPORTED
    assert call(N=1 << 30, d=64) == UNSUPPORTED                 # N*d/8 = 2^33 vectors
    assert call(g=p + 4) == ALIGN and call(idx=p + 8) == ALIGN and call(out=p + 4) == ALIGN
    assert lib.mac_b200_launch_count() == before
    if not torch.cuda.is_available():
        # every argument check passed (N*d/8 = 2^31 - 1 vectors included): only the CUDA runtime's call fails here
        for kw in (dict(), dict(N=(2 ** 31 - 1), d=8), dict(B=70000, U=70000)):
            assert call(**kw) not in (0, INVALID, ALIGN, UNSUPPORTED), kw


# ------------------------------------------------------------------------------------------------ the trainer
def _net(monkeypatch, **kw):
    """A MACnet over the dry-run library, its calls recorded with their arguments."""
    rec = _recorder(monkeypatch)
    log = _fake_cuda(monkeypatch)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True), raising=False)
    from mac_network_b200.config import MACConfig
    from mac_network_b200.model import MACnet
    cfg = MACConfig.args("args", netLength=L, memDim=128, ctrlDim=128, attDim=128)
    net = MACnet(cfg, L, V, A, wrd_emb_dim=E, image_in_dim=C, classifier_dims=(16,), prec="bf16", device="cpu", **kw)
    return rec, net, log


def _data(k, index):
    return {"questions": torch.ones(B, S, dtype=torch.int32), "questionLengths": torch.full((B,), S, dtype=torch.int32),
            "answers": torch.zeros(B, dtype=torch.int32), "images_nchw": torch.zeros(k, C, H, W),
            "imageIndex": torch.tensor(index, dtype=torch.int32)}


def test_trainer_refuses_a_malformed_index_before_any_launch(monkeypatch):
    rec, net, _ = _net(monkeypatch, stem_prec="bf16")
    t = net.trainer
    good = _data(2, [0, 1, 1, 0])
    wide = torch.zeros(B, 2, dtype=torch.int32)
    bad = [dict(good, imageIndex=good["imageIndex"].float()), dict(good, imageIndex=good["imageIndex"].long()),
           dict(good, imageIndex=good["imageIndex"].bool()), dict(good, imageIndex=good["imageIndex"][:3]),
           dict(good, imageIndex=torch.zeros(B + 1, dtype=torch.int32)), dict(good, imageIndex=wide[:, 0]),
           dict(good, imageIndex=[0, 1, 1, 0]), dict(good, images_nchw=torch.zeros(B + 1, C, H, W)),
           dict(good, images_nchw=torch.zeros(0, C, H, W)),
           # the NHWC layout takes the index too, with the same rules
           dict({k: v for k, v in good.items() if k != "images_nchw"}, images=torch.zeros(B + 1, H, W, C))]
    rec.log.clear()
    for d in bad:
        with pytest.raises(ValueError):
            t.full_forward_backward((B, S), d, global_batch=B)
    assert rec.log == [] and t.step_id == 0


def test_indexed_step_launch_order(monkeypatch):
    """encoder -> the stem over the k images -> mac_kb_gather into the cell's input -> the cell ... the cell's backward ->
    mac_kb_gather_bwd over [B] -> [k] -> the stem's backward over k rows -> the encoder's backward."""
    rec, net, _ = _net(monkeypatch, stem_prec="bf16")
    t = net.trainer
    k = 3
    for step in range(2):
        rec.log.clear()
        t.train_step_full((B, S), _data(k, [2, 0, 2, 1]), global_batch=B)
        names = [n for n, _ in rec.log]
        at = lambda n: names.index(n)
        last = lambda n: len(names) - 1 - names[::-1].index(n)
        assert names.count("mac_kb_gather") == 1 and names.count("mac_kb_gather_bwd") == 1
        (ing,) = rec.args_of("mac_ingest_nchw_train")
        assert ing[8] == k                                                       # the stem's rows: the k images
        assert at("mac_lstm_fwd") < at("mac_ingest_nchw_train") < last("mac_linear_tc_fwd") < at("mac_kb_gather")
        assert at("mac_kb_gather") < at("mac_read_fwd")
        assert last("mac_read_bwd") < at("mac_kb_gather_bwd") < at("mac_conv3x3_bwd_tc") < at("mac_lstm_bwd")
        (gat,) = rec.args_of("mac_kb_gather")
        assert gat[3:8] == (0, B, k, H * W, 128)                             # fp32 out, B questions from k images
        (bwd,) = rec.args_of("mac_kb_gather_bwd")
        assert bwd[3:7] == (B, k, H * W, 128)
        assert all(a[-6] == k for a in rec.args_of("mac_conv3x3_bwd_tc"))       # the stem's backward over k rows
        cell, bufs = t._cells[(B, S)]
        if step:     # the cell exists: the gather writes straight into its persistent input, which cell_for does not copy
            assert gat[2].value == bufs["knowledgeBase"].data_ptr()
            assert cell.knowledgeBase.data_ptr() == bufs["knowledgeBase"].data_ptr()
        assert gat[1].value == bwd[1].value                                      # one index for both
    assert t.step_id == 2


def test_step_without_an_index_makes_neither_launch(monkeypatch):
    rec, net, _ = _net(monkeypatch, stem_prec="bf16x3")
    d = _data(B, [0, 1, 2, 3])
    del d["imageIndex"]
    net.trainer.train_step_full((B, S), d, global_batch=B)
    names = [n for n, _ in rec.log]
    assert "mac_kb_gather" not in names and "mac_kb_gather_bwd" not in names
    assert rec.args_of("mac_ingest_nchw_train")[0][8] == B


# ------------------------------------------------------------------------------------------------ the pipeline
def _shared(seed, k, longest=S):
    b = _batch(seed, longest=longest)
    rng = np.random.RandomState(seed + 100)
    idx = rng.randint(0, k, size=(B,)).astype(np.int32)
    idx[:k] = np.arange(k)
    return dict(b, images=rng.standard_normal((k, C, H, W)).astype(np.float32), imageIndex=idx)


def test_pipeline_refusals_precede_any_library_call(monkeypatch):
    from mac_network_b200.serving import TrainPipeline
    rec, net, log = _net(monkeypatch, stem_prec="bf16")
    rec.log.clear()
    for images in (0, B + 1, -1, 2.0, True, "2"):
        with pytest.raises(ValueError):
            TrainPipeline(net, (B, S, H, W), images=images)
    U = 3
    pipe = TrainPipeline(net, (B, S, H, W), depth=2, stage_threads=2, images=U)
    good = _shared(0, 2)
    bad = [{k: v for k, v in good.items() if k != "imageIndex"},                    # no index
           dict(good, images=np.zeros((U + 1, C, H, W), np.float32)),                 # k > U
           dict(good, images=np.zeros((0, C, H, W), np.float32)),                     # k = 0
           dict(good, images=np.zeros((2, C, H + 1, W), np.float32)),
           dict(good, images=np.zeros((2 * C * H * W,), np.float32)),
           dict(good, imageIndex=np.array([0, 1, 2, 0], np.int32)),                  # 2 outside [0, k = 2)
           dict(good, imageIndex=np.array([0, -1, 1, 0], np.int32)),
           dict(good, imageIndex=good["imageIndex"].astype(np.float32)),
           dict(good, imageIndex=good["imageIndex"].astype(bool)),
           dict(good, imageIndex=good["imageIndex"][:3]),
           dict(good, imageIndex=good["imageIndex"].reshape(2, 2))]
    for b in bad:
        with pytest.raises(ValueError):
            pipe.submit(b)
    plain = TrainPipeline(net, (B, S, H, W), depth=1)
    with pytest.raises(ValueError, match="images=U"):
        plain.submit(dict(_batch(0), imageIndex=np.zeros(B, np.int32)))
    assert rec.log == [] and pipe._next == 0 and plain._next == 0
    assert not [e for e in log if e[0] in ("wait", "sync")]


def test_pipeline_sizes_its_buffers_from_u_and_copies_k_images(monkeypatch):
    from mac_network_b200.serving import TrainPipeline
    rec, net, log = _net(monkeypatch, stem_prec="bf16x3")
    U = 3
    pipe = TrainPipeline(net, (B, S, H, W), depth=2, stage_threads=2, images=U)
    per = C * H * W
    for s in pipe.slots:
        assert s.host["images"].numel() == U * per and s.dev["images"].numel() == U * per
        assert s.host["imageIndex"].numel() == B and s.dev["imageIndex"].dtype == torch.int32
        s.dev["images"].fill_(-7.0)
    plain = TrainPipeline(net, (B, S, H, W), depth=1)
    assert plain.slots[0].host["images"].numel() == B * per and "imageIndex" not in plain.slots[0].host
    for i, k in enumerate((U, U - 2, 1)):
        rec.log.clear()
        b = _shared(i, k)
        if i == 1:                                              # a pinned tensor is copied from where it lies
            pinned = torch.from_numpy(b["images"])
            monkeypatch.setattr(torch.Tensor, "is_pinned", lambda self: self.data_ptr() == pinned.data_ptr())
            b = dict(b, images=pinned)
        pipe.submit(b)
        slot = pipe.slots[i % 2]
        assert torch.equal(slot.dev["images"][:k * per], torch.as_tensor(b["images"]).reshape(-1)), i
        # only k images were copied: the rest of the slot still holds what was there before
        prev = -7.0 if i < 2 else _shared(0, U)["images"].reshape(-1)[k * per:]
        assert torch.equal(slot.dev["images"][k * per:], torch.as_tensor(prev).expand(U * per - k * per)), i
        assert torch.equal(slot.dev["imageIndex"], torch.from_numpy(b["imageIndex"]))
        (ing,) = rec.args_of("mac_ingest_nchw_train")
        assert ing[8] == k
        (bwd,) = rec.args_of("mac_kb_gather_bwd")
        assert bwd[3:5] == (B, k) and bwd[1].value == slot.dev["imageIndex"].data_ptr()
    assert net.trainer.step_id == 3
