"""CPU side of whole-model training from host buffers (serving.TrainPipeline, mac_ingest_nchw_train, Stem.forward_nchw in
training): the new entry point's declaration and its refusals through the real library (each status comes back before any
CUDA call), the stem's and the trainer's calls into it over the dry-run library (tests/_mocklib.py), and the pipeline's host
logic -- refusals before any library call, ticket rules, the order in which a slot's buffers are written, copied, read and
written again -- with the CUDA stream / event objects replaced by a log."""
import contextlib
import ctypes

import numpy as np
import pytest
import torch

from mac_network_b200 import _lib as L_
from tests import _mocklib
from tests.test_stem_tc_training import _cpu_params, _fake_ptr, _recorder

INVALID, ALIGN, UNSUPPORTED = -1, -2, -3


# ------------------------------------------------------------------------------------------------ the C boundary
def test_prototype_is_declared_bound_and_exported():
    from tests.test_abi import _declared
    lib = L_.load()
    assert "mac_ingest_nchw_train" in _declared() and hasattr(lib, "mac_ingest_nchw_train")
    c = ctypes
    assert L_.PROTOTYPES["mac_ingest_nchw_train"] == (c.c_int, [c.c_void_p, c.c_void_p, c.c_void_p, c.c_int, c.c_float,
                                                                c.c_uint64] + [c.c_int] * 6 + [c.c_void_p])
    assert lib.mac_b200_abi_version() == 1


def test_ingest_train_refuses_before_any_cuda_call():
    lib = L_.load()
    buf = (ctypes.c_float * 4096)()
    p = _fake_ptr(buf)

    def call(x=p, y=p, cols=p, form=0, keep=0.82, B=2, C=64, H=7, W=7):
        return lib.mac_ingest_nchw_train(x, y, cols, form, keep, 7, 32, 3, B, C, H, W, None)
    before = lib.mac_b200_launch_count()
    assert call(x=None) == INVALID and call(y=None) == INVALID and call(cols=None) == INVALID
    assert call(B=0) == INVALID and call(C=0) == INVALID and call(H=-1) == INVALID and call(W=0) == INVALID
    for keep in (0.0, -0.5, 1.0001, 2.0, float("nan")):
        assert call(keep=keep) == INVALID, keep
    assert call(x=p + 4) == ALIGN and call(y=p + 8) == ALIGN and call(cols=p + 2) == ALIGN
    assert call(C=96) == UNSUPPORTED and call(C=32) == UNSUPPORTED
    assert call(form=2) == UNSUPPORTED and call(form=-1) == UNSUPPORTED
    assert call(B=65536) == UNSUPPORTED
    # shared memory per pixel: 672 bytes (bf16 patches), 816 (split); 227 KB less the 128 static bytes
    assert call(H=2, W=173) == UNSUPPORTED and call(form=1, H=5, W=57) == UNSUPPORTED      # 346 / 285 pixels
    assert call(H=100, W=100) == UNSUPPORTED and call(H=1 << 16, W=1 << 16) == UNSUPPORTED
    assert lib.mac_b200_launch_count() == before
    if not torch.cuda.is_available():
        # every argument check passed: the largest slabs, keep = 1, 1x1 images; only the CUDA runtime's call fails here
        for kw in (dict(H=15, W=23), dict(form=1, H=4, W=71), dict(keep=1.0, H=1, W=1), dict(C=2048, B=65535)):
            assert call(**kw) not in (0, INVALID, ALIGN, UNSUPPORTED), kw


# ------------------------------------------------------------------------------------------------ the stem
def _stem(prec, cin=128, cout=128):
    from mac_network_b200.stem import Stem, init_stem_params, stem_specs
    return Stem(_cpu_params(init_stem_params(stem_specs(cin, cout), seed=1)), relu="ELU", prec=prec, seed=11)


@pytest.mark.parametrize("prec,form", [("bf16", 0), ("bf16x3", 1)])
def test_forward_nchw_training_passes_seed_site_and_step(monkeypatch, prec, form):
    rec = _recorder(monkeypatch)
    from mac_network_b200.stem import SITE_STEM
    st = _stem(prec)
    kb = st.forward_nchw(torch.zeros(2, 128, 5, 7), keep=0.82, step=9, save_for_backward=True)
    assert kb.shape == (2, 35, 128)
    (a,) = rec.args_of("mac_ingest_nchw_train")
    assert a[3] == form and a[4] == pytest.approx(0.82) and a[5:8] == (11, SITE_STEM, 9) and a[8:12] == (2, 128, 5, 7)
    # layer 0's patch pass is the ingest's; layer 1 builds its own from layer 0's output
    patch = "mac_im2col3x3_split" if prec == "bf16x3" else "mac_im2col3x3"
    assert len(rec.args_of(patch)) == 1 and rec.args_of(patch)[0][4 if prec == "bf16x3" else 5] == SITE_STEM + 1
    assert not rec.args_of("mac_ingest_nchw")
    x0 = st._saved["xs"][0]
    assert x0.shape == (2, 5, 7, 128) and x0.dtype == torch.float32 and x0.is_contiguous()
    assert st._saved["keep"] == pytest.approx(0.82) and st._saved["step"] == 9
    # a dropout alone (no save) takes the training ingest too; the default call keeps the inference ingest
    rec.log.clear()
    st.forward_nchw(torch.zeros(2, 128, 5, 7), keep=0.5, step=2)
    assert len(rec.args_of("mac_ingest_nchw_train")) == 1 and rec.args_of("mac_ingest_nchw_train")[0][7] == 2
    rec.log.clear()
    st.forward_nchw(torch.zeros(2, 128, 5, 7))
    assert not rec.args_of("mac_ingest_nchw_train") and len(rec.args_of("mac_ingest_nchw")) == 1


def test_forward_nchw_training_fp32_stem_and_refusals(monkeypatch):
    rec = _recorder(monkeypatch)
    from mac_network_b200.stem import INGEST_NHWC_F32
    st = _stem("fp32")
    st.forward_nchw(torch.zeros(2, 128, 5, 7), keep=0.82, step=4, save_for_backward=True)
    assert [n for n, _ in rec.log if n.startswith(("mac_ingest", "mac_im2col"))] == \
        ["mac_ingest_nchw", "mac_im2col3x3", "mac_im2col3x3"]
    assert rec.args_of("mac_ingest_nchw")[0][3] == INGEST_NHWC_F32
    assert [a[3] == pytest.approx(0.82) and a[6] == 4 for a in rec.args_of("mac_im2col3x3")] == [True, True]
    assert st._saved["xs"][0].shape == (2, 5, 7, 128)
    rec.log.clear()
    st16 = _stem("bf16")
    for kw in (dict(save_for_backward=True), dict(keep=0.82)):
        with pytest.raises(ValueError, match="bf16 images"):
            st16.forward_nchw(torch.zeros(2, 128, 5, 7, dtype=torch.bfloat16), **kw)
    with pytest.raises(NotImplementedError):                     # the e4m3 stem is inference only
        _stem("fp8").forward_nchw(torch.zeros(2, 128, 5, 7), keep=0.82)
    with pytest.raises(NotImplementedError, match="multiples of 128"):
        _stem("bf16", cin=64).forward_nchw(torch.zeros(2, 64, 5, 7), save_for_backward=True)
    assert rec.log == []


def test_trainer_takes_exactly_one_image_layout(monkeypatch):
    mock, net, _ = _net(monkeypatch, stem_prec="bf16")
    t = net.trainer
    B, S = 4, 6
    data = {"questions": torch.ones(B, S, dtype=torch.int32), "questionLengths": torch.full((B,), S, dtype=torch.int32),
            "answers": torch.zeros(B, dtype=torch.int32)}
    mock.calls.clear()
    for imgs in ({}, {"images": torch.zeros(B, H, W, C), "images_nchw": torch.zeros(B, C, H, W)},
                 {"images_nchw": torch.zeros(B, H, W, C).permute(0, 3, 1, 2)}, {"images_nchw": torch.zeros(B, C, H, W).double()}):
        with pytest.raises(ValueError):
            t.full_forward_backward((B, S), dict(data, **imgs), global_batch=B)
    assert mock.calls == [] and t.step_id == 0
    t.train_step_full((B, S), dict(data, images_nchw=torch.zeros(B, C, H, W)), global_batch=B)
    assert mock.calls.count("mac_ingest_nchw_train") == 1 and "mac_im2col3x3" in mock.calls      # layer 1's own pass
    assert t.step_id == 1


# ------------------------------------------------------------------------------------------------ the pipeline
B, S, V, E, H, W, C, A, L = 4, 6, 9, 12, 3, 3, 128, 8, 2


def _fake_cuda(monkeypatch):
    """Streams and events that log what is enqueued where: ("record", event, stream name), ("wait", stream name, event)
    and ("sync", event)."""
    from mac_network_b200 import serving
    log = []
    state = {"stream": None}

    class Stream(object):
        def __init__(self, name="copy"):
            self.name = name

        def wait_event(self, ev):
            log.append(("wait", self.name, ev))

        def wait_stream(self, other):
            pass

        def synchronize(self):
            pass

    main = Stream("main")

    class Event(object):
        def record(self, stream=None):
            log.append(("record", self, (stream or main).name))

        def synchronize(self):
            log.append(("sync", self))

    @contextlib.contextmanager
    def stream_ctx(s):
        prev, state["stream"] = state["stream"], s
        try:
            yield
        finally:
            state["stream"] = prev

    monkeypatch.setattr(torch.cuda, "Event", Event)
    monkeypatch.setattr(torch.cuda, "Stream", Stream)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda: main)
    monkeypatch.setattr(torch.cuda, "stream", stream_ctx)
    monkeypatch.setattr(serving, "_pinned", lambda numel, dtype: torch.empty(numel, dtype=dtype))
    return log


def _net(monkeypatch, **kw):
    mock = _mocklib.install(monkeypatch)
    log = _fake_cuda(monkeypatch)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True), raising=False)
    from mac_network_b200.config import MACConfig
    from mac_network_b200.model import MACnet
    cfg = MACConfig.args("args", netLength=L, memDim=128, ctrlDim=128, attDim=128)
    net = MACnet(cfg, L, V, A, wrd_emb_dim=E, image_in_dim=C, classifier_dims=(16,), prec="bf16", device="cpu", **kw)
    return mock, net, log


def _batch(seed, longest=S, width=S):
    rng = np.random.RandomState(seed)
    lengths = rng.randint(1, longest + 1, size=(B,)).astype(np.int32)
    lengths[seed % B] = longest
    q = rng.randint(1, V + 1, size=(B, width)).astype(np.int32)
    q[np.arange(width)[None, :] >= lengths[:, None]] = 0
    return {"questions": q, "questionLengths": lengths, "answers": rng.randint(0, A, size=(B,)).astype(np.int32),
            "images": rng.standard_normal((B, C, H, W)).astype(np.float32)}


def test_pipeline_refusals_precede_any_library_call(monkeypatch):
    from mac_network_b200.serving import TrainPipeline
    mock, net, log = _net(monkeypatch, stem_prec="bf16")
    mock.calls.clear()
    for shape, kw in (((B, 0, H, W), {}), ((B, S, H, W), dict(depth=0))):
        with pytest.raises(ValueError):
            TrainPipeline(net, shape, **kw)
    pipe = TrainPipeline(net, (B, S, H, W), depth=2, stage_threads=3)
    good = _batch(0)
    bad = [dict(good, questions=good["questions"][:2]), dict(good, questions=np.zeros((B, S + 1), np.int32)),
           dict(good, questions=good["questions"].astype(np.float32)), dict(good, questionLengths=good["questionLengths"][:3]),
           dict(good, questionLengths=np.full(B, S + 1, np.int32)), dict(good, questionLengths=np.zeros(B, np.int32)),
           dict(good, questionLengths=np.array([-1, 2, 3, 4], np.int32)), dict(good, answers=np.full(B, A, np.int32)),
           dict(good, answers=-np.ones(B, np.int32)), dict(good, images=good["images"][:, :64]),
           dict(good, images=good["images"].transpose(0, 2, 3, 1)), {k: v for k, v in good.items() if k != "answers"},
           # a question trimmed narrower than its length
           dict(good, questions=good["questions"][:, :3], questionLengths=np.array([5, 2, 2, 3], np.int32))]
    for b in bad:
        with pytest.raises(ValueError):
            pipe.submit(b)
    assert mock.calls == [] and pipe._next == 0 and not [e for e in log if e[0] in ("wait", "sync")]
    with pytest.raises(ValueError):
        pipe.result(0)


def test_pipeline_steps_tickets_and_buffer_reuse_order(monkeypatch):
    from mac_network_b200.serving import TrainPipeline
    mock, net, log = _net(monkeypatch, stem_prec="bf16x3")
    tr = net.trainer
    pipe = TrainPipeline(net, (B, S, H, W), depth=2, stage_threads=2)
    longest = [S, 4, 4, 2, S]
    tickets = []
    for i, n in enumerate(longest):
        log.clear()
        mock.calls.clear()
        tickets.append(pipe.submit(_batch(i, longest=n)))
        slot = pipe.slots[i % 2]
        kinds = [e[0] for e in log]
        # written only after the step that read the slot (two submits back) is done; copied; the step waits for the copy
        first = ["record", "wait"] if i < 2 else ["sync", "record", "wait"]
        assert kinds[:len(first)] == first, (i, kinds)
        if i >= 2:
            assert log[0][1] is slot.done
        assert log[len(first) - 2][1:] == (slot.copied, "copy") and log[len(first) - 1][1:] == ("main", slot.copied)
        assert log[-1][1:] == (slot.done, "main")                                 # after the step and its result copies
        # one step of the trimmed shape, with the NCHW features through the training ingest (split form)
        assert tuple(tr._cells) [-1] == (B, n) and net.macCell is tr._cells[(B, n)][0]
        (a,) = [c for c in mock.calls if c.startswith("mac_ingest")]
        assert a == "mac_ingest_nchw_train" and mock.calls.count("mac_clip_adam_ema_step") == 1
        assert int(slot.dev["questionLengths"].max()) == n
        assert torch.equal(slot.host["questions"][:B * n].view(B, n), torch.from_numpy(_batch(i, longest=n)["questions"][:, :n]))
        assert torch.equal(slot.host["images"], torch.from_numpy(_batch(i, longest=n)["images"]).reshape(-1))
        assert tr.step_id == i + 1
    assert tickets == list(range(5))
    for t in (3, 4):
        res = pipe.result(t)
        assert set(res) == {"loss", "correctNum", "acc", "gradNorm", "predictions"}
        assert res["predictions"] is pipe.slots[t % 2].out["predictions"] and res["predictions"].dtype == torch.int32
        assert len(pipe.predictions(res)) == B and res["acc"] == res["correctNum"] / B
    for t in (2, 5, -1):
        with pytest.raises(ValueError):
            pipe.result(t)
    log.clear()
    pipe.drain()
    assert [e[0] for e in log] == ["sync", "sync"]


def test_pipeline_pinned_images_are_copied_from_where_they_lie(monkeypatch):
    from mac_network_b200.serving import TrainPipeline
    mock, net, log = _net(monkeypatch)
    pipe = TrainPipeline(net, (B, S, H, W), depth=1, stage_threads=1)
    b = _batch(3)
    img = torch.from_numpy(b["images"])
    staged = []
    monkeypatch.setattr(pipe, "_stage_images", lambda dst, src: staged.append(src))
    monkeypatch.setattr(torch.Tensor, "is_pinned", lambda self: self.data_ptr() == img.data_ptr())
    pipe.submit(dict(b, images=img))
    assert staged == [] and torch.equal(pipe.slots[0].dev["images"], img.reshape(-1))
    pipe.submit(_batch(4))                                       # numpy (pageable): staged into the slot's pinned buffer
    assert len(staged) == 1
    # depth 1: the second submit waited for the first step before it wrote the slot again
    assert [e[0] for e in log].count("sync") == 1
    # the fp32 stem: NHWC ingest, then its own patch pass for layer 0 and layer 1
    assert mock.calls.count("mac_ingest_nchw") == 2 and "mac_ingest_nchw_train" not in mock.calls
