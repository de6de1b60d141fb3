"""CPU side of image features stored in fp16 (mac_ingest_nchw_f16, mac_ingest_nchw_train_f16, Stem.forward_nchw with
torch.float16 images, the pipelines' image_dtype): the two entry points' declarations and their refusals through the real
library (each status comes back before any CUDA call, the shared-memory limits on both sides), the stem's launches over the
dry-run library (tests/_mocklib.py) against the fp32 images' launches, and the pipelines' fp16 staging and refusals with
the CUDA stream / event / graph objects replaced by counters."""
import ctypes

import numpy as np
import pytest
import torch

from mac_network_b200 import _lib as L_
from tests import test_kb_cache_host as KB
from tests import test_model_pipeline_host as MP
from tests import test_train_pipeline_host as TP
from tests.test_stem_tc_training import _cpu_params, _fake_ptr, _recorder

INVALID, ALIGN, UNSUPPORTED = -1, -2, -3
ERRORS = (0, INVALID, ALIGN, UNSUPPORTED)


# ------------------------------------------------------------------------------------------------ the C boundary
def test_prototypes_match_the_header_and_are_exported():
    from tests.test_abi import _declared
    lib = L_.load()
    c = ctypes
    assert L_.PROTOTYPES["mac_ingest_nchw_f16"] == (c.c_int, [c.c_void_p, c.c_void_p] + [c.c_int] * 5 + [c.c_void_p])
    assert L_.PROTOTYPES["mac_ingest_nchw_train_f16"] == (c.c_int, [c.c_void_p] * 3 + [c.c_int, c.c_float, c.c_uint64]
                                                          + [c.c_int] * 6 + [c.c_void_p])
    # the fp32 entry points' arguments, less mac_ingest_nchw's x_bf16
    fp32 = L_.PROTOTYPES["mac_ingest_nchw"][1]
    assert L_.PROTOTYPES["mac_ingest_nchw_f16"][1] == fp32[:1] + fp32[2:]
    assert L_.PROTOTYPES["mac_ingest_nchw_train_f16"] == L_.PROTOTYPES["mac_ingest_nchw_train"]
    for name in ("mac_ingest_nchw_f16", "mac_ingest_nchw_train_f16"):
        assert name in _declared() and hasattr(lib, name)
    assert lib.mac_b200_abi_version() == 1


def test_ingest_f16_refuses_before_any_cuda_call():
    lib = L_.load()
    buf = (ctypes.c_float * 4096)()
    p = _fake_ptr(buf)

    def call(x=p, out=p, mode=0, B=2, C=64, H=7, W=7):
        return lib.mac_ingest_nchw_f16(x, out, mode, B, C, H, W, None)
    before = lib.mac_b200_launch_count()
    assert call(x=None) == INVALID and call(out=None) == INVALID
    assert call(B=0) == INVALID and call(C=0) == INVALID and call(H=0) == INVALID and call(W=-3) == INVALID
    assert call(x=p + 2) == ALIGN and call(x=p + 8) == ALIGN and call(out=p + 4, mode=1) == ALIGN
    assert call(C=32) == UNSUPPORTED and call(C=96) == UNSUPPORTED
    assert call(mode=2) == UNSUPPORTED and call(mode=-1) == UNSUPPORTED
    assert call(B=65536) == UNSUPPORTED and call(H=100, W=100) == UNSUPPORTED and call(H=1 << 16, W=1 << 16) == UNSUPPORTED
    # shared memory per pixel: 128 + 272 bytes (-> NHWC), 128 + 144 (-> patches); 227 KB less the 128 static bytes
    assert call(mode=0, H=7, W=83) == UNSUPPORTED and call(mode=1, H=9, W=95) == UNSUPPORTED      # 581 / 855 pixels
    # the refusal classes in their order: INVALID before ALIGN before UNSUPPORTED
    assert call(x=p + 2, B=0) == INVALID and call(x=p + 2, C=96) == ALIGN
    assert lib.mac_b200_launch_count() == before
    if not torch.cuda.is_available():
        # every argument check passed -- the largest slabs, 1x1 images, the largest grid; only the CUDA runtime fails here
        for kw in (dict(mode=0, H=20, W=29), dict(mode=1, H=14, W=61), dict(H=1, W=1), dict(C=2048, B=65535)):
            assert call(**kw) not in ERRORS, kw


def test_ingest_train_f16_refuses_before_any_cuda_call():
    lib = L_.load()
    buf = (ctypes.c_float * 4096)()
    p = _fake_ptr(buf)

    def call(x=p, y=p, cols=p, form=0, keep=0.82, B=2, C=64, H=7, W=7):
        return lib.mac_ingest_nchw_train_f16(x, y, cols, form, keep, 7, 32, 3, B, C, H, W, None)
    before = lib.mac_b200_launch_count()
    assert call(x=None) == INVALID and call(y=None) == INVALID and call(cols=None) == INVALID
    assert call(B=0) == INVALID and call(C=0) == INVALID and call(H=-1) == INVALID and call(W=0) == INVALID
    for keep in (0.0, -0.5, 1.0001, 2.0, float("nan")):
        assert call(keep=keep) == INVALID, keep
    assert call(x=p + 2) == ALIGN and call(y=p + 8) == ALIGN and call(cols=p + 2) == ALIGN
    assert call(C=96) == UNSUPPORTED and call(C=32) == UNSUPPORTED
    assert call(form=2) == UNSUPPORTED and call(form=-1) == UNSUPPORTED and call(B=65536) == UNSUPPORTED
    # shared memory per pixel: 544 bytes (bf16 patches), 688 (split)
    assert call(H=4, W=107) == UNSUPPORTED and call(form=1, H=2, W=169) == UNSUPPORTED      # 428 / 338 pixels
    assert call(H=100, W=100) == UNSUPPORTED and call(H=1 << 16, W=1 << 16) == UNSUPPORTED
    assert call(x=p + 2, keep=0.0) == INVALID and call(x=p + 2, form=2) == ALIGN
    assert lib.mac_b200_launch_count() == before
    if not torch.cuda.is_available():
        for kw in (dict(H=7, W=61), dict(form=1, H=337, W=1), dict(keep=1.0, H=1, W=1), dict(C=2048, B=65535)):
            assert call(**kw) not in ERRORS, kw


# ------------------------------------------------------------------------------------------------ the stem
def _stem(prec, cin=128, cout=128):
    from mac_network_b200.stem import Stem, init_stem_params, stem_specs
    return Stem(_cpu_params(init_stem_params(stem_specs(cin, cout), seed=1)), relu="ELU", prec=prec, seed=11)


def _scalars(args):
    return tuple(a for a in args if isinstance(a, (int, float)))


FP32_OF = {"mac_ingest_nchw_f16": "mac_ingest_nchw", "mac_ingest_nchw_train_f16": "mac_ingest_nchw_train"}


@pytest.mark.parametrize("prec,train", [("fp32", False), ("bf16", False), ("bf16x3", False), ("fp8", False),
                                        ("fp32", True), ("bf16", True), ("bf16x3", True)])
def test_forward_nchw_f16_launches_what_fp32_launches_but_the_ingest(monkeypatch, prec, train):
    rec = _recorder(monkeypatch)
    st = _stem(prec)
    kw = dict(keep=0.82, step=5, save_for_backward=True) if train else {}
    st.forward_nchw(torch.zeros(2, 128, 5, 7), **kw)                   # the weight packs, built once
    runs = {}
    for dtype in (torch.float32, torch.float16):
        rec.log.clear()
        kb = st.forward_nchw(torch.zeros(2, 128, 5, 7, dtype=dtype), **kw)
        assert kb.shape == (2, 35, 128) and kb.dtype == torch.float32
        if train:
            runs[dtype] = (list(rec.log), [t.dtype for t in st._saved["xs"]], [t.shape for t in st._saved["xs"]])
        else:
            runs[dtype] = (list(rec.log), None, None)
    (log32, dt32, sh32), (log16, dt16, sh16) = runs[torch.float32], runs[torch.float16]
    assert dt16 == dt32 and sh16 == sh32                                # the saved layer inputs: fp32 NHWC either way
    names16 = [n for n, _ in log16]
    ingest = [n for n in names16 if n.startswith("mac_ingest")]
    assert ingest == ["mac_ingest_nchw_train_f16" if train and prec != "fp32" else "mac_ingest_nchw_f16"]
    assert [FP32_OF.get(n, n) for n in names16] == [n for n, _ in log32]
    for (n16, a16), (n32, a32) in zip(log16, log32):
        if n16 == "mac_ingest_nchw_f16":
            assert _scalars(a16) == _scalars(a32)[1:]                   # mac_ingest_nchw's x_bf16 = 0 dropped
        else:
            assert _scalars(a16) == _scalars(a32), n16


def test_forward_nchw_f16_backward_launches_what_fp32_launches(monkeypatch):
    rec = _recorder(monkeypatch)
    for prec in ("fp32", "bf16", "bf16x3"):
        st = _stem(prec)
        st.forward_nchw(torch.zeros(2, 128, 5, 7))                      # the weight packs, built once
        logs = []
        for dtype in (torch.float32, torch.float16):
            kb = st.forward_nchw(torch.zeros(2, 128, 5, 7, dtype=dtype), keep=0.82, step=5, save_for_backward=True)
            grads = {k: torch.zeros_like(v) for k, v in st.p.items()}
            rec.log.clear()
            dx = st.backward(torch.zeros_like(kb), grads, need_d_images=True)
            assert dx.dtype == torch.float32 and dx.shape == (2, 5, 7, 128)
            logs.append([(n, _scalars(a)) for n, a in rec.log])
        assert logs[0] == logs[1], prec


def test_forward_nchw_refusals_keep_their_rules(monkeypatch):
    rec = _recorder(monkeypatch)
    for bad in (torch.zeros(2, 128, 5, 7, dtype=torch.float64), torch.zeros(2, 5, 7, 128, dtype=torch.float16).permute(0, 3, 1, 2)):
        with pytest.raises(ValueError):
            _stem("bf16").forward_nchw(bad)
    with pytest.raises(NotImplementedError):                    # the e4m3 stem is inference only, whatever the images
        _stem("fp8").forward_nchw(torch.zeros(2, 128, 5, 7, dtype=torch.float16), keep=0.82)
    with pytest.raises(NotImplementedError, match="multiple of 64"):
        _stem("fp32", cin=96).forward_nchw(torch.zeros(2, 96, 5, 7, dtype=torch.float16))
    with pytest.raises(ValueError, match="bf16 images"):        # bf16 images keep their own rules
        _stem("bf16").forward_nchw(torch.zeros(2, 128, 5, 7, dtype=torch.bfloat16), keep=0.82)
    assert rec.log == []


def test_trainer_takes_fp16_nchw_images(monkeypatch):
    mock, net, _ = TP._net(monkeypatch, stem_prec="bf16")
    t = net.trainer
    B, S, H, W, C = TP.B, TP.S, TP.H, TP.W, TP.C
    data = {"questions": torch.ones(B, S, dtype=torch.int32), "questionLengths": torch.full((B,), S, dtype=torch.int32),
            "answers": torch.zeros(B, dtype=torch.int32)}
    mock.calls.clear()
    with pytest.raises(ValueError):
        t.train_step_full((B, S), dict(data, images_nchw=torch.zeros(B, C, H, W, dtype=torch.bfloat16)), global_batch=B)
    assert mock.calls == [] and t.step_id == 0
    t.train_step_full((B, S), dict(data, images_nchw=torch.zeros(B, C, H, W, dtype=torch.float16)), global_batch=B)
    ingest = [c for c in mock.calls if c.startswith("mac_ingest")]
    assert ingest == ["mac_ingest_nchw_train_f16"] and t.step_id == 1
    mock.calls.clear()
    t.train_step_full((B, S), dict(data, images_nchw=torch.zeros(2, C, H, W, dtype=torch.float16),
                                   imageIndex=torch.tensor([0, 1, 1, 0], dtype=torch.int32)), global_batch=B)
    assert [c for c in mock.calls if c.startswith("mac_ingest")] == ["mac_ingest_nchw_train_f16"]
    assert mock.calls.count("mac_kb_gather") == 1 and mock.calls.count("mac_kb_gather_bwd") == 1


# ------------------------------------------------------------------------------------------------ ModelPipeline
B, S, H, W, C = MP.B, MP.S, MP.H, MP.W, MP.C
BAD_DTYPES = (torch.bfloat16, torch.float64, torch.int32, "float16", np.float16, None)


def _half(batch):
    return dict(batch, images=batch["images"].astype(np.float16))


def test_model_pipeline_constructor_refusals(monkeypatch):
    from mac_network_b200.serving import ModelPipeline
    mock, n, net = MP._model(monkeypatch)
    del mock.calls[:]
    for dt in BAD_DTYPES:
        with pytest.raises(ValueError, match="image_dtype"):
            ModelPipeline(net, (B, S, H, W), slots=1, image_dtype=dt)
    with pytest.raises(ValueError, match="host_cast"):
        ModelPipeline(net, (B, S, H, W), slots=1, host_cast=True, image_dtype=torch.float16)
    with pytest.raises(ValueError, match="host_cast"):
        ModelPipeline(net, (B, S, H, W), slots=1, images=2, cache=B, host_cast=True, image_dtype=torch.float16)
    assert mock.calls == [] and n.streams == 0


@pytest.mark.parametrize("prec,images", [("bf16", None), ("bf16", 2), ("fp32", None)])
def test_model_pipeline_f16_stages_and_ingests_fp16(monkeypatch, prec, images):
    from mac_network_b200.serving import ModelPipeline
    mock, n, net = MP._model(monkeypatch, prec=prec)
    plain = ModelPipeline(net, (B, S, H, W), slots=2, host_cast=False, images=images)
    del mock.calls[:]
    pipe = ModelPipeline(net, (B, S, H, W), slots=2, images=images, image_dtype=torch.float16)
    assert not pipe.host_cast and pipe._ring is None and pipe.image_dtype == torch.float16
    k = B if images is None else images
    for s in pipe.slots:
        assert s.x["images"].dtype == torch.float16 and s.x["images"].shape == (k, C, H, W)
    assert mock.calls.count("mac_ingest_nchw_f16") == 4 and "mac_ingest_nchw" not in mock.calls     # eager + captured, two slots
    assert pipe.h2d_bytes - (B * S * 4 + B * 4 + (0 if images is None else B * 4)) == k * C * H * W * 2
    assert plain.h2d_bytes - pipe.h2d_bytes == k * C * H * W * 2          # half the fp32 image bytes
    b = _half(MP._batch(0))
    if images is not None:
        b = dict(b, images=b["images"][:2], imageIndex=np.array([0, 1, 1, 0], np.int32))
    del mock.calls[:]
    t = pipe.submit(b)
    assert mock.calls == [] and n.replays >= 1
    slot = pipe.slots[t % 2]
    assert torch.equal(slot.x["images"][:b["images"].shape[0]], torch.from_numpy(b["images"]))
    # the fp32 pipeline still takes an fp16 batch and widens it on the host
    plain.submit(b)
    assert plain.slots[0].x["images"].dtype == torch.float32
    assert torch.equal(plain.slots[0].x["images"][:b["images"].shape[0]], torch.from_numpy(b["images"]).float())


def test_model_pipeline_f16_refuses_other_batches_before_staging(monkeypatch):
    from mac_network_b200.serving import ModelPipeline
    mock, n, net = MP._model(monkeypatch)
    pipe = ModelPipeline(net, (B, S, H, W), slots=1, image_dtype=torch.float16)
    before = pipe.slots[0].x["images"].clone()
    del mock.calls[:]
    good = MP._batch(0)
    for img in (good["images"], good["images"].astype(np.float64), torch.from_numpy(good["images"]).bfloat16(),
                good["images"].astype(np.int16)):
        with pytest.raises(ValueError, match="fp16"):
            pipe.submit(dict(good, images=img))
    with pytest.raises(ValueError):
        pipe.submit(dict(_half(good), images=_half(good)["images"][:, :64]))
    assert mock.calls == [] and n.replays == 0 and pipe._next == 0 and torch.equal(pipe.slots[0].x["images"], before)


def test_model_pipeline_f16_cache(monkeypatch):
    from mac_network_b200.serving import ModelPipeline
    mock, n, net = KB._model(monkeypatch)
    pipe = ModelPipeline(net, (B, S, H, W), slots=2, images=2, cache=6, image_dtype=torch.float16)
    assert pipe.slots[0].x["images"].dtype == torch.float16 and pipe.h2d_bytes == B * S * 4 + B * 4 + B * 4
    del mock.calls[:]
    pipe.slots[0]._stem_pass()
    assert mock.calls[0] == "mac_ingest_nchw_f16" and mock.calls[-1] == "mac_kb_pool_insert"
    load = KB.Loader(dtype=np.float16)
    pipe.submit(KB._batch([7, 3, 7, 9], load))
    assert load.calls == [[7, 3, 9]]
    assert pipe.cache_stats()["image_bytes"] == 3 * C * H * W * 2
    assert torch.equal(pipe.slots[0].x["images"][0], torch.full((C, H, W), 9.0, dtype=torch.float16))
    snap = lambda: (list(pipe._cache.rows.items()), list(pipe._cache.key), [list(r) for r in pipe._cache.reader],
                    pipe.cache_stats(), pipe._next, n.replays, pipe.slots[1].x["images"].clone())
    before = snap()
    for dt in (np.float32, np.float64):                         # never rounded to fp16 silently
        with pytest.raises(ValueError, match="fp16"):
            pipe.submit(KB._batch([1, 2, 7, 1], KB.Loader(dtype=dt)))
        s = snap()
        assert s[:6] == before[:6] and torch.equal(s[6], before[6])
    with pytest.raises(ValueError):
        pipe.submit(KB._batch([1, 2, 7, 1], lambda ids: torch.zeros(len(ids), C, H, W, dtype=torch.bfloat16)))
    assert snap()[:6] == before[:6]
    pipe.submit(KB._batch([1, 2, 7, 1], load))
    assert pipe.cache_stats()["misses"] == 5 and pipe.cache_stats()["image_bytes"] == 5 * C * H * W * 2


# ------------------------------------------------------------------------------------------------ TrainPipeline
def test_train_pipeline_f16_stages_and_refuses(monkeypatch):
    from mac_network_b200.serving import TrainPipeline
    mock, net, log = TP._net(monkeypatch, stem_prec="bf16x3")
    mock.calls.clear()
    for dt in BAD_DTYPES:
        with pytest.raises(ValueError, match="image_dtype"):
            TrainPipeline(net, (TP.B, TP.S, TP.H, TP.W), image_dtype=dt)
    assert mock.calls == []
    pipe = TrainPipeline(net, (TP.B, TP.S, TP.H, TP.W), depth=2, stage_threads=2, image_dtype=torch.float16)
    for s in pipe.slots:
        assert s.host["images"].dtype == torch.float16 and s.dev["images"].dtype == torch.float16
        assert s.host["images"].numel() == TP.B * TP.C * TP.H * TP.W
    good = TP._batch(0)
    for img in (good["images"], good["images"].astype(np.float64), torch.from_numpy(good["images"]).bfloat16()):
        with pytest.raises(ValueError, match="fp16"):
            pipe.submit(dict(good, images=img))
    assert mock.calls == [] and pipe._next == 0 and not [e for e in log if e[0] in ("wait", "sync")]
    b = dict(good, images=good["images"].astype(np.float16))
    pipe.submit(b)
    assert [c for c in mock.calls if c.startswith("mac_ingest")] == ["mac_ingest_nchw_train_f16"]
    assert torch.equal(pipe.slots[0].host["images"], torch.from_numpy(b["images"]).reshape(-1))
    assert torch.equal(pipe.slots[0].dev["images"], torch.from_numpy(b["images"]).reshape(-1))
    assert net.trainer.step_id == 1


def test_train_pipeline_f16_with_shared_images(monkeypatch):
    from mac_network_b200.serving import TrainPipeline
    mock, net, log = TP._net(monkeypatch, stem_prec="bf16")
    pipe = TrainPipeline(net, (TP.B, TP.S, TP.H, TP.W), depth=1, stage_threads=1, images=3, image_dtype=torch.float16)
    assert pipe.slots[0].host["images"].numel() == 3 * TP.C * TP.H * TP.W
    good = TP._batch(1)
    b = dict(good, images=good["images"][:2].astype(np.float16), imageIndex=np.array([1, 0, 0, 1], np.int32))
    with pytest.raises(ValueError, match="fp16"):
        pipe.submit(dict(b, images=good["images"][:2]))
    mock.calls.clear()
    pipe.submit(b)
    assert [c for c in mock.calls if c.startswith("mac_ingest")] == ["mac_ingest_nchw_train_f16"]
    assert mock.calls.count("mac_kb_gather") == 1 and mock.calls.count("mac_kb_gather_bwd") == 1
    n = 2 * TP.C * TP.H * TP.W
    assert torch.equal(pipe.slots[0].dev["images"][:n], torch.from_numpy(b["images"]).reshape(-1))
    # the default pipeline widens an fp16 batch on the host, as before
    plain = TrainPipeline(net, (TP.B, TP.S, TP.H, TP.W), depth=1, stage_threads=1, images=3)
    mock.calls.clear()
    plain.submit(b)
    assert plain.slots[0].dev["images"].dtype == torch.float32
    assert [c for c in mock.calls if c.startswith("mac_ingest")] == ["mac_ingest_nchw_train"]
