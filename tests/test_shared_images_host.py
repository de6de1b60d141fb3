"""CPU side of several questions per image (mac_kb_gather, MACCell(kbIndex=), ModelPipeline(images=U), runBatch by
imageIds): the entry point's declaration and its refusals (which return before any CUDA call), the cell's refusals, and
the host logic of the pipeline and of runBatch over the dry-run library (tests/_mocklib.py)."""
import ctypes

import numpy as np
import pytest
import torch

from mac_network_b200 import _lib as L_
from tests import _mocklib

INVALID, ALIGN, UNSUPPORTED = -1, -2, -3


# ------------------------------------------------------------------------------------------------ the C boundary
def test_kb_gather_is_declared_bound_and_exported():
    from tests.test_abi import _declared
    lib = L_.load()
    assert "mac_kb_gather" in _declared() and "mac_kb_gather" in L_.PROTOTYPES and hasattr(lib, "mac_kb_gather")
    assert lib.mac_b200_abi_version() == 1


def test_kb_gather_refuses_before_any_cuda_call():
    lib = L_.load()
    buf = (ctypes.c_float * 4096)()
    p = (ctypes.addressof(buf) + 15) & ~15                  # 16-byte aligned fake "device" pointer, never dereferenced
    g = lambda kb, idx, out, bf, B, U, N, d: lib.mac_kb_gather(kb, idx, out, bf, B, U, N, d, None)
    assert g(None, p, p, 0, 2, 1, 4, 8) == INVALID and g(p, None, p, 0, 2, 1, 4, 8) == INVALID
    assert g(p, p, None, 1, 2, 1, 4, 8) == INVALID
    for B, U, N, d in ((0, 1, 4, 8), (2, 0, 4, 8), (2, 1, 0, 8), (2, 1, 4, 0), (-1, 1, 4, 8), (2, 1, 4, -8)):
        assert g(p, p, p, 0, B, U, N, d) == INVALID, (B, U, N, d)
    assert g(p, p, p, 2, 2, 1, 4, 8) == UNSUPPORTED and g(p, p, p, -1, 2, 1, 4, 8) == UNSUPPORTED
    assert g(p, p, p, 0, 2, 1, 4, 12) == UNSUPPORTED and g(p, p, p, 1, 2, 1, 4, 4) == UNSUPPORTED
    assert g(p, p, p, 0, 2, 1, 1 << 20, 1 << 14) == UNSUPPORTED          # a run of 2^31 vectors
    assert g(p + 4, p, p, 0, 2, 1, 4, 8) == ALIGN and g(p, p + 8, p, 0, 2, 1, 4, 8) == ALIGN
    assert g(p, p, p + 2, 1, 2, 1, 4, 8) == ALIGN
    # the refusal classes in their order: INVALID before UNSUPPORTED before ALIGN
    assert g(p + 4, p, p, 2, 0, 1, 4, 8) == INVALID and g(p + 4, p, p, 2, 2, 1, 4, 8) == UNSUPPORTED


# ------------------------------------------------------------------------------------------------ the cell
def _cell_inputs(B, U, N=4, d=128, S=3):
    x = {"vq": torch.zeros(B, d), "w": torch.zeros(B, S, d), "len": torch.full((B,), S, dtype=torch.int32),
         "kb": torch.zeros(U, N, d)}
    return x


ARGS = ["--memoryVariationalDropout", "--relu=ELU", "--controlContextual", "--readProjInputs", "--readMemConcatKB",
        "--readMemConcatProj", "--readMemProj", "--readCtrl", "--writeMemProj", "--initCtrl=Q", "--controlInputUnshared"]
P2 = {"p2_unshared": ARGS + ["--unsharedCells", "1", "--initMem=ZERO"],              # the fused read unit, per-step weights
      "p2_read_bl": ARGS + ["--readMemAttType=BL", "--readCtrlAttType=BL", "--readProjShared", "--readMemAct=TANH",
                            "--readCtrlAct=NON"]}                                    # the composed read unit


def config(variant, **kw):
    """A shipped flag file (MACConfig.args) or one of the P2 flag sets above."""
    from mac_network_b200.config import MACConfig
    if variant in P2:
        return MACConfig.from_flags(P2[variant], **kw)
    return MACConfig.args(variant, **kw)


def _cfg(d=128, L=2):
    return config("args", netLength=L, memDim=d, ctrlDim=d, attDim=d)


def _cell(x, B, prec="bf16", cfg=None, kbIndex=None, drop=(1.0, 1.0, 1.0), **kw):
    from mac_network_b200.mac_cell import MACCell, MACParams
    cfg = cfg or _cfg()
    params = MACParams(cfg, cfg.netLength, device="cpu")
    return MACCell(x["vq"], x["w"], x["w"], x["len"], x["kb"], *drop, B, False, config=cfg, params=params, prec=prec,
                   kbIndex=kbIndex, **kw)


@pytest.fixture
def mock(monkeypatch):
    m = _mocklib.install(monkeypatch)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True), raising=False)
    return m


def test_cell_refusals(mock):
    B, U = 6, 2
    x = _cell_inputs(B, U)
    idx = torch.zeros(B, dtype=torch.int32)
    with pytest.raises(NotImplementedError):
        _cell(x, B, prec="fp32", kbIndex=idx, save_for_backward=True)
    for drop in ((0.9, 1.0, 1.0), (1.0, 0.85, 1.0), (1.0, 1.0, 0.9)):
        with pytest.raises(NotImplementedError):
            _cell(x, B, kbIndex=idx, drop=drop)
    with pytest.raises(NotImplementedError):
        _cell(dict(x, kb=x["kb"].to(torch.bfloat16)), B, kbIndex=idx)
    for bad in (idx.long(), idx[:B - 1], torch.zeros(B + 1, dtype=torch.int32), torch.zeros(B, 1, dtype=torch.int32),
                torch.zeros(2 * B, dtype=torch.int32)[::2], idx.float(), [0] * B):
        with pytest.raises(ValueError):
            _cell(x, B, kbIndex=bad)
    assert mock.calls.count("mac_kb_gather") == 0
    # rebind: the same index rules, and an index exactly when the cell was built with one
    cell = _cell(x, B, kbIndex=idx)
    with pytest.raises(ValueError):
        cell.rebind(x["vq"], x["w"], x["w"], x["kb"])
    with pytest.raises(ValueError):
        cell.rebind(x["vq"], x["w"], x["w"], x["kb"], kbIndex=idx[:B - 1])
    with pytest.raises(ValueError):
        cell.rebind(x["vq"], x["w"], x["w"], torch.zeros(U + 1, 4, 128), kbIndex=idx)
    plain = _cell(dict(x, kb=torch.zeros(B, 4, 128)), B)
    with pytest.raises(ValueError):
        plain.rebind(x["vq"], x["w"], x["w"], torch.zeros(B, 4, 128), kbIndex=idx)
    idx2 = torch.ones(B, dtype=torch.int32)
    cell.rebind(x["vq"], x["w"], x["w"], torch.zeros(U, 4, 128), kbIndex=idx2)
    assert cell.kbIndex is idx2


@pytest.mark.parametrize("prec,variant,bf16_out", [("bf16", "args", True), ("fp8", "args", True), ("fp32", "args", False),
                                                   ("tc32", "args", False), ("bf16", "p2_unshared", False),
                                                   ("bf16", "p2_read_bl", False)])
def test_cell_gathers_into_the_operand_its_form_reads(mock, prec, variant, bf16_out):
    from mac_network_b200.mac_cell import mac_network
    B, U, d = 6, 2, 512 if prec == "fp8" else 128
    N = 4
    x = _cell_inputs(B, U, N=N, d=d)
    cfg = config(variant, netLength=2, memDim=d, ctrlDim=d, attDim=d)
    cell = _cell(x, B, prec=prec, cfg=cfg, kbIndex=torch.zeros(B, dtype=torch.int32))
    assert cell.B == B and cell.U == U and cell.N == N
    del mock.calls[:]
    mac_network(cell, 2)
    assert mock.calls.count("mac_kb_gather") == 1 and mock.calls[0] == "mac_kb_gather"
    assert (cell._kb_rows is None) == bf16_out
    if bf16_out:                  # the gather writes the bf16 operand: no cast launch, no fp32 buffer
        assert "mac_cast_bf16" not in mock.calls
        assert cell._kb_q is cell.kb_bf16 and cell.kb_bf16.shape == (B, N, d) and cell.kb_bf16.dtype == torch.bfloat16
    else:
        assert cell._kb_q is cell._kb_rows and cell._kb_rows.shape == (B, N, d) and cell._kb_rows.dtype == torch.float32
        assert mock.calls.count("mac_cast_bf16") == (1 if prec == "bf16" and variant == "p2_unshared" else 0)
    # without kbIndex the same forward makes no gather
    plain = _cell(dict(x, kb=torch.zeros(B, N, d)), B, prec=prec, cfg=cfg)
    del mock.calls[:]
    mac_network(plain, 2)
    assert "mac_kb_gather" not in mock.calls and plain._kb_q is plain.knowledgeBase


# ------------------------------------------------------------------------------------------------ runBatch
def test_shared_images_keeps_first_occurrences():
    from mac_network_b200.model import MACnet
    assert MACnet.shared_images({"images": None}) is None
    assert MACnet.shared_images({"images": None, "imageIds": [3, 1, 2]}) is None            # all distinct
    rows, inv = MACnet.shared_images({"images": None, "imageIds": ["b", "a", "b", "c", "a", "a"]})
    assert rows.tolist() == [1, 0, 3] and inv.tolist() == [1, 0, 1, 2, 0, 0] and inv.dtype == np.int32
    ids = np.array([7, 7, 2, 9, 2, 7])
    rows, inv = MACnet.shared_images({"imageIds": ids})
    assert np.array_equal(ids[rows][inv], ids) and all(ids[r] not in ids[:r] for r in rows)


def _model(monkeypatch, prec="bf16", d=128, **kw):
    from tests import test_model_pipeline_host as H
    return H._model(monkeypatch, prec=prec, d=d, **kw)


def test_run_batch_copies_only_the_first_rows(monkeypatch):
    from tests.test_model_pipeline_host import B, C, H, W, S
    mock, n, net = _model(monkeypatch)
    seen = {}
    orig = net._to_device

    def spy(data, images, rows=None):
        dev = orig(data, images, rows)
        seen["rows"], seen["images"] = rows, dev["images"]
        return dev
    net._to_device = spy
    rng = np.random.RandomState(0)
    imgs = rng.standard_normal((B, C, H, W)).astype(np.float32)
    data = {"questions": rng.randint(1, 9, size=(B, S)).astype(np.int32), "questionLengths": np.full(B, S, np.int32),
            "answers": np.zeros(B, np.int32)}
    ids = [5, 3, 5, 3]
    del mock.calls[:]
    net.runBatch(None, data, {"images": imgs, "imageIds": ids}, train=False)
    assert seen["rows"].tolist() == [1, 0]
    assert np.array_equal(seen["images"].numpy(), imgs[[1, 0]].transpose(0, 2, 3, 1))
    assert net.macCell.kbIndex.tolist() == [1, 0, 1, 0] and net.macCell.U == 2 and net.macCell.B == B
    assert mock.calls.count("mac_kb_gather") == 1
    # all distinct, or no ids: today's path, no gather
    for imgs_dict in ({"images": imgs, "imageIds": [1, 2, 3, 4]}, {"images": imgs}):
        del mock.calls[:]
        net.runBatch(None, data, imgs_dict, train=False)
        assert seen["rows"] is None and seen["images"].shape[0] == B and net.macCell.kbIndex is None
        assert "mac_kb_gather" not in mock.calls


# ------------------------------------------------------------------------------------------------ the pipeline
def _batch(k, index, seed=0):
    from tests.test_model_pipeline_host import B, C, H, W, S, V
    rng = np.random.RandomState(seed)
    return {"questions": rng.randint(1, V + 1, size=(B, S)).astype(np.int32), "questionLengths": np.full(B, S, np.int32),
            "images": rng.standard_normal((k, C, H, W)).astype(np.float32), "imageIndex": np.asarray(index, np.int32)}


@pytest.mark.parametrize("host_cast", [False, True])
def test_pipeline_sizes_from_u_and_refuses_bad_batches(monkeypatch, host_cast):
    from mac_network_b200.serving import ModelPipeline
    from tests.test_model_pipeline_host import B, C, H, W, S
    U = 3
    mock, n, net = _model(monkeypatch)
    for bad in (0, B + 1, 2.0):
        with pytest.raises(ValueError):
            ModelPipeline(net, (B, S, H, W), slots=1, images=bad)
    pipe = ModelPipeline(net, (B, S, H, W), slots=2, images=U, host_cast=host_cast, stage_ring=2, cast_threads=2)
    for s in pipe.slots:
        assert s.x["images"].shape == (U, C, H, W) and s.x["imageIndex"].shape == (B,)
        assert s.x["imageIndex"].dtype == torch.int32 and s.cell.kbIndex is s.x["imageIndex"]
    if host_cast:
        assert all(st.numel() == U * C * H * W for st in pipe._ring.stages)
    assert pipe.h2d_bytes == U * C * H * W * (2 if host_cast else 4) + B * S * 4 + B * 4 + B * 4
    # eager pass and capture per slot: ingest over U images, one gather each
    assert mock.calls.count("mac_kb_gather") == 4 and mock.calls.count("mac_ingest_nchw") == 4
    del mock.calls[:]
    good = _batch(2, [0, 1, 1, 0])
    bads = [{k: v for k, v in good.items() if k != "imageIndex"},           # no index
            dict(_batch(U + 1, [0, 1, 2, 3])),                              # k > U
            dict(good, imageIndex=np.array([0, 1, 2, 0], np.int32)),        # index == k
            dict(good, imageIndex=np.array([0, -1, 1, 0], np.int32)),       # negative
            dict(good, imageIndex=np.array([0, 1, 1], np.int32)),           # wrong length
            dict(good, imageIndex=np.array([0.0, 1, 1, 0])),                # not integers
            dict(good, images=good["images"][:0])]                          # no image
    for bad in bads:
        with pytest.raises(ValueError):
            pipe.submit(bad)
        if host_cast:               # the next batch is read (its cast started) only with the host cast
            with pytest.raises(ValueError):
                pipe.submit(good, next_batch=bad)
    assert mock.calls == [] and n.replays == 0 and pipe._next == 0
    # valid batches with any k <= U and any index pattern: replays only, no library call, no capture
    caps = n.captures
    for i, (k, index) in enumerate(((1, [0, 0, 0, 0]), (2, [1, 0, 1, 1]), (3, [2, 2, 1, 0]))):
        pipe.submit(_batch(k, index, seed=i))
    assert n.replays == 3 and n.captures == caps and mock.calls.count("mac_host_cast_bf16_begin") == (3 if host_cast else 0)
    assert [c for c in mock.calls if not c.startswith("mac_host_cast")] == []
    # an index without images=
    plain = ModelPipeline(net, (B, S, H, W), slots=1, host_cast=False)
    with pytest.raises(ValueError):
        plain.submit(dict(_batch(B, [0, 1, 2, 3])))
    assert plain._next == 0


def test_pipeline_copies_k_images_and_the_index(monkeypatch):
    from mac_network_b200 import serving
    from tests.test_model_pipeline_host import B, C, H, W, S
    mock, n, net = _model(monkeypatch)
    pipe = serving.ModelPipeline(net, (B, S, H, W), slots=1, images=3, host_cast=False)
    slot = pipe.slots[0]
    slot.x["images"].fill_(-5.0)
    b = _batch(2, [1, 0, 1, 1])
    pipe.submit(b)
    got = slot.x["images"]
    assert torch.equal(got[:2], torch.from_numpy(b["images"])) and bool((got[2] == -5.0).all())
    assert slot.x["imageIndex"].tolist() == [1, 0, 1, 1]
