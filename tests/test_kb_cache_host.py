"""CPU side of the device-resident knowledge-base cache (mac_kb_pool_insert, mac_kb_gather_bf16, ModelPipeline(cache=C)):
the entry points' declarations and refusals (which return before any CUDA call), and the pipeline's host logic over the
dry-run library (tests/_mocklib.py) with the CUDA stream / event / graph objects replaced by counters: which images the
loader is asked for, which rows are evicted, which launches and replays a batch makes, the pool's dtype per cell form, the
stream waits between slots, and what a bad batch, a weight update or clear_cache() does to the cache."""
import ctypes

import numpy as np
import pytest
import torch

from mac_network_b200 import _lib as L_
from tests import test_model_pipeline_host as MP
from tests.test_shared_images_host import config

INVALID, ALIGN, UNSUPPORTED = -1, -2, -3
B, S, H, W, C = MP.B, MP.S, MP.H, MP.W, MP.C


# ------------------------------------------------------------------------------------------------ the C boundary
def test_new_entry_points_are_declared_bound_and_exported():
    from tests.test_abi import _declared
    lib = L_.load()
    c = ctypes
    assert L_.PROTOTYPES["mac_kb_pool_insert"] == (c.c_int, [c.c_void_p] * 3 + [c.c_int] * 5 + [c.c_void_p])
    assert L_.PROTOTYPES["mac_kb_gather_bf16"] == (c.c_int, [c.c_void_p] * 3 + [c.c_int] * 4 + [c.c_void_p])
    for name in ("mac_kb_pool_insert", "mac_kb_gather_bf16"):
        assert name in _declared() and hasattr(lib, name)
    assert lib.mac_b200_abi_version() == 1


def _fake_pointer():
    buf = (ctypes.c_float * 4096)()
    return buf, (ctypes.addressof(buf) + 15) & ~15      # 16-byte aligned fake "device" pointer, never dereferenced


def test_pool_insert_refuses_before_any_cuda_call():
    lib = L_.load()
    buf, p = _fake_pointer()
    f = lambda kb, sl, pool, bf, U, cap, N, d: lib.mac_kb_pool_insert(kb, sl, pool, bf, U, cap, N, d, None)
    assert f(None, p, p, 0, 2, 4, 4, 8) == INVALID and f(p, None, p, 0, 2, 4, 4, 8) == INVALID
    assert f(p, p, None, 1, 2, 4, 4, 8) == INVALID
    for U, cap, N, d in ((0, 4, 4, 8), (2, 0, 4, 8), (2, 4, 0, 8), (2, 4, 4, 0), (-1, 4, 4, 8), (2, -4, 4, 8)):
        assert f(p, p, p, 0, U, cap, N, d) == INVALID, (U, cap, N, d)
    assert f(p, p, p, 2, 2, 4, 4, 8) == UNSUPPORTED and f(p, p, p, -1, 2, 4, 4, 8) == UNSUPPORTED
    assert f(p, p, p, 0, 2, 4, 4, 12) == UNSUPPORTED and f(p, p, p, 1, 2, 4, 4, 4) == UNSUPPORTED
    assert f(p, p, p, 0, 2, 4, 1 << 20, 1 << 14) == UNSUPPORTED          # a run of 2^31 vectors
    assert f(p + 4, p, p, 0, 2, 4, 4, 8) == ALIGN and f(p, p + 8, p, 0, 2, 4, 4, 8) == ALIGN
    assert f(p, p, p + 2, 1, 2, 4, 4, 8) == ALIGN
    # the refusal classes in their order: INVALID before UNSUPPORTED before ALIGN
    assert f(p + 4, p, p, 2, 0, 4, 4, 8) == INVALID and f(p + 4, p, p, 2, 2, 4, 4, 8) == UNSUPPORTED


def test_gather_bf16_refuses_before_any_cuda_call():
    lib = L_.load()
    buf, p = _fake_pointer()
    g = lambda kb, idx, out, B_, U, N, d: lib.mac_kb_gather_bf16(kb, idx, out, B_, U, N, d, None)
    assert g(None, p, p, 2, 1, 4, 8) == INVALID and g(p, None, p, 2, 1, 4, 8) == INVALID and g(p, p, None, 2, 1, 4, 8) == INVALID
    for B_, U, N, d in ((0, 1, 4, 8), (2, 0, 4, 8), (2, 1, 0, 8), (2, 1, 4, 0), (-1, 1, 4, 8)):
        assert g(p, p, p, B_, U, N, d) == INVALID, (B_, U, N, d)
    assert g(p, p, p, 2, 1, 4, 12) == UNSUPPORTED and g(p, p, p, 2, 1, 1 << 20, 1 << 14) == UNSUPPORTED
    assert g(p + 2, p, p, 2, 1, 4, 8) == ALIGN and g(p, p + 4, p, 2, 1, 4, 8) == ALIGN and g(p, p, p + 8, 2, 1, 4, 8) == ALIGN
    assert g(p + 2, p, p, 0, 1, 4, 8) == INVALID and g(p + 2, p, p, 2, 1, 4, 4) == UNSUPPORTED


# ------------------------------------------------------------------------------------------------ the bookkeeping
def test_lru_victims_are_never_rows_the_batch_reads():
    from mac_network_b200.serving import _KBCache
    c = _KBCache(4, 3)
    p = c.plan([10, 11, 12, 13])
    assert p.hits == [] and p.miss == [10, 11, 12, 13] and p.rows == [0, 1, 2, 3] and p.victims == []
    c.commit(p, 0)
    # 10 and 11 are read again, then 13: least recently used is now 12, then 10, 11, 13
    c.commit(c.plan([10, 11]), 1)
    c.commit(c.plan([13]), 2)
    p = c.plan([12, 20, 21])            # 12 is read: the victims are 10 and 11, not 12 although it is the oldest
    assert p.hits == [2] and p.miss == [20, 21] and p.victims == [0, 1] and p.rows == [0, 1]
    rng = np.random.RandomState(0)
    for t in range(3, 200):
        keys = list(dict.fromkeys(rng.randint(0, 9, size=4).tolist()))
        p = c.plan(keys)
        assert not set(p.victims) & set(p.hits) and len(p.rows) == len(p.miss) and len(set(p.rows)) == len(p.rows)
        c.commit(p, t)
        assert all(c.key[c.rows[k]] == k for k in keys) and all(c.reader[c.rows[k]][t % 3][0] == t for k in keys)
        assert len(c.rows) + len(c.free) == 4 and sorted(list(c.rows.values()) + c.free) == [0, 1, 2, 3]
    st = c.stats
    assert st["hits"] + st["misses"] > 0 and st["evictions"] == st["misses"] - 4


# ------------------------------------------------------------------------------------------------ the pipeline
def _model(monkeypatch, variant="args", prec="bf16", d=128, **kw):
    """MP._model with another flag set, a patched stream handle in serving, and streams that record their waits."""
    mock, n, net = MP._model(monkeypatch, prec=prec, d=d, **kw)
    from mac_network_b200 import serving
    from mac_network_b200.model import MACnet
    monkeypatch.setattr(serving, "stream_ptr", lambda: None)
    n.waits = []
    monkeypatch.setattr(torch.cuda.Stream, "wait_event", lambda self, ev: n.waits.append((self, ev)), raising=False)
    if variant != "args":
        cfg = config(variant, netLength=MP.L, memDim=d, ctrlDim=d, attDim=d)
        net = MACnet(cfg, MP.L, MP.V, MP.A, wrd_emb_dim=MP.E, image_in_dim=C, classifier_dims=(16,), prec=prec, device="cpu",
                     **kw)
    return mock, n, net


class Loader(object):
    def __init__(self, dtype=np.float32, shape=None):
        self.calls, self.dtype, self.shape = [], dtype, shape

    def __call__(self, ids):
        assert isinstance(ids, np.ndarray) and ids.dtype == np.int64 and ids.ndim == 1
        self.calls.append(ids.tolist())
        shp = self.shape or (len(ids), C, H, W)
        return np.stack([np.full(shp[1:], float(i), dtype=self.dtype) for i in ids]) if shp[0] == len(ids) else \
            np.zeros(shp, self.dtype)


def _batch(ids, load, seed=0):
    rng = np.random.RandomState(seed)
    return {"questions": rng.randint(1, MP.V + 1, size=(B, S)).astype(np.int32), "questionLengths": np.full(B, S, np.int32),
            "imageIds": np.asarray(ids), "images": load}


def test_constructor_refusals(monkeypatch):
    from mac_network_b200.serving import ModelPipeline
    mock, n, net = _model(monkeypatch)
    del mock.calls[:]
    for kw in (dict(cache=B), dict(images=2, cache=B - 1), dict(images=2, cache=0), dict(images=2, cache=float(B)),
               dict(images=2, cache=True), dict(images=2, cache="8")):
        with pytest.raises(ValueError):
            ModelPipeline(net, (B, S, H, W), slots=1, **kw)
    assert mock.calls == [] and n.streams == 0
    pipe = ModelPipeline(net, (B, S, H, W), slots=1, images=2, cache=B, host_cast=True)
    assert not pipe.host_cast and pipe._ring is None            # host_cast is off with a cache
    plain = ModelPipeline(net, (B, S, H, W), slots=1, host_cast=False)
    for f in (plain.cache_stats, plain.clear_cache):
        with pytest.raises(ValueError):
            f()


@pytest.mark.parametrize("use_graph", [True, False])
def test_loader_gets_the_misses_and_an_all_hit_batch_runs_no_stem(monkeypatch, use_graph):
    from mac_network_b200.serving import ModelPipeline
    U = 2
    mock, n, net = _model(monkeypatch)
    pipe = ModelPipeline(net, (B, S, H, W), slots=2, images=U, cache=6, host_cast=False, use_graph=use_graph)
    slot0 = pipe.slots[0]
    assert slot0.x["insertSlot"].shape == (U,) and slot0.x["kbSlot"].shape == (B,) and slot0.x["images"].shape == (U, C, H, W)
    assert pipe.pool.shape == (6, H * W, 128) and pipe.h2d_bytes == B * S * 4 + B * 4 + B * 4
    if use_graph:
        assert slot0.stem_graph is not None and slot0.graph is not None and n.captures == 4
    # the launches of one stem pass and of one cell pass, eagerly
    del mock.calls[:]
    slot0._stem_pass()
    stem_calls = list(mock.calls)
    del mock.calls[:]
    slot0._forward()
    cell_calls = list(mock.calls)
    assert stem_calls[0] == "mac_ingest_nchw" and stem_calls[-1] == "mac_kb_pool_insert"
    assert "mac_ingest_nchw" not in cell_calls and "mac_kb_pool_insert" not in cell_calls
    assert cell_calls.count("mac_kb_gather_bf16") == 1 and "mac_kb_gather" not in cell_calls

    def run(ids, passes):
        load = Loader()
        del mock.calls[:]
        r0 = n.replays
        pipe.submit(_batch(ids, load))
        if use_graph:
            assert mock.calls == [] and n.replays - r0 == passes + 1
        else:
            assert mock.calls == stem_calls * passes + cell_calls
        return load.calls
    # three misses in first-occurrence order -> two stem passes of U = 2
    assert run([7, 3, 7, 9], 2) == [[7, 3, 9]]
    assert slot0.x["kbSlot"].tolist() == [0, 1, 0, 2]
    assert slot0.x["insertSlot"].tolist() == [2, -1]                  # the second pass: one image, a padding row
    assert torch.equal(slot0.x["images"][0], torch.full((C, H, W), 9.0))
    assert run([9, 3, 3, 7], 0) == []                                 # every image cached: no loader call, no stem
    assert pipe.slots[1].x["kbSlot"].tolist() == [2, 1, 1, 0]
    assert run([1, 9, 2, 1], 1) == [[1, 2]]
    st = pipe.cache_stats()
    assert st == {"hits": 4, "misses": 5, "evictions": 0, "image_bytes": 5 * C * H * W * 4, "resident": 5}
    assert run([4, 5, 6, 8], 2) == [[4, 5, 6, 8]]                     # 4 misses, 6 rows: 3 evictions
    assert pipe.cache_stats()["evictions"] == 3 and pipe.cache_stats()["resident"] == 6


def test_pool_dtype_follows_the_cell_form(monkeypatch):
    from mac_network_b200.serving import ModelPipeline
    for variant, prec, d, kw, bf16 in (("args", "bf16", 128, {}, True),
                                       ("args", "fp8", 512, dict(eval_stem_prec="fp8", eval_enc_prec="bf16"), True),
                                       ("args", "fp32", 128, {}, False), ("args", "tc32", 128, {}, False),
                                       ("p2_unshared", "bf16", 128, {}, False), ("p2_read_bl", "bf16", 128, {}, False)):
        mock, n, net = _model(monkeypatch, variant=variant, prec=prec, d=d, **kw)
        pipe = ModelPipeline(net, (B, S, H, W), slots=1, images=2, cache=B, host_cast=False, use_graph=False)
        s = pipe.slots[0]
        assert pipe.pool.dtype == (torch.bfloat16 if bf16 else torch.float32), (variant, prec)
        assert pipe.pool.shape == (B, H * W, d)
        del mock.calls[:]
        pipe.submit(_batch([1, 2, 1, 2], Loader()))
        if bf16:        # the cell graph gathers the bf16 rows; the cell reads them as a bf16 knowledge base
            assert s.cell.knowledgeBase is s.kb16 and s.cell.kbIndex is None and s.kb16.shape == (B, H * W, d)
            assert mock.calls.count("mac_kb_gather_bf16") == 1 and "mac_kb_gather" not in mock.calls
        else:           # the cell gathers its fp32 rows from the pool itself
            assert s.kb16 is None and s.cell.knowledgeBase is pipe.pool and s.cell.kbIndex is s.x["kbSlot"]
            assert mock.calls.count("mac_kb_gather") == 1 and "mac_kb_gather_bf16" not in mock.calls
        assert "mac_cast_bf16" not in mock.calls or variant == "p2_unshared"
        assert mock.calls.count("mac_kb_pool_insert") == 1


def test_bad_batches_leave_the_cache_unchanged(monkeypatch):
    from mac_network_b200.serving import ModelPipeline
    mock, n, net = _model(monkeypatch)
    pipe = ModelPipeline(net, (B, S, H, W), slots=2, images=2, cache=B, host_cast=False)
    pipe.submit(_batch([1, 2, 3, 1], Loader()))
    snap = lambda: (list(pipe._cache.rows.items()), list(pipe._cache.key), [list(r) for r in pipe._cache.reader],
                    pipe.cache_stats(),
                    pipe._next, n.replays)
    before = snap()
    good = _batch([1, 5, 6, 7], Loader())

    def raising(ids):
        raise TypeError("cannot read")
    bads = [dict(good, imageIds=np.array([1, 5, 6])), dict(good, imageIds=np.array([1.0, 5, 6, 7])),
            dict(good, imageIds=np.array([[1, 5], [6, 7]])), dict(good, imageIds=np.array([True, False, True, True])),
            dict(good, images=np.zeros((3, C, H, W), np.float32)), {k: v for k, v in good.items() if k != "imageIds"},
            dict(good, imageIndex=np.zeros(B, np.int32)), dict(good, questions=good["questions"][:, :S - 1]),
            dict(good, images=Loader(dtype=np.float64)), dict(good, images=Loader(shape=(2, C, H, W))),
            dict(good, images=Loader(shape=(3, C, H, W + 1))), dict(good, images=lambda ids: "features")]
    for bad in bads:
        with pytest.raises(ValueError):
            pipe.submit(bad)
        assert snap() == before
    with pytest.raises(TypeError):          # the loader's own errors pass through, and change nothing either
        pipe.submit(dict(good, images=raising))
    assert snap() == before
    pipe.submit(good)
    assert pipe.cache_stats()["misses"] == before[3]["misses"] + 3


def test_weight_update_and_clear_cache_empty_the_cache(monkeypatch):
    from mac_network_b200.serving import ModelPipeline
    mock, n, net = _model(monkeypatch)
    pipe = ModelPipeline(net, (B, S, H, W), slots=2, images=2, cache=B, host_cast=False)
    load = Loader()
    pipe.submit(_batch([1, 2, 3, 4], load))
    pipe.submit(_batch([1, 2, 3, 4], load))
    assert load.calls == [[1, 2, 3, 4]] and pipe.cache_stats()["resident"] == 4
    caps, syncs = n.captures, n.event_syncs
    net.trainer.params.touch()
    pipe.submit(_batch([1, 2, 3, 4], load))
    assert load.calls[-1] == [1, 2, 3, 4] and n.captures == caps + 4 and n.event_syncs > syncs    # drained, captured again
    pipe.submit(_batch([4, 3, 4, 3], load))
    assert len(load.calls) == 2
    pipe.clear_cache()
    assert pipe.cache_stats()["resident"] == 0 and pipe._cache.free == list(range(B))
    pipe.submit(_batch([4, 3, 4, 3], load))
    assert load.calls[-1] == [4, 3] and n.captures == caps + 4
    st = pipe.cache_stats()
    assert st["misses"] == 4 + 4 + 2 and st["hits"] == 4 + 2


def test_stream_waits_between_slots(monkeypatch):
    """Write after read: evicting a row another slot's batch read waits for that slot's done event.  Read after write: a
    hit on a row another slot's stem pass wrote waits for that pass's event.  Waits already covered are not repeated."""
    from mac_network_b200.serving import ModelPipeline
    mock, n, net = _model(monkeypatch)
    pipe = ModelPipeline(net, (B, S, H, W), slots=2, images=2, cache=4, host_cast=False)
    s0, s1 = pipe.slots
    n.waits = []
    pipe.submit(_batch([0, 1, 2, 3], Loader()))         # ticket 0, slot 0: rows 0..3 in two stem passes
    assert n.waits == []
    w = pipe._cache.written
    assert w[0][:2] == (0, 0) and w[1][2] is w[0][2] and w[2][:2] == (0, 1) and w[3][2] is w[2][2]
    pipe.submit(_batch([0, 1, 4, 5], Loader()))         # ticket 1, slot 1: evicts rows 2, 3 (read by ticket 0), hits 0, 1
    assert n.waits == [(s1.stream, s0.done)]            # the done event covers the stem passes of ticket 0 as well
    n.waits = []
    pipe.submit(_batch([4, 6, 0, 1], Loader()))         # ticket 2, slot 0: hit 4 (written by ticket 1), evicts row of 5
    assert n.waits == [(s0.stream, s1.done)]            # evicts 5 (read by ticket 1), which also covers the write of 4
    n.waits = []
    pipe.submit(_batch([6, 6, 6, 6], Loader()))         # ticket 3, slot 1: hit 6 (written by ticket 2 on slot 0)
    ev6 = pipe._cache.written[pipe._cache.rows[6]][2]
    assert n.waits == [(s1.stream, ev6)]
    n.waits = []
    pipe.submit(_batch([6, 0, 1, 4], Loader()))         # ticket 4, slot 0: everything it reads is covered or its own
    assert n.waits == []


def test_eviction_waits_for_every_slot_that_read_the_row(monkeypatch):
    """Reads of one row on two other slots are not ordered with each other: evicting it waits for both."""
    from mac_network_b200.serving import ModelPipeline
    mock, n, net = _model(monkeypatch)
    pipe = ModelPipeline(net, (B, S, H, W), slots=3, images=2, cache=4, host_cast=False)
    s0, s1, s2 = pipe.slots
    pipe.submit(_batch([0, 1, 2, 3], Loader()))         # ticket 0, slot 0
    ev0 = pipe._cache.written[0][2]
    n.waits = []
    pipe.submit(_batch([0, 0, 0, 0], Loader()))         # ticket 1, slot 1 reads row 0
    pipe.submit(_batch([0, 0, 0, 0], Loader()))         # ticket 2, slot 2 reads row 0
    assert n.waits == [(s1.stream, ev0), (s2.stream, ev0)]
    assert [rd[0] for rd in pipe._cache.reader[0]] == [0, 1, 2]
    n.waits = []
    pipe.submit(_batch([4, 5, 6, 7], Loader()))         # ticket 3, slot 0 evicts every row, row 0 last
    assert n.waits == [(s0.stream, s1.done), (s0.stream, s2.done)]


def test_eviction_waits_for_the_readers_own_batch_not_the_slots_latest(monkeypatch):
    """A victim last read by an old batch of another slot: the wait is on that batch's done event, not on the batch the slot
    runs now, and none at all once this slot's stream has already waited for that batch."""
    from mac_network_b200.serving import ModelPipeline
    mock, n, net = _model(monkeypatch)
    pipe = ModelPipeline(net, (B, S, H, W), slots=2, images=2, cache=6, host_cast=False)
    s0, s1 = pipe.slots
    pipe.submit(_batch([0, 1, 2, 3], Loader()))         # ticket 0, slot 0: rows 0..3
    done0 = s0.done
    pipe.submit(_batch([0, 1, 2, 3], Loader()))         # ticket 1, slot 1: hits, waits for ticket 0's two stem passes
    pipe.submit(_batch([10, 11, 10, 11], Loader()))     # ticket 2, slot 0: free rows 4, 5
    assert s0.done is not done0
    n.waits = []
    pipe.submit(_batch([12, 13, 12, 13], Loader()))     # ticket 3, slot 1: evicts keys 0, 1, read by ticket 0 on slot 0
    assert n.waits == [(s1.stream, done0)]              # not s0.done, the batch slot 0 runs now (ticket 2)
    pipe.submit(_batch([10, 11, 10, 11], Loader()))     # ticket 4, slot 0: hits its own rows
    n.waits = []
    pipe.submit(_batch([14, 15, 14, 15], Loader()))     # ticket 5, slot 1: evicts keys 2, 3, read by ticket 0 (covered)
    assert n.waits == [] and pipe.cache_stats()["evictions"] == 4
