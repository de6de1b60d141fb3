"""Knowledge bases kept on the device across batches, on the GPU: mac_kb_pool_insert, mac_kb_gather_bf16 and
ModelPipeline(images=U, cache=C).

- mac_kb_pool_insert bit for bit kb_u[u] into pool row slot[u] (fp32) and mac_cast_bf16 of it (bf16); rows named by no
  valid slot, and the rows around the pool, untouched.  mac_kb_gather_bf16 bit for bit indexing, NaN rows out of range.
- The cached pipeline bit for bit ModelPipeline(images=U) fed the same stream without a cache (the stem runs over the same
  U rows), for the bf16, e4m3, split-bf16 and fp32 stems and on the fp32-pool path of a flag set with per-step cells; and
  against ModelPipeline() fed one image per question, with several stem passes per batch.
- Four slots with C = B, every batch evicting rows the batches in flight read: still bit for bit.
- A weight update mid-stream and clear_cache() give what a fresh pipeline gives.
- A batch whose images are all cached launches no ingest or stem kernel."""
import numpy as np
import pytest
import torch

from tests.test_gpu_shared_images import FP32_SKINNY_BOUND, _cast_bf16, _net, _rel

pytestmark = pytest.mark.gpu

C_IN, V = 128, 90


def _lib():
    from mac_network_b200 import _lib as L_
    return L_, L_.load()


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("U,cap,N,d", [(1, 1, 1, 8), (5, 9, 196, 512), (3, 4, 49, 8), (16, 40, 196, 512), (7, 70000, 1, 8)])
def test_pool_insert_equals_numpy_bit_for_bit(U, cap, N, d):
    L_, lib = _lib()
    rng = np.random.RandomState(U * 100 + cap)
    g = torch.Generator(device="cuda").manual_seed(N * d + U)
    kb_u = torch.randn(U, N, d, device="cuda", generator=g)
    kb_u.view(-1)[::5] = kb_u.view(-1)[::5].to(torch.bfloat16).float() + 2.0 ** -9 * kb_u.view(-1)[::5].abs()  # near ties
    slot = rng.permutation(cap)[:U].astype(np.int64)
    bad = np.array([-1, cap, cap + 5, 2 ** 31 - 1, -2 ** 31])
    slot[1::3] = bad[np.arange(len(slot[1::3])) % len(bad)]                 # padding rows and out-of-range slots
    slot_d = torch.from_numpy(slot.astype(np.int32)).cuda()
    want32 = kb_u.cpu().numpy()
    for bf16 in (0, 1):
        dt = torch.bfloat16 if bf16 else torch.float32
        buf = torch.full((cap + 2, N, d), -3.0, dtype=dt, device="cuda")          # canary rows around the pool
        st = lib.mac_kb_pool_insert(L_.ptr(kb_u), L_.ptr(slot_d), L_.ptr(buf[1:cap + 1]), bf16, U, cap, N, d,
                                    L_.stream_ptr())
        torch.cuda.synchronize()
        assert st == 0
        ref = _cast_bf16(kb_u).view(torch.int16).cpu().numpy() if bf16 else want32.view(np.int32)
        got = (buf.view(torch.int16) if bf16 else buf.view(torch.int32)).cpu().numpy()
        canary = np.full((N, d), -3.0, dtype=np.float32)
        canary = torch.from_numpy(canary).to(dt).view(torch.int16 if bf16 else torch.int32).numpy()
        written = set()
        for u, s in enumerate(slot):
            if 0 <= s < cap:
                assert np.array_equal(got[1 + s], ref[u]), (bf16, u, s)
                written.add(int(s))
        for r in range(cap + 2):
            if r - 1 not in written:
                assert np.array_equal(got[r], canary), (bf16, "untouched row", r)


@pytest.mark.parametrize("B,U,N,d", [(1, 1, 1, 8), (64, 40, 196, 512), (13, 29, 49, 128), (70000, 3, 1, 8)])
def test_kb_gather_bf16_equals_indexing_bit_for_bit(B, U, N, d):
    L_, lib = _lib()
    rng = np.random.RandomState(B + U)
    g = torch.Generator(device="cuda").manual_seed(B * 7 + d)
    src = torch.randn(U, N, d, device="cuda", generator=g).to(torch.bfloat16)
    index = rng.randint(0, U, size=B)
    index[::3] = np.array([-1, U, 2 ** 31 - 1, -2 ** 31])[np.arange(len(index[::3])) % 4]
    index_d = torch.from_numpy(index.astype(np.int32)).cuda()
    buf = torch.full((B + 2, N, d), -3.0, dtype=torch.bfloat16, device="cuda")
    st = lib.mac_kb_gather_bf16(L_.ptr(src), L_.ptr(index_d), L_.ptr(buf[1:B + 1]), B, U, N, d, L_.stream_ptr())
    torch.cuda.synchronize()
    assert st == 0
    ok = torch.from_numpy((index >= 0) & (index < U)).cuda()
    got = buf[1:B + 1]
    want = src[torch.where(ok, index_d, torch.zeros_like(index_d)).long()]
    assert torch.equal(got[ok].view(torch.int16), want[ok].view(torch.int16))
    assert bool((got[~ok].view(torch.int16) == 0x7fc0).all()) and bool(got[~ok].isnan().all())
    assert bool((buf[0] == -3.0).all()) and bool((buf[B + 1] == -3.0).all())


# ------------------------------------------------------------------------------------------------ the pipeline
def _stream(n, B, S, H, W, I, kmax, seed, kmin=1):
    """n batches of B questions about 1..kmax of I images each (every chosen image asked about at least once, the questions
    shuffled), image keys that are not 0..I-1, and the features of every key."""
    rng = np.random.RandomState(seed)
    keys = (1000 + 7 * np.arange(I)).tolist()
    feats = {k: np.maximum(rng.standard_normal((C_IN, H, W)), 0).astype(np.float32) for k in keys}
    out = []
    for _ in range(n):
        k = rng.randint(kmin, kmax + 1)
        chosen = rng.choice(keys, size=k, replace=False)
        pick = np.concatenate([np.arange(k), rng.randint(0, k, size=B - k)])
        rng.shuffle(pick)
        lengths = rng.randint(1, S + 1, size=(B,)).astype(np.int32)
        lengths[rng.randint(B)] = S
        q = rng.randint(1, V + 1, size=(B, S)).astype(np.int32)
        q[np.arange(S)[None, :] >= lengths[:, None]] = 0
        out.append({"questions": q, "questionLengths": lengths, "ids": chosen[pick]})
    return out, feats


class _Loader(object):
    def __init__(self, feats):
        self.feats, self.calls = feats, []

    def __call__(self, ids):
        self.calls.append(ids.tolist())
        return torch.from_numpy(np.stack([self.feats[int(i)] for i in ids])).pin_memory()


def _form(b, feats, how, load=None):
    base = {"questions": b["questions"], "questionLengths": b["questionLengths"]}
    if how == "cache":
        return dict(base, imageIds=b["ids"], images=load)
    if how == "shared":                      # images=U without a cache: the batch's distinct images, first occurrence
        distinct = list(dict.fromkeys(b["ids"].tolist()))
        index = np.array([distinct.index(i) for i in b["ids"]], dtype=np.int32)
        return dict(base, images=np.stack([feats[i] for i in distinct]), imageIndex=index)
    return dict(base, images=np.stack([feats[int(i)] for i in b["ids"]]))          # one image per question


def _run(pipe, subs):
    """Submit every batch, reading each result before its slot is taken again; numpy copies of the outputs."""
    n, tickets, outs = len(pipe.slots), [], []
    for b in subs:
        tickets.append(pipe.submit(b))
        if len(tickets) >= n:
            outs.append({k: v.numpy().copy() for k, v in pipe.result(tickets[len(outs)]).items()})
    while len(outs) < len(tickets):
        outs.append({k: v.numpy().copy() for k, v in pipe.result(tickets[len(outs)]).items()})
    pipe.drain()
    return outs


def _equal(got, want, what):
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert set(g) == set(w), (what, i)
        for k in w:
            assert np.array_equal(g[k], w[k]), (what, i, k)


@pytest.mark.parametrize("variant,model,pool_bf16", [("args", "bf16", True), ("args", "fp8", True), ("args", "bf16x3", False),
                                                     ("args", "fp32", False), ("p2_unshared", "bf16", False)])
def test_cached_pipeline_equals_images_u_without_a_cache(variant, model, pool_bf16):
    """Ten images cached of fourteen, batches of up to U = 4 images: hits across batches, evictions, partial stem passes."""
    from mac_network_b200.serving import ModelPipeline
    B, S, L, U, H, W = 8, 10, 3, 4, 14, 14
    net = _net(variant, model, L)
    batches, feats = _stream(10, B, S, H, W, I=14, kmax=U, seed=101)
    want = _run(ModelPipeline(net, (B, S, H, W), slots=2, images=U, host_cast=False),
                [_form(b, feats, "shared") for b in batches])
    load = _Loader(feats)
    pipe = ModelPipeline(net, (B, S, H, W), slots=2, images=U, cache=10)
    assert pipe.pool.dtype == (torch.bfloat16 if pool_bf16 else torch.float32)
    got = _run(pipe, [_form(b, feats, "cache", load) for b in batches])
    _equal(got, want, model)
    st = pipe.cache_stats()
    assert st["hits"] > 0 and st["evictions"] > 0 and st["misses"] == sum(len(c) for c in load.calls)
    assert st["image_bytes"] == st["misses"] * C_IN * H * W * 4


@pytest.mark.parametrize("model,H,W,U", [("bf16", 14, 14, 2), ("fp32", 14, 14, 2), ("fp8", 14, 14, 3), ("bf16", 7, 7, 1),
                                         ("fp32", 7, 7, 1)])
def test_cached_pipeline_against_duplicated_features(model, H, W, U):
    """Up to 5 images per batch through stem passes of U: up to five passes a batch.  Bit for bit ModelPipeline() fed one
    image per question, but for the fp32 stem over one 7x7 image (FP32_SKINNY_MEASURED in test_gpu_shared_images.py)."""
    from mac_network_b200.serving import ModelPipeline
    B, S, L = 8, 10, 3
    net = _net("args" if H == 14 else "gqa", model, L)
    batches, feats = _stream(8, B, S, H, W, I=9, kmax=5, seed=111)
    want = _run(ModelPipeline(net, (B, S, H, W), slots=1, host_cast=False), [_form(b, feats, "dup") for b in batches])
    pipe = ModelPipeline(net, (B, S, H, W), slots=3, images=U, cache=B)
    got = _run(pipe, [_form(b, feats, "cache", _Loader(feats)) for b in batches])
    if model == "fp32" and U * H * W < 64:
        for g, w in zip(got, want):
            errs = {k: _rel(g[k], w[k]) for k in ("logits", "memory", "att_kb", "att_question")}
            assert max(errs.values()) <= FP32_SKINNY_BOUND, errs
    else:
        _equal(got, want, model)
    assert pipe.cache_stats()["hits"] > 0


def test_four_slots_evicting_rows_the_batches_in_flight_read():
    """C = B = U = 8 and every batch keeps four images of the previous one and brings four new: each batch evicts the rows
    the batch before it read (write after read) and reads rows it wrote (read after write), on another slot each time."""
    from mac_network_b200.serving import ModelPipeline
    B, S, L, H, W = 8, 10, 3, 14, 14
    net = _net("args", "bf16", L)
    rng = np.random.RandomState(121)
    _, feats = _stream(0, B, S, H, W, I=60, kmax=1, seed=121)
    keys, batches, prev = sorted(feats), [], []
    fresh = iter(keys)
    for i in range(12):
        ids = prev[4:] + [next(fresh) for _ in range(8 - len(prev[4:]))]
        rng.shuffle(ids)
        prev = ids
        lengths = rng.randint(1, S + 1, size=(B,)).astype(np.int32)
        q = rng.randint(1, V + 1, size=(B, S)).astype(np.int32)
        q[np.arange(S)[None, :] >= lengths[:, None]] = 0
        batches.append({"questions": q, "questionLengths": lengths, "ids": np.array(ids)})
    want = _run(ModelPipeline(net, (B, S, H, W), slots=1, images=B, host_cast=False),
                [_form(b, feats, "shared") for b in batches])
    pipe = ModelPipeline(net, (B, S, H, W), slots=4, images=B, cache=B)
    got = _run(pipe, [_form(b, feats, "cache", _Loader(feats)) for b in batches])
    _equal(got, want, "ordering")
    st = pipe.cache_stats()
    assert st["hits"] == 4 * 11 and st["evictions"] == 4 * 11


def test_weight_update_and_clear_cache_equal_a_fresh_pipeline():
    from mac_network_b200.serving import ModelPipeline
    B, S, L, U, H, W = 8, 10, 3, 4, 14, 14
    net = _net("args", "bf16", L)
    batches, feats = _stream(9, B, S, H, W, I=6, kmax=U, seed=131)
    subs = lambda bs: [_form(b, feats, "cache", _Loader(feats)) for b in bs]
    pipe = ModelPipeline(net, (B, S, H, W), slots=2, images=U, cache=B)
    _run(pipe, subs(batches[:3]))
    p = net.trainer.params
    with torch.no_grad():
        p.flat.mul_(1.03)
    p.touch()
    got = _run(pipe, subs(batches[3:6]))                 # every cached row came from the old weights
    _equal(got, _run(ModelPipeline(net, (B, S, H, W), slots=2, images=U, cache=B), subs(batches[3:6])), "touch")
    # rows of another image file under the same keys: clear_cache() forgets the old ones
    other = {k: np.ascontiguousarray(v[:, ::-1]) for k, v in feats.items()}
    pipe.clear_cache()
    assert pipe.cache_stats()["resident"] == 0
    got = _run(pipe, [_form(b, other, "cache", _Loader(other)) for b in batches[6:]])
    want = _run(ModelPipeline(net, (B, S, H, W), slots=1, images=U, host_cast=False),
                [_form(b, other, "shared") for b in batches[6:]])
    _equal(got, want, "clear_cache")


def test_an_all_hit_batch_launches_no_ingest_or_stem_kernel():
    from mac_network_b200 import _lib as L_
    from mac_network_b200.serving import ModelPipeline
    B, S, L, U, H, W = 8, 10, 3, 2, 14, 14
    lib = L_.load()
    net = _net("args", "bf16", L)
    batches, feats = _stream(1, B, S, H, W, I=3, kmax=3, seed=141, kmin=3)
    pipe = ModelPipeline(net, (B, S, H, W), slots=1, images=U, cache=B, use_graph=False)
    s = pipe.slots[0]

    def launches(fn):
        torch.cuda.synchronize()
        n0 = lib.mac_b200_launch_count()
        fn()
        torch.cuda.synchronize()
        return lib.mac_b200_launch_count() - n0
    with torch.cuda.stream(s.stream):
        s.x["insertSlot"].fill_(-1)
        stem = launches(s._stem_pass)                    # writes no pool row: every insert slot is -1
        cell = launches(s._forward)
    assert stem >= 3 and cell > 0                        # ingest, the stem's GEMMs, the insert
    b = _form(batches[0], feats, "cache", _Loader(feats))
    miss = launches(lambda: pipe.result(pipe.submit(b)))
    hit = launches(lambda: pipe.result(pipe.submit(b)))
    assert miss == 2 * stem + cell and hit == cell       # three images: two stem passes of U = 2, then none
    assert pipe.cache_stats()["hits"] == 3 and pipe.cache_stats()["misses"] == 3
