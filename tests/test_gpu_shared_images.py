"""Several questions per image on the GPU: mac_kb_gather, MACCell(kbIndex=), ModelPipeline(images=U) and runBatch by
imageIds.

- mac_kb_gather bit for bit kb_u[index] (fp32) and mac_cast_bf16 of it (bf16), NaN rows for indices outside [0, U), the
  rows around the output untouched.
- MACCell(kb_u, kbIndex=idx) bit for bit MACCell(kb_u[idx]) in control, memory and every attention map of every step, on
  every inference form.
- ModelPipeline(images=U) bit for bit runBatch(train=False) with repeated imageIds, for every evaluation stem precision;
  against ModelPipeline() fed the duplicated features, bit for bit where the stem's GEMMs do not choose their schedule from
  M (bf16, e4m3, split bf16), bounded for the fp32 stem, whose sgemm does.
- New index patterns and k < U need no new capture; a weight update captures every slot again.
- runBatch with all-distinct imageIds launches what it launches without them."""
import numpy as np
import pytest
import torch

from tests.test_gpu_model_pipeline import A, C, E, V, _assert_same
from tests.test_shared_images_host import config

pytestmark = pytest.mark.gpu


def _lib():
    from mac_network_b200 import _lib as L_
    return L_, L_.load()


# ------------------------------------------------------------------------------------------------ mac_kb_gather
def _cast_bf16(x):
    L_, lib = _lib()
    out = torch.empty(x.shape, dtype=torch.bfloat16, device="cuda")
    L_.check(lib.mac_cast_bf16(L_.ptr(x), L_.ptr(out), x.numel(), L_.stream_ptr()), "mac_cast_bf16")
    return out


def _gather(kb_u, index, bf16, B):
    """mac_kb_gather into rows 1..B of a canary-filled buffer of B + 2 rows; returns (all rows, status)."""
    L_, lib = _lib()
    U, N, d = kb_u.shape
    dt = torch.bfloat16 if bf16 else torch.float32
    buf = torch.full((B + 2, N, d), -3.0, dtype=dt, device="cuda")
    st = lib.mac_kb_gather(L_.ptr(kb_u), L_.ptr(index), L_.ptr(buf[1:B + 1]), int(bf16), B, U, N, d, L_.stream_ptr())
    torch.cuda.synchronize()
    return buf, st


def _index_patterns(B, U, rng):
    pats = {"random": rng.randint(0, U, size=B)}
    if U > 1:
        pats["unused"] = rng.randint(0, max(1, U // 2), size=B)             # the upper images never read
    if U == B:
        pats["permutation"] = rng.permutation(B)
    bad = rng.randint(0, U, size=B)
    bad[::3] = np.array([-1, U, 2 ** 31 - 1, -2 ** 31])[np.arange(len(bad[::3])) % 4]
    pats["out_of_range"] = bad
    return pats


@pytest.mark.parametrize("d", [8, 128, 512])
@pytest.mark.parametrize("N", [1, 49, 196, 257])
@pytest.mark.parametrize("B,U", [(1, 1), (5, 1), (7, 7), (64, 8), (13, 29)])
def test_kb_gather_equals_indexing_bit_for_bit(B, U, N, d):
    rng = np.random.RandomState(B * 1000 + U * 10 + N + d)
    g = torch.Generator(device="cuda").manual_seed(N * d + B)
    kb_u = torch.randn(U, N, d, device="cuda", generator=g)
    kb_u.view(-1)[::5] = kb_u.view(-1)[::5].to(torch.bfloat16).float() + 2.0 ** -9 * kb_u.view(-1)[::5].abs()  # near ties
    kb_before = kb_u.clone()
    for name, pat in _index_patterns(B, U, rng).items():
        index = torch.from_numpy(pat.astype(np.int32)).cuda()
        ok = (index >= 0) & (index < U)
        safe = torch.where(ok, index, torch.zeros_like(index)).long()
        want = kb_u[safe].clone()
        want[~ok] = float("nan")
        for bf16 in (0, 1):
            buf, st = _gather(kb_u, index, bf16, B)
            assert st == 0, (name, bf16, st)
            got = buf[1:B + 1]
            ref = _cast_bf16(want) if bf16 else want
            if bf16:   # what mac_cast_bf16 makes of the gathered rows, NaN rows included
                assert torch.equal(got.view(torch.int16), ref.view(torch.int16)), (name, "bf16")
                assert bool(got[~ok].isnan().all()), (name, "bf16 NaN rows")
            else:
                assert torch.equal(got[ok].view(torch.int32), ref[ok].view(torch.int32)), (name, "fp32")
                assert bool((got[~ok].view(torch.int32) == 0x7fc00000).all()), (name, "fp32 NaN rows")
            assert bool((buf[0] == -3.0).all()) and bool((buf[B + 1] == -3.0).all()), (name, bf16, "neighbour rows")
    assert torch.equal(kb_u, kb_before)


def test_kb_gather_refusals_leave_the_output_untouched():
    L_, lib = _lib()
    kb = torch.ones(2, 4, 8, device="cuda")
    idx = torch.zeros(3, dtype=torch.int32, device="cuda")
    out = torch.full((3, 4, 8), 7.0, device="cuda")
    k, i, o = kb.data_ptr(), idx.data_ptr(), out.data_ptr()
    g = lambda kp, ip, op, bf, B, U, N, d: lib.mac_kb_gather(kp, ip, op, bf, B, U, N, d, None)
    assert g(None, i, o, 0, 3, 2, 4, 8) == -1 and g(k, i, o, 0, 3, 0, 4, 8) == -1
    assert g(k, i, o, 2, 3, 2, 4, 8) == -3 and g(k, i, o, 0, 3, 2, 8, 4) == -3
    assert g(k + 4, i, o, 0, 3, 2, 4, 8) == -2 and g(k, i, o + 8, 0, 3, 2, 4, 8) == -2
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())


# ------------------------------------------------------------------------------------------------ the cell
def _cell_pair(variant, prec, B, U, N, d=512, L=4, seed=0):
    from mac_network_b200.mac_cell import MACCell, MACParams, mac_network
    from mac_network_b200.params import init_params, perturb_biases
    from mac_network_b200.synthetic import make_inputs
    cfg = config(variant, netLength=L, memDim=d, ctrlDim=d, attDim=d)
    params = MACParams(cfg, L, values=perturb_biases(init_params(cfg, L, seed=seed + 1), seed=seed + 2))
    inp = make_inputs(B, 7, N, d, seed=seed + 3)
    x = {k: torch.from_numpy(v).cuda() for k, v in inp.items() if k != "knowledgeBase"}
    kb_u = torch.from_numpy(make_inputs(U, 2, N, d, seed=seed + 4)["knowledgeBase"]).cuda()
    rng = np.random.RandomState(seed + 5)
    idx = torch.from_numpy(rng.randint(0, max(1, U - 1), size=B).astype(np.int32)).cuda()     # image U-1 unused
    outs = []
    for kb, kbIndex in ((kb_u, idx), (kb_u[idx.long()].contiguous(), None)):
        cell = MACCell(x["vecQuestions"], x["questionWords"], x["questionCntxWords"], x["questionLengths"], kb, 1.0, 1.0,
                       1.0, B, False, config=cfg, params=params, prec=prec, kbIndex=kbIndex)
        control, memory = mac_network(cell, L)
        torch.cuda.synchronize()
        outs.append((cell, control.clone(), memory.clone(), {k: [a.clone() for a in v] for k, v in cell.attentions.items()}))
    return outs


def _assert_cells_equal(outs, L):
    (c1, ctl1, mem1, att1), (c2, ctl2, mem2, att2) = outs
    assert c1.kbIndex is not None and c2.kbIndex is None
    assert torch.equal(ctl1, ctl2) and torch.equal(mem1, mem2)
    assert torch.equal(c1._hc, c2._hc) and torch.equal(c1._hm, c2._hm) and torch.equal(c1._hi, c2._hi)
    assert set(att1) == set(att2)
    for k in att1:
        assert len(att1[k]) == len(att2[k]), k
        for i, (a, b) in enumerate(zip(att1[k], att2[k])):
            assert torch.equal(a, b), (k, i)
    assert len(att1["kb"]) == L and torch.isfinite(mem1).all()


@pytest.mark.parametrize("N", [196, 49])
@pytest.mark.parametrize("variant", ["args", "args1", "gqa"])
@pytest.mark.parametrize("prec", ["fp32", "tc32", "bf16", "fp8"])
def test_cell_with_kb_index_equals_the_gathered_cell(prec, variant, N):
    outs = _cell_pair(variant, prec, B=24, U=7, N=N)
    assert (outs[0][0]._kb_rows is None) == (prec in ("bf16", "fp8"))
    _assert_cells_equal(outs, 4)


@pytest.mark.parametrize("N", [196, 49])
@pytest.mark.parametrize("variant", ["p2_read_bl", "p2_unshared"])
@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_cell_with_kb_index_equals_the_gathered_cell_p2(prec, variant, N):
    outs = _cell_pair(variant, prec, B=12, U=5, N=N, L=3)
    assert outs[0][0]._kb_rows is not None                # these forms read the fp32 per-question knowledge base
    _assert_cells_equal(outs, 3)


def test_cell_with_kb_index_unfused_bf16_chain():
    """N > 256: the bf16 read unit's unfused chain (BF16_INV), which also reads only the bf16 knowledge base."""
    from mac_network_b200 import _lib as L_
    assert not L_.load().mac_read_step_fused_supported(10, 260, 512)
    outs = _cell_pair("args", "bf16", B=10, U=4, N=260)
    assert outs[0][0]._kb_rows is None
    _assert_cells_equal(outs, 4)


# ------------------------------------------------------------------------------------------------ whole model
MODELS = {"fp32": dict(prec="fp32"), "bf16": dict(prec="bf16"),
          "fp8": dict(prec="fp8", eval_stem_prec="fp8", eval_enc_prec="bf16"),
          "bf16x3": dict(prec="tc32", eval_stem_prec="bf16x3")}


def _net(variant, model, L=3, seed=3):
    from mac_network_b200.model import MACnet
    cfg = config(variant, netLength=L)
    return MACnet(cfg, L, V, A, wrd_emb_dim=E, image_in_dim=C, classifier_dims=(512,), seed=seed, **MODELS[model])


def _shared_batches(n, B, S, H, W, ks, seed):
    """n batches of B questions over k = ks[i] distinct images: `ids` per question (repeats), `images` one row per question
    (the reference's loader form), `distinct`/`index` the pipeline's form in runBatch's order (ascending id)."""
    rng = np.random.RandomState(seed)
    out = []
    for i in range(n):
        k = ks[i % len(ks)]
        lengths = rng.randint(1, S + 1, size=(B,)).astype(np.int32)
        lengths[rng.randint(B)] = S
        q = rng.randint(1, V + 1, size=(B, S)).astype(np.int32)
        q[np.arange(S)[None, :] >= lengths[:, None]] = 0
        id_values = np.sort(rng.choice(1000, size=k, replace=False))
        pick = np.concatenate([np.arange(k), rng.randint(0, k, size=B - k)])      # every image asked about at least once
        rng.shuffle(pick)
        distinct = np.maximum(rng.standard_normal((k, C, H, W)), 0).astype(np.float32)
        ids, index, images = id_values[pick], pick.astype(np.int32), distinct[pick]
        out.append({"questions": q, "questionLengths": lengths, "ids": ids, "dup": images,
                    "distinct": np.ascontiguousarray(distinct), "index": index})
    return out


def _pipe_batch(b, shared):
    base = {"questions": b["questions"], "questionLengths": b["questionLengths"]}
    return dict(base, images=b["distinct"], imageIndex=b["index"]) if shared else dict(base, images=b["dup"])


def _run_batch_reference(net, b):
    data = {"questions": b["questions"], "questionLengths": b["questionLengths"],
            "answers": np.zeros(len(b["questionLengths"]), dtype=np.int32)}
    net.runBatch(None, data, {"images": b["dup"], "imageIds": b["ids"]}, train=False, getAtt=True)
    torch.cuda.synchronize()
    cell = net.macCell
    assert cell.kbIndex is not None and cell.U == len(b["distinct"])
    assert np.array_equal(cell.kbIndex.cpu().numpy(), b["index"])
    ref = {"answers": net._out.last_logits.argmax(-1).int().cpu().numpy(),
           "logits": net._out.last_logits.cpu().numpy(), "memory": cell._hm[net.L].cpu().numpy(),
           "att_kb": torch.stack(cell.attentions["kb"]).cpu().numpy(),
           "att_question": torch.stack(cell.attentions["question"]).cpu().numpy()}
    if cell.attentions["gate"]:
        ref["gate"] = torch.stack(cell.attentions["gate"]).cpu().numpy()
    if cell.attentions["self"]:
        ref["self"] = [a.cpu().numpy() for a in cell.attentions["self"]]
    return ref


@pytest.mark.parametrize("variant,H,W", [("args", 14, 14), ("gqa", 7, 7)])
@pytest.mark.parametrize("model", ["fp32", "bf16", "fp8", "bf16x3"])
def test_pipeline_with_images_equals_run_batch_by_image_ids(variant, H, W, model):
    """k = U distinct images per batch, so the stem of both runs over the same rows; the longest question fills S."""
    from mac_network_b200.serving import ModelPipeline
    B, S, L, U = 8, 10, 3, 3
    net = _net(variant, model, L)
    batches = _shared_batches(5, B, S, H, W, ks=[U], seed=61)
    refs = [_run_batch_reference(net, b) for b in batches]
    for slots, host_cast in ((2, True), (1, False)):
        pipe = ModelPipeline(net, (B, S, H, W), slots=slots, images=U, host_cast=host_cast, cast_threads=3)
        assert pipe.host_cast == (host_cast and model == "bf16")
        tickets = []
        for i, b in enumerate(batches):
            nxt = _pipe_batch(batches[i + 1], True) if i + 1 < len(batches) else None
            tickets.append(pipe.submit(_pipe_batch(b, True), next_batch=nxt))
            if len(tickets) >= slots:
                j = len(tickets) - slots
                _assert_same(pipe.result(tickets[j]), refs[j], L)
        for j in range(len(batches) - slots + 1, len(batches)):
            _assert_same(pipe.result(tickets[j]), refs[j], L)
        pipe.drain()


def _rel(a, b):
    return float(np.abs(a.astype(np.float64) - b).max() / max(np.abs(b).max(), 1e-30))


# The fp32 stem's sgemm (sgemm_launch) chooses its kernel from M.  With M > 64 rows it runs one CTA per output tile with no
# split-K (the stem passes no workspace), and the tile height it picks from M does not change the order of a row's k-loop:
# at 14x14 (M >= 196) a stem over U images and one over B duplicated images agree bit for bit.  With M <= 64 (one 7x7
# image) it runs the cluster split-K kernel (skinny_launch), which sums the k-slices in another order than the tiled
# kernel the duplicated stem (M = 8 * 49) runs.  Measured on an H100 80GB HBM3 the two then differ by FP32_SKINNY_MEASURED
# (largest relative difference over logits, memory and attention maps); the bound is three times that.
FP32_SKINNY_MEASURED = 4.0e-7
FP32_SKINNY_BOUND = 3 * FP32_SKINNY_MEASURED


@pytest.mark.parametrize("model,H,W", [("fp32", 14, 14), ("bf16", 14, 14), ("fp8", 14, 14), ("bf16x3", 14, 14),
                                       ("fp32", 7, 7), ("bf16", 7, 7)])
def test_pipeline_with_images_against_duplicated_features(model, H, W):
    """images=U against ModelPipeline() fed one image per question: at 14x14 U = 4 with k in {4, 2, 1}, at 7x7 U = k = 1.  The bf16 (tc_gemm), e4m3
    (mac_linear_fp8_fwd) and split-bf16 (tc3_gemm) stems give each output row one CTA's k-loop over its own patch row,
    whatever M is, and the gather hands the cell the same bits as the duplicated stem output: bit for bit.  The fp32 stem:
    see FP32_SKINNY_MEASURED."""
    from mac_network_b200.serving import ModelPipeline
    B, S, L, U = 8, 10, 3, (4 if H == 14 else 1)
    net = _net("args" if H == 14 else "gqa", model, L)
    batches = _shared_batches(6, B, S, H, W, ks=[U, 2, 1] if U == 4 else [1], seed=71)
    skinny = model == "fp32" and U * H * W <= 64
    dup = ModelPipeline(net, (B, S, H, W), slots=1, host_cast=False)
    shared = ModelPipeline(net, (B, S, H, W), slots=2, images=U, host_cast=False)
    worst = 0.0
    for b in batches:
        want = {k: v.numpy().copy() for k, v in dup.result(dup.submit(_pipe_batch(b, False))).items()}
        got = {k: v.numpy().copy() for k, v in shared.result(shared.submit(_pipe_batch(b, True))).items()}
        assert set(got) == set(want)
        if not skinny:
            for k in want:
                assert np.array_equal(got[k], want[k]), (model, k)
        else:
            errs = {k: _rel(got[k], want[k]) for k in ("logits", "memory", "att_kb", "att_question")}
            worst = max(worst, max(errs.values()))
            assert max(errs.values()) <= FP32_SKINNY_BOUND, errs
    print("%s: images=U against duplicated features, largest relative difference %.3g" % (model, worst))
    dup.drain()
    shared.drain()


def test_new_index_patterns_need_no_capture_and_weight_updates_capture_again():
    from mac_network_b200.serving import ModelPipeline
    B, S, L, U, H, W = 8, 10, 3, 4, 14, 14
    net = _net("args", "bf16", L)
    batches = _shared_batches(6, B, S, H, W, ks=[4, 1, 3, 2], seed=81)
    dup = ModelPipeline(net, (B, S, H, W), slots=1, host_cast=False)
    pipe = ModelPipeline(net, (B, S, H, W), slots=2, images=U, host_cast=True, cast_threads=3)
    graphs = [s.graph for s in pipe.slots]
    assert all(g is not None for g in graphs)
    for b in batches[:4]:                   # k = 4, 1, 3, 2 with their own index patterns
        got = pipe.result(pipe.submit(_pipe_batch(b, True)))
        want = dup.result(dup.submit(_pipe_batch(b, False)))
        for k in want:
            assert torch.equal(got[k], want[k]), k
    assert [s.graph for s in pipe.slots] == graphs          # same graph objects: nothing captured again
    p = net.trainer.params
    with torch.no_grad():
        p.flat.mul_(1.03)
    p.touch()
    for b in batches[4:]:
        got = {k: v.clone() for k, v in pipe.result(pipe.submit(_pipe_batch(b, True))).items()}
        want = dup.result(dup.submit(_pipe_batch(b, False)))
        for k in want:
            assert torch.equal(got[k], want[k]), k
        ref = _run_batch_reference(net, dict(b, distinct=b["distinct"]))
        assert np.array_equal(got["logits"].numpy(), ref["logits"])
    assert all(s.graph is not g for s, g in zip(pipe.slots, graphs))      # every slot captured again
    pipe.drain()
    dup.drain()


def test_run_batch_with_distinct_image_ids_launches_the_same_kernels():
    from mac_network_b200 import _lib as L_
    B, S, H, W = 8, 10, 14, 14
    net = _net("args", "bf16", 3)
    b = _shared_batches(1, B, S, H, W, ks=[B], seed=91)[0]
    assert len(set(b["ids"].tolist())) == B
    data = {"questions": b["questions"], "questionLengths": b["questionLengths"], "answers": np.zeros(B, dtype=np.int32)}
    lib = L_.load()
    net.runBatch(None, data, {"images": b["dup"]}, train=False)          # warm-up: packs
    counts, logits = [], []
    for images in ({"images": b["dup"]}, {"images": b["dup"], "imageIds": b["ids"]}):
        torch.cuda.synchronize()
        n0 = lib.mac_b200_launch_count()
        net.runBatch(None, data, images, train=False)
        torch.cuda.synchronize()
        counts.append(lib.mac_b200_launch_count() - n0)
        logits.append(net._out.last_logits.clone())
        assert net.macCell.kbIndex is None
    assert counts[0] == counts[1] and torch.equal(logits[0], logits[1])
    # with repeats the shared path runs: one gather launch more, no bf16 cast launch
    ids = b["ids"].copy()
    ids[1] = ids[0]
    n0 = lib.mac_b200_launch_count()
    net.runBatch(None, data, {"images": b["dup"], "imageIds": ids}, train=False)
    torch.cuda.synchronize()
    assert net.macCell.kbIndex is not None and net.macCell.U == B - 1
    assert lib.mac_b200_launch_count() - n0 == counts[0]
