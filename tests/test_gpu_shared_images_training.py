"""Several questions per image in training on the GPU: mac_kb_gather_bwd, DPTrainer with data["imageIndex"] and
serving.TrainPipeline(images=U).

- mac_kb_gather_bwd bit for bit the sequential float32 sum that starts from each image's first question row and adds the
  later ones in ascending question order, over index patterns with lone terms (signed zeros kept), images with no question
  (zero rows) and out-of-range entries (ignored); reruns bit-identical; the rows around the output untouched; refusals leave
  the output untouched.
- The stem over k images, gathered to B questions and differentiated through the per-image sum, against fp64 autograd with
  the per-image dropout masks, within the bars each stem precision meets alone.
- train_step_full with imageIndex = arange(B) bit for bit the step without an index (stem keep 0.82), over three steps.
- A many-to-one index at stem keep 1.0 against a twin fed images[imageIndex]: everything but the stem's gradients bit for
  bit; those within the stem's bars (they differ in summation order only).
- TrainPipeline(images=U) bit for bit train_step_full on device copies of the same batches; library launches per step."""
import numpy as np
import pytest
import torch

from mac_network_b200 import _lib as L_
from oracle.model_torch_autograd import mask_uniforms, stem_grads
from tests.test_gpu_stem_bf16x3 import BAR_FWD, BAR_GRAD, _mr
from tests.test_stem_tc_training import TOL_STEM_BF16, _uniform_mask

pytestmark = pytest.mark.gpu

INVALID, ALIGN, UNSUPPORTED = -1, -2, -3


# ------------------------------------------------------------------------------------------------ mac_kb_gather_bwd
def _gather_bwd(d_out, index, U):
    """mac_kb_gather_bwd into rows 1..U of a NaN-filled buffer of U + 2 rows; returns (all rows, status)."""
    lib = L_.load()
    B, N, d = d_out.shape
    buf = torch.full((U + 2, N, d), float("nan"), device="cuda")
    st = lib.mac_kb_gather_bwd(L_.ptr(d_out), L_.ptr(index), L_.ptr(buf[1:U + 1]), B, U, N, d, L_.stream_ptr())
    torch.cuda.synchronize()
    return buf, st


def _sequential_sum(g, index, U):
    """numpy float32: each image's first question row, then the later ones added in ascending b; zeros for unused images."""
    out = np.zeros((U,) + g.shape[1:], np.float32)
    seen = np.zeros(U, bool)
    for b, u in enumerate(index):
        if 0 <= u < U:
            if seen[u]:
                out[u] = out[u] + g[b]
            else:
                out[u], seen[u] = g[b], True
    return out


def _grad_rows(B, N, d, seed):
    """Random rows with signed zeros and subnormals sprinkled in: a lone term must keep -0.0, a sum must not start from 0."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    g = torch.randn(B, N, d, device="cuda", generator=gen)
    flat = g.view(-1)
    flat[::7] = -0.0
    flat[3::11] = 0.0
    flat[5::13] = torch.sign(flat[5::13]) * 3e-39
    return g


def _patterns(B, U, rng):
    pats = {"random": rng.randint(0, U, size=B), "one_image": np.full(B, U - 1)}
    if U == B:
        pats["identity"] = np.arange(B)
    if U > 1:
        pats["unused"] = rng.randint(0, max(1, U // 2), size=B)              # the upper images get no question
    bad = rng.randint(0, U, size=B)
    bad[::3] = np.array([-1, U, 2 ** 31 - 1, -2 ** 31])[np.arange(len(bad[::3])) % 4]
    pats["out_of_range"] = bad
    return pats


@pytest.mark.parametrize("d", [8, 136, 512])
@pytest.mark.parametrize("N", [1, 49, 196])
@pytest.mark.parametrize("B,U", [(1, 1), (1, 3), (7, 1), (7, 3), (7, 7), (64, 1), (64, 3), (64, 64), (300, 1), (300, 3),
                                 (300, 300)])
def test_kb_gather_bwd_is_the_sequential_float32_sum(B, U, N, d):
    rng = np.random.RandomState(B * 1000 + U * 10 + N + d)
    g = _grad_rows(B, N, d, seed=N * d + B)
    g_np = g.cpu().numpy()
    for name, pat in _patterns(B, U, rng).items():
        index = torch.from_numpy(pat.astype(np.int32)).cuda()
        want = _sequential_sum(g_np, pat, U)
        buf, st = _gather_bwd(g, index, U)
        assert st == 0, (name, st)
        got = buf[1:U + 1]
        assert np.array_equal(got.cpu().numpy().view(np.int32), want.view(np.int32)), name
        if name == "identity":
            assert torch.equal(got.view(torch.int32), g.view(torch.int32))
        assert bool(buf[0].isnan().all()) and bool(buf[U + 1].isnan().all()), (name, "neighbour rows")
        again, _ = _gather_bwd(g, index, U)
        assert torch.equal(again.view(torch.int32), buf.view(torch.int32)), (name, "rerun")


def test_kb_gather_bwd_refusals_leave_the_output_untouched():
    lib = L_.load()
    g = torch.ones(3, 4, 8, device="cuda")
    idx = torch.zeros(3, dtype=torch.int32, device="cuda")
    out = torch.full((2, 4, 8), 7.0, device="cuda")
    gp, i, o = g.data_ptr(), idx.data_ptr(), out.data_ptr()
    f = lambda gp, ip, op, B, U, N, d: lib.mac_kb_gather_bwd(gp, ip, op, B, U, N, d, None)
    before = lib.mac_b200_launch_count()
    assert f(None, i, o, 3, 2, 4, 8) == INVALID and f(gp, None, o, 3, 2, 4, 8) == INVALID and f(gp, i, None, 3, 2, 4, 8) == INVALID
    assert f(gp, i, o, 0, 2, 4, 8) == INVALID and f(gp, i, o, 3, 0, 4, 8) == INVALID and f(gp, i, o, 3, 2, 4, -8) == INVALID
    assert f(gp, i, o, 3, 2, 8, 4) == UNSUPPORTED and f(gp, i, o, 3, 2, 1 << 30, 64) == UNSUPPORTED
    assert f(gp + 4, i, o, 3, 2, 4, 8) == ALIGN and f(gp, i + 4, o, 3, 2, 4, 8) == ALIGN and f(gp, i, o + 8, 3, 2, 4, 8) == ALIGN
    torch.cuda.synchronize()
    assert lib.mac_b200_launch_count() == before
    assert bool((out == 7.0).all())


# ------------------------------------------------------------------------------------------------ the stem through gather and sum
@pytest.mark.parametrize("k", [8, 16])
@pytest.mark.parametrize("prec", ["fp32", "bf16", "bf16x3"])
def test_stem_through_gather_and_sum_against_fp64_autograd(prec, k):
    from mac_network_b200.stem import SITE_STEM, Stem, init_stem_params, stem_specs
    lib = L_.load()
    B, H, W, cin, cout, keep, seed, step = 64, 14, 14, 1024, 512, 0.82, 13, 4
    params = {k_: torch.from_numpy(v).cuda() for k_, v in init_stem_params(stem_specs(cin, cout), seed=8).items()}
    gen = torch.Generator(device="cuda").manual_seed(9 + k)
    images = torch.relu(torch.randn(k, cin, H, W, device="cuda", generator=gen))
    rng = np.random.RandomState(k)
    pat = rng.randint(0, k, size=B)
    pat[rng.permutation(B)[:k]] = np.arange(k)                                   # every image has a question
    index = torch.from_numpy(pat.astype(np.int32)).cuda()
    st = Stem(params, relu="ELU", prec=prec, seed=seed)
    kb_u = st.forward_nchw(images, keep=keep, step=step, save_for_backward=True)
    N = H * W
    kb = torch.empty(B, N, cout, device="cuda")
    L_.check(lib.mac_kb_gather(L_.ptr(kb_u), L_.ptr(index), L_.ptr(kb), 0, B, k, N, cout, L_.stream_ptr()), "mac_kb_gather")
    d_kb = torch.randn(B, N, cout, device="cuda", generator=gen)                 # one upstream gradient per question
    d_kb_u = torch.empty(k, N, cout, device="cuda")
    L_.check(lib.mac_kb_gather_bwd(L_.ptr(d_kb), L_.ptr(index), L_.ptr(d_kb_u), B, k, N, cout, L_.stream_ptr()),
             "mac_kb_gather_bwd")
    grads = {k_: torch.zeros_like(v) for k_, v in params.items()}
    st.backward(d_kb_u, grads)
    torch.cuda.synchronize()
    assert torch.equal(kb, kb_u[index.long()])
    # the fp64 model: the per-image masks (the Philox numbering over the k-row tensor), each image's gradient summed over its
    # questions in fp64
    us = [mask_uniforms(_uniform_mask(lib, seed, SITE_STEM + i, step, (k, H, W, c), keep)) for i, c in ((0, cin), (1, cout))]
    d_ref = torch.zeros(k, N, cout, dtype=torch.float64, device="cuda").index_add_(0, index.long(), d_kb.double())
    kb_ref, gref, _ = stem_grads("ELU", params, images.permute(0, 2, 3, 1), keep, us, d_ref)
    errs = {"kb": _mr(kb, kb_ref[index.long()])}
    errs.update({n: _mr(grads[n], gref[n]) for n in gref})
    print("%s stem, %d images for %d questions: %s" % (prec, k, B, ", ".join(
        "%s %.2e" % (n.split("/")[1] + "/" + n.split("/")[-1] if "/" in n else n, v) for n, v in errs.items())))
    fwd, grad = (TOL_STEM_BF16, TOL_STEM_BF16) if prec == "bf16" else (BAR_FWD, BAR_GRAD)
    assert errs.pop("kb") < fwd
    bad = {n: v for n, v in errs.items() if not v < grad}
    assert not bad, bad


# ------------------------------------------------------------------------------------------------ the trainer
TRAINERS = {"bf16": dict(prec="bf16", bwd_tc=True, stem_prec="bf16"),
            "tc32_bf16x3": dict(prec="tc32", bwd_tc=True, stem_prec="bf16x3"),
            "tc32_fp32": dict(prec="tc32", bwd_tc=True, stem_prec="fp32")}
TB, TS, TV, TE, TD, TH, TW, TC, TA, TL = 16, 7, 13, 16, 128, 4, 4, 128, 8, 2     # TB*TH*TW % 64 == 0 (mac_read_bwd_tc)


def _trainer(config, stem_dropout):
    from mac_network_b200.dp import DPTrainer
    from tests.test_full_model import _make
    cfg, _ = _make(TB, TS, TV, TE, TD, TH, TW, TC, TA, TL, seed=0)
    return DPTrainer(cfg, TL, seed=7, lr=1e-3, classifier=(TA, [32]), encoder=(TV, TE), stem=(TC, 2),
                     stem_dropout=stem_dropout, **TRAINERS[config])


def _device_batch(seed):
    from tests.test_full_model import _make
    _, data = _make(TB, TS, TV, TE, TD, TH, TW, TC, TA, TL, seed=seed)
    dev = {k: torch.from_numpy(v).cuda() for k, v in data.items() if k != "images"}
    dev["images_nchw"] = torch.from_numpy(data["images"]).cuda().permute(0, 3, 1, 2).contiguous()
    return dev


def _same_trainer_state(a, b):
    for x, y, n in ((a.params.flat, b.params.flat, "flat"), (a.adam_m, b.adam_m, "adam_m"), (a.adam_v, b.adam_v, "adam_v"),
                    (a.ema, b.ema, "ema"), (a.norm, b.norm, "norm")):
        assert torch.equal(x, y), n
    assert a.step_id == b.step_id


@pytest.mark.parametrize("config", list(TRAINERS))
def test_identity_index_is_the_step_without_an_index(config):
    plain, indexed = _trainer(config, 0.82), _trainer(config, 0.82)
    for s in range(3):
        data = _device_batch(40 + s)
        ident = dict(data, imageIndex=torch.arange(TB, dtype=torch.int32, device="cuda"))
        lp, sp = plain.train_step_full("k", data, global_batch=TB)
        li, si = indexed.train_step_full("k", ident, global_batch=TB)
        torch.cuda.synchronize()
        assert torch.equal(lp, li) and torch.equal(sp, si), s
        assert torch.equal(plain.bucket, indexed.bucket), s
        _same_trainer_state(plain, indexed)


@pytest.mark.parametrize("config", list(TRAINERS))
def test_many_to_one_index_against_a_twin_fed_the_duplicated_images(config):
    """Stem keep 1.0 (the other dropouts as in training, numbered by question row in both arms).  The stems' products give
    each output row one CTA's k-loop whatever the row count (the fp32 stem above 64 rows), so the gathered knowledge base
    is the twin's bit for bit and so is everything computed from it; the stems' own gradients differ in summation order."""
    shared, twin = _trainer(config, 1.0), _trainer(config, 1.0)
    data = _device_batch(50)
    k = 6                                                        # 96 stem rows against the twin's 256
    rng = np.random.RandomState(5)
    pat = rng.randint(0, k, size=TB)
    pat[:k] = rng.permutation(k)
    index = torch.from_numpy(pat.astype(np.int32)).cuda()
    images_k = data["images_nchw"][:k].contiguous()
    ls, ss = shared.full_forward_backward("k", dict(data, images_nchw=images_k, imageIndex=index), global_batch=TB)
    lt, st = twin.full_forward_backward("k", dict(data, images_nchw=images_k[index.long()].contiguous()), global_batch=TB)
    torch.cuda.synchronize()
    assert torch.equal(ls, lt) and torch.equal(ss, st)
    p = shared.params
    errs, bar = {}, TOL_STEM_BF16 if TRAINERS[config]["stem_prec"] == "bf16" else BAR_GRAD
    for n in p.specs:
        o, size = p.offsets[n], int(np.prod(p.specs[n][0]))
        a, b = shared.bucket[o:o + size], twin.bucket[o:o + size]
        if n.startswith("stem/"):
            errs[n] = _mr(a, b)
        else:
            assert torch.equal(a, b), n
    print("%s: stem gradients, %d images against %d duplicated rows: %s" % (config, k, TB, ", ".join(
        "%s %.2e" % (n.split("/")[1] + "/" + n.split("/")[-1], v) for n, v in errs.items())))
    assert len(errs) == 4
    bad = {n: v for n, v in errs.items() if not v < bar}
    assert not bad, bad


# ------------------------------------------------------------------------------------------------ the pipeline
U = 5


def _shared_batches(ks, seed):
    from tests.test_gpu_train_pipeline import _batches
    rng = np.random.RandomState(seed)
    out = []
    for b, k in zip(_batches(len(ks), seed=seed), ks):
        pat = rng.randint(0, k, size=b["questions"].shape[0]).astype(np.int32)
        pat[rng.permutation(len(pat))[:k]] = np.arange(k)
        out.append(dict(b, images=np.ascontiguousarray(b["images"][:k]), imageIndex=pat))
    return out


def _direct_step(net, b):
    """train_step_full on device copies of the batch, trimmed as the pipeline trims it; the pipeline's reported values."""
    t = net.trainer
    S = int(b["questionLengths"].max())
    B = b["questions"].shape[0]
    data = {"questions": torch.from_numpy(np.ascontiguousarray(b["questions"][:, :S])).cuda(),
            "questionLengths": torch.from_numpy(b["questionLengths"]).cuda(),
            "answers": torch.from_numpy(b["answers"]).cuda(),
            "images_nchw": torch.from_numpy(np.asarray(b["images"])).cuda(),
            "imageIndex": torch.from_numpy(b["imageIndex"]).cuda()}
    logits, losses = t.train_step_full((B, S), data, global_batch=B * t.world)
    preds = torch.argmax(logits, dim=-1).to(torch.int32)
    return {"loss": float(losses.mean()), "correctNum": int((preds == data["answers"]).sum()), "gradNorm": float(t.norm[0]),
            "predictions": preds.cpu()}


@pytest.mark.parametrize("config", ["fp32", "all_tc", "tc32"])
def test_pipeline_with_images_equals_direct_steps_bit_for_bit(config):
    from mac_network_b200.serving import TrainPipeline
    from tests.test_gpu_train_pipeline import BS, HW, SMAX, _net, _pinned, _same_state
    net, twin = _net(config), _net(config)
    pipe = TrainPipeline(net, (BS, SMAX, HW, HW), depth=2, stage_threads=3, images=U)
    for i, b in enumerate(_shared_batches([U, U - 3, 1, U, U - 3, 1], seed=91)):
        got = pipe.result(pipe.submit(_pinned(b) if i % 2 else b))     # numpy and pinned images alternate
        want = _direct_step(twin, b)
        assert (got["loss"], got["correctNum"], got["gradNorm"]) == (want["loss"], want["correctNum"], want["gradNorm"]), i
        assert torch.equal(got["predictions"], want["predictions"]), i
        pipe.drain()
        _same_state(net, twin)


@pytest.mark.parametrize("stem_prec", ["fp32", "bf16", "bf16x3"])
def test_pipeline_with_images_launches_two_more_per_step(stem_prec):
    """The gather and the per-image sum are the only launches an indexed step adds to the step on duplicated features."""
    from mac_network_b200.serving import TrainPipeline
    from tests.test_gpu_train_pipeline import BS, HW, SMAX, _net_with
    lib = L_.load()
    net, twin = _net_with(stem_prec), _net_with(stem_prec)
    pipe = TrainPipeline(net, (BS, SMAX, HW, HW), depth=2, images=U)
    plain = TrainPipeline(twin, (BS, SMAX, HW, HW), depth=2)
    counts = {"shared": [], "plain": []}
    for b in _shared_batches([U, 2, U], seed=93):
        n0 = lib.mac_b200_launch_count()
        pipe.result(pipe.submit(b))
        counts["shared"].append(lib.mac_b200_launch_count() - n0)
        dup = {k: v for k, v in b.items() if k != "imageIndex"}
        dup["images"] = np.ascontiguousarray(b["images"][b["imageIndex"]])
        n0 = lib.mac_b200_launch_count()
        plain.result(plain.submit(dup))
        counts["plain"].append(lib.mac_b200_launch_count() - n0)
    assert [s - p for s, p in zip(counts["shared"], counts["plain"])] == [2] * 3, (stem_prec, counts)
