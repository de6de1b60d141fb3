"""Whole-model training from host buffers (serving.TrainPipeline) and the training ingest under it, on the GPU.

- mac_ingest_nchw_train, both patch forms, bit for bit permute + mac_im2col3x3(cols_bf16 = 1) / mac_im2col3x3_split, NHWC
  output included, at keep 1, 0.82 and 0.5 and the shapes the stem meets (1024x14x14, 2048x7x7, B = 1, odd and 1x1 images,
  64..192 channels); canary bytes around both outputs stay; refusals leave the outputs untouched.
- Stem.forward_nchw in training: forward, saved tensors, weight and image gradients bit for bit the NHWC path's.
- The pipeline against a twin MACnet looping over runBatch(train=True): loss, correctNum, gradNorm, predictions, then
  weights, Adam m / v and EMA, bit for bit, over pageable and pinned batches of three question lengths; with drained
  evaluations (live and EMA) between steps and across save_training_state / resume; library launches per step."""
import numpy as np
import pytest
import torch

from tests.test_gpu_model_pipeline import _features

pytestmark = pytest.mark.gpu

INVALID, ALIGN, UNSUPPORTED = -1, -2, -3
CANARY = 16                     # elements of sentinel on each side of an output


def _lib():
    from mac_network_b200 import _lib as L_
    return L_, L_.load()


def _padded(n, dtype, fill):
    buf = torch.full((n + 2 * CANARY,), fill, dtype=dtype, device="cuda")
    return buf, buf[CANARY:CANARY + n]


def _untouched(buf, n, fill):
    return bool((buf[:CANARY] == fill).all()) and bool((buf[CANARY + n:] == fill).all())


@pytest.mark.parametrize("keep", [1.0, 0.82, 0.5])
@pytest.mark.parametrize("B,C,H,W", [(64, 1024, 14, 14), (64, 2048, 7, 7), (1, 64, 14, 14), (3, 128, 5, 3), (2, 192, 1, 1),
                                     (5, 64, 3, 5)])
def test_ingest_train_equals_permute_and_patch_passes(B, C, H, W, keep):
    L_, lib = _lib()
    x = _features(B, C, H, W, seed=B + C + H)
    nhwc = x.permute(0, 2, 3, 1).contiguous()
    M, K = B * H * W, 9 * C
    seed, site, step = 0x1234567890AB, 32, 7
    for form in (0, 1):
        width = K * (2 if form else 1)
        want = torch.empty((M, width), dtype=torch.bfloat16, device="cuda")
        if form:
            L_.check(lib.mac_im2col3x3_split(L_.ptr(nhwc), L_.ptr(want), keep, seed, site, step, B, H, W, C, L_.stream_ptr()),
                     "mac_im2col3x3_split")
        else:
            L_.check(lib.mac_im2col3x3(L_.ptr(nhwc), L_.ptr(want), 1, keep, seed, site, step, B, H, W, C, L_.stream_ptr()),
                     "mac_im2col3x3")
        ybuf, y = _padded(nhwc.numel(), torch.float32, -3.0)
        cbuf, cols = _padded(M * width, torch.bfloat16, -5.0)
        st = lib.mac_ingest_nchw_train(L_.ptr(x), L_.ptr(y), L_.ptr(cols), form, keep, seed, site, step, B, C, H, W,
                                       L_.stream_ptr())
        assert st == 0
        assert torch.equal(y.view(B, H, W, C), nhwc), form
        assert torch.equal(cols.view(M, width).view(torch.int16), want.view(torch.int16)), (form, keep)
        assert _untouched(ybuf, y.numel(), -3.0) and _untouched(cbuf, cols.numel(), -5.0), form
        if keep < 1:                                 # the mask did something, and what it dropped is exactly 0
            dropped = (cols.view(M, width)[:, :K] == 0).float().mean().item()
            assert dropped > (1 - keep) * 0.5, dropped
        del want, cols, cbuf
    torch.cuda.synchronize()


def test_ingest_train_refusals_leave_the_outputs_untouched():
    L_, lib = _lib()
    x = torch.ones(2, 64, 3, 3, device="cuda")
    y = torch.full((2, 3, 3, 64), 7.0, device="cuda")
    cols = torch.full((18, 18 * 64), 7.0, dtype=torch.bfloat16, device="cuda")
    p, o, c = x.data_ptr(), y.data_ptr(), cols.data_ptr()
    before = lib.mac_b200_launch_count()

    def call(xp=p, op=o, cp=c, form=0, keep=0.82, B=2, C=64, H=3, W=3):
        return lib.mac_ingest_nchw_train(xp, op, cp, form, keep, 1, 32, 0, B, C, H, W, None)
    assert call(xp=None) == INVALID and call(op=None) == INVALID and call(cp=None) == INVALID
    assert call(keep=0.0) == INVALID and call(keep=1.5) == INVALID and call(B=0) == INVALID
    assert call(xp=p + 4) == ALIGN and call(op=o + 4) == ALIGN and call(cp=c + 2) == ALIGN
    assert call(C=96) == UNSUPPORTED and call(form=2) == UNSUPPORTED and call(B=70000) == UNSUPPORTED
    assert call(H=40, W=40) == UNSUPPORTED and call(form=1, H=17, W=17) == UNSUPPORTED
    torch.cuda.synchronize()
    assert lib.mac_b200_launch_count() == before
    assert bool((y == 7.0).all()) and bool((cols == 7.0).all())


@pytest.mark.parametrize("prec", ["fp32", "bf16", "bf16x3"])
def test_stem_forward_nchw_training_equals_the_nhwc_path(prec):
    from mac_network_b200.stem import Stem, init_stem_params, stem_specs
    B, C, H, W = 3, 128, 7, 7
    p = {k: torch.from_numpy(v).cuda() for k, v in init_stem_params(stem_specs(C, 128), seed=6, bias_scale=0.1).items()}
    x = _features(B, C, H, W, seed=12)
    g = torch.Generator(device="cuda").manual_seed(3)
    d_kb = torch.randn(B, H * W, 128, device="cuda", generator=g)
    res = []
    for nchw in (False, True):
        st = Stem(p, relu="ELU", prec=prec, seed=41)
        if nchw:
            kb = st.forward_nchw(x, keep=0.82, step=5, save_for_backward=True)
        else:
            kb = st.forward(x.permute(0, 2, 3, 1).contiguous(), keep=0.82, step=5, save_for_backward=True)
        grads = {k: torch.zeros_like(v) for k, v in p.items()}
        d_img = st.backward(d_kb, grads, need_d_images=True)
        torch.cuda.synchronize()
        res.append((kb, st._saved, grads, d_img))
    (kb0, s0, g0, d0), (kb1, s1, g1, d1) = res
    assert torch.equal(kb0, kb1)
    for k in ("xs", "ys"):
        assert all(torch.equal(a, b) for a, b in zip(s0[k], s1[k])), k
    assert all(torch.equal(g0[k], g1[k]) for k in g0)
    assert torch.equal(d0, d1)
    assert not torch.equal(kb1, Stem(p, relu="ELU", prec=prec, seed=41).forward_nchw(x))       # the dropout was applied


# ------------------------------------------------------------------------------------------------ the pipeline
CONFIGS = {"fp32": dict(),
           "all_tc": dict(train_prec="bf16", bwd_tc=True, stem_prec="bf16", enc_prec="bf16"),
           "tc32": dict(train_prec="tc32", bwd_tc=True, stem_prec="bf16x3")}
V, E, C, A, L = 90, 300, 128, 28, 3
BS, SMAX, HW = 8, 12, 8          # B * H * W a multiple of 64: the bf16 tensor-core read backward
LENGTHS = [12, 7, 12, 4, 7, 4]                  # six steps over three trimmed question lengths
HP = dict(lr=1e-3, clip=1.0, ema_decay=0.99)


def _net(config, seed=3):
    from mac_network_b200.config import MACConfig
    from mac_network_b200.model import MACnet
    cfg = MACConfig.args("args", netLength=L)
    return MACnet(cfg, L, V, A, wrd_emb_dim=E, image_in_dim=C, classifier_dims=(512,), seed=seed, prec="bf16", **HP,
                  **CONFIGS[config])


def _batches(n, seed=61):
    rng = np.random.RandomState(seed)
    out = []
    for i in range(n):
        longest = LENGTHS[i % len(LENGTHS)]
        lengths = rng.randint(1, longest + 1, size=(BS,)).astype(np.int32)
        lengths[rng.randint(BS)] = longest
        q = rng.randint(1, V + 1, size=(BS, SMAX)).astype(np.int32)
        q[np.arange(SMAX)[None, :] >= lengths[:, None]] = 0
        out.append({"questions": q, "questionLengths": lengths, "answers": rng.randint(0, A, size=(BS,)).astype(np.int32),
                    "images": np.maximum(rng.standard_normal((BS, C, HW, HW)), 0).astype(np.float32)})
    return out


def _pinned(b):
    return dict(b, images=torch.from_numpy(b["images"]).pin_memory())


def _twin_step(net, b):
    r = net.runBatch(None, {k: b[k] for k in ("questions", "questionLengths", "answers")}, {"images": b["images"]}, train=True)
    return {"loss": r["loss"], "correctNum": r["correctNum"], "gradNorm": r["gradNorm"],
            "predictions": [p["prediction"] for p in r["preds"]]}


def _same_state(a, b):
    ta, tb = a.trainer, b.trainer
    for x, y, k in ((ta.params.flat, tb.params.flat, "flat"), (ta.adam_m, tb.adam_m, "adam_m"), (ta.adam_v, tb.adam_v, "adam_v"),
                    (ta.ema, tb.ema, "ema")):
        assert torch.equal(x, y), k
    assert ta.step_id == tb.step_id


def _check(got, want, pipe, i):
    assert (got["loss"], got["correctNum"], got["gradNorm"]) == (want["loss"], want["correctNum"], want["gradNorm"]), i
    assert got["acc"] == want["correctNum"] / BS
    assert pipe.predictions(got) == want["predictions"], i


@pytest.mark.parametrize("config", list(CONFIGS))
def test_pipeline_equals_run_batch_training_bit_for_bit(config):
    from mac_network_b200.serving import TrainPipeline
    net, twin = _net(config), _net(config)
    batches = _batches(6)
    pipe = TrainPipeline(net, (BS, SMAX, HW, HW), depth=2, stage_threads=3)
    tickets, wants = [], []
    for i, b in enumerate(batches):
        tickets.append(pipe.submit(_pinned(b) if i % 2 else b))           # pageable and pinned batches alternate
        wants.append(_twin_step(twin, b))
        if i >= 1:                                                        # read each result before its slot is taken again
            _check(pipe.result(tickets[i - 1]), wants[i - 1], pipe, i - 1)
    _check(pipe.result(tickets[-1]), wants[-1], pipe, len(batches) - 1)
    pipe.drain()
    _same_state(net, twin)
    assert sorted(k[1] for k in net.trainer._cells) == [4, 7, 12]


@pytest.mark.parametrize("config", ["fp32", "tc32"])
def test_pipeline_with_evaluations_between_steps_and_resume(config, tmp_path):
    """Drained runBatch(train=False) on the live weights and on the EMA shadows between steps equal the twin's and do not
    disturb training; a training state saved after a drain and loaded into a fresh model continues in a new pipeline
    exactly as the uninterrupted twin does."""
    from mac_network_b200.checkpoint import load_training_state, save_training_state
    from mac_network_b200.serving import TrainPipeline
    from tests.test_gpu_model_pipeline import _reference
    net, twin = _net(config), _net(config)
    batches = _batches(6, seed=71)
    ev = {k: batches[0][k] for k in ("questions", "questionLengths", "images")}
    pipe = TrainPipeline(net, (BS, SMAX, HW, HW), depth=2)
    for i, b in enumerate(batches[:3]):
        t = pipe.submit(b)
        want = _twin_step(twin, b)
        _check(pipe.result(t), want, pipe, i)
        pipe.drain()
        for use_ema in (False, True):
            net.use_ema = twin.use_ema = use_ema
            got, ref = _reference(net, ev), _reference(twin, ev)
            net.use_ema = twin.use_ema = False
            for k in ref:
                assert np.array_equal(got[k], ref[k]), (i, use_ema, k)
        _same_state(net, twin)
    path = str(tmp_path / "state")
    save_training_state(path, net.trainer)
    fresh = _net(config)
    assert load_training_state(path, fresh.trainer) == 3
    pipe2 = TrainPipeline(fresh, (BS, SMAX, HW, HW), depth=2)
    for i, b in enumerate(batches[3:], 3):
        t = pipe2.submit(_pinned(b))
        _check(pipe2.result(t), _twin_step(twin, b), pipe2, i)
    pipe2.drain()
    _same_state(fresh, twin)


@pytest.mark.parametrize("stem_prec,extra", [("fp32", 1), ("bf16", 0), ("bf16x3", 0)])
def test_pipeline_launches_per_step(stem_prec, extra):
    """The training ingest replaces the permute (a torch kernel) and layer 0's patch pass: as many library launches per step
    as runBatch for the bf16 and bf16x3 stems; one more for the fp32 stem (the NHWC ingest in place of torch's permute)."""
    from mac_network_b200.serving import TrainPipeline
    L_, lib = _lib()
    net, twin = _net_with(stem_prec), _net_with(stem_prec)
    pipe = TrainPipeline(net, (BS, SMAX, HW, HW), depth=2)
    counts = {"pipe": [], "run": []}
    for b in _batches(3, seed=81):
        n0 = lib.mac_b200_launch_count()
        pipe.result(pipe.submit(b))
        counts["pipe"].append(lib.mac_b200_launch_count() - n0)
        n0 = lib.mac_b200_launch_count()
        _twin_step(twin, b)
        counts["run"].append(lib.mac_b200_launch_count() - n0)
    assert [p - r for p, r in zip(counts["pipe"], counts["run"])] == [extra] * 3, (stem_prec, counts)
    pipe.drain()
    _same_state(net, twin)


def _net_with(stem_prec):
    from mac_network_b200.config import MACConfig
    from mac_network_b200.model import MACnet
    cfg = MACConfig.args("args", netLength=L)
    return MACnet(cfg, L, V, A, wrd_emb_dim=E, image_in_dim=C, classifier_dims=(512,), seed=3, prec="bf16", stem_prec=stem_prec,
                  **HP)
