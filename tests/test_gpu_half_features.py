"""Image features stored in fp16, on the GPU.  Every comparison is bit for bit against the fp32 path fed `x.float()`:

- mac_ingest_nchw_f16 (both modes) and mac_ingest_nchw_train_f16 (both forms, keep 1 and 0.82) against the fp32 entry
  points, at B = 1 and 64, C = 64, 1024 and 2048, H x W = 1x1, 7x7, 13x17, 14x14, 8x32 and the largest each accepts, with
  fp16 subnormals, +-0, +-65504, infinities and NaNs in the input; every output element written, the guard bytes around
  every output untouched.
- Stem.forward_nchw of fp16 images: the result, the saved tensors and the backward's gradients, for every precision.
- ModelPipeline(image_dtype=torch.float16) against the fp32 pipeline (bf16 and e4m3 forms, CLEVR and GQA shapes, with
  images=None, images=U and cache=C), every output; TrainPipeline over two steps; MACModel's forward and backward.
- The cost of the storage itself: the stem's output from fp16-rounded features against fp32 features, bounded."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GUARD = 256          # guard elements on each side of every output (a multiple of 16 bytes for every element size)
FILL = 0xA5


def _lib():
    from mac_network_b200 import _lib as L_
    return L_, L_.load()


def _half_features(B, C, H, W, seed):
    """fp16 NCHW features: a spread of normal values with subnormals, +-0, +-65504, infinities and NaNs (two payloads, both
    signs) planted at interior and border pixels."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.randn(B, C, H, W, device="cuda", generator=g) * 8).half()
    flat = x.view(-1).view(torch.int16)
    n = flat.numel()
    sub = torch.randint(1, 1024, (n,), device="cuda", generator=g, dtype=torch.int16)
    sub = sub | (torch.randint(0, 2, (n,), device="cuda", generator=g, dtype=torch.int16) << 15)
    flat[::7] = sub[::7]                                                          # subnormals of both signs
    special = torch.tensor([0x0000, -0x8000, 0x7bff, -0x0401, 0x7c00, -0x0400, 0x7e00, 0x7c01, -0x0200, 0x7fff,
                            0x0001, -0x7fff, 0x03ff, 0x0400], dtype=torch.int16, device="cuda")
    pos = torch.randint(0, n, (max(64, n // 50),), device="cuda", generator=g)
    flat[pos] = special[torch.arange(pos.numel(), device="cuda") % special.numel()]
    flat[:special.numel()] = special                                              # the first pixel's channels
    flat[-special.numel():] = special                                             # the last pixel's
    return x


def _guarded(n, dtype):
    buf = torch.empty(n + 2 * GUARD, dtype=dtype, device="cuda")
    buf.view(torch.uint8).fill_(FILL)
    return buf, buf[GUARD:GUARD + n]


def _guards_untouched(buf):
    raw = buf.view(torch.uint8)
    k = GUARD * buf.element_size()
    return bool((raw[:k] == FILL).all()) and bool((raw[-k:] == FILL).all())


def _bits(t):
    return t.view(torch.int32) if t.element_size() == 4 else t.view(torch.int16)


def _ref_fill(out):
    out.view(torch.uint8).fill_(0x5A)          # another pattern: an element neither call writes differs


SHAPES = [(1, 64, 1, 1), (64, 64, 7, 7), (1, 1024, 13, 17), (64, 1024, 14, 14), (1, 2048, 8, 32), (64, 2048, 1, 1),
          (1, 2048, 14, 14), (64, 64, 13, 17)]
LARGEST = {"nhwc": (20, 29), "patch": (14, 61), "cols": (7, 61), "split": (337, 1)}       # 580, 854, 427, 337 pixels


@pytest.mark.parametrize("mode", ["nhwc", "patch"])
@pytest.mark.parametrize("B,C,H,W", SHAPES + [(2, 128, "largest", None)])
def test_ingest_f16_equals_fp32_ingest_of_the_widened_features(mode, B, C, H, W):
    L_, lib = _lib()
    if H == "largest":
        H, W = LARGEST[mode]
    m = 0 if mode == "nhwc" else 1
    x16 = _half_features(B, C, H, W, seed=B * 31 + C + H * 7 + W)
    x32 = x16.float()
    n, dt = (B * H * W * C, torch.float32) if m == 0 else (B * H * W * 9 * C, torch.bfloat16)
    buf, out = _guarded(n, dt)
    ref = torch.empty(n, dtype=dt, device="cuda")
    _ref_fill(ref)
    s = L_.stream_ptr()
    assert lib.mac_ingest_nchw_f16(L_.ptr(x16), L_.ptr(out), m, B, C, H, W, s) == 0
    st = lib.mac_ingest_nchw(L_.ptr(x32), 0, L_.ptr(ref), m, B, C, H, W, s)
    if st != 0:         # beyond the fp32 slab's limit: the fp32 stem's own path, permute and mac_im2col3x3
        assert st == -3 and (H, W) == LARGEST[mode]
        nhwc = x32.permute(0, 2, 3, 1).contiguous()
        if m == 0:
            ref.copy_(nhwc.view(-1))
        else:
            assert lib.mac_im2col3x3(L_.ptr(nhwc), L_.ptr(ref), 1, 1.0, 0, 32, 0, B, H, W, C, s) == 0
    torch.cuda.synchronize()
    assert torch.equal(_bits(out), _bits(ref))
    assert _guards_untouched(buf)
    if m == 0:          # the widening itself: NHWC of x.float(), NaN payloads included
        assert torch.equal(_bits(out.view(B, H, W, C)), _bits(x32.permute(0, 2, 3, 1).contiguous()))
    if (H, W) == LARGEST[mode]:                         # one pixel more is refused
        assert lib.mac_ingest_nchw_f16(L_.ptr(x16), L_.ptr(out), m, B, C, 1, H * W + 1, s) == -3


@pytest.mark.parametrize("keep", [1.0, 0.82])
@pytest.mark.parametrize("form", ["cols", "split"])
@pytest.mark.parametrize("B,C,H,W", SHAPES + [(2, 128, "largest", None)])
def test_ingest_train_f16_equals_fp32_training_ingest(form, keep, B, C, H, W):
    L_, lib = _lib()
    if H == "largest":
        H, W = LARGEST[form]
    f = 0 if form == "cols" else 1
    x16 = _half_features(B, C, H, W, seed=B * 37 + C + H * 5 + W + f)
    x32 = x16.float()
    n_x, n_c = B * H * W * C, B * H * W * 9 * C * (2 if f else 1)
    xbuf, xo = _guarded(n_x, torch.float32)
    cbuf, co = _guarded(n_c, torch.bfloat16)
    xr, cr = torch.empty(n_x, device="cuda"), torch.empty(n_c, dtype=torch.bfloat16, device="cuda")
    _ref_fill(xr)
    _ref_fill(cr)
    s = L_.stream_ptr()
    args = (f, keep, 1234567, 32, 3, B, C, H, W, s)
    assert lib.mac_ingest_nchw_train_f16(L_.ptr(x16), L_.ptr(xo), L_.ptr(co), *args) == 0
    st = lib.mac_ingest_nchw_train(L_.ptr(x32), L_.ptr(xr), L_.ptr(cr), *args)
    if st != 0:         # beyond the fp32 slab's limit: the stem's own path, permute and the patch pass with the same mask
        assert st == -3 and (H, W) == LARGEST[form]
        xr.copy_(x32.permute(0, 2, 3, 1).contiguous().view(-1))
        if f:
            assert lib.mac_im2col3x3_split(L_.ptr(xr), L_.ptr(cr), keep, 1234567, 32, 3, B, H, W, C, s) == 0
        else:
            assert lib.mac_im2col3x3(L_.ptr(xr), L_.ptr(cr), 1, keep, 1234567, 32, 3, B, H, W, C, s) == 0
    torch.cuda.synchronize()
    assert torch.equal(_bits(xo), _bits(xr)) and torch.equal(_bits(co), _bits(cr))
    assert _guards_untouched(xbuf) and _guards_untouched(cbuf)
    if (H, W) == LARGEST[form]:
        assert lib.mac_ingest_nchw_train_f16(L_.ptr(x16), L_.ptr(xo), L_.ptr(co), f, keep, 1, 32, 3, B, C, 1, H * W + 1, s) == -3
        torch.cuda.synchronize()
        assert torch.equal(_bits(xo), _bits(xr)) and _guards_untouched(xbuf)


# ------------------------------------------------------------------------------------------------ the stem
def _stem(prec, C=256, out=128, seed=41):
    from mac_network_b200.stem import Stem, init_stem_params, stem_specs
    p = {k: torch.from_numpy(v).cuda() for k, v in init_stem_params(stem_specs(C, out), seed=6).items()}
    return Stem(p, relu="ELU", prec=prec, seed=seed), p


def _features(B, C, H, W, seed):
    rng = np.random.RandomState(seed)
    return torch.from_numpy(np.maximum(rng.standard_normal((B, C, H, W)), 0).astype(np.float16)).cuda()


@pytest.mark.parametrize("prec", ["fp32", "bf16", "bf16x3", "fp8"])
@pytest.mark.parametrize("B,H,W", [(4, 14, 14), (3, 7, 7)])
def test_stem_inference_from_fp16_features(prec, B, H, W):
    st, _ = _stem(prec)
    x16 = _features(B, 256, H, W, seed=B + H)
    assert torch.equal(_bits(st.forward_nchw(x16)), _bits(st.forward_nchw(x16.float())))


@pytest.mark.parametrize("prec", ["fp32", "bf16", "bf16x3"])
def test_stem_training_from_fp16_features(prec):
    st, p = _stem(prec)
    x16 = _features(4, 256, 8, 8, seed=5)
    runs = []
    for x in (x16.float(), x16):
        kb = st.forward_nchw(x, keep=0.82, step=3, save_for_backward=True)
        saved = {k: [t.clone() for t in st._saved[k]] for k in ("xs", "ys")}
        grads = {k: torch.zeros_like(v) for k, v in p.items()}
        d_kb = torch.from_numpy(np.random.RandomState(9).standard_normal(tuple(kb.shape)).astype(np.float32)).cuda()
        dx = st.backward(d_kb, grads, need_d_images=True)
        torch.cuda.synchronize()
        runs.append((kb, saved, grads, dx))
    (kb0, s0, g0, d0), (kb1, s1, g1, d1) = runs
    assert torch.equal(_bits(kb0), _bits(kb1))
    for k in ("xs", "ys"):
        assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(s0[k], s1[k])), k
    assert all(torch.equal(_bits(g0[k]), _bits(g1[k])) for k in g0)
    assert torch.equal(_bits(d0), _bits(d1))


# ------------------------------------------------------------------------------------------------ ModelPipeline
def _as_half(b):
    return dict(b, images=b["images"].astype(np.float16))


def _widened(b):
    return dict(b, images=b["images"].astype(np.float32))


def _same_outputs(a, b):
    assert set(a) == set(b)
    for k in a:
        assert torch.equal(a[k], b[k]), k


def _run(pipe, batches):
    outs = []
    for b in batches:       # one slot's results are read before it is taken again: copy them out
        outs.append({k: v.clone() for k, v in pipe.result(pipe.submit(b)).items()})
    pipe.drain()
    return outs


@pytest.mark.parametrize("variant,H,W", [("args", 14, 14), ("gqa", 7, 7)])
@pytest.mark.parametrize("model", ["bf16", "fp8"])
@pytest.mark.parametrize("arm", ["plain", "images", "cache"])
def test_model_pipeline_f16_equals_the_fp32_pipeline(variant, H, W, model, arm):
    from mac_network_b200.serving import ModelPipeline
    from tests.test_gpu_model_pipeline import _batches, _net
    B, S, L, U = 8, 10, 3, 3
    net = _net(variant, model, L)
    base = [_as_half(b) for b in _batches(6, B, S, H, W, seed=23, longest=S)]
    kw = {}
    if arm == "plain":
        b16 = base
    elif arm == "images":
        kw = dict(images=U)
        idx = np.random.RandomState(4).randint(0, U, size=(len(base), B)).astype(np.int32)
        b16 = [dict(b, images=b["images"][:U], imageIndex=idx[i]) for i, b in enumerate(base)]
    else:
        kw = dict(images=U, cache=2 * B)
        store = np.maximum(np.random.RandomState(8).standard_normal((24, 128, H, W)), 0).astype(np.float16)
        ids = np.random.RandomState(5).randint(0, 24, size=(len(base), B))

        def loader(dtype):
            return lambda m: store[m].astype(dtype)
    if arm == "cache":
        mk = lambda i, dt: {"questions": base[i]["questions"], "questionLengths": base[i]["questionLengths"],
                            "imageIds": ids[i], "images": loader(dt)}
        b16 = [mk(i, np.float16) for i in range(len(base))]
        b32 = [mk(i, np.float32) for i in range(len(base))]
    else:
        b32 = [_widened(b) for b in b16]
    pipe16 = ModelPipeline(net, (B, S, H, W), slots=4, topk=3, image_dtype=torch.float16, **kw)
    pipe32 = ModelPipeline(net, (B, S, H, W), slots=4, topk=3, host_cast=False, **kw)
    assert pipe16.slots[0].x["images"].dtype == torch.float16 and pipe32.slots[0].x["images"].dtype == torch.float32
    k = B if arm == "plain" else U
    if arm != "cache":
        assert pipe32.h2d_bytes - pipe16.h2d_bytes == k * 128 * H * W * 2
    for a, b in zip(_run(pipe16, b16), _run(pipe32, b32)):
        _same_outputs(a, b)
    if arm == "cache":
        s16, s32 = pipe16.cache_stats(), pipe32.cache_stats()
        assert s16["image_bytes"] * 2 == s32["image_bytes"] and s16["misses"] == s32["misses"] > 0 and s16["hits"] > 0


# ------------------------------------------------------------------------------------------------ TrainPipeline
@pytest.mark.parametrize("config", ["all_tc", "tc32", "fp32"])
@pytest.mark.parametrize("images", [None, 3])
def test_train_pipeline_f16_equals_the_fp32_pipeline(config, images):
    from mac_network_b200.serving import TrainPipeline
    from tests.test_gpu_train_pipeline import BS, HW, SMAX, _batches, _net, _same_state
    net16, net32 = _net(config), _net(config)
    batches = [_as_half(b) for b in _batches(2, seed=67)]
    if images is not None:
        idx = np.random.RandomState(2).randint(0, images, size=(2, BS)).astype(np.int32)
        batches = [dict(b, images=b["images"][:images], imageIndex=idx[i]) for i, b in enumerate(batches)]
    p16 = TrainPipeline(net16, (BS, SMAX, HW, HW), depth=2, images=images, image_dtype=torch.float16)
    p32 = TrainPipeline(net32, (BS, SMAX, HW, HW), depth=2, images=images)
    for i, b in enumerate(batches):
        src = dict(b, images=torch.from_numpy(b["images"]).pin_memory()) if i % 2 else b      # pageable, then pinned
        r16 = p16.result(p16.submit(src))
        r32 = p32.result(p32.submit(_widened(b)))
        assert (r16["loss"], r16["gradNorm"], r16["correctNum"]) == (r32["loss"], r32["gradNorm"], r32["correctNum"]), i
        assert torch.equal(r16["predictions"], r32["predictions"])
    p16.drain()
    p32.drain()
    _same_state(net16, net32)


# ------------------------------------------------------------------------------------------------ MACModel
@pytest.mark.parametrize("kw", [dict(), dict(prec="bf16", bwd_tc=True, stem_prec="bf16", enc_prec="bf16")])
def test_mac_model_forward_and_backward_from_fp16_features(kw):
    from mac_network_b200.modules import MACModel, answer_loss
    from tests.test_gpu_modules import B, S, _data, _trainer
    t = _trainer("args", 512 if kw else 128, kw)
    models = [MACModel.from_trainer(t), MACModel.from_trainer(t)]
    data = _data(2)
    x16 = data["images_nchw"].half()
    res = []
    for m, x in zip(models, (x16.float(), x16)):
        x = x.clone().requires_grad_(True)
        logits, memory = m(data["questions"], data["questionLengths"], images_nchw=x)
        answer_loss(logits, data["answers"]).backward()
        torch.cuda.synchronize()
        res.append((logits.detach(), memory.detach(), {n: p.grad.clone() for n, p in m.named_parameters()}, x.grad))
    (l0, m0, g0, d0), (l1, m1, g1, d1) = res
    assert torch.equal(l0, l1) and torch.equal(m0, m1)
    assert all(torch.equal(g0[n], g1[n]) for n in g0)
    assert d1.dtype == torch.float16 and torch.equal(_bits(d1), _bits(d0.half()))       # autograd's cast to the input dtype
    with torch.no_grad():
        e0 = models[0](data["questions"], data["questionLengths"], images_nchw=x16.float())
        e1 = models[1](data["questions"], data["questionLengths"], images_nchw=x16)
    assert torch.equal(e0[0], e1[0]) and torch.equal(e0[1], e1[1])


# ------------------------------------------------------------------------------------------------ the storage error
# max-norm relative error of the stem's output from fp16-rounded features against fp32 features, B = 64, 1024 x 14 x 14 ->
# 512, ReLU-like features; measured on an H100 80GB HBM3 by profiles/half_features.py (profiles/half_features_h100.json)
# (2.0e-4 fp32, 2.0e-4 bf16x3, 2.3e-3 bf16, 1.7e-2 fp8); the bars are about three times those
STORAGE_BOUND = {"fp32": 6e-4, "bf16x3": 6e-4, "bf16": 7e-3, "fp8": 5e-2}


@pytest.mark.parametrize("prec", list(STORAGE_BOUND))
def test_fp16_storage_error_of_the_stem_output_is_bounded(prec):
    st, _ = _stem(prec, C=1024, out=512)
    x = torch.from_numpy(np.maximum(np.random.RandomState(3).standard_normal((64, 1024, 14, 14)), 0).astype(np.float32)).cuda()
    kb32 = st.forward_nchw(x).double()
    kb16 = st.forward_nchw(x.half()).double()
    err = float((kb16 - kb32).abs().max() / kb32.abs().max())
    assert err < STORAGE_BOUND[prec], (prec, err)
