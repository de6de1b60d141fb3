"""The stem's kernel sizes, strides and linear form on the GPU (--stemKernelSize(s), --stemStrideSizes, --stemLinear).

- mac_im2col at k = 3, s = 1: bit for bit mac_im2col3x3 (fp32, bf16) and mac_im2col3x3_split; at every other geometry bit
  for bit a host restatement with the Philox keep-mask; mac_im2col_t bit for bit the transpose of the bf16 / split patch
  matrix with zero padding columns (odd M); mac_col2im against fp64; reruns bit-identical.
- Stem(prec="fp32") against every geometry fixture of the reference (forward 1e-4, gradients 2e-4 of each tensor's maximum,
  training fixtures with the device's own masks); bf16x3 inside the same bars and bf16 inside the bf16 stem's bounds, against
  fp64 autograd at B = 64, 1024 -> 512 -> 512 on the 14 x 14 grid.
- MACnet.runBatch(train=False) against ModelPipeline bit for bit with a stride-2 and a linear stem, with and without
  images=U / cache=C; attention maps on the stem's output grid.
- Refusals before any launch."""
import numpy as np
import pytest
import torch

from oracle.philox import philox_uniform
from oracle.stem_geometry import same_pads, stem_grads
from mac_network_b200.stem import SITE_STEM, Stem, init_stem_params, stem_grid, stem_specs
from tests._util import max_rel
from tests.test_stem_geometry import CASES, case_specs, load_case

pytestmark = pytest.mark.gpu

INVALID, ALIGN, UNSUPPORTED = -1, -2, -3
F32, BF16, SPLIT = 0, 1, 2
GEOMS = [(1, 1), (2, 1), (4, 1), (5, 1), (3, 2), (5, 2), (1, 2), (2, 2), (7, 3)]


def _lib():
    from mac_network_b200 import _lib as L_
    return L_, L_.load()


def _x(B, H, W, C, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(B, H, W, C, device="cuda", generator=g)


def _im2col(x, form, keep, k, s, seed=5, site=SITE_STEM, step=3):
    L_, lib = _lib()
    B, H, W, C = x.shape
    Ho, Wo = stem_grid(H, W, [s])
    K = k * k * C
    cols = torch.empty((B * Ho * Wo, K * (2 if form == SPLIT else 1)), dtype=torch.float32 if form == F32 else torch.bfloat16,
                       device="cuda")
    L_.check(lib.mac_im2col(L_.ptr(x), L_.ptr(cols), form, keep, seed, site, step, B, H, W, C, k, s, L_.stream_ptr()),
             "mac_im2col")
    return cols


def _host_dropped(x, keep, seed, site, step):
    """dropout(x) in fp32 as the kernels compute it: keep-mask (p >> 8) >= ceil((1 - keep) 2^24), value * fp32(1 / keep)."""
    xn = x.cpu().numpy()
    if keep == 1.0:
        return xn
    u = philox_uniform(seed, site, step, xn.size).reshape(xn.shape)
    thr = np.ceil((1.0 - float(np.float32(keep))) * 16777216.0)
    scale = np.float32(1.0) / np.float32(keep)
    return np.where(u * 16777216.0 >= thr, xn * scale, np.float32(0)).astype(np.float32)


def _host_cols(xd, k, s):
    """The fp32 patch matrix [B*Ho*Wo, k*k*C] of the dropped-out NHWC input, TF SAME padding."""
    B, H, W, C = xd.shape
    Ho, Wo = stem_grid(H, W, [s])
    (pt, pb), (pl, pr) = same_pads(H, k, s), same_pads(W, k, s)
    xp = np.zeros((B, H + pt + pb, W + pl + pr, C), np.float32)
    xp[:, pt:pt + H, pl:pl + W] = xd
    taps = [xp[:, i:i + (Ho - 1) * s + 1:s, j:j + (Wo - 1) * s + 1:s] for i in range(k) for j in range(k)]
    return np.concatenate(taps, axis=-1).reshape(B * Ho * Wo, k * k * C)


def _bits(t):
    return t.view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


@pytest.mark.parametrize("keep", [1.0, 0.82])
@pytest.mark.parametrize("form", [F32, BF16, SPLIT])
def test_im2col_at_3x3_stride_1_equals_the_3x3_passes(form, keep):
    L_, lib = _lib()
    x = _x(3, 7, 5, 64, seed=1)
    got = _im2col(x, form, keep, 3, 1)
    want = torch.empty_like(got)
    if form == SPLIT:
        L_.check(lib.mac_im2col3x3_split(L_.ptr(x), L_.ptr(want), keep, 5, SITE_STEM, 3, 3, 7, 5, 64, L_.stream_ptr()))
    else:
        L_.check(lib.mac_im2col3x3(L_.ptr(x), L_.ptr(want), form, keep, 5, SITE_STEM, 3, 3, 7, 5, 64, L_.stream_ptr()))
    assert torch.equal(_bits(got), _bits(want))


@pytest.mark.parametrize("keep", [1.0, 0.82])
@pytest.mark.parametrize("k,s", GEOMS)
@pytest.mark.parametrize("form,C", [(F32, 12), (BF16, 12), (BF16, 64), (SPLIT, 64)])
def test_im2col_equals_host_restatement(form, C, k, s, keep):
    x = _x(2, 7, 6, C, seed=k * 10 + s)
    got = _im2col(x, form, keep, k, s)
    ref = torch.from_numpy(_host_cols(_host_dropped(x, keep, 5, SITE_STEM, 3), k, s))
    if form == F32:
        assert torch.equal(_bits(got.cpu()), _bits(ref))
        return
    hi = ref.to(torch.bfloat16)
    if form == BF16:
        assert torch.equal(_bits(got.cpu()), _bits(hi))
        return
    lo = (ref - hi.float()).to(torch.bfloat16)
    assert torch.equal(_bits(got.cpu()), _bits(torch.cat([hi, lo], dim=1)))
    assert torch.equal(_bits(_im2col(x, form, keep, k, s)), _bits(got))                # rerun


@pytest.mark.parametrize("split", [0, 1])
@pytest.mark.parametrize("k,s,B,H,W", [(1, 1, 1, 7, 5), (5, 2, 1, 7, 5), (2, 1, 3, 5, 3), (3, 2, 1, 14, 14), (3, 1, 1, 3, 5)])
def test_im2col_t_is_the_transposed_patch_matrix(split, k, s, B, H, W):
    L_, lib = _lib()
    C, keep = 128, 0.82
    x = _x(B, H, W, C, seed=7)
    M = B * np.prod(stem_grid(H, W, [s]))
    Mp = (M + 63) // 64 * 64
    K = k * k * C
    colsT = torch.full((K, Mp * (2 if split else 1)), float("nan"), dtype=torch.bfloat16, device="cuda")
    L_.check(lib.mac_im2col_t(L_.ptr(x), L_.ptr(colsT), split, keep, 5, SITE_STEM, 3, B, H, W, C, k, s, L_.stream_ptr()))
    cols = _im2col(x, SPLIT if split else BF16, keep, k, s)
    segs = [cols[:, :K], cols[:, K:]] if split else [cols]
    for j, seg in enumerate(segs):
        part = colsT[:, j * Mp:(j + 1) * Mp]
        assert torch.equal(_bits(part[:, :M]), _bits(seg.t()))
        assert not _bits(part[:, M:]).any()                                           # the padding columns are zeros


@pytest.mark.parametrize("keep", [1.0, 0.82])
@pytest.mark.parametrize("k,s,B,H,W", [(1, 1, 1, 7, 5), (5, 2, 2, 7, 6), (4, 1, 1, 5, 3), (3, 2, 1, 14, 14), (2, 2, 3, 5, 5)])
def test_col2im_against_fp64(k, s, B, H, W, keep):
    L_, lib = _lib()
    C = 8
    Ho, Wo = stem_grid(H, W, [s])
    g = torch.Generator(device="cuda").manual_seed(11)
    dcols = torch.randn(B * Ho * Wo, k * k * C, device="cuda", generator=g)
    dx = torch.empty(B, H, W, C, device="cuda")
    args = (keep, 5, SITE_STEM, 3, B, H, W, C, k, s, L_.stream_ptr())
    L_.check(lib.mac_col2im(L_.ptr(dcols), L_.ptr(dx), *args))
    # fp64: scatter each patch entry back to the pixel it copied, then the forward's mask and 1 / keep
    (pt, pb), (pl, pr) = same_pads(H, k, s), same_pads(W, k, s)
    acc = np.zeros((B, H + pt + pb, W + pl + pr, C))
    d = dcols.cpu().numpy().astype(np.float64).reshape(B, Ho, Wo, k, k, C)
    for i in range(k):
        for j in range(k):
            acc[:, i:i + (Ho - 1) * s + 1:s, j:j + (Wo - 1) * s + 1:s] += d[:, :, :, i, j]
    ref = acc[:, pt:pt + H, pl:pl + W]
    mask = _host_dropped(torch.ones(B, H, W, C), keep, 5, SITE_STEM, 3).astype(np.float64)
    ref = ref * (mask * keep if keep < 1 else 1.0) / keep
    assert max_rel(dx.cpu().numpy(), ref) < 1e-6
    dx2 = torch.empty_like(dx)
    L_.check(lib.mac_col2im(L_.ptr(dcols), L_.ptr(dx2), *args))
    assert torch.equal(_bits(dx), _bits(dx2))


def _uniforms(seed, step, shapes):
    L_, lib = _lib()
    us = []
    for layer, shape in enumerate(shapes):
        u = torch.empty(int(np.prod(shape)), device="cuda")
        L_.check(lib.mac_dropout_uniform(seed, SITE_STEM + layer, step, L_.ptr(u), u.numel(), L_.stream_ptr()))
        us.append(u.double().view(*shape))
    return us


def _layer_inputs(B, H, W, cin, cout, nlayers, strides):
    shapes, c = [], cin
    for i in range(nlayers):
        shapes.append((B, H, W, c))
        H, W = stem_grid(H, W, [strides[i]])
        c = cout
    return shapes


def _check_stem(st, pv, images, keep, strides, linear, relu, fwd_tol, grad_tol, seed, step=4):
    """Forward (save) + backward of `st` against stem_grads on the device's own keep-masks."""
    B, H, W, cin = images.shape
    x = images.float().contiguous()
    kb = st.forward(x, keep=keep, step=step, save_for_backward=True)
    d_kb = torch.randn(kb.shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(seed))
    grads = {k: torch.zeros_like(v) for k, v in st.p.items()}
    d_img = st.backward(d_kb, grads, need_d_images=True)
    torch.cuda.synchronize()
    cout = kb.shape[-1]
    us = [] if (keep == 1.0 or linear) else _uniforms(st.seed, step, _layer_inputs(B, H, W, cin, cout, st.nlayers, strides))
    pref = {k: torch.as_tensor(v, dtype=torch.float64, device="cuda") for k, v in pv.items()}
    kb_ref, gref, dimg_ref = stem_grads(relu, pref, images.double(), keep, us, d_kb.double(), strides, linear)
    errs = {"kb": max_rel(kb.cpu().numpy(), kb_ref), "d_images": max_rel(d_img.cpu().numpy(), dimg_ref)}
    for k in gref:
        errs[k] = max_rel(grads[k].cpu().numpy(), gref[k])
    print(" ".join("%s %.2e" % kv for kv in errs.items()))
    assert errs["kb"] < fwd_tol, errs
    assert all(v < grad_tol for k, v in errs.items() if k != "kb"), errs


@pytest.mark.parametrize("case", CASES)
def test_fp32_stem_matches_reference_fixture(case):
    meta, g = load_case(case)
    pv = init_stem_params(case_specs(meta), seed=meta["param_seed"], dtype=np.float64)
    params = {k: torch.from_numpy(v.astype(np.float32)).cuda() for k, v in pv.items()}
    strides = None if meta["linear"] else meta["strides"]
    st = Stem(params, relu=meta["relu"], prec="fp32", seed=17, strides=strides, linear=meta["linear"])
    images = torch.from_numpy(g["images"]).cuda()
    if not meta["train"]:
        kb = st.forward(images.float())
        assert max_rel(kb.cpu().numpy(), g["kb"]) < 1e-4
    _check_stem(st, pv, images, meta["keep"], strides, meta["linear"], meta["relu"], 1e-4, 2e-4, seed=3)


BIG = [dict(ksizes=[1, 1]), dict(ksizes=[3, 3], strides=[2, 1]), dict(ksizes=[5, 3], strides=[2, 1]),
       dict(ksizes=[4, 2]), dict(linear=True)]


@pytest.mark.parametrize("prec,keep", [("bf16x3", 0.82), ("bf16", 0.82), ("bf16x3", 1.0)])
@pytest.mark.parametrize("geom", range(len(BIG)))
def test_tensor_core_stem_against_fp64(prec, keep, geom):
    """B = 64, 1024 -> 512 -> 512 on the 14 x 14 grid: bf16x3 inside the fp32 bars, bf16 inside the bf16 stem's (forward
    2e-2 as the bf16 stem test, gradients 1.2e-2 as the bf16 stem training test)."""
    gm = BIG[geom]
    linear = gm.get("linear", False)
    strides = gm.get("strides", [1] if linear else [1, 1])
    pv = init_stem_params(stem_specs(1024, 512, ksizes=gm.get("ksizes"), linear=linear), seed=19 + geom, dtype=np.float64)
    params = {k: torch.from_numpy(v.astype(np.float32)).cuda() for k, v in pv.items()}
    st = Stem(params, relu="ELU", prec=prec, seed=23, strides=strides, linear=linear)
    g = torch.Generator(device="cuda").manual_seed(29)
    images = torch.randn(64, 14, 14, 1024, device="cuda", generator=g, dtype=torch.float64).clamp_(min=0)
    fwd, grad = (1e-4, 2e-4) if prec == "bf16x3" else (2e-2, 1.2e-2)
    _check_stem(st, pv, images, keep, strides, linear, "ELU", fwd, grad, seed=31)


def test_nchw_forward_of_other_geometries_equals_nhwc_forward():
    for gm in BIG[1:]:
        linear = gm.get("linear", False)
        strides = gm.get("strides", [1] if linear else [1, 1])
        pv = init_stem_params(stem_specs(128, 128, ksizes=gm.get("ksizes"), linear=linear), seed=2, dtype=np.float32)
        params = {k: torch.from_numpy(v).cuda() for k, v in pv.items()}
        x = torch.rand(3, 128, 7, 6, device="cuda")
        for prec in ("fp32", "bf16", "bf16x3"):
            st = Stem(params, prec=prec, seed=4, strides=strides, linear=linear)
            for keep, save in ((1.0, False), (0.82, True)):
                a = st.forward_nchw(x, keep=keep, step=2, save_for_backward=save)
                b = st.forward(x.permute(0, 2, 3, 1).contiguous(), keep=keep, step=2, save_for_backward=save)
                assert a.shape == (3, int(np.prod(st.grid(7, 6))), 128)
                assert torch.equal(a, b), (gm, prec, keep)
            if prec == "bf16":
                a = st.forward_nchw(x.half())
                assert torch.equal(a, st.forward(x.half().float().permute(0, 2, 3, 1).contiguous()))


# ------------------------------------------------------------------------------------------------ refusals
def test_entry_points_refuse_before_any_launch():
    L_, lib = _lib()
    x = torch.zeros(2, 5, 5, 64, device="cuda")
    out = torch.full((4096 * 64,), 7.0, device="cuda")
    sp = L_.stream_ptr()
    launches = lib.mac_b200_launch_count()
    for k, s, C, form, want in ((0, 1, 64, F32, INVALID), (3, 0, 64, F32, INVALID), (17, 1, 64, F32, UNSUPPORTED),
                                (3, 17, 64, F32, UNSUPPORTED), (3, 1, 6, F32, UNSUPPORTED), (3, 2, 32, SPLIT, UNSUPPORTED),
                                (3, 2, 64, 3, UNSUPPORTED)):
        assert lib.mac_im2col(L_.ptr(x), L_.ptr(out), form, 1.0, 0, 0, 0, 2, 5, 5, C, k, s, sp) == want
    assert lib.mac_im2col(L_.ptr(x), L_.ptr(out), F32, 0.0, 0, 0, 0, 2, 5, 5, 64, 3, 2, sp) == INVALID
    assert lib.mac_col2im(L_.ptr(out), L_.ptr(x), 1.0, 0, 0, 0, 2, 5, 5, 6, 3, 2, sp) == UNSUPPORTED
    assert lib.mac_col2im(L_.ptr(out), L_.ptr(x), 1.0, 0, 0, 0, 2, 5, 5, 64, 0, 2, sp) == INVALID
    assert lib.mac_im2col_t(L_.ptr(x), L_.ptr(out), 0, 1.0, 0, 0, 0, 2, 5, 5, 32, 3, 2, sp) == UNSUPPORTED
    assert lib.mac_conv_bwd_tc(L_.ptr(x), L_.ptr(out), L_.ptr(out), L_.ptr(out), 3, 1.0, 0, 0, 0, L_.ptr(out), L_.ptr(out),
                               None, L_.ptr(out), 1 << 30, 2, 5, 5, 64, 128, 3, 2, sp) == UNSUPPORTED
    assert lib.mac_conv_bwd_tc_workspace_bytes(2, 5, 5, 128, 128, 0, 1, 0) == 0
    torch.cuda.synchronize()
    assert lib.mac_b200_launch_count() == launches
    assert bool((out == 7.0).all())


def test_stem_refusals_before_any_launch():
    L_, lib = _lib()
    pv = init_stem_params(stem_specs(128, 128, ksizes=[3, 3]), seed=1, dtype=np.float32)
    params = {k: torch.from_numpy(v).cuda() for k, v in pv.items()}
    x = torch.rand(2, 7, 7, 128, device="cuda")
    launches = lib.mac_b200_launch_count()
    with pytest.raises(NotImplementedError):
        Stem(params, prec="fp8", strides=[2, 1]).forward(x)
    with pytest.raises(NotImplementedError):
        Stem(params, prec="fp8", strides=[2, 1]).forward_nchw(x.permute(0, 3, 1, 2).contiguous())
    lin = init_stem_params(stem_specs(128, 128, linear=True), seed=1, dtype=np.float32)
    with pytest.raises(NotImplementedError):
        Stem({k: torch.from_numpy(v).cuda() for k, v in lin.items()}, prec="fp8", linear=True).forward(x)
    p64 = {k: torch.from_numpy(v).cuda() for k, v in init_stem_params(stem_specs(64, 128, ksizes=[1, 1]), seed=1).items()}
    with pytest.raises(NotImplementedError):
        Stem(p64, prec="bf16x3").forward(torch.rand(2, 7, 7, 64, device="cuda"))
    with pytest.raises(NotImplementedError):
        Stem(p64, prec="bf16", strides=[2, 1]).forward(torch.rand(2, 7, 7, 64, device="cuda"), save_for_backward=True)
    with pytest.raises(ValueError):
        Stem(params, strides=[2])
    with pytest.raises(ValueError):
        Stem({k: torch.from_numpy(v).cuda() for k, v in lin.items()}, linear=True, strides=[2])
    torch.cuda.synchronize()
    assert lib.mac_b200_launch_count() == launches


# ------------------------------------------------------------------------------------------------ whole model
V, E, C, A = 90, 300, 128, 28


def _net(geom, L=3, seed=3, prec="fp32"):
    from mac_network_b200.config import MACConfig
    from mac_network_b200.model import MACnet
    cfg = MACConfig.args("args", netLength=L)
    return MACnet(cfg, L, V, A, wrd_emb_dim=E, image_in_dim=C, classifier_dims=(512,), seed=seed, prec=prec, **geom)


GEOM_NETS = {"stride2": dict(stem_kernel_sizes=[3, 3], stem_strides=[2, 1]), "linear": dict(stem_linear=True)}


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("geom", sorted(GEOM_NETS))
def test_pipeline_equals_run_batch_with_the_stem_geometry(geom, prec):
    from mac_network_b200.serving import ModelPipeline
    from tests.test_gpu_model_pipeline import _assert_same, _batches, _reference
    net = _net(GEOM_NETS[geom], prec=prec)
    B, S, H, W = 8, 7, 14, 14
    Ho, Wo = net._stem.grid(H, W)
    assert (Ho * Wo) == (49 if geom == "stride2" else 196)
    batches = _batches(3, B, S, H, W, seed=5, longest=S)
    refs = [_reference(net, b) for b in batches]
    assert refs[0]["att_kb"].shape == (3, B, Ho * Wo)
    res = net.runBatch(None, dict(batches[0], answers=np.zeros(B, np.int32)), {"images": batches[0]["images"]}, train=False,
                       getAtt=True)
    assert np.array(res["preds"][0]["attentions"]["kb"]).shape == (3, Ho, Wo)
    pipe = ModelPipeline(net, (B, S, H, W), slots=2)
    for b, r in zip(batches, refs):
        _assert_same(pipe.result(pipe.submit(b)), r, net.L)
    # several questions per image, and the knowledge-base cache: the reference is runBatch on the gathered images
    U = 3
    idx = np.array([0, 1, 2, 0, 1, 2, 2, 0], np.int32)
    for kw in (dict(images=U), dict(images=U, cache=10)):
        pipe = ModelPipeline(net, (B, S, H, W), slots=1, **kw)
        for j, b in enumerate(batches[:2]):
            imgs = b["images"][:U]
            sub = {"questions": b["questions"], "questionLengths": b["questionLengths"], "images": imgs, "imageIndex": idx}
            if "cache" in kw:
                sub = {"questions": b["questions"], "questionLengths": b["questionLengths"],
                       "imageIds": (10 * j + idx).astype(np.int64),
                       "images": (lambda imgs_: (lambda ids: imgs_[np.asarray(ids) % 10]))(imgs)}
            ref = _reference(net, dict(b, images=imgs[idx]))
            _assert_same(pipe.result(pipe.submit(sub)), ref, net.L)
