"""The location-aware stem (--locationAware) on the GPU.

- mac_loc_cols bit for bit a host restatement (grid, SAME patches, the location site's Philox mask) in every form, L and PE,
  at the geometries of the stem, odd M, padding columns zero after a dirty buffer; mac_loc_cols_t its transpose with zero
  padding; reruns bit-identical.  The _acc GEMMs against fp64.
- Stem(prec="fp32") against every location fixture of the reference with the device's own masks (forward 1e-4, gradients
  2e-4 of each tensor's maximum); bf16x3 inside the same bars and bf16 inside the bf16 stem's bounds against fp64 autograd
  at B = 64, 1024 -> 512 -> 512 on 14 x 14 and 2048 on 7 x 7, L and PE.
- K_loc = 0: output, image gradient, dK_img and bias gradient bit for bit the location-free stem's, in every precision and
  with dropout.  forward_nchw (fp32 and fp16 images) bit for bit forward of the permuted tensor.
- Whole model: DPTrainer and MACModel steps against the fp64 graph, ModelPipeline and TrainPipeline bit for bit runBatch,
  and a reference-named checkpoint with a 1026-channel layer-0 kernel loading with strict=True."""
import numpy as np
import pytest
import torch

from oracle import model_torch_autograd as MA
from oracle.stem_location import stem_loc_grads, stem_loc_torch
from mac_network_b200.stem import (SITE_LOCATION, SITE_STEM, Stem, init_stem_params, location_channels, location_grid,
                                   location_width, stem_grid, stem_specs)
from tests._util import max_rel
from tests.test_gpu_stem_geometry import _bits, _host_cols, _host_dropped, _lib, _x
from tests.test_stem_location import CASES, case_specs, load_case

pytestmark = pytest.mark.gpu

F32, BF16, SPLIT = 0, 1, 2
LOCS = {"L": ("L", 1.0, 32), "PE3": ("PE", 0.5, 3), "PE": ("PE", 1.0, 32)}


def _host_q(loc, B, H, W, k, s, keep, seed, step):
    """Q [M, Kq] fp32 on the host: the dropped-out location tensor's SAME patches, zero columns up to Kq."""
    g = np.ascontiguousarray(location_grid(loc, H, W), dtype=np.float32)
    xl = torch.from_numpy(np.ascontiguousarray(np.broadcast_to(g, (B,) + g.shape)))
    cols = _host_cols(_host_dropped(xl, keep, seed, SITE_LOCATION, step), k, s)
    l = g.shape[-1]
    return np.concatenate([cols, np.zeros((cols.shape[0], location_width(l, k) - cols.shape[1]), np.float32)], axis=1)


def _dev_grid(loc, H, W):
    return torch.from_numpy(np.ascontiguousarray(location_grid(loc, H, W), dtype=np.float32)).cuda()


@pytest.mark.parametrize("keep", [1.0, 0.82])
@pytest.mark.parametrize("k,s", [(3, 1), (1, 1), (5, 2), (4, 1), (2, 2)])
@pytest.mark.parametrize("loc", sorted(LOCS))
@pytest.mark.parametrize("form", [F32, BF16, SPLIT])
def test_loc_cols_equals_host_restatement(form, loc, k, s, keep):
    L_, lib = _lib()
    B, H, W = 3, 5, 7                                       # M = 105 at stride 1: odd
    grid = _dev_grid(LOCS[loc], H, W)
    l = grid.shape[-1]
    M, Kq = B * int(np.prod(stem_grid(H, W, [s]))), location_width(l, k)
    ref = torch.from_numpy(_host_q(LOCS[loc], B, H, W, k, s, keep, 5, 3))

    def run():
        q = torch.full((M, Kq * (2 if form == SPLIT else 1)), float("nan"), device="cuda",
                       dtype=torch.float32 if form == F32 else torch.bfloat16)
        L_.check(lib.mac_loc_cols(L_.ptr(grid), L_.ptr(q), form, keep, 5, SITE_LOCATION, 3, B, H, W, l, k, s,
                                  L_.stream_ptr()), "mac_loc_cols")
        return q.cpu()
    got = run()
    hi = ref.to(torch.bfloat16)
    want = {F32: ref, BF16: hi, SPLIT: torch.cat([hi, (ref - hi.float()).to(torch.bfloat16)], dim=1)}[form]
    assert torch.equal(_bits(got), _bits(want))
    assert torch.equal(_bits(run()), _bits(got))


@pytest.mark.parametrize("split", [0, 1])
@pytest.mark.parametrize("loc", sorted(LOCS))
@pytest.mark.parametrize("k,s", [(3, 1), (5, 2), (1, 1)])
def test_loc_cols_t_is_the_transpose(split, loc, k, s):
    L_, lib = _lib()
    B, H, W, keep = 1, 7, 5, 0.82
    grid = _dev_grid(LOCS[loc], H, W)
    l = grid.shape[-1]
    M, Kq = B * int(np.prod(stem_grid(H, W, [s]))), location_width(l, k)
    Mp = (M + 63) // 64 * 64
    qT = torch.full((Kq, Mp * (2 if split else 1)), float("nan"), dtype=torch.bfloat16, device="cuda")
    L_.check(lib.mac_loc_cols_t(L_.ptr(grid), L_.ptr(qT), split, keep, 5, SITE_LOCATION, 3, B, H, W, l, k, s,
                                L_.stream_ptr()))
    ref = torch.from_numpy(_host_q(LOCS[loc], B, H, W, k, s, keep, 5, 3))
    pad = torch.zeros(Kq, Mp - M)
    hi = ref.to(torch.bfloat16)
    want = torch.cat([hi.float().t(), pad], 1).to(torch.bfloat16)
    if split:
        lo = (ref - hi.float()).to(torch.bfloat16)
        want = torch.cat([want, torch.cat([lo.float().t(), pad], 1).to(torch.bfloat16)], 1)
    assert torch.equal(_bits(qT.cpu()), _bits(want))


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("M,K,N,act", [(129, 128, 128, 3), (12544, 9216, 512, 3), (64, 256, 256, 0), (77, 64, 384, 4)])
def test_acc_gemms_against_fp64(split, M, K, N, act):
    from mac_network_b200 import packs
    L_, lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(M + K)
    a = torch.randn(M, K, device="cuda", generator=g)
    w = torch.randn(K, N, device="cuda", generator=g) / K ** 0.5
    y0 = torch.randn(M, N, device="cuda", generator=g)
    y = y0.clone()
    if split:
        hi = a.to(torch.bfloat16)
        a2 = torch.cat([hi, (a - hi.float()).to(torch.bfloat16)], 1).contiguous()
        L_.check(lib.mac_linear_tc32_fwd_acc(L_.ptr(a2), L_.ptr(packs.split3(w, L_.stream_ptr())), act, L_.ptr(y), M, K, N,
                                             L_.stream_ptr()))
        ref, tol = a.double() @ w.double() + y0.double(), 1e-5
    else:
        ab = a.to(torch.bfloat16)
        wb = packs.bf16(w, L_.stream_ptr())
        L_.check(lib.mac_linear_tc_fwd_acc(L_.ptr(ab), L_.ptr(wb), act, L_.ptr(y), M, K, N, L_.stream_ptr()))
        ref, tol = ab.double() @ wb.double().t() + y0.double(), 1e-5
    ref = {0: ref, 3: torch.nn.functional.elu(ref), 4: ref.clamp(min=0)}[act]
    assert max_rel(y.cpu().numpy(), ref.cpu().numpy()) < tol


# ------------------------------------------------------------------------------------------------ the stem
def _uniforms(seed, step, B, shapes, l):
    """The device's own draws: layer 0's input is [image | location], each from its own site; then each later layer's."""
    L_, lib = _lib()

    def draw(site, shape):
        u = torch.empty(int(np.prod(shape)), device="cuda")
        L_.check(lib.mac_dropout_uniform(seed, site, step, L_.ptr(u), u.numel(), L_.stream_ptr()))
        return u.double().view(*shape)
    us = [torch.cat([draw(SITE_STEM, shapes[0]), draw(SITE_LOCATION, shapes[0][:3] + (l,))], dim=-1)]
    return us + [draw(SITE_STEM + i, sh) for i, sh in enumerate(shapes) if i > 0]


def _check_stem(st, pv, images, keep, strides, fwd_tol, grad_tol, seed, step=4):
    B, H, W, cin = images.shape
    kb = st.forward(images.float().contiguous(), keep=keep, step=step, save_for_backward=True)
    d_kb = torch.randn(kb.shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(seed))
    grads = {k: torch.zeros_like(v) for k, v in st.p.items()}
    d_img = st.backward(d_kb, grads, need_d_images=True)
    torch.cuda.synchronize()
    shapes, h, w, c = [], H, W, cin
    for i, s in enumerate(strides):
        shapes.append((B, h, w, c))
        h, w = stem_grid(h, w, [s])
        c = kb.shape[-1]
    us = [] if keep == 1.0 else _uniforms(st.seed, step, B, shapes, st.nloc)
    pref = {k: torch.as_tensor(v, dtype=torch.float64, device="cuda") for k, v in pv.items()}
    kb_ref, gref, dimg_ref = stem_loc_grads("ELU", pref, images.double(), st.location, keep, us, d_kb.double(), strides)
    errs = {"kb": max_rel(kb.cpu().numpy(), kb_ref), "d_images": max_rel(d_img.cpu().numpy(), dimg_ref)}
    for k in gref:
        errs[k] = max_rel(grads[k].cpu().numpy(), gref[k])
    K0 = "stem/cnnLayercnn_0/kernels/kernel"
    C = images.shape[-1]
    errs["location rows"] = max_rel(grads[K0][:, :, C:].cpu().numpy(), gref[K0][:, :, C:])
    print(" ".join("%s %.2e" % kv for kv in errs.items()))
    assert errs["kb"] < fwd_tol, errs
    assert all(v < grad_tol for k, v in errs.items() if k != "kb"), errs


@pytest.mark.parametrize("case", CASES)
def test_fp32_stem_matches_reference_fixture(case):
    meta, g = load_case(case)
    pv = init_stem_params(case_specs(meta), seed=meta["param_seed"], dtype=np.float64)
    params = {k: torch.from_numpy(v.astype(np.float32)).cuda() for k, v in pv.items()}
    st = Stem(params, relu=meta["relu"], prec="fp32", seed=17, strides=meta["strides"], location=tuple(meta["location"]))
    images = torch.from_numpy(g["images"]).cuda()
    if not meta["train"]:
        assert max_rel(st.forward(images.float()).cpu().numpy(), g["kb"]) < 1e-4
    _check_stem(st, pv, images, meta["keep"], meta["strides"], 1e-4, 2e-4, seed=3)


@pytest.mark.parametrize("prec,keep", [("bf16x3", 0.82), ("bf16", 0.82), ("bf16x3", 1.0), ("bf16", 1.0)])
@pytest.mark.parametrize("loc", ["L", "PE"])
@pytest.mark.parametrize("C,HW", [(1024, 14), (2048, 7)])
def test_tensor_core_stem_against_fp64(prec, keep, loc, C, HW):
    pv = init_stem_params(stem_specs(C, 512, location=LOCS[loc]), seed=19, dtype=np.float64)
    params = {k: torch.from_numpy(v.astype(np.float32)).cuda() for k, v in pv.items()}
    st = Stem(params, relu="ELU", prec=prec, seed=23, location=LOCS[loc])
    g = torch.Generator(device="cuda").manual_seed(29)
    images = torch.randn(64, HW, HW, C, device="cuda", generator=g, dtype=torch.float64).clamp_(min=0)
    fwd, grad = (1e-4, 2e-4) if prec == "bf16x3" else (2e-2, 1.2e-2)
    _check_stem(st, pv, images, keep, [1, 1], fwd, grad, seed=31)


@pytest.mark.parametrize("geom", [dict(), dict(ksizes=[5, 3], strides=[2, 1])])
@pytest.mark.parametrize("prec", ["fp32", "bf16", "bf16x3"])
def test_zero_location_kernel_leaves_the_image_path_bit_for_bit(prec, geom):
    C, l = 128, location_channels("PE")
    pv = init_stem_params(stem_specs(C, 128, ksizes=geom.get("ksizes"), location="PE"), seed=3)
    K0 = "stem/cnnLayercnn_0/kernels/kernel"
    pv[K0][:, :, C:] = 0
    loc_p = {k: torch.from_numpy(v).cuda() for k, v in pv.items()}
    plain_p = dict(loc_p, **{K0: loc_p[K0][:, :, :C].contiguous()})
    a = Stem(loc_p, prec=prec, seed=5, strides=geom.get("strides"), location="PE")
    b = Stem(plain_p, prec=prec, seed=5, strides=geom.get("strides"))
    x = torch.rand(4, 7, 6, C, device="cuda")
    ka = a.forward(x, keep=0.82, step=2, save_for_backward=True)
    kb = b.forward(x, keep=0.82, step=2, save_for_backward=True)
    assert torch.equal(ka, kb)
    d = torch.randn_like(ka)
    ga = {k: torch.zeros_like(v) for k, v in loc_p.items()}
    gb = {k: torch.zeros_like(v) for k, v in plain_p.items()}
    assert torch.equal(a.backward(d, ga, need_d_images=True), b.backward(d, gb, need_d_images=True))
    assert torch.equal(ga[K0][:, :, :C], gb[K0])
    assert float(ga[K0][:, :, C:].abs().max()) > 0                      # the location rows do get a gradient
    for k in gb:
        if k != K0:
            assert torch.equal(ga[k], gb[k]), k


def test_nchw_forward_equals_nhwc_forward():
    for geom in (dict(), dict(ksizes=[5, 3], strides=[2, 1])):
        pv = init_stem_params(stem_specs(128, 128, ksizes=geom.get("ksizes"), location="L"), seed=2)
        params = {k: torch.from_numpy(v).cuda() for k, v in pv.items()}
        x = torch.rand(3, 128, 7, 6, device="cuda")
        for prec in ("fp32", "bf16", "bf16x3"):
            st = Stem(params, prec=prec, seed=4, strides=geom.get("strides"), location="L")
            for keep, save in ((1.0, False), (0.82, True)):
                for img in (x, x.half()):
                    a = st.forward_nchw(img, keep=keep, step=2, save_for_backward=save)
                    b = st.forward(img.float().permute(0, 2, 3, 1).contiguous(), keep=keep, step=2, save_for_backward=save)
                    assert torch.equal(a, b), (geom, prec, keep, img.dtype)


# ------------------------------------------------------------------------------------------------ whole model
from tests import test_gpu_model_gradients as MG                       # noqa: E402
from tests import test_gpu_stem_geometry_training as GT                # noqa: E402
from tests.test_model_autograd_oracle import training_keeps            # noqa: E402

MODEL_LOCS = {"L": {"location": "L"}, "PE": {"location": "PE", "location_bias": 0.5, "location_dim": 4}}


def _stem_oracle(monkeypatch, geom):
    loc = (geom["location"], geom.get("location_bias", 1.0), geom.get("location_dim", 32))

    def graph(relu, p, images, keep=1.0, uniforms=None):
        us = list(uniforms or [])
        if us:                                  # [image draw, location draw, layer 1 ...] -> layer 0's whole input
            us = [torch.cat([torch.as_tensor(us[0]).to(images), torch.as_tensor(us[1]).to(images)], dim=-1)] + us[2:]
        return stem_loc_torch(relu, {k: v for k, v in p.items() if k.startswith("stem/")}, images, loc, keep, us)
    monkeypatch.setattr(MA, "stem_graph", graph)


def _plan(cfg, values, keeps, k, H, W, C, geom, step):
    plan = GT._plan(cfg, values, keeps, k, H, W, C, geom, step)
    if plan["stem"]:
        l = location_channels((geom["location"], geom.get("location_bias", 1.0), geom.get("location_dim", 32)))
        plan["stem"].insert(1, (SITE_LOCATION, step, (k, H, W, l)))
    return plan


@pytest.mark.parametrize("loc", sorted(MODEL_LOCS))
def test_trainer_step_with_location_against_the_fp64_graph(loc, monkeypatch):
    geom = MODEL_LOCS[loc]
    c = dict(MG.DEFAULT, flags="args", HW=(5, 4))
    _stem_oracle(monkeypatch, geom)
    cfg, cell_dp, tr, data = GT._trainer(c, geom)
    keeps = training_keeps(cell_dp)
    H, W = c["HW"]
    dev = MG._device(data, c["layout"])
    values = tr.params.numpy()
    logits, losses = tr.full_forward_backward("t", dev, global_batch=GT.B)
    torch.cuda.synchronize()
    plan = _plan(cfg, values, keeps, GT.B, H, W, c["C"], geom, tr.step_id)
    raw = MG.draws(plan, MG.philox_seed(MG.BASE_SEED, tr.step_id, 0))
    ref = MA.run(cfg, GT.L, values, MG._oracle_data(data, dev), keeps, MG.kernel_masks(plan, raw, keeps),
                 global_batch=GT.B, device="cuda")
    p = tr.params
    got = {n: tr.bucket[p.offsets[n]:p.offsets[n] + max(1, int(np.prod(p.specs[n][0])))] for n in p.specs}
    errs, null = MG._compare(got, ref, logits, losses)
    MG._report("location " + loc, errs, null, MG._kind(c))


def test_mac_model_with_location_against_the_fp64_graph(monkeypatch):
    from mac_network_b200.modules import MACModel, answer_loss
    geom = MODEL_LOCS["PE"]
    c = dict(MG.DEFAULT, flags="args", HW=(5, 4), C=64)
    _stem_oracle(monkeypatch, geom)
    cfg, cell_dp, tr, data = GT._trainer(c, geom)
    keeps = training_keeps(cell_dp)
    H, W = c["HW"]
    model = MACModel.from_trainer(tr)
    assert model._stem.location == ("PE", 0.5, 4)
    model.train()
    dev = MG._device(data, "nchw")
    x = dev["images_nchw"].clone().requires_grad_(True)
    values = {n: v.detach().cpu().numpy().astype(np.float64) for n, v in model.named_parameters()}
    step = model.step
    logits, _ = model(dev["questions"], dev["questionLengths"], images_nchw=x)
    answer_loss(logits, dev["answers"]).backward()
    torch.cuda.synchronize()
    plan = _plan(cfg, values, keeps, GT.B, H, W, c["C"], geom, step)
    raw = MG.draws(plan, MG.philox_seed(MG.BASE_SEED, step, 0))
    ref = MA.run(cfg, GT.L, values, MG._oracle_data(data, dict(dev, images_nchw=x.detach())), keeps,
                 MG.kernel_masks(plan, raw, keeps), device="cuda")
    errs, null = MG._compare({n: v.grad for n, v in model.named_parameters()}, ref, logits, None)
    errs["d_images"] = float((x.grad.double() - ref["d_images"]).abs().max()) / float(ref["d_images"].abs().max())
    MG._report("MACModel location PE", errs, null, "fp32")


NET_LOCS = {"L": dict(stem_location="L"), "PE": dict(stem_location="PE", stem_location_dim=8, stem_location_bias=0.5)}


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("loc", sorted(NET_LOCS))
def test_pipeline_equals_run_batch_with_location(loc, prec):
    from mac_network_b200.serving import ModelPipeline
    from tests.test_gpu_model_pipeline import _assert_same, _batches, _reference
    from tests.test_gpu_stem_geometry import _net
    net = _net(NET_LOCS[loc], prec=prec)
    B, S, H, W = 8, 7, 14, 14
    batches = _batches(3, B, S, H, W, seed=5, longest=S)
    refs = [_reference(net, b) for b in batches]
    pipe = ModelPipeline(net, (B, S, H, W), slots=2)
    for b, r in zip(batches, refs):
        _assert_same(pipe.result(pipe.submit(b)), r, net.L)
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
            _assert_same(pipe.result(pipe.submit(sub)), _reference(net, dict(b, images=imgs[idx])), net.L)


@pytest.mark.parametrize("config", ["fp32", "tc32"])
@pytest.mark.parametrize("loc", sorted(NET_LOCS))
def test_train_pipeline_equals_run_batch_training_with_location(loc, config):
    from mac_network_b200.config import MACConfig
    from mac_network_b200.model import MACnet
    from mac_network_b200.serving import TrainPipeline
    TP = GT.TP

    def make():
        cfg = MACConfig.args("args", netLength=TP.L)
        return MACnet(cfg, TP.L, TP.V, TP.A, wrd_emb_dim=TP.E, image_in_dim=TP.C, classifier_dims=(512,), seed=3,
                      prec="bf16", **TP.HP, **TP.CONFIGS[config], **NET_LOCS[loc])
    net, twin = make(), make()
    batches = TP._batches(4)
    pipe = TrainPipeline(net, (TP.BS, TP.SMAX, TP.HW, TP.HW), depth=2)
    tickets, wants = [], []
    for i, b in enumerate(batches):
        tickets.append(pipe.submit(TP._pinned(b) if i % 2 else b))
        wants.append(TP._twin_step(twin, b))
        if i >= 1:
            TP._check(pipe.result(tickets[i - 1]), wants[i - 1], pipe, i - 1)
    TP._check(pipe.result(tickets[-1]), wants[-1], pipe, len(batches) - 1)
    pipe.drain()
    TP._same_state(net, twin)


def test_reference_checkpoint_with_1026_channels_loads_strictly(tmp_path, monkeypatch):
    from mac_network_b200.checkpoint import load_tf_checkpoint, save_tf_checkpoint
    from mac_network_b200.modules import MACModel
    geom = MODEL_LOCS["L"]
    c = dict(MG.DEFAULT, flags="args", HW=(5, 4), C=1024)
    _stem_oracle(monkeypatch, geom)
    cfg, cell_dp, tr, data = GT._trainer(c, geom)
    values = {k: v.reshape(tr.params.specs[k][0]) for k, v in tr.params.numpy().items()}
    assert values["stem/cnnLayercnn_0/kernels/kernel"].shape == (3, 3, 1026, c["d"])
    prefix = str(tmp_path / "weights.ckpt")
    save_tf_checkpoint(prefix, values)
    back = load_tf_checkpoint(prefix)
    model = MACModel(cfg, GT.L, MG.V, MG.A, wrd_emb_dim=MG.E, image_in_dim=1024, classifier_dims=MG.HIDDEN, seed=1,
                     stem_geometry=geom)
    missing, unexpected = model.load_state_dict({k: torch.from_numpy(v) for k, v in back.items()}, strict=True)
    assert not missing and not unexpected
    model.eval()
    dev = MG._device(data, "nhwc")
    with torch.no_grad():
        logits, _ = model(dev["questions"], dev["questionLengths"], images=dev["images"])
    ref = MA.run(cfg, GT.L, {k: v.astype(np.float64) for k, v in back.items()}, data,
                 {"encoder": (1.0, 1.0), "stem": 1.0, "cell": (1.0, 1.0, 1.0), "output": 1.0}, device="cuda", grad=False)
    assert MG._rowwise(logits, ref["logits"]) < 1e-4
