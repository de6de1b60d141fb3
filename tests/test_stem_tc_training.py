"""Mixed-precision training of the image stem (DESIGN.md section 9, item 2): `mac_conv3x3_bwd_tc`, `Stem(prec="bf16")`
forward(save) + backward, and `DPTrainer(stem_prec="bf16")`.

CPU: the entry point's status codes (returned before any CUDA call) and the host plumbing against the dry-run library.
GPU: the entry point against fp64 references of its OWN operation -- computed on exactly the operands the kernels see,
bf16(dropout(x)) with the keep-masks `mac_dropout_uniform` draws, bf16(dZ) and bf16(kernel) -- with the element-wise bound
of tests/test_gpu_backward_kernels.py, |got - ref| <= tol * absref (absref: the same reference on absolute values); then the
composition (the stem against the fp64 autograd restatement, the whole-model trainer against its fp32-stem twin).
Each `tol` is a few times the worst value measured on an H100 80GB HBM3 (SXM, 132 SMs), written beside it."""
import ctypes

import numpy as np
import pytest
import torch

from mac_network_b200 import _lib as L_
from tests import _mocklib

INVALID, ALIGN, UNSUPPORTED, WORKSPACE = -1, -2, -3, -4
ACT_ELU = L_.ACT["ELU"]

# ---- bounds; measured worst value on the H100 beside each
# mac_conv3x3_bwd_tc against fp64 of its own bf16 operands (fraction of absref)             measured
TOL_CONV = {"dkernel": 6e-6,         # K = Mp = 12 544 in one slice at the headline layers           1.9e-6
            "dbias": 1.5e-7,                                                                # 4.0e-8
            "dx": 3e-7}                                                                     # 1.0e-7
# Stem(prec="bf16") gradients against the fp64 restatement of the fp32 model (max-rel per tensor)
TOL_STEM_BF16 = 1.2e-2                                                                      # 4.2e-3
# stem slice of the whole-model gradient bucket, stem_prec="bf16" against "fp32" (max-rel per tensor)
TOL_TRAINER_STEM = 1e-2                                                                     # 2.8e-3


# ------------------------------------------------------------------------------------------------ CPU
def _fake_ptr(buf):
    return (ctypes.addressof(buf) + 15) & ~15          # 16-byte aligned fake "device" pointer (never dereferenced)


def test_conv3x3_bwd_tc_status_codes():
    """Bad arguments come back as MAC_ERR_* before any launch, so this runs without a GPU."""
    lib = L_.load()
    buf = (ctypes.c_float * 4096)()
    p = _fake_ptr(buf)

    def call(x=p, C=128, Cout=128, ws_bytes=1 << 40, dx=p, keep=0.82, kernel=p):
        return lib.mac_conv3x3_bwd_tc(x, p, p, kernel, ACT_ELU, keep, 7, 32, 1, p, p, dx, p, ws_bytes, 2, 5, 7, C, Cout, None)

    assert call(C=96) == UNSUPPORTED
    assert call(Cout=96) == UNSUPPORTED
    assert call(x=None) == INVALID
    assert call(kernel=None) == INVALID
    assert call(keep=0.0) == INVALID
    assert call(kernel=p + 4) == ALIGN
    need = lib.mac_conv3x3_bwd_tc_workspace_bytes(2, 5, 7, 128, 128, 1)
    assert call(ws_bytes=need - 1) == WORKSPACE
    # the data gradient's operands (bf16 kernel, fp32 patch gradient) are part of the workspace only when dx is asked for
    no_dx = lib.mac_conv3x3_bwd_tc_workspace_bytes(2, 5, 7, 128, 128, 0)
    assert no_dx + 9 * 128 * 128 * 2 + 70 * 9 * 128 * 4 <= need
    assert call(ws_bytes=no_dx - 1, dx=None) == WORKSPACE
    # the transposed operands cover Mp = 128 columns (M = 70 rounded up to the 64-row k-block)
    assert no_dx >= 128 * 128 * 2 + 9 * 128 * 128 * 2 + 70 * 128 * 2 + 9 * 128 * 128 * 4


class _Recorder(object):
    """Wraps the dry-run library and keeps each call's arguments."""

    def __init__(self, mock):
        self.mock, self.log = mock, []

    def __getattr__(self, name):
        fn = getattr(self.mock, name)

        def rec(*args):
            self.log.append((name, args))
            return fn(*args)
        return rec

    def args_of(self, name):
        return [a for n, a in self.log if n == name]


def _recorder(monkeypatch):
    rec = _Recorder(_mocklib.install(monkeypatch))
    monkeypatch.setattr(L_, "load", lambda: rec)
    return rec


def _cpu_params(specs_values):
    return {k: torch.from_numpy(np.ascontiguousarray(v, dtype=np.float32)) for k, v in specs_values.items()}


def test_stem_bf16_training_host_calls(monkeypatch):
    rec = _recorder(monkeypatch)
    from mac_network_b200.stem import Stem, SITE_STEM, stem_specs, init_stem_params
    p = _cpu_params(init_stem_params(stem_specs(128, 256), seed=1))
    st = Stem(p, relu="ELU", prec="bf16", seed=1)
    kb = st.forward(torch.zeros(2, 5, 7, 128), keep=0.82, step=3, save_for_backward=True)
    assert kb.shape == (2, 35, 256)
    assert len(rec.args_of("mac_linear_tc_fwd")) == 2 and not rec.args_of("mac_linear_fwd")
    grads = {k: torch.zeros_like(v) for k, v in p.items()}
    for need in (False, True):
        rec.log.clear()
        d_img = st.backward(torch.zeros_like(kb), grads, need_d_images=need)
        calls = rec.args_of("mac_conv3x3_bwd_tc")
        assert len(calls) == 2                                  # one per layer
        assert not rec.args_of("mac_linear_bwd") and not rec.args_of("mac_col2im3x3")
        layer1, layer0 = calls                                  # last layer first
        assert layer1[7] == SITE_STEM + 1 and layer0[7] == SITE_STEM
        assert layer1[-6:-1] == (2, 5, 7, 256, 256) and layer0[-6:-1] == (2, 5, 7, 128, 256)
        assert layer1[5] == pytest.approx(0.82) and layer1[8] == 3
        assert layer1[11] is not None                           # layer 1 always passes dx (layer 0's dy)
        assert (layer0[11] is not None) == need                 # the image gradient only when asked for
        assert [a[-1] for a in rec.args_of("mac_conv3x3_bwd_tc_workspace_bytes")] == [1, int(need)]
        assert (d_img is not None) == need
        if need:
            assert d_img.shape == (2, 5, 7, 128)


def test_stem_bf16_training_rejects_channel_counts(monkeypatch):
    mock = _mocklib.install(monkeypatch)
    from mac_network_b200.stem import Stem, stem_specs, init_stem_params
    for cin, cout in ((96, 128), (128, 64)):
        p = _cpu_params(init_stem_params(stem_specs(cin, cout), seed=1))
        st = Stem(p, relu="ELU", prec="bf16", seed=1)
        mock.calls.clear()
        with pytest.raises(NotImplementedError, match="multiples of 128"):
            st.forward(torch.zeros(1, 3, 3, cin), keep=0.82, step=0, save_for_backward=True)
        assert not mock.calls
        st.forward(torch.zeros(1, 3, 3, cin))                   # inference is unchanged
    p = _cpu_params(init_stem_params(stem_specs(128, 128), seed=1))
    with pytest.raises(NotImplementedError):
        Stem(p, relu="ELU", prec="tc32", seed=1).forward(torch.zeros(1, 3, 3, 128), save_for_backward=True)


def _host_trainer(monkeypatch, **kw):
    from mac_network_b200 import dp
    from mac_network_b200.config import MACConfig
    cfg = MACConfig.args("args", netLength=2, memDim=128, ctrlDim=128, attDim=128)
    return dp.DPTrainer(cfg, 2, seed=1, device="cpu", classifier=(8, [16]), encoder=(9, 12), **kw)


def test_trainer_stem_prec_validation(monkeypatch):
    _mocklib.install(monkeypatch)
    with pytest.raises(ValueError, match="stem_prec"):
        _host_trainer(monkeypatch, stem=(128, 2), stem_prec="fp16")
    with pytest.raises(ValueError, match="stem_prec"):
        _host_trainer(monkeypatch, stem=(128, 2), stem_prec="tc32")
    with pytest.raises(NotImplementedError, match="multiples of 128"):
        _host_trainer(monkeypatch, stem=(96, 2), stem_prec="bf16")
    assert _host_trainer(monkeypatch, stem=(96, 2)).stem.prec == "fp32"        # the default is unchanged
    assert _host_trainer(monkeypatch, stem=(128, 2), stem_prec="bf16").stem.prec == "bf16"


def test_full_model_trainer_bf16_stem_host_calls(monkeypatch):
    """DPTrainer(stem_prec="bf16").train_step_full with the already GPU-validated cell stubbed out."""
    rec = _recorder(monkeypatch)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True), raising=False)
    from mac_network_b200 import autograd, dp, mac_cell
    from mac_network_b200.config import MACConfig
    B, S, V, E, d, H, W, C, A, L = 4, 6, 9, 12, 128, 3, 3, 128, 8, 2
    cfg = MACConfig.args("args", netLength=L, memDim=d, ctrlDim=d, attDim=d)
    tr = dp.DPTrainer(cfg, L, seed=1, device="cpu", classifier=(A, [16]), encoder=(V, E), stem=(C, 2), stem_prec="bf16")

    class _Cell(object):
        _rw = {}
        seed = 0
    monkeypatch.setattr(tr, "cell_for", lambda key, batch: _Cell())
    monkeypatch.setattr(mac_cell, "mac_network", lambda cell, L_: (torch.zeros(B, d), torch.zeros(B, d)))
    monkeypatch.setattr(autograd, "mac_backward", lambda cell, dc, dm, bucket=None, zero_bucket=True, d_vecq=None, tc=False: {
        "knowledgeBase": torch.zeros(B, H * W, d), "questionCntxWords": torch.zeros(B, S, d), "vecQuestions": torch.zeros(B, d)})
    data = {"questions": torch.randint(0, V + 1, (B, S), dtype=torch.int32),
            "questionLengths": torch.randint(1, S + 1, (B,), dtype=torch.int32),
            "images": torch.zeros(B, H, W, C), "answers": torch.randint(0, A, (B,), dtype=torch.int32)}
    logits, losses = tr.train_step_full("k", data, global_batch=B)
    assert logits.shape == (B, A) and losses.shape == (B,)
    conv = rec.args_of("mac_conv3x3_bwd_tc")
    assert len(conv) == 2 and conv[1][11] is None               # the image gradient is not needed
    im2col = rec.args_of("mac_im2col3x3")
    assert len(im2col) == 2 and all(a[2] == 1 for a in im2col)  # bf16 patch matrices for the tensor-core forward
    assert not rec.args_of("mac_col2im3x3")
    assert "mac_clip_adam_ema_step" in [n for n, _ in rec.log] and tr.step_id == 1


# ------------------------------------------------------------------------------------------------ GPU
def _gpu_helpers():
    from tests.test_gpu_wgmma import bf16_round, excess, keep_threshold
    return bf16_round, excess, keep_threshold


def _uniform_mask(lib, seed, site, step, shape, keep):
    """the keep-mask of `mac_im2col3x3` from the uniforms `mac_dropout_uniform` draws (u = (philox word >> 8) * 2^-24)"""
    _, _, keep_threshold = _gpu_helpers()
    u = torch.empty(int(np.prod(shape)), device="cuda")
    L_.check(lib.mac_dropout_uniform(seed, site, step, L_.ptr(u), u.numel(), L_.stream_ptr()), "mac_dropout_uniform")
    return (u.double() * 16777216.0 >= keep_threshold(keep)).view(*shape)


def _patches(xd):
    """fp64 [B,H,W,C] -> [B*H*W, 9C] patch matrix, tap-major (kh*3 + kw), SAME padding"""
    B, H, W, C = xd.shape
    xp = torch.nn.functional.pad(xd, (0, 0, 1, 1, 1, 1))
    return torch.cat([xp[:, kh:kh + H, kw:kw + W, :].reshape(-1, C) for kh in range(3) for kw in range(3)], 1)


def _col2im(dcols, B, H, W, C):
    acc = torch.zeros(B, H + 2, W + 2, C, dtype=dcols.dtype, device=dcols.device)
    for tap in range(9):
        kh, kw = divmod(tap, 3)
        acc[:, kh:kh + H, kw:kw + W, :] += dcols[:, tap * C:(tap + 1) * C].reshape(B, H, W, C)
    return acc[:, 1:H + 1, 1:W + 1, :]


def _run_conv(lib, x, y, dy, kernel, keep, seed, site, step, dkernel, dbias, dx, shape):
    B, H, W, C, Cout = shape
    nbytes = int(lib.mac_conv3x3_bwd_tc_workspace_bytes(B, H, W, C, Cout, int(dx is not None)))
    ws = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device="cuda")    # NaN everywhere: the workspace is not assumed zero
    L_.check(lib.mac_conv3x3_bwd_tc(L_.ptr(x), L_.ptr(y), L_.ptr(dy), L_.ptr(kernel), ACT_ELU, keep, seed, site, step,
                                    L_.ptr(dkernel), L_.ptr(dbias), L_.ptr(dx), L_.ptr(ws), nbytes, B, H, W, C, Cout,
                                    L_.stream_ptr()), "mac_conv3x3_bwd_tc")


@pytest.mark.gpu
@pytest.mark.parametrize("shape,keep,with_dx", [((2, 5, 7, 128, 128), 0.82, True),      # M = 70: not a multiple of 64
                                                ((3, 14, 14, 256, 128), 1.0, True),     # tc_pick_ksplit picks 5 slices
                                                ((64, 14, 14, 1024, 512), 0.82, False),  # headline layer 0
                                                ((64, 14, 14, 512, 512), 0.82, True)])   # headline layer 1
def test_conv3x3_bwd_tc_against_fp64(shape, keep, with_dx):
    bf16_round, excess, _ = _gpu_helpers()
    lib = L_.load()
    B, H, W, C, Cout = shape
    M = B * H * W
    g = torch.Generator(device="cuda").manual_seed(sum(shape))
    x = torch.relu(torch.randn(B, H, W, C, device="cuda", generator=g))
    kernel = torch.randn(3, 3, C, Cout, device="cuda", generator=g) * (2.0 / (9 * (C + Cout))) ** 0.5
    y = torch.nn.functional.elu(torch.randn(M, Cout, device="cuda", generator=g))
    dy = torch.randn(M, Cout, device="cuda", generator=g)
    seed, site, step = 4321, 33, 5
    pre_k = torch.randn(3, 3, C, Cout, device="cuda", generator=g) * 0.1
    pre_b = torch.randn(Cout, device="cuda", generator=g)
    runs = []
    for _ in range(2):
        dkernel, dbias = pre_k.clone(), pre_b.clone()
        dx = torch.full((B, H, W, C), float("nan"), device="cuda") if with_dx else None
        _run_conv(lib, x, y, dy, kernel, keep, seed, site, step, dkernel, dbias, dx, shape)
        runs.append((dkernel, dbias, dx))
    torch.cuda.synchronize()
    same = lambda a, b: torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert same(runs[0][0], runs[1][0]) and same(runs[0][1], runs[1][1])
    if with_dx:
        assert same(runs[0][2], runs[1][2])
    dkernel, dbias, dx = runs[0]
    # the operands the kernels see
    dz32 = dy * torch.where(y > 0, torch.ones_like(y), y + 1)                    # fp32, as mac_activation_bwd forms it
    dz16 = bf16_round(dz32)
    scale = float(np.float32(1.0) / np.float32(keep))
    mask = _uniform_mask(lib, seed, site, step, (B, H, W, C), keep) if keep < 1.0 else torch.ones(B, H, W, C, device="cuda",
                                                                                                     dtype=torch.bool)
    xd16 = bf16_round(x * np.float32(scale)) * mask                               # bf16(dropout(x))
    cols = _patches(xd16)
    ref_k, abs_k = cols.t() @ dz16, cols.abs().t() @ dz16.abs()
    del cols
    rows = {}
    rows["dkernel"] = excess(dkernel.view(-1, Cout), pre_k.double().view(-1, Cout) + ref_k,
                             abs_k + pre_k.double().view(-1, Cout).abs())
    ref_b, abs_b = dz32.double().sum(0), dz32.double().abs().sum(0)
    rows["dbias"] = excess(dbias, pre_b.double() + ref_b, abs_b + pre_b.double().abs())
    if with_dx:
        k16 = bf16_round(kernel.view(-1, Cout))
        f = mask.double() * scale
        ref_x = _col2im(dz16 @ k16.t(), B, H, W, C) * f
        abs_x = _col2im(dz16.abs() @ k16.abs().t(), B, H, W, C) * f
        assert bool(torch.isfinite(dx).all())                                     # every element written
        rows["dx"] = excess(dx, ref_x, abs_x)
    print("conv3x3_bwd_tc %s keep=%s: %s" % (shape, keep, ", ".join("%s %.2e" % kv for kv in rows.items())))
    bad = {k: v for k, v in rows.items() if not v <= TOL_CONV[k]}
    assert not bad, bad


@pytest.mark.gpu
@pytest.mark.parametrize("keep,shape", [(0.82, (2, 5, 7, 128, 128)), (1.0, (4, 14, 14, 256, 256))])
def test_stem_bf16_training_against_fp64_autograd(keep, shape):
    """Stem(prec="bf16") forward(save) + backward against torch.autograd on the fp64 restatement of the fp32 model."""
    from mac_network_b200.stem import Stem, SITE_STEM, stem_specs, init_stem_params
    from tests._util import max_rel
    from oracle.model_torch_autograd import stem_grads
    lib = L_.load()
    B, H, W, cin, cout = shape
    pv = init_stem_params(stem_specs(cin, cout), seed=8, dtype=np.float64)
    images = np.maximum(np.random.RandomState(9).standard_normal((B, H, W, cin)), 0)
    params = {k: torch.from_numpy(v.astype(np.float32)).cuda() for k, v in pv.items()}
    st = Stem(params, relu="ELU", prec="bf16", seed=13)
    kb = st.forward(torch.from_numpy(images.astype(np.float32)).cuda(), keep=keep, step=4, save_for_backward=True)
    d_kb = np.random.RandomState(10).standard_normal(tuple(kb.shape))
    grads = {k: torch.zeros_like(v) for k, v in params.items()}
    d_img = st.backward(torch.from_numpy(d_kb.astype(np.float32)).cuda(), grads, need_d_images=True)
    torch.cuda.synchronize()
    us = []
    if keep < 1.0:
        for layer, c in ((0, cin), (1, cout)):
            u = torch.empty(B * H * W * c, device="cuda")
            L_.check(lib.mac_dropout_uniform(13, SITE_STEM + layer, 4, L_.ptr(u), u.numel(), L_.stream_ptr()))
            us.append(u.cpu().numpy().astype(np.float64).reshape(B, H, W, c))
    kb_ref, gref, dimg_ref = stem_grads("ELU", pv, images, keep, us, d_kb)
    errs = {"kb": max_rel(kb.cpu().numpy(), kb_ref), "d_images": max_rel(d_img.cpu().numpy(), dimg_ref)}
    for k in gref:
        errs[k] = max_rel(grads[k].cpu().numpy(), gref[k])
    print("bf16 stem keep=%s %s: %s" % (keep, shape, ", ".join("%s %.2e" % (k.split("/")[1] if "/" in k else k, v)
                                                               for k, v in errs.items())))
    assert errs["kb"] < 2e-2
    bad = {k: v for k, v in errs.items() if not v < TOL_STEM_BF16}
    assert not bad, bad


def _full_setup(seed):
    from tests.test_full_model import _make
    B, S, V, E, d, H, W, C, A, L = 16, 7, 13, 16, 128, 4, 4, 128, 8, 2      # B*H*W % 64 == 0 (mac_read_bwd_tc)
    cfg, data = _make(B, S, V, E, d, H, W, C, A, L, seed=seed)
    return cfg, data, dict(classifier=(A, [32]), encoder=(V, E), stem=(C, 2)), B, L


@pytest.mark.gpu
def test_full_model_bf16_stem_train_steps_reduce_loss():
    """12 whole-model steps with the cell and the stem on tensor cores: the loss goes down, every sub-model moves."""
    from mac_network_b200.dp import DPTrainer
    cfg, data, kw, B, L = _full_setup(21)
    tr = DPTrainer(cfg, L, seed=6, lr=3e-3, prec="bf16", bwd_tc=True, stem_prec="bf16", **kw)
    dev = {k: torch.from_numpy(v).cuda() for k, v in data.items()}
    before = {k: v.clone() for k, v in tr.params.t.items()}
    hist = []
    for _ in range(12):
        _, losses = tr.train_step_full("t", dev, global_batch=B)
        hist.append(float(losses.mean().item()))
    print("losses", [round(h, 4) for h in hist])
    assert np.all(np.isfinite(hist)) and min(hist[-3:]) < hist[0], hist
    for prefix in ("encoder/", "qEmbeddings/", "stem/", "MACnetwork/", "classifier/"):
        moved = [float((tr.params.t[k] - before[k]).abs().max().item()) for k in before if k.startswith(prefix)]
        assert moved and max(moved) > 0, prefix


@pytest.mark.gpu
def test_full_model_bf16_stem_gradient_matches_fp32_stem():
    """Dropouts off, same parameters and data: the stem's slice of the gradient bucket with stem_prec="bf16" against the
    stem_prec="fp32" trainer (the cell is bf16 / tensor-core in both)."""
    from mac_network_b200.dp import DPTrainer
    cfg, data, kw, B, L = _full_setup(31)
    off = dict(dropouts=(1.0, 1.0, 1.0), output_dropout=1.0, enc_dropouts=(1.0, 1.0), stem_dropout=1.0)
    dev = {k: torch.from_numpy(v).cuda() for k, v in data.items()}
    buckets = {}
    ref_flat = None
    for sp in ("fp32", "bf16"):
        tr = DPTrainer(cfg, L, seed=7, prec="bf16", bwd_tc=True, stem_prec=sp, **kw, **off)
        if ref_flat is None:
            ref_flat = tr.params.flat.clone()
        tr.params.flat.copy_(ref_flat)
        tr.params.touch()
        tr.full_forward_backward("t", dev, global_batch=B)
        torch.cuda.synchronize()
        buckets[sp] = tr.bucket.double().cpu()
    errs = {}
    for n in (n for n in tr.params.specs if n.startswith("stem/")):
        o, k = tr.params.offsets[n], int(np.prod(tr.params.specs[n][0]))
        ref = buckets["fp32"][o:o + k]
        errs[n] = float((buckets["bf16"][o:o + k] - ref).abs().max() / ref.abs().max())
    print("stem gradient bf16 vs fp32 stem:", {k: "%.2e" % v for k, v in errs.items()})
    bad = {k: v for k, v in errs.items() if not v < TOL_TRAINER_STEM}
    assert not bad, bad
