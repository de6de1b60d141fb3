"""CPU side of the e4m3 inference stem (Stem(prec="fp8"), csrc/tc_gemm_fp8.cuh): the restatement of the scheme
(oracle/fp8_stem_oracle.py) against the fp64 convolution, the host plumbing of Stem and MACnet(eval_stem_prec="fp8") against
the dry-run library (tests/_mocklib.py), and the C entry points' rejections, which return before any CUDA call."""
import ctypes

import numpy as np
import pytest
import torch

from mac_network_b200 import _lib as L_
from oracle import fp8_stem_oracle as F8S
from oracle.stem_oracle import stem_forward as stem_fp64
from tests import _mocklib

INVALID, ALIGN, UNSUPPORTED, WORKSPACE = -1, -2, -3, -4
FP8_STEM_CALLS = ("mac_im2col3x3_fp8", "mac_linear_fp8_fwd", "mac_pack_weight_fp8")


def _params(cin, cout, seed=1, bias_scale=0.1):
    from mac_network_b200.stem import init_stem_params, stem_specs
    return init_stem_params(stem_specs(cin, cout), seed=seed, bias_scale=bias_scale)


def test_patch_quantisation_scales_and_zero_windows():
    """sA is the window amax over 448 in fp32; each row's largest element maps to 448; a window with no nonzero pixel has
    sA = 0 and zero bytes; the patch layout is mac_im2col3x3's (tap-major, channel fastest)."""
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 6, 5, 128, generator=g)
    x[1] = 0
    x[1, 0, 0] = torch.randn(128, generator=g)                # one pixel: only its neighbours' windows are nonzero
    cols8, sA = F8S.quant_patches(x)
    assert cols8.shape == (60, 9 * 128) and sA.dtype == torch.float32
    am = F8S.window_amax(x)
    assert torch.equal(sA, am / torch.full_like(am, 448.0))
    nz = sA > 0
    assert int(nz[30:].sum()) == 4                           # pixel (0, 0) lies in the windows of (0,0), (0,1), (1,0), (1,1)
    assert bool((cols8[~nz] == 0).all())
    assert bool((cols8[nz].abs().amax(1) == 448.0).all())
    ref = F8S.im2col3x3(x.double())
    err = (cols8 * sA.double()[:, None] - ref).abs().amax(1) / ref.abs().amax(1).clamp_min(1e-300)
    assert float(err[nz].max()) <= 2 ** -4                   # half an e4m3 step (3 mantissa bits)


def test_restatement_is_within_e4m3_distance_of_fp64_conv():
    """The two-layer e4m3 stem (128 -> 256 -> 256, xavier kernels as the model initialises them) against the fp64 convolution
    of oracle/stem_oracle.py: a few per cent (max-norm), the size of e4m3's 3-bit mantissa on both operands.  Measured 5.3e-2;
    below 1e-2 the operands would not be e4m3 at all."""
    rng = np.random.RandomState(4)
    p = _params(128, 256, seed=2)
    images = np.maximum(rng.standard_normal((2, 7, 7, 128)), 0).astype(np.float32)
    ref = stem_fp64("ELU", p, images)
    got = F8S.stem_forward("ELU", p, images).numpy()
    err = float(np.abs(got - ref).max() / np.abs(ref).max())
    assert 1e-2 < err < 1e-1, err


def _counter_stem(monkeypatch, cin=128, cout=256, **kw):
    mock = _mocklib.install(monkeypatch)
    from mac_network_b200.stem import Stem
    p = {k: torch.from_numpy(v) for k, v in _params(cin, cout).items()}
    version = [0]
    st = Stem(p, relu="ELU", prec="fp8", version=lambda: version[0], **kw)
    return mock, st, version


def test_stem_fp8_host_calls(monkeypatch):
    """Per layer: im2col in e4m3 with its workspace query, then the e4m3 GEMM; the weights are packed once per layer per
    parameter version and again after the version moves."""
    mock, st, version = _counter_stem(monkeypatch)
    seen = []
    for name in ("mac_im2col3x3_fp8", "mac_linear_fp8_fwd", "mac_pack_weight_fp8"):
        fn = getattr(mock, name)

        def spy(*a, _fn=fn, _name=name):
            seen.append((_name, a))
            return _fn(*a)
        setattr(mock, name, spy)
    kb = st.forward(torch.zeros(2, 5, 7, 128))
    assert kb.shape == (2, 35, 256)
    assert mock.calls == ["mac_pack_weight_fp8", "mac_im2col3x3_fp8_workspace_bytes", "mac_im2col3x3_fp8",
                          "mac_linear_fp8_fwd"] * 2
    assert [a[-5:-1] for n, a in seen if n == "mac_im2col3x3_fp8"] == [(2, 5, 7, 128), (2, 5, 7, 256)]
    assert [(a[5], a[-4], a[-3], a[-2]) for n, a in seen if n == "mac_linear_fp8_fwd"] == \
        [(L_.ACT["ELU"], 70, 9 * 128, 256), (L_.ACT["ELU"], 70, 9 * 256, 256)]
    assert [a[-3:-1] for n, a in seen if n == "mac_pack_weight_fp8"] == [(9 * 128, 256), (9 * 256, 256)]
    assert "mac_im2col3x3" not in mock.calls and "mac_linear_tc_fwd" not in mock.calls
    st.forward(torch.zeros(2, 5, 7, 128))
    assert mock.calls.count("mac_pack_weight_fp8") == 2                  # same version: the packs are reused
    version[0] += 1
    st.forward(torch.zeros(2, 5, 7, 128))
    assert mock.calls.count("mac_pack_weight_fp8") == 4                  # a parameter update repacks both layers
    version[0] += 1                                                      # as MACnet._swap_ema's touch() does
    st.forward(torch.zeros(2, 5, 7, 128))
    assert mock.calls.count("mac_pack_weight_fp8") == 6


@pytest.mark.parametrize("what", ["train", "keep", "cin", "cout"])
def test_stem_fp8_rejections_before_any_launch(monkeypatch, what):
    """Training (forward with save_for_backward), dropout and channel counts that are not multiples of 128 raise
    NotImplementedError before the library is asked to compute anything."""
    cin, cout = {"cin": (96, 128), "cout": (128, 64)}.get(what, (128, 128))
    mock, st, _ = _counter_stem(monkeypatch, cin=cin, cout=cout)
    kw = {"train": dict(save_for_backward=True), "keep": dict(keep=0.82)}.get(what, {})
    with pytest.raises(NotImplementedError):
        st.forward(torch.zeros(1, 3, 3, cin), **kw)
    assert mock.calls == []


def _macnet(monkeypatch, d, prec, **kw):
    mock = _mocklib.install(monkeypatch)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True), raising=False)
    from mac_network_b200.config import MACConfig
    from mac_network_b200.model import MACnet
    B, S, V, E, H, W, C, A, L = 4, 6, 9, 12, 3, 3, 128, 8, 2
    cfg = MACConfig.args("args", netLength=L, memDim=d, ctrlDim=d, attDim=d)
    net = MACnet(cfg, L, V, A, wrd_emb_dim=E, image_in_dim=C, classifier_dims=(16,), prec=prec, device="cpu", **kw)
    rng = np.random.RandomState(0)
    lengths = np.array([5, 6, 2, 4], dtype=np.int32)
    q = rng.randint(1, V + 1, size=(B, S)).astype(np.int32)
    q[np.arange(S)[None, :] >= lengths[:, None]] = 0
    data = {"questions": q, "questionLengths": lengths, "answers": rng.randint(0, A, size=(B,)).astype(np.int32)}
    images = {"images": rng.standard_normal((B, C, H, W)).astype(np.float32)}
    return mock, net, data, images


def test_macnet_eval_stem_fp8_host_calls(monkeypatch):
    """MACnet(eval_stem_prec="fp8"): the evaluation stem runs in e4m3 (one pack per layer per parameter version, a repack
    after touch()); training keeps its own stem and makes no e4m3 stem call."""
    mock, net, data, images = _macnet(monkeypatch, 128, "bf16", eval_stem_prec="fp8")
    assert net._stem.prec == "fp8" and net.trainer.stem.prec == "fp32"
    net.runBatch(None, data, images, train=False)
    assert mock.calls.count("mac_im2col3x3_fp8") == 2 and mock.calls.count("mac_linear_fp8_fwd") == 2
    assert mock.calls.count("mac_pack_weight_fp8") == 2
    assert "mac_im2col3x3" not in mock.calls and "mac_read_invariant" in mock.calls
    net.runBatch(None, data, images, train=False)
    assert mock.calls.count("mac_pack_weight_fp8") == 2
    net.trainer.params.touch()
    net.runBatch(None, data, images, train=False)
    assert mock.calls.count("mac_pack_weight_fp8") == 4
    mock.calls.clear()
    net.runBatch(None, data, images, train=True)
    assert not any(c in mock.calls for c in FP8_STEM_CALLS) and "mac_im2col3x3" in mock.calls


def test_macnet_default_eval_stem_is_unchanged(monkeypatch):
    """eval_stem_prec=None keeps today's mapping: under prec="fp8" the stem runs in bf16, with no e4m3 stem call."""
    mock, net, data, images = _macnet(monkeypatch, 512, "fp8")
    assert net._stem.prec == "bf16"
    net.runBatch(None, data, images, train=False)
    assert not any(c in mock.calls for c in ("mac_im2col3x3_fp8", "mac_linear_fp8_fwd"))
    assert mock.calls.count("mac_linear_tc_fwd") == 2 and mock.calls.count("mac_pack_weight_fp8") == 2   # the read step's


def test_bad_eval_stem_prec_and_fp8_stem_training_raise(monkeypatch):
    for bad in ("bf16", "fp32", "e4m3"):
        with pytest.raises(ValueError, match="eval_stem_prec"):
            _macnet(monkeypatch, 128, "bf16", eval_stem_prec=bad)
    from mac_network_b200 import dp
    from mac_network_b200.config import MACConfig
    cfg = MACConfig.args("args", netLength=2, memDim=128, ctrlDim=128, attDim=128)
    with pytest.raises(ValueError, match="stem_prec"):
        dp.DPTrainer(cfg, 2, seed=1, device="cpu", classifier=(8, [16]), encoder=(9, 12), stem=(128, 2), stem_prec="fp8")


def _fake_ptr(buf):
    return (ctypes.addressof(buf) + 15) & ~15          # 16-byte aligned fake "device" pointer (never dereferenced)


def test_im2col3x3_fp8_status_codes():
    lib = L_.load()
    buf = (ctypes.c_float * 4096)()
    p = _fake_ptr(buf)
    need = lib.mac_im2col3x3_fp8_workspace_bytes(2, 5, 7, 128)
    assert need >= 2 * 5 * 7 * 4
    assert lib.mac_im2col3x3_fp8_workspace_bytes(0, 5, 7, 128) == 0

    def call(x=p, cols=p, sa=p, ws=p, ws_bytes=need, B=2, H=5, W=7, C=128):
        return lib.mac_im2col3x3_fp8(x, cols, sa, ws, ws_bytes, B, H, W, C, None)
    assert call(x=None) == INVALID and call(cols=None) == INVALID and call(sa=None) == INVALID and call(ws=None) == INVALID
    assert call(B=0) == INVALID and call(H=0) == INVALID and call(W=-1) == INVALID and call(C=0) == INVALID
    assert call(C=96) == UNSUPPORTED and call(C=64) == UNSUPPORTED
    assert call(x=p + 4) == ALIGN and call(cols=p + 8) == ALIGN
    assert call(ws_bytes=need - 1) == WORKSPACE


def test_linear_fp8_fwd_status_codes():
    lib = L_.load()
    buf = (ctypes.c_float * 4096)()
    p = _fake_ptr(buf)

    def call(x=p, sa=p, w=p, sw=p, b=p, act=L_.ACT["ELU"], y=p, M=70, K=1152, N=256):
        return lib.mac_linear_fp8_fwd(x, sa, w, sw, b, act, y, M, K, N, None)
    assert call(x=None) == INVALID and call(sa=None) == INVALID and call(w=None) == INVALID
    assert call(sw=None) == INVALID and call(y=None) == INVALID
    assert call(M=0) == INVALID and call(M=-3) == INVALID and call(K=0) == INVALID and call(N=0) == INVALID
    assert call(K=1088) == UNSUPPORTED and call(N=192) == UNSUPPORTED
    assert call(act=L_.ACT["TANH"]) == UNSUPPORTED and call(act=L_.ACT["SIGMOID"]) == UNSUPPORTED
    assert call(x=p + 4) == ALIGN and call(y=p + 8) == ALIGN
