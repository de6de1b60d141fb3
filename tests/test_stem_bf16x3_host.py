"""Host side of the split-bf16 image stem (`Stem(prec="bf16x3")`, DESIGN.md section 9 item 6), without a GPU: the call
sequence of the stem, `DPTrainer(stem_prec="bf16x3")` and `MACnet(eval_stem_prec="bf16x3")` against the dry-run library,
every refusal of `mac_im2col3x3_split`, `mac_linear_tc32_fwd`, `mac_conv3x3_bwd_tc32` and its workspace query through the
real library (each status comes back before any CUDA call), and the Python-level refusals before the library is called."""
import ctypes

import numpy as np
import pytest
import torch

from mac_network_b200 import _lib as L_
from tests import _mocklib
from tests.test_stem_fp8_host import _macnet
from tests.test_stem_tc_training import _cpu_params, _fake_ptr, _host_trainer, _recorder

INVALID, ALIGN, UNSUPPORTED, WORKSPACE, ARCH = -1, -2, -3, -4, -5
ACT_ELU = L_.ACT["ELU"]


def _stem(cin=128, cout=256, **kw):
    from mac_network_b200.stem import Stem, stem_specs, init_stem_params
    p = _cpu_params(init_stem_params(stem_specs(cin, cout), seed=1))
    return Stem(p, relu="ELU", prec="bf16x3", seed=1, **kw), p


# ------------------------------------------------------------------------------------------------ the stem's calls
def test_stem_bf16x3_forward_calls_and_pack_cache(monkeypatch):
    """Per layer: one split3 pack per parameter version, the hi | lo patch matrix, the split-bf16 GEMM."""
    rec = _recorder(monkeypatch)
    from mac_network_b200.stem import SITE_STEM
    version = [0]
    st, _ = _stem(version=lambda: version[0])
    kb = st.forward(torch.zeros(2, 5, 7, 128), keep=0.82, step=3)
    assert kb.shape == (2, 35, 256)
    assert [n for n, _ in rec.log] == ["mac_pack_weight_split3", "mac_im2col3x3_split", "mac_linear_tc32_fwd"] * 2
    assert [a[2:4] for a in rec.args_of("mac_pack_weight_split3")] == [(9 * 128, 256), (9 * 256, 256)]
    _, W3 = st._weights(0)
    assert W3.shape == (256, 3 * 9 * 128) and W3.dtype == torch.bfloat16
    im = rec.args_of("mac_im2col3x3_split")
    assert [a[-5:-1] for a in im] == [(2, 5, 7, 128), (2, 5, 7, 256)]
    assert [a[4] for a in im] == [SITE_STEM, SITE_STEM + 1] and all(a[2] == pytest.approx(0.82) and a[5] == 3 for a in im)
    assert [a[3:4] + a[5:8] for a in rec.args_of("mac_linear_tc32_fwd")] == [(ACT_ELU, 70, 9 * 128, 256),
                                                                            (ACT_ELU, 70, 9 * 256, 256)]
    count = lambda: len(rec.args_of("mac_pack_weight_split3"))
    st.forward(torch.zeros(2, 5, 7, 128))
    assert count() == 2                                      # same version: the packs are reused
    version[0] += 1
    st.forward(torch.zeros(2, 5, 7, 128))
    assert count() == 4                                      # a parameter update repacks both layers
    assert not rec.args_of("mac_im2col3x3") and not rec.args_of("mac_linear_fwd") and not rec.args_of("mac_linear_tc_fwd")


def test_stem_bf16x3_training_calls(monkeypatch):
    rec = _recorder(monkeypatch)
    from mac_network_b200.stem import SITE_STEM
    st, p = _stem()
    x = torch.zeros(2, 5, 7, 128)
    kb = st.forward(x, keep=0.82, step=3, save_for_backward=True)
    sv = st._saved
    assert sv["xs"][0] is x and [tuple(t.shape) for t in sv["xs"]] == [(2, 5, 7, 128), (2, 5, 7, 256)]
    assert [(tuple(t.shape), t.dtype) for t in sv["ys"]] == [((70, 256), torch.float32)] * 2      # fp32, as every precision
    grads = {k: torch.zeros_like(v) for k, v in p.items()}
    for need in (False, True):
        rec.log.clear()
        d_img = st.backward(torch.zeros_like(kb), grads, need_d_images=need)
        layer1, layer0 = rec.args_of("mac_conv3x3_bwd_tc32")                                        # last layer first
        assert [n for n, _ in rec.log] == ["mac_conv3x3_bwd_tc32_workspace_bytes", "mac_conv3x3_bwd_tc32"] * 2
        assert layer1[7] == SITE_STEM + 1 and layer0[7] == SITE_STEM
        assert layer1[-6:-1] == (2, 5, 7, 256, 256) and layer0[-6:-1] == (2, 5, 7, 128, 256)
        assert layer1[4] == ACT_ELU and layer1[5] == pytest.approx(0.82) and layer1[8] == 3
        assert layer1[11] is not None and (layer0[11] is not None) == need
        assert [a[-1] for a in rec.args_of("mac_conv3x3_bwd_tc32_workspace_bytes")] == [1, int(need)]
        assert (d_img is not None) == need


@pytest.mark.parametrize("cin,cout", [(96, 128), (128, 64), (64, 128)])
def test_stem_bf16x3_refuses_channel_counts_before_any_call(monkeypatch, cin, cout):
    """inference and training alike: every channel count a multiple of 128"""
    mock = _mocklib.install(monkeypatch)
    st, _ = _stem(cin, cout)
    for kw in ({}, dict(keep=0.82, save_for_backward=True)):
        with pytest.raises(NotImplementedError, match="multiples of 128"):
            st.forward(torch.zeros(1, 3, 3, cin), **kw)
    assert mock.calls == []


def test_trainer_and_macnet_accept_bf16x3_and_refuse_the_rest(monkeypatch):
    mock = _mocklib.install(monkeypatch)
    tr = _host_trainer(monkeypatch, stem=(128, 2), stem_prec="bf16x3")
    assert tr.stem.prec == "bf16x3" and tr.prec == "fp32" and not tr.bwd_tc           # independent of prec and bwd_tc
    assert _host_trainer(monkeypatch, stem=(128, 2), stem_prec="bf16x3", prec="tc32", bwd_tc=True).stem.prec == "bf16x3"
    mock.calls.clear()
    with pytest.raises(NotImplementedError, match="multiples of 128"):
        _host_trainer(monkeypatch, stem=(96, 2), stem_prec="bf16x3")
    with pytest.raises(ValueError, match="needs stem="):
        _host_trainer(monkeypatch, stem_prec="bf16x3")
    for bad in ("fp16", "fp8", "tc32", "bf16x2"):
        with pytest.raises(ValueError, match="stem_prec"):
            _host_trainer(monkeypatch, stem=(128, 2), stem_prec=bad)
    assert mock.calls == []
    for bad in ("bf16", "fp32", "e4m3", "tc32"):
        with pytest.raises(ValueError, match="eval_stem_prec"):
            _macnet(monkeypatch, 128, "bf16", eval_stem_prec=bad)
    # "tc32" on the stem itself keeps constructing and keeps refusing to train
    from mac_network_b200.stem import Stem, stem_specs, init_stem_params
    p = _cpu_params(init_stem_params(stem_specs(128, 128), seed=1))
    with pytest.raises(NotImplementedError):
        Stem(p, relu="ELU", prec="tc32", seed=1).forward(torch.zeros(1, 3, 3, 128), save_for_backward=True)


def test_macnet_eval_stem_bf16x3_host_calls(monkeypatch):
    mock, net, data, images = _macnet(monkeypatch, 128, "bf16", eval_stem_prec="bf16x3")
    assert net._stem.prec == "bf16x3" and net.trainer.stem.prec == "fp32"
    net.runBatch(None, data, images, train=False)
    assert mock.calls.count("mac_im2col3x3_split") == 2 and mock.calls.count("mac_linear_tc32_fwd") == 2
    assert "mac_im2col3x3" not in mock.calls
    net.trainer.params.touch()
    n = mock.calls.count("mac_pack_weight_split3")
    net.runBatch(None, data, images, train=False)
    assert mock.calls.count("mac_pack_weight_split3") == n + 2
    mock.calls.clear()
    net.runBatch(None, data, images, train=True)                 # training keeps its own (fp32) stem
    assert "mac_im2col3x3_split" not in mock.calls and "mac_im2col3x3" in mock.calls
    _, net, _, _ = _macnet(monkeypatch, 128, "tc32")             # no new mapping: the tc32 cell keeps the stem it had
    assert net._stem.prec == "tc32"


def test_train_step_full_reaches_conv3x3_bwd_tc32_once_per_layer(monkeypatch):
    """DPTrainer(stem_prec="bf16x3").train_step_full with the cell stubbed out."""
    rec = _recorder(monkeypatch)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True), raising=False)
    from mac_network_b200 import autograd, dp, mac_cell
    from mac_network_b200.config import MACConfig
    B, S, V, E, d, H, W, C, A, L = 4, 6, 9, 12, 128, 3, 3, 128, 8, 2
    cfg = MACConfig.args("args", netLength=L, memDim=d, ctrlDim=d, attDim=d)
    tr = dp.DPTrainer(cfg, L, seed=1, device="cpu", classifier=(A, [16]), encoder=(V, E), stem=(C, 2), stem_prec="bf16x3")

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
    tr.train_step_full("k", data, global_batch=B)
    conv = rec.args_of("mac_conv3x3_bwd_tc32")
    assert len(conv) == 2 and conv[0][11] is not None and conv[1][11] is None      # the image gradient is not needed
    assert len(rec.args_of("mac_im2col3x3_split")) == 2 and len(rec.args_of("mac_linear_tc32_fwd")) == 2
    assert not rec.args_of("mac_im2col3x3") and not rec.args_of("mac_col2im3x3") and not rec.args_of("mac_conv3x3_bwd_tc")
    assert tr.step_id == 1


# ------------------------------------------------------------------------------------------------ the library's refusals
def _p():
    buf = (ctypes.c_float * 4096)()
    return buf, _fake_ptr(buf)


def test_im2col3x3_split_status_codes():
    lib = L_.load()
    buf, p = _p()

    def call(x=p, cols=p, keep=0.82, B=2, H=5, W=7, C=128):
        return lib.mac_im2col3x3_split(x, cols, keep, 7, 32, 1, B, H, W, C, None)
    assert call(x=None) == INVALID and call(cols=None) == INVALID
    assert call(B=0) == INVALID and call(H=0) == INVALID and call(W=-1) == INVALID and call(C=0) == INVALID
    assert call(keep=0.0) == INVALID and call(keep=1.5) == INVALID
    assert call(C=96) == UNSUPPORTED and call(C=32) == UNSUPPORTED
    assert call(x=p + 4) == ALIGN and call(cols=p + 8) == ALIGN


def test_linear_tc32_fwd_status_codes():
    lib = L_.load()
    buf, p = _p()

    def call(a=p, w=p, b=p, act=ACT_ELU, y=p, M=70, K=1152, N=256):
        return lib.mac_linear_tc32_fwd(a, w, b, act, y, M, K, N, None)
    assert call(a=None) == INVALID and call(w=None) == INVALID and call(y=None) == INVALID
    assert call(M=0) == INVALID and call(K=0) == INVALID and call(N=-128) == INVALID
    assert call(K=1120) == UNSUPPORTED and call(N=192) == UNSUPPORTED and call(act=5) == UNSUPPORTED
    assert call(a=p + 4) == ALIGN and call(w=p + 8) == ALIGN and call(y=p + 4) == ALIGN
    if not torch.cuda.is_available():
        # every argument check passed: K = 1088 is 17 whole 64-element k-blocks, the bias is optional, any M
        assert call(K=1088, b=None, M=1) == ARCH


def test_conv3x3_bwd_tc32_status_codes():
    lib = L_.load()
    buf, p = _p()

    def call(x=p, C=128, Cout=128, ws_bytes=1 << 40, dx=p, keep=0.82, kernel=p, ws=p):
        return lib.mac_conv3x3_bwd_tc32(x, p, p, kernel, ACT_ELU, keep, 7, 32, 1, p, p, dx, ws, ws_bytes, 2, 5, 7, C, Cout, None)
    assert call(C=96) == UNSUPPORTED and call(Cout=96) == UNSUPPORTED and call(C=64) == UNSUPPORTED
    assert call(x=None) == INVALID and call(kernel=None) == INVALID and call(ws=None) == INVALID and call(keep=0.0) == INVALID
    assert call(kernel=p + 4) == ALIGN and call(dx=p + 8) == ALIGN
    q = lib.mac_conv3x3_bwd_tc32_workspace_bytes
    assert q(0, 5, 7, 128, 128, 1) == 0 and q(2, 5, 7, 128, 0, 1) == 0
    need, no_dx = q(2, 5, 7, 128, 128, 1), q(2, 5, 7, 128, 128, 0)
    assert call(ws_bytes=need - 1) == WORKSPACE and call(ws_bytes=no_dx - 1, dx=None) == WORKSPACE
    if not torch.cuda.is_available():
        assert call(ws_bytes=need) == ARCH and call(ws_bytes=no_dx, dx=None) == ARCH
    # M = 70, Mp = 128, K = 9C = 1152: [dZ^T] x 3, [cols^T] x 2, one slice of fp32 partials at least
    assert no_dx >= 128 * 128 * 2 * 3 + 1152 * 128 * 2 * 2 + 1152 * 128 * 4
    # with dx: the [hi | lo] rows of dZ, the kernel as [hi | hi | lo] and the fp32 patch gradient
    assert need >= no_dx + 70 * 128 * 2 * 2 + 1152 * 128 * 2 * 3 + 70 * 1152 * 4
    assert need > lib.mac_conv3x3_bwd_tc_workspace_bytes(2, 5, 7, 128, 128, 1)
