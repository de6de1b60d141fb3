"""CPU side of the tensor-core question encoder (QuestionEncoder(prec="bf16"), csrc/encoder_tc.cuh): the fp64 restatement
(oracle/encoder_tc_oracle.py) without rounding against the encoder oracle and torch.autograd, the host plumbing of the
encoder, DPTrainer(enc_prec="bf16") and MACnet(eval_enc_prec="bf16") against the dry-run library (tests/_mocklib.py), and the
C entry points' rejections, which return before any CUDA call."""
import ctypes

import numpy as np
import pytest
import torch

from mac_network_b200 import _lib as L_
from mac_network_b200.encoder import encoder_specs, init_encoder_params
from oracle import encoder_torch_autograd
from oracle.encoder_oracle import encoder_forward
from oracle.encoder_tc_oracle import EncoderTC
from tests import _mocklib

INVALID, ALIGN, UNSUPPORTED, WORKSPACE = -1, -2, -3, -4
TC_CALLS = ("mac_embed_fwd_tc", "mac_pack_weight_bf16_kpad", "mac_lstm_fwd_tc", "mac_lstm_bwd_tc")


def _batch(B, S, V, seed):
    rng = np.random.RandomState(seed)
    lengths = rng.randint(1, S + 1, size=(B,)).astype(np.int32)
    lengths[0] = S
    q = rng.randint(1, V + 1, size=(B, S)).astype(np.int32)
    q[np.arange(S)[None, :] >= lengths[:, None]] = 0
    return q, lengths


@pytest.mark.parametrize("bi", [True, False])
def test_restatement_without_rounding_is_the_encoder(bi):
    """bf16=False: outputs equal encoder_forward and gradients equal torch.autograd on the fp64 restatement."""
    B, S, V, E, D = 5, 6, 9, 8, 12
    pv = init_encoder_params(encoder_specs(V, E, D, bi=bi), seed=3, dtype=np.float64)
    q, lengths = _batch(B, S, V, 4)
    rng = np.random.RandomState(5)
    us = [rng.uniform(size=(B, S, E)), rng.uniform(size=(B, D))]
    ref = encoder_forward(pv, q, lengths, 0.8, 0.9, uniforms=[u.copy() for u in us])
    tc = EncoderTC(pv, 0.8, 0.9, uniforms=us, bf16=False)
    out = tc.forward(q, lengths)
    for k in ("questionWords", "questionCntxWords", "vecQuestions"):
        assert np.max(np.abs(out[k] - ref[k])) < 1e-12, k
    if not bi:
        return
    d_cntx, d_vecq = rng.standard_normal((B, S, D)), rng.standard_normal((B, D))
    _, _, gref = encoder_torch_autograd.run(pv, q, lengths, 0.8, 0.9, us, d_cntx=d_cntx, d_vecq=d_vecq)
    got = tc.backward(d_cntx, d_vecq)
    for k, g in gref.items():
        assert np.max(np.abs(got[k] - g)) < 1e-10 * max(1.0, np.max(np.abs(g))), k


def test_restatement_rounds_products_to_bf16():
    """With rounding the restatement moves by about bf16's resolution, not more."""
    B, S, V, E, D = 4, 5, 7, 20, 16
    pv = init_encoder_params(encoder_specs(V, E, D), seed=6, dtype=np.float64)
    q, lengths = _batch(B, S, V, 7)
    a = EncoderTC(pv, bf16=False).forward(q, lengths)["questionCntxWords"]
    b = EncoderTC(pv, bf16=True).forward(q, lengths)["questionCntxWords"]
    err = np.max(np.abs(a - b)) / np.max(np.abs(a))
    assert 1e-4 < err < 3e-2, err


def _aligned():
    buf = (ctypes.c_float * 8192)()
    return (ctypes.addressof(buf) + 15) & ~15, buf


def test_entry_point_status_codes_without_gpu():
    """Bad arguments, unsupported h and short workspaces come back as MAC_ERR_* before any CUDA call."""
    lib = L_.load()
    p, _keep = _aligned()
    fwd = lambda gx_bw, h, nd, out=p, sg=None, sc=None, shp=None: lib.mac_lstm_fwd_tc(
        p, gx_bw, p, gx_bw, p, 1.0, out, None, sg, sc, shp, 2, 3, h, nd, None)
    assert fwd(p, 128, 2) == UNSUPPORTED
    assert fwd(p, 512, 2) == UNSUPPORTED
    assert fwd(None, 256, 2) == INVALID                           # two directions need both
    assert fwd(p, 256, 3) == INVALID
    assert fwd(p, 256, 2, out=None) == INVALID
    assert fwd(p, 256, 2, sg=p) == INVALID                        # saved tensors: all or none
    assert fwd(p, 256, 2, out=p + 4) == ALIGN
    assert lib.mac_lstm_fwd_tc(p, p, p, p, p, 1.0, p, None, None, None, None, 0, 3, 256, 2, None) == INVALID
    ws = lambda B, S, E, h, nd: lib.mac_lstm_bwd_tc_workspace_bytes(B, S, E, h, nd)
    assert ws(64, 40, 300, 128, 2) == 0 and ws(64, 40, 300, 256, 3) == 0
    need = ws(64, 40, 300, 256, 2)
    assert need > 2 * 64 * 40 * 1024 * 4                         # at least the fp32 gate gradients of both directions
    bwd = lambda wsb, h=256, E=300, x=p, dx=p: lib.mac_lstm_bwd_tc(
        x, p, p, p, p, p, p, p, None, p, p, p, p, dx, p, wsb, 64, 40, E, h, 2, None)
    assert bwd(need - 1) == WORKSPACE
    assert bwd(need, h=128) == UNSUPPORTED
    assert bwd(need, E=302) == INVALID                            # E % 4
    assert bwd(need, x=None) == INVALID
    assert bwd(need, dx=p + 4) == ALIGN
    emb = lambda keep, E, out=p: lib.mac_embed_fwd_tc(p, p, keep, 1, 48, 0, out, p, 2, 3, 5, E, None)
    assert emb(1.0, 6) == INVALID and emb(0.0, 8) == INVALID and emb(1.0, 8, out=None) == INVALID
    assert emb(1.0, 8, out=p + 4) == ALIGN
    assert lib.mac_pack_weight_bf16_kpad(p, p, 300, 256, 1024, None) == INVALID


def _encoder(monkeypatch, D=512, E=300, bi=True, **kw):
    mock = _mocklib.install(monkeypatch)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True), raising=False)
    from mac_network_b200.encoder import QuestionEncoder
    pv = init_encoder_params(encoder_specs(9, E, D, bi=bi), seed=1)
    version = [0]
    enc = QuestionEncoder({k: torch.from_numpy(v) for k, v in pv.items()}, prec="bf16", version=lambda: version[0], **kw)
    return mock, enc, version


def test_encoder_bf16_host_calls(monkeypatch):
    """Forward: one embed pass, one packed projection per direction, one recurrence launch; backward: one call, then the
    embedding gradient.  kernel[0:E] is packed once per direction per parameter version."""
    mock, enc, version = _encoder(monkeypatch, keep_input=0.85, keep_question=0.92)
    seen = []
    for name in ("mac_pack_weight_bf16_kpad", "mac_linear_tc_fwd", "mac_lstm_fwd_tc", "mac_lstm_bwd_tc"):
        fn = getattr(mock, name)

        def spy(*a, _fn=fn, _name=name):
            seen.append((_name, a))
            return _fn(*a)
        setattr(mock, name, spy)
    q = torch.ones(3, 7, dtype=torch.int32)
    words, cntx, vecq = enc.forward(q, torch.tensor([7, 1, 4]), step=2, save_for_backward=True)
    assert words.shape == (3, 7, 300) and cntx.shape == (3, 7, 512) and vecq.shape == (3, 512)
    assert mock.calls == ["mac_embed_fwd_tc", "mac_pack_weight_bf16_kpad", "mac_linear_tc_fwd", "mac_pack_weight_bf16_kpad",
                          "mac_linear_tc_fwd", "mac_lstm_fwd_tc", "mac_dropout_fwd"]
    assert [a[-4:-1] for n, a in seen if n == "mac_pack_weight_bf16_kpad"] == [(300, 384, 1024)] * 2
    assert [a[-4:-1] for n, a in seen if n == "mac_linear_tc_fwd"] == [(21, 384, 1024)] * 2
    assert [a[-5:-1] for n, a in seen if n == "mac_lstm_fwd_tc"] == [(3, 7, 256, 2)]
    mock.calls.clear()
    grads = {k: torch.zeros_like(v) for k, v in enc.p.items()}
    enc.backward(torch.zeros(3, 7, 512), torch.zeros(3, 512), grads)
    assert mock.calls == ["mac_dropout_fwd", "mac_lstm_bwd_tc_workspace_bytes", "mac_lstm_bwd_tc", "mac_embed_bwd"]
    assert [a[-6:-1] for n, a in seen if n == "mac_lstm_bwd_tc"] == [(3, 7, 300, 256, 2)]
    mock.calls.clear()
    enc.forward(q, torch.tensor([7, 1, 4]))
    assert "mac_pack_weight_bf16_kpad" not in mock.calls                # same version: packs reused
    version[0] += 1
    enc.forward(q, torch.tensor([7, 1, 4]))
    assert mock.calls.count("mac_pack_weight_bf16_kpad") == 2


def test_encoder_bf16_unidirectional_host_calls(monkeypatch):
    mock, enc, _ = _encoder(monkeypatch, D=256, E=256, bi=False)
    enc.forward(torch.ones(2, 3, dtype=torch.int32), torch.tensor([3, 2]))
    assert mock.calls.count("mac_linear_tc_fwd") == 1 and mock.calls.count("mac_lstm_fwd_tc") == 1


@pytest.mark.parametrize("what", ["h", "prec"])
def test_encoder_rejections_before_any_launch(monkeypatch, what):
    """An unsupported hidden size raises NotImplementedError and an unknown prec ValueError, before any library call."""
    mock = _mocklib.install(monkeypatch)
    from mac_network_b200.encoder import QuestionEncoder
    D = 64 if what == "h" else 512
    p = {k: torch.from_numpy(v) for k, v in init_encoder_params(encoder_specs(9, 12, D), seed=1).items()}
    with pytest.raises(NotImplementedError if what == "h" else ValueError):
        QuestionEncoder(p, prec="bf16" if what == "h" else "fp16")
    assert mock.calls == []


def _macnet(monkeypatch, d=512, **kw):
    mock = _mocklib.install(monkeypatch)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True), raising=False)
    from mac_network_b200.config import MACConfig
    from mac_network_b200.model import MACnet
    B, S, V, E, H, W, C, A, L = 4, 6, 9, 12, 3, 3, 128, 8, 2
    cfg = MACConfig.args("args", netLength=L, memDim=d, ctrlDim=d, attDim=d)
    net = MACnet(cfg, L, V, A, wrd_emb_dim=E, image_in_dim=C, classifier_dims=(16,), prec="bf16", device="cpu", **kw)
    rng = np.random.RandomState(0)
    lengths = np.array([5, 6, 2, 4], dtype=np.int32)
    q = rng.randint(1, V + 1, size=(B, S)).astype(np.int32)
    q[np.arange(S)[None, :] >= lengths[:, None]] = 0
    data = {"questions": q, "questionLengths": lengths, "answers": rng.randint(0, A, size=(B,)).astype(np.int32)}
    images = {"images": rng.standard_normal((B, C, H, W)).astype(np.float32)}
    return mock, net, data, images


def test_dptrainer_enc_prec_bf16_train_step_full(monkeypatch):
    """DPTrainer(enc_prec="bf16").train_step_full: the encoder forward and backward run on the tensor-core entry points and
    the fp32 LSTM entry points are not called; the evaluation encoder stays fp32."""
    mock, net, data, images = _macnet(monkeypatch, enc_prec="bf16")
    assert net.trainer.enc.prec == "bf16" and net._enc.prec == "fp32"
    net.runBatch(None, data, images, train=True)
    assert all(c in mock.calls for c in TC_CALLS)
    assert "mac_lstm_fwd" not in mock.calls and "mac_lstm_bwd" not in mock.calls


def test_macnet_eval_enc_prec_bf16_run_batch(monkeypatch):
    mock, net, data, images = _macnet(monkeypatch, eval_enc_prec="bf16")
    assert net._enc.prec == "bf16" and net.trainer.enc.prec == "fp32"
    net.runBatch(None, data, images, train=False)
    assert "mac_lstm_fwd_tc" in mock.calls and "mac_lstm_fwd" not in mock.calls
    assert mock.calls.count("mac_pack_weight_bf16_kpad") == 2
    net.runBatch(None, data, images, train=False)
    assert mock.calls.count("mac_pack_weight_bf16_kpad") == 2
    net.trainer.params.touch()
    net.runBatch(None, data, images, train=False)
    assert mock.calls.count("mac_pack_weight_bf16_kpad") == 4


def test_defaults_leave_the_encoder_fp32(monkeypatch):
    mock, net, data, images = _macnet(monkeypatch)
    assert net._enc.prec == "fp32" and net.trainer.enc.prec == "fp32"
    net.runBatch(None, data, images, train=True)
    net.runBatch(None, data, images, train=False)
    assert not any(c in mock.calls for c in TC_CALLS)


@pytest.mark.parametrize("kw,exc", [(dict(eval_enc_prec="fp8"), ValueError), (dict(enc_prec="fp16"), ValueError)])
def test_prec_arguments_reject_unknown_values(monkeypatch, kw, exc):
    with pytest.raises(exc):
        _macnet(monkeypatch, **kw)


def test_dptrainer_enc_prec_bf16_needs_h_256(monkeypatch):
    with pytest.raises(NotImplementedError):
        _macnet(monkeypatch, d=128, enc_prec="bf16")
