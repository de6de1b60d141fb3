"""Host-side plumbing of the GPU-only paths on a box without a GPU: the encoder / stem / output unit / full-model trainer
run against a dry-run library (tests/_mocklib.py) that validates every C-ABI call against the prototype table.  Numerics
are the business of the `-m gpu` tests; this catches marshalling mistakes (arity, pointer kinds, buffer shapes, call order)."""
import numpy as np
import pytest
import torch

from tests import _mocklib


def _params(specs_values):
    return {k: torch.from_numpy(np.ascontiguousarray(v, dtype=np.float32)) for k, v in specs_values.items()}


def test_encoder_host_calls(monkeypatch):
    mock = _mocklib.install(monkeypatch)
    from mac_network_b200.encoder import QuestionEncoder, encoder_specs, init_encoder_params
    for proj, keeps in ((False, (1.0, 1.0)), (True, (0.85, 0.92))):
        pv = init_encoder_params(encoder_specs(11, 12, 16, ctrl_dim=20 if proj else 16, proj=proj), seed=1)
        p = _params(pv)
        enc = QuestionEncoder(p, keep_input=keeps[0], keep_question=keeps[1], seed=3)
        q = torch.randint(0, 12, (5, 7), dtype=torch.int32)
        lens = torch.randint(1, 8, (5,), dtype=torch.int32)
        mock.calls.clear()
        # the mock cannot tell a CPU tensor from a CUDA one; bypass the device check only
        monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True), raising=False)
        words, cntx, vecq = enc.forward(q, lens, step=2, save_for_backward=True)
        assert words.shape == (5, 7, 12) and cntx.shape == (5, 7, 20 if proj else 16) and vecq.shape == (5, 20 if proj else 16)
        assert mock.calls.count("mac_lstm_fwd") == 1 and mock.calls.count("mac_embed_fwd") == 1
        assert mock.calls.count("mac_linear_fwd") == (4 if proj else 2)
        grads = {k: torch.zeros_like(v) for k, v in p.items()}
        enc.backward(torch.zeros_like(cntx), torch.zeros_like(vecq), grads)
        assert mock.calls.count("mac_lstm_bwd") == 1 and mock.calls.count("mac_embed_bwd") == 1
        assert mock.calls.count("mac_linear_bwd") == (4 if proj else 2)
        assert len(enc.dropout_uniforms(5, 7, step=2)) == (2 if keeps[0] < 1 else 0)


def test_stem_host_calls(monkeypatch):
    mock = _mocklib.install(monkeypatch)
    from mac_network_b200.stem import Stem, stem_specs, init_stem_params
    p = _params(init_stem_params(stem_specs(8, 16), seed=1))
    st = Stem(p, relu="ELU", prec="fp32", seed=1)
    kb = st.forward(torch.zeros(2, 5, 4, 8), keep=0.82, step=1, save_for_backward=True)
    assert kb.shape == (2, 20, 16)
    grads = {k: torch.zeros_like(v) for k, v in p.items()}
    assert st.backward(torch.zeros_like(kb), grads) is None
    assert mock.calls.count("mac_col2im3x3") == 1            # layer 1 only: the image gradient is not needed
    d_img = st.backward(torch.zeros_like(kb), grads, need_d_images=True)
    assert d_img.shape == (2, 5, 4, 8)
    assert mock.calls.count("mac_linear_bwd") == 4


def test_full_model_trainer_host_calls(monkeypatch):
    """DPTrainer.train_step_full up to (and after) the cell, with the already GPU-validated cell stubbed out."""
    mock = _mocklib.install(monkeypatch)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True), raising=False)
    from mac_network_b200 import autograd, dp, mac_cell
    from mac_network_b200.config import MACConfig
    B, S, V, E, d, H, W, C, A, L = 4, 6, 9, 12, 32, 3, 3, 8, 8, 2
    cfg = MACConfig.args("args", netLength=L, memDim=d, ctrlDim=d, attDim=d)
    tr = dp.DPTrainer(cfg, L, seed=1, device="cpu", classifier=(A, [16]), encoder=(V, E), stem=(C, 2))
    names = list(tr.params.specs)
    assert any(n.startswith("encoder/") for n in names) and any(n.startswith("stem/") for n in names)
    assert any(n.startswith("MACnetwork/") for n in names) and "qEmbeddings/emb" in names

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
    for name in ("mac_embed_fwd", "mac_lstm_fwd", "mac_im2col3x3", "mac_softmax_xent", "mac_lstm_bwd", "mac_embed_bwd",
                 "mac_col2im3x3", "mac_clip_adam_ema_step"):
        assert name in mock.calls, name
    assert tr.step_id == 1


@pytest.mark.parametrize("flags,prec,train", [("args", "fp32", False), ("args", "bf16", False), ("gqa", "fp32", False),
                                              ("gqa", "bf16", False), ("args1", "fp32", True), ("gqa", "fp32", True)])
def test_cell_host_calls(monkeypatch, flags, prec, train):
    """The cell's forward (hoisted eval form, per-step train form) and backward sweep against the prototype table."""
    mock = _mocklib.install(monkeypatch)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True), raising=False)
    from mac_network_b200.autograd import mac_backward
    from mac_network_b200.config import MACConfig
    from mac_network_b200.mac_cell import MACCell, MACParams, mac_network
    from mac_network_b200.synthetic import make_inputs
    B, S, N, d, L = 4, 6, 9, 64, 3
    cfg = MACConfig.args(flags, netLength=L, memDim=d, ctrlDim=d, attDim=d)
    params = MACParams(cfg, L, seed=1, device="cpu")
    x = {k: torch.from_numpy(v) for k, v in make_inputs(B, S, N, d, seed=2).items()}
    keeps = (0.85, 0.85, 1.0) if train else (1.0, 1.0, 1.0)
    cell = MACCell(x["vecQuestions"], x["questionWords"], x["questionCntxWords"], x["questionLengths"], x["knowledgeBase"],
                   keeps[0], keeps[1], keeps[2], B, train, config=cfg, params=params, prec=prec, save_for_backward=train)
    control, memory = mac_network(cell, L)
    assert control.shape == (B, d) and memory.shape == (B, d)
    assert len(cell.attentions["kb"]) == L and len(cell.attentions["question"]) == L
    if train:
        g = mac_backward(cell, torch.zeros(B, d), torch.zeros(B, d))
        assert g["knowledgeBase"].shape == (B, N, d) and g["vecQuestions"].shape == (B, d)
        assert mock.calls.count("mac_read_bwd") == L
    else:
        assert mock.calls.count("mac_read_invariant") == 1 and mock.calls.count("mac_read_fwd_inv") == L


def test_training_state_roundtrip(monkeypatch, tmp_path):
    """Checkpoint / resume of the whole-model trainer (weights, EMA shadows, Adam slots under TF's slot names, step)."""
    _mocklib.install(monkeypatch)
    from mac_network_b200 import dp
    from mac_network_b200.checkpoint import load_checkpoint, load_training_state, save_training_state
    from mac_network_b200.config import MACConfig
    cfg = MACConfig.args("gqa", netLength=2, memDim=32, ctrlDim=32, attDim=32)
    kw = dict(device="cpu", classifier=(8, [16]), encoder=(9, 12), stem=(8, 2))
    a = dp.DPTrainer(cfg, 2, seed=1, **kw)
    g = torch.Generator().manual_seed(0)
    for t in (a.adam_m, a.adam_v, a.ema):
        t.copy_(torch.randn(t.shape, generator=g))
    a.step_id = 17
    names = save_training_state(str(tmp_path / "state.npz"), a)
    wname = "macModel/MACnetwork/MACCell/read/linearLayermemKbProj/weights/weight"
    assert wname in names and wname + "/Adam" in names and wname + "/Adam_1" in names
    assert wname + "/ExponentialMovingAverage" in names and "beta1_power" in names
    assert "macModel/encoder/birnnLayer/bidirectional_rnn/fw/basic_lstm_cell/kernel/Adam" in names
    b = dp.DPTrainer(cfg, 2, seed=2, **kw)                      # different initial weights
    assert not torch.equal(a.params.flat, b.params.flat)
    assert load_training_state(str(tmp_path / "state.npz"), b) == 17
    for x, y in ((a.params.flat, b.params.flat), (a.adam_m, b.adam_m), (a.adam_v, b.adam_v), (a.ema, b.ema)):
        for name, (shape, _) in a.params.specs.items():          # the 64-element padding between variables is not state
            o, n = a.params.offsets[name], max(1, int(np.prod(shape)) if shape else 1)
            assert torch.equal(x[o:o + n], y[o:o + n]), name
    # the weights-only reader skips the optimizer slots and can swap in the EMA shadows (main.py:717-719)
    vals = load_checkpoint(str(tmp_path / "state.npz"), use_ema=True)
    assert set(vals) == set(a.params.specs)
    k = "MACnetwork/MACCell/read/linearLayermemKbProj/weights/weight"
    o = a.params.offsets[k]
    assert np.array_equal(vals[k].reshape(-1), a.ema[o:o + vals[k].size].numpy())
    # a path without the extension round-trips too (numpy appends ".npz" on save, not on load: ADVICE r1)
    save_training_state(str(tmp_path / "bare"), a)
    assert load_training_state(str(tmp_path / "bare"), b) == 17
    # weight-derived caches of the stem / output unit follow the parameter version, whoever changed the values (ADVICE r1)
    wt = b.out._wt_of("classifier/linearLayerfc_0/weights/weight")
    assert b.out._wt_of("classifier/linearLayerfc_0/weights/weight") is wt          # cached while nothing changes
    b.params.touch()
    assert b.out._wt_of("classifier/linearLayerfc_0/weights/weight") is not wt      # rebuilt after a restore / step


@pytest.mark.parametrize("prec,tc", [("fp32", True), ("bf16", False), ("bf16", True)])
def test_cell_tensor_core_training_host_calls(monkeypatch, prec, tc):
    """Mixed-precision training forms: bf16 forward with the saved activations widened for the backward, and the backward
    with its six big products on tensor cores (mac_read_bwd_tc)."""
    mock = _mocklib.install(monkeypatch)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True), raising=False)
    from mac_network_b200.autograd import mac_backward
    from mac_network_b200.config import MACConfig
    from mac_network_b200.mac_cell import MACCell, MACParams, mac_network
    from mac_network_b200.synthetic import make_inputs
    B, S, N, d, L = 4, 6, 16, 128, 2                     # B*N % 64 == 0, d % 128 == 0
    cfg = MACConfig.args("args", netLength=L, memDim=d, ctrlDim=d, attDim=d)
    params = MACParams(cfg, L, seed=1, device="cpu")
    x = {k: torch.from_numpy(v) for k, v in make_inputs(B, S, N, d, seed=2).items()}
    cell = MACCell(x["vecQuestions"], x["questionWords"], x["questionCntxWords"], x["questionLengths"], x["knowledgeBase"],
                   0.85, 0.85, 1.0, B, True, config=cfg, params=params, prec=prec, save_for_backward=True)
    mac_network(cell, L)
    g = mac_backward(cell, torch.zeros(B, d), torch.zeros(B, d), tc=tc)
    assert g["knowledgeBase"].shape == (B, N, d)
    assert mock.calls.count("mac_read_bwd_tc" if tc else "mac_read_bwd") == L
    assert mock.calls.count("mac_read_bwd" if tc else "mac_read_bwd_tc") == 0


def test_macnet_run_batch_host_calls(monkeypatch):
    """model.MACnet.runBatch (the reference's per-batch call, model.py:732-760): train and eval, trimming, predictions,
    attention maps -- through the dry-run library, nothing stubbed."""
    mock = _mocklib.install(monkeypatch)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True), raising=False)
    import importlib
    m = importlib.import_module("mac_network_b200.model")
    from mac_network_b200.config import MACConfig
    B, S, V, E, d, H, W, C, A, L = 4, 9, 11, 12, 64, 3, 3, 8, 8, 2
    cfg = MACConfig.args("gqa", netLength=L, memDim=d, ctrlDim=d, attDim=d)
    net = m.MACnet(cfg, L, V, A, wrd_emb_dim=E, image_in_dim=C, classifier_dims=(16,), prec="fp32", device="cpu",
                   answer_decoder=lambda i: "ans%d" % i)
    rng = np.random.RandomState(0)
    lengths = np.array([5, 7, 2, 6], dtype=np.int32)                     # longest question 7 < S: the batch is trimmed
    q = rng.randint(1, V + 1, size=(B, S)).astype(np.int32)
    q[np.arange(S)[None, :] >= lengths[:, None]] = 0
    data = {"questions": q, "questionLengths": lengths, "answers": rng.randint(0, A, size=(B,)).astype(np.int32),
            "instances": [{"questionId": i} for i in range(B)]}
    images = {"images": rng.standard_normal((B, C, H, W)).astype(np.float32)}
    res = net.runBatch(None, data, images, train=True)
    assert set(res) == {"loss", "correctNum", "acc", "preds", "gradNorm", "readTime", "trainTime"}
    assert "mac_lstm_bwd" in mock.calls and "mac_clip_adam_ema_step" in mock.calls and res["gradNorm"] != -1
    assert data["questions"].shape == (B, S)                              # the caller's batch is not modified
    mock.calls.clear()
    res = net.runBatch(None, data, images, train=False, getAtt=True)
    assert res["gradNorm"] == -1 and 0 <= res["correctNum"] <= B and len(res["preds"]) == B
    assert "mac_read_invariant" in mock.calls and "mac_lstm_bwd" not in mock.calls      # inference form, no backward
    rec = res["preds"][1]
    assert rec["questionId"] == 1 and rec["prediction"].startswith("ans")
    att = rec["attentions"]
    assert set(att) == {"kb", "question", "self", "gate"} and len(att["kb"]) == L
    assert np.asarray(att["kb"][0]).shape == (H, W) and len(att["question"][0]) == 7     # trimmed to the longest question


@pytest.mark.filterwarnings("ignore:invalid value")          # the dry-run library leaves the drawn uniforms uninitialised
@pytest.mark.parametrize("case", ["p2_read_add_train", "p2_read_plain_train"])
def test_general_path_training_dropout_host_calls(monkeypatch, case):
    """Composed (P2) read unit in training mode: the dropouts the reference applies there (ops.py:678-679 on both operands of
    the projected interaction; mac_cell.py:266 on the concatenated interactions) and their draw order / widths."""
    mock = _mocklib.install(monkeypatch)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True), raising=False)
    from mac_network_b200.mac_cell import MACCell, MACParams, mac_network
    from tests._util import load_golden, rebuild
    meta, arrays = load_golden(case)
    cfg, inputs, pv = rebuild(meta, dtype=np.float32)
    sh = meta["shape"]
    B, N, d, L = sh["B"], sh["N"], sh["d"], sh["L"]
    params = MACParams(cfg, L, values=pv, device="cpu")
    x = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in inputs.items()}
    dp = meta["dropouts"]
    cell = MACCell(x["vecQuestions"], x["questionWords"], x["questionCntxWords"], x["questionLengths"], x["knowledgeBase"],
                   dp["memory"], dp["read"], dp["write"], B, True, config=cfg, params=params)
    assert not cell._fused_read
    mac_network(cell, L)
    draws = cell.dropout_uniforms()
    # same number and shapes of uniform draws as the reference made on the shim for this flag set
    assert len(draws) == meta["n_uniform"]
    for i, u in enumerate(draws):
        assert tuple(u.shape) == tuple(arrays["uniform_%03d" % i].shape), i


def test_device_for_rank_spreads_over_numa_nodes(monkeypatch):
    """serving.device_for_rank: fewer ranks than GPUs -> round-robin over the sockets; all GPUs used / unknown topology /
    one socket -> the identity (so LOCAL_RANK keeps its usual meaning)."""
    from mac_network_b200 import serving
    assert serving.spread_order([0, 0, 0, 0, 1, 1, 1, 1]) == [0, 4, 1, 5, 2, 6, 3, 7]
    assert serving.spread_order([1, 1, 0]) == [0, 2, 1]
    assert serving._parse_cpulist("0-3,8,10-11\n") == {0, 1, 2, 3, 8, 10, 11}
    monkeypatch.setattr(serving.torch.cuda, "device_count", lambda: 8)
    monkeypatch.setattr(serving, "gpu_numa_nodes", lambda: [0, 0, 0, 0, 1, 1, 1, 1])
    assert [serving.device_for_rank(r, 2) for r in range(2)] == [0, 4]
    assert [serving.device_for_rank(r, 4) for r in range(4)] == [0, 4, 1, 5]
    assert [serving.device_for_rank(r, 8) for r in range(8)] == list(range(8))
    monkeypatch.setattr(serving, "gpu_numa_nodes", lambda: [0] * 8)
    assert [serving.device_for_rank(r, 2) for r in range(2)] == [0, 1]
    monkeypatch.setattr(serving, "gpu_numa_nodes", lambda: [-1] * 8)
    assert [serving.device_for_rank(r, 4) for r in range(4)] == [0, 1, 2, 3]


P2_CASES = ["p2_control", "p2_control_feed", "p2_ablations", "p2_wholeq", "p2_unshared", "p2_read_bl", "p2_read_add",
            "p2_read_plain", "p2_read_noproj", "p2_write_info", "p2_write_sum", "p2_write_mem", "p2_write_mul",
            "p2_read_add_train", "p2_read_plain_train", "p2_memory_bn", "p2_memory_bn_train"]


@pytest.mark.filterwarnings("ignore:invalid value")
@pytest.mark.parametrize("case", P2_CASES + ["args_train_small", "args1_train_small", "gqa_train_small"])
def test_tape_bwd_host_calls(monkeypatch, case):
    """Backward of the flag combinations outside the hand-scheduled sweep (tape.py): every forward launch leaves a node, the
    sweep calls the matching backward entry points with well-formed arguments, and every parameter the flag set creates that
    the forward read has a gradient slot.  (The shipped flag files go through the same tape with tape_bwd=True.)"""
    mock = _mocklib.install(monkeypatch)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True), raising=False)
    from mac_network_b200.autograd import mac_backward
    from mac_network_b200.mac_cell import MACCell, MACParams, mac_network
    from tests._util import load_golden, rebuild
    meta, _ = load_golden(case)
    cfg, inputs, pv = rebuild(meta, dtype=np.float32)
    sh = meta["shape"]
    B, N, d, L = sh["B"], sh["N"], sh["d"], sh["L"]
    params = MACParams(cfg, L, values=pv, device="cpu")
    x = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in inputs.items()}
    dp = meta["dropouts"]
    cell = MACCell(x["vecQuestions"], x["questionWords"], x["questionCntxWords"], x["questionLengths"], x["knowledgeBase"],
                   dp["memory"], dp["read"], dp["write"], B, True, config=cfg, params=params, save_for_backward=True,
                   tape_bwd=True)
    assert cell._use_tape
    mac_network(cell, L)
    n_nodes = len(cell._tape.nodes)
    assert n_nodes >= 3 * L
    fwd_calls = len(mock.calls)
    g = mac_backward(cell, torch.zeros(B, d), torch.zeros(B, d))
    assert g["knowledgeBase"].shape == (B, N, d) and g["vecQuestions"].shape == (B, d)
    assert len(mock.calls) - fwd_calls >= n_nodes           # at least one backward launch per node
    assert set(params.t) <= set(g)
    if not cell._fused_read:
        assert mock.calls.count("mac_rowdot_bwd") >= L and mock.calls.count("mac_kb_attend_bwd") >= L
    else:
        assert mock.calls.count("mac_read_bwd") == L
