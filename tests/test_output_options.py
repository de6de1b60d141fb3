"""The output unit's layouts (--outQuestion, --outQuestionMul, --outputBN) on a box without a GPU: the fp64 oracles against
the reference's own outputOp / classifier on the TF1 shim (tests/golden/output_<layout>_<widths>_<mode>.npz), and the host
plumbing of the unit, the trainer and the checkpoints against the dry-run library (tests/_mocklib.py)."""
import json
import os

import numpy as np
import pytest
import torch

from tests import _mocklib

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LAYOUTS = {"q0": dict(question=False, mul=False), "q1": dict(question=True, mul=False), "qmul": dict(question=True, mul=True)}
WIDTHS = {"h0": (), "h8": (8,), "h8_6": (8, 6)}
CASES = [(l, bn, w, mode) for l in LAYOUTS for bn in (False, True) for w in WIDTHS for mode in ("eval", "train")]


def _load(layout, bn, widths, mode):
    z = np.load(os.path.join(GOLDEN, "output_%s%s_%s_%s.npz" % (layout, "_bn" if bn else "", widths, mode)))
    return z, json.loads(bytes(z["meta_json"]).decode())


def _fixture_params(meta, opts, bn):
    from mac_network_b200.output_unit import init_output_params, output_specs
    specs = output_specs(meta["d"], meta["d"], meta["hidden"], meta["A"], bn=bn, **opts)
    return specs, init_output_params(specs, seed=meta["param_seed"], dtype=np.float64)


@pytest.mark.parametrize("layout,bn,widths,mode", CASES)
def test_output_oracle_matches_reference(layout, bn, widths, mode):
    from oracle.output_options import output_forward
    z, meta = _load(layout, bn, widths, mode)
    opts = LAYOUTS[layout]
    specs, params = _fixture_params(meta, opts, bn)
    assert {k: list(v[0]) for k, v in specs.items()} == meta["variables"]          # names and shapes as the reference's
    us = [z["uniform_%03d" % i] for i in range(meta["n_uniform"])]
    assert (len(us) > 0) == (mode == "train")
    r = output_forward(meta["relu"], params, z["memory"], z["vecQuestions"], z["answers"], keep=meta["keep"], uniforms=us,
                       bn=bn, train=(mode == "train"), decay=meta.get("bnDecay", 0.999), **opts)
    for k in ("logits", "losses", "loss"):
        ref = np.asarray(z[k])
        assert np.max(np.abs(r[k] - ref)) <= 1e-12 * max(1.0, np.max(np.abs(ref))), k
    if bn:
        stats = [k for k in z.files if k.startswith("final/")]
        assert len(stats) == 2 * (len(WIDTHS[widths]) + 1)
        for k in stats:
            name = k[len("final/"):]
            assert np.max(np.abs(r["moving"][name] - z[k])) <= 1e-12, name
            assert np.array_equal(z["initial/" + name], params[name])
            assert np.array_equal(z[k], z["initial/" + name]) == (mode == "eval")       # moved by the training call only


@pytest.mark.parametrize("layout,bn,widths", [(l, bn, w) for l in LAYOUTS for bn in (False, True) for w in WIDTHS])
def test_output_autograd_graph_matches_oracle(layout, bn, widths):
    """oracle/output_options.output_graph (the gradient oracle of the GPU tests) against the reference's fixtures."""
    from oracle.output_options import output_graph
    opts = LAYOUTS[layout]
    for mode in ("eval", "train"):
        z, meta = _load(layout, bn, widths, mode)
        _, params = _fixture_params(meta, opts, bn)
        us = [z["uniform_%03d" % i] for i in range(meta["n_uniform"])]
        t = {k: torch.from_numpy(v) for k, v in params.items()}
        moving = {}
        logits, losses = output_graph(meta["relu"], t, torch.from_numpy(z["memory"]), torch.from_numpy(z["vecQuestions"]),
                                      torch.from_numpy(z["answers"]).long(), meta["keep"], us, bn=bn,
                                      train=(mode == "train"), decay=meta.get("bnDecay", 0.999), moving=moving, **opts)
        assert np.max(np.abs(logits.numpy() - z["logits"])) <= 1e-12 * max(1.0, np.max(np.abs(z["logits"])))
        if bn and mode == "train":
            for k, v in moving.items():
                assert np.max(np.abs(v.numpy() - z["final/" + k])) <= 1e-12, k


@pytest.mark.parametrize("mode", ["eval", "train"])
def test_default_options_are_the_shipped_oracles(mode):
    """With the default keywords the options' oracles are the shipped layout's (`oracle/output_oracle.py`,
    `model_torch_autograd.output_graph`) on that layout's own fixtures."""
    from oracle import model_torch_autograd as MA, output_options as OO
    from oracle.output_oracle import output_forward
    z = np.load(os.path.join(GOLDEN, "output_%s.npz" % mode))
    meta = json.loads(bytes(z["meta_json"]).decode())
    _, params = _fixture_params(meta, LAYOUTS["q1"], False)
    us = [z["uniform_%03d" % i] for i in range(meta["n_uniform"])]
    args = (meta["relu"], params, z["memory"], z["vecQuestions"], z["answers"])
    want, got = output_forward(*args, keep=meta["keep"], uniforms=us), OO.output_forward(*args, keep=meta["keep"], uniforms=us)
    assert all(np.array_equal(got[k], want[k]) for k in ("logits", "losses", "loss"))
    t = {k: torch.from_numpy(v) for k, v in params.items()}
    targs = ("ELU", t, torch.from_numpy(z["memory"]), torch.from_numpy(z["vecQuestions"]), torch.from_numpy(z["answers"]).long(),
             meta["keep"], us)
    assert all(torch.equal(a, b) for a, b in zip(MA.output_graph(*targs), OO.output_graph(*targs)))


def test_output_specs_per_option():
    from mac_network_b200.output_unit import is_moving_stat, output_specs
    shipped = output_specs(24, 16, [8], 12)
    assert output_specs(24, 16, [8], 12, question=True, mul=False, bn=False) == shipped
    assert shipped["classifier/linearLayerfc_0/weights/weight"][0] == (32, 8)
    q0 = output_specs(24, 16, [8], 12, question=False)
    assert not any(k.startswith("outputUnit/") for k in q0) and q0["classifier/linearLayerfc_0/weights/weight"][0] == (16, 8)
    assert output_specs(24, 16, [8], 12, question=False, mul=True) == q0          # the product needs the question
    qm = output_specs(24, 16, [8], 12, mul=True)
    assert qm["classifier/linearLayerfc_0/weights/weight"][0] == (48, 8)
    bn = output_specs(24, 16, [8, 4], 12, mul=True, bn=True)
    for i, width in enumerate((48, 8, 4)):
        for n in ("beta", "gamma", "moving_mean", "moving_variance"):
            assert bn["classifier/linearLayerfc_%d/BatchNorm/%s" % (i, n)][0] == (width,)
    assert [k for k in bn if is_moving_stat(k)] == [k for k in bn if "/moving_" in k] and len(bn) == 2 + 3 * 6
    assert not any(is_moving_stat(k) for k in ("MACnetwork/MACCell/write/BatchNorm/moving_mean",
                                                "classifier/linearLayerfc_0/BatchNorm/gamma"))


def _params(values):
    return {k: torch.from_numpy(np.ascontiguousarray(v, dtype=np.float32)) for k, v in values.items()}


# the launches of the shipped layout (question on, no product, no batch norm) at classifier widths (16,), as the unit made
# them before the options existed: forward to the loss, then the backward
SHIPPED_CALLS = {
    1.0: ["mac_linear_fwd", "mac_linear_fwd", "mac_linear_fwd", "mac_softmax_xent",
          "mac_linear_bwd", "mac_activation_bwd", "mac_linear_bwd", "mac_axpy", "mac_linear_bwd"],
    0.85: ["mac_linear_fwd", "mac_dropout_fwd", "mac_linear_fwd", "mac_dropout_fwd", "mac_linear_fwd", "mac_softmax_xent",
           "mac_linear_bwd", "mac_dropout_fwd", "mac_activation_bwd", "mac_linear_bwd", "mac_dropout_fwd", "mac_axpy",
           "mac_linear_bwd"],
}


@pytest.mark.parametrize("keep", [1.0, 0.85])
def test_shipped_layout_launches_unchanged(monkeypatch, keep):
    mock = _mocklib.install(monkeypatch)
    from mac_network_b200.output_unit import OutputUnit, init_output_params, output_specs
    p = _params(init_output_params(output_specs(16, 16, [16], 12), seed=1))
    out = OutputUnit(p, keep=keep, seed=3)
    B = 4
    mem, q = torch.zeros(B, 16), torch.zeros(B, 16)
    out.forward(mem, q, torch.zeros(B, dtype=torch.int32), step=1)
    out.backward({k: torch.zeros_like(v) for k, v in p.items()}, torch.zeros(B, 16), torch.zeros(B, 16))
    assert mock.calls == SHIPPED_CALLS[keep]
    mock.calls.clear()
    out.logits(mem, q)
    assert mock.calls == ["mac_linear_fwd"] * 3


@pytest.mark.parametrize("layout,bn", [(l, bn) for l in LAYOUTS for bn in (False, True)])
def test_layout_host_calls(monkeypatch, layout, bn):
    mock = _mocklib.install(monkeypatch)
    from mac_network_b200.output_unit import OutputUnit, init_output_params, output_specs
    opts = LAYOUTS[layout]
    p = _params(init_output_params(output_specs(16, 16, [16, 8], 12, bn=bn, **opts), seed=1))
    out = OutputUnit(p, keep=0.85, seed=3, bn=bn, **opts)
    B = 4
    logits, _, _ = out.forward(torch.zeros(B, 16), torch.zeros(B, 16), torch.zeros(B, dtype=torch.int32), step=1)
    assert logits.shape == (B, 12)
    d_mem, d_q = torch.zeros(B, 16), torch.zeros(B, 16)
    out.backward({k: torch.zeros_like(v) for k, v in p.items()}, d_mem, d_q)
    c = list(mock.calls)
    nseg = 1 + int(opts["question"]) + int(opts["mul"])                  # layer 0 normalises each feature segment
    assert c.count("mac_batchnorm_fwd") == (nseg + 2) * bn
    assert c.count("mac_batchnorm_bwd") == c.count("mac_batchnorm_fwd")
    assert c.count("mac_bcast_mul") == c.count("mac_bcast_op_bwd") == int(opts["mul"])
    assert c.count("mac_linear_fwd") == 3 + int(opts["question"])
    assert c.count("mac_linear_bwd") == 3 + int(opts["question"])
    assert c.count("mac_dropout_fwd") == 6
    mock.calls.clear()
    out.logits(torch.zeros(B, 16), torch.zeros(B, 16))
    assert "mac_dropout_fwd" not in mock.calls and mock.calls.count("mac_batchnorm_fwd") == c.count("mac_batchnorm_bwd")


def test_invalid_options_refused_before_any_launch(monkeypatch):
    mock = _mocklib.install(monkeypatch)
    from mac_network_b200 import dp
    from mac_network_b200.config import MACConfig
    from mac_network_b200.output_unit import OutputUnit, init_output_params, output_options, output_specs
    p = _params(init_output_params(output_specs(16, 16, [8], 12), seed=1))
    for kw in (dict(question=False), dict(bn=True), dict(mul=True)):
        with pytest.raises(ValueError):
            OutputUnit(p, **kw)
    pb = _params(init_output_params(output_specs(16, 16, [8], 12, bn=True), seed=1))
    with pytest.raises(ValueError):
        OutputUnit(pb)
    with pytest.raises(ValueError):
        OutputUnit(p, bn="yes")
    with pytest.raises(ValueError):
        output_options({"outQuestion": False})
    q0 = OutputUnit(_params(init_output_params(output_specs(16, 16, [8], 12, question=False), seed=1)), question=False)
    with pytest.raises(ValueError):
        q0.logits(torch.zeros(4, 8), None)                                  # memory too narrow for fc_0
    cfg = MACConfig.args("gqa", netLength=2, memDim=32, ctrlDim=32, attDim=32)
    for opts in ({"bogus": True}, {"bn": 1}):
        with pytest.raises(ValueError):
            dp.DPTrainer(cfg, 2, device="cpu", classifier=(8, [16], opts), encoder=(9, 12), stem=(8, 2))
    assert mock.calls == []


def test_trainer_layout_and_checkpoint(monkeypatch, tmp_path):
    """The stored statistics sit at the end of the flat buffer, outside the optimizer's and the EMA's range; the checkpoints
    hold them under the reference's names with no EMA shadow or Adam slot, and restore them."""
    _mocklib.install(monkeypatch)
    from mac_network_b200 import dp
    from mac_network_b200.checkpoint import (load_checkpoint, load_training_state, save_checkpoint, save_training_state,
                                             save_tf_checkpoint, load_tf_checkpoint)
    from mac_network_b200.config import MACConfig
    from mac_network_b200.output_unit import is_moving_stat
    cfg = MACConfig.args("gqa", netLength=2, memDim=32, ctrlDim=32, attDim=32)
    kw = dict(device="cpu", classifier=(8, [16], {"question": True, "mul": True, "bn": True}), encoder=(9, 12), stem=(8, 2))
    a = dp.DPTrainer(cfg, 2, seed=1, **kw)
    moving = [k for k in a.params.specs if is_moving_stat(k)]
    assert len(moving) == 4 and list(a.params.specs)[-4:] == moving
    assert a.n_train == min(a.params.offsets[k] for k in moving) < a.params.numel
    assert a.out.options == {"question": True, "mul": True, "bn": True}
    shipped = dp.DPTrainer(cfg, 2, seed=1, device="cpu", classifier=(8, [16]), encoder=(9, 12), stem=(8, 2))
    assert shipped.n_train == shipped.params.numel
    assert list(shipped.params.specs) == list(dp.DPTrainer(cfg, 2, seed=1, device="cpu", classifier=(8, [16], {}),
                                                           encoder=(9, 12), stem=(8, 2)).params.specs)
    g = torch.Generator().manual_seed(0)
    for t in (a.params.flat, a.adam_m, a.adam_v, a.ema):
        t.copy_(torch.rand(t.shape, generator=g) + 0.5)
    a.step_id = 5
    names = save_training_state(str(tmp_path / "state.npz"), a)
    for k in moving:
        assert "macModel/" + k in names
        assert not any(n.startswith("macModel/" + k + "/") for n in names), k
    assert "macModel/classifier/linearLayerfc_0/BatchNorm/gamma/ExponentialMovingAverage" in names
    b = dp.DPTrainer(cfg, 2, seed=2, **kw)
    assert load_training_state(str(tmp_path / "state.npz"), b) == 5
    for name in a.params.specs:
        assert torch.equal(a.params.t[name], b.params.t[name]), name
    n = a.n_train
    for x, y in ((a.adam_m, b.adam_m), (a.adam_v, b.adam_v), (a.ema, b.ema)):
        for name, (shape, _) in a.params.specs.items():
            o = a.params.offsets[name]
            if o < n:
                assert torch.equal(x[o:o + int(np.prod(shape))], y[o:o + int(np.prod(shape))]), name
    # the EMA-swapping readers fall back to the live statistics, which have no shadow
    vals = load_checkpoint(str(tmp_path / "state.npz"), use_ema=True)
    for k in moving:
        assert np.array_equal(vals[k], a.params.t[k].numpy())
    written = save_checkpoint(str(tmp_path / "w.npz"), a.params, a.ema)
    assert not any(w.endswith(k + "/ExponentialMovingAverage") for w in written for k in moving)
    values = {k: v.numpy() for k, v in a.params.t.items()}
    tf_names = save_tf_checkpoint(str(tmp_path / "ckpt"), values, ema_values=values)
    assert not any(w.endswith("moving_mean/ExponentialMovingAverage") for w in tf_names)
    back = load_tf_checkpoint(str(tmp_path / "ckpt"), use_ema=True)
    assert set(back) == set(values) and all(np.array_equal(back[k], values[k]) for k in moving)
