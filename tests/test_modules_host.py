"""CPU side of the `torch.nn` modules (mac_network_b200/modules.py) over the dry-run library (tests/_mocklib.py): parameter
names and state dicts, the launches of a training step against DPTrainer.full_forward_backward's, the inference forms, the
refusals before any launch, the version refresh and the graph's one backward."""
import numpy as np
import pytest
import torch

from tests._util import load_golden
from tests.test_stem_tc_training import _recorder
from tests.test_train_pipeline_host import A, B, C, E, L, S, V

H = W = 4                 # B * H * W = 64: the bf16 tensor-core backward's rows

D = 128
# the loss's own launches, which DPTrainer (no scalar loss) has not: the reduction of the per-sample losses after
# mac_softmax_xent, and the incoming gradient's product with dlogits at the head of the backward
LOSS_LAUNCHES = ["mac_colsum", "mac_axpy", "mac_bcast_op"]


def _launches(rec):
    """The library calls that launch: everything but the workspace-size queries."""
    return [n for n, _ in rec.log if not n.endswith("_bytes")]


def _mock(monkeypatch):
    rec = _recorder(monkeypatch)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True), raising=False)
    from mac_network_b200 import modules
    monkeypatch.setattr(modules, "stream_ptr", lambda: None)
    return rec


def _cfg(variant="args", **kw):
    from mac_network_b200.config import MACConfig
    if variant.startswith("p2_"):
        meta, _ = load_golden(variant)
        return MACConfig(**dict(meta["cell_flags"], memDim=D, ctrlDim=D, attDim=D, netLength=L, **kw)).validate()
    return MACConfig.args(variant, netLength=L, memDim=D, ctrlDim=D, attDim=D, **kw)


def _trainer(cfg, **kw):
    from mac_network_b200.dp import DPTrainer
    return DPTrainer(cfg, L, seed=5, device="cpu", classifier=(A, [16]), encoder=(V, E), stem=(C, 2), **kw)


def _data(k=B, index=None, nchw=True):
    rng = np.random.RandomState(1)
    d = {"questions": torch.from_numpy(rng.randint(1, V + 1, size=(B, S)).astype(np.int32)),
         "questionLengths": torch.full((B,), S, dtype=torch.int32), "answers": torch.zeros(B, dtype=torch.int32)}
    d["images_nchw" if nchw else "images"] = torch.zeros((k, C, H, W) if nchw else (k, H, W, C))
    if index is not None:
        d["imageIndex"] = torch.tensor(index, dtype=torch.int32)
    return d


def _model_step(model, d):
    from mac_network_b200.modules import answer_loss
    imgs = {k: d[k] for k in ("images", "images_nchw") if k in d}
    logits, _ = model(d["questions"], d["questionLengths"], imageIndex=d.get("imageIndex"), **imgs)
    loss = answer_loss(logits, d["answers"])
    loss.backward()
    return loss


# ------------------------------------------------------------------------------------------------ parameters
def test_parameter_names_are_the_spec_names_and_a_tf_checkpoint_loads(monkeypatch, tmp_path):
    _mock(monkeypatch)
    from mac_network_b200.checkpoint import load_tf_checkpoint, save_tf_checkpoint
    from mac_network_b200.modules import MACModel, MACNetwork
    from mac_network_b200.params import param_specs
    t = _trainer(_cfg())
    m = MACModel.from_trainer(t)
    names = [n for n, _ in m.named_parameters()]
    assert names == list(t.params.specs) and list(m.state_dict()) == names
    for n, p in m.named_parameters():            # views of the one flat buffer, in MACParams' layout
        assert p.data_ptr() == m.params.flat[m.params.offsets[n]:].data_ptr() and p.shape == tuple(t.params.specs[n][0])
        assert torch.equal(p.detach().reshape(-1), t.params.t[n].reshape(-1))
    net = MACNetwork(_cfg(), L, device="cpu")
    assert [n for n, _ in net.named_parameters()] == list(param_specs(_cfg(), L))
    # the reference's checkpoint format: load_tf_checkpoint's output loads strictly
    other = MACModel.from_trainer(_trainer(_cfg()))
    with torch.no_grad():
        for p in other.parameters():
            p.uniform_(-1, 1)
    save_tf_checkpoint(str(tmp_path / "model"), {n: p.detach().numpy() for n, p in other.named_parameters()})
    vals = load_tf_checkpoint(str(tmp_path / "model"))
    v0 = m.params.flat._version
    m.load_state_dict({k: torch.from_numpy(v) for k, v in vals.items()}, strict=True)
    assert m.params.flat._version != v0
    assert all(torch.equal(a, b) for a, b in zip(m.state_dict().values(), other.state_dict().values()))


# ------------------------------------------------------------------------------------------------ the training step
@pytest.mark.parametrize("variant,kw,index,nchw", [
    ("args", dict(), None, True),
    ("args", dict(prec="bf16", bwd_tc=True, stem_prec="bf16"), None, True),
    ("args", dict(prec="tc32", bwd_tc=True, stem_prec="bf16x3"), None, False),
    ("args", dict(prec="bf16", bwd_tc=True, stem_prec="bf16"), [2, 0, 2, 1], True),
    ("args1", dict(prec="tc32", bwd_tc=True), None, True),
    ("args3", dict(), [0, 0, 1, 0], False),
    ("p2_read_add", dict(), None, True),
])
def test_training_step_launches_what_the_trainer_launches(monkeypatch, variant, kw, index, nchw):
    """forward + answer_loss + backward: the entry points of DPTrainer.full_forward_backward in the same order, with the
    loss's own three launches after mac_softmax_xent."""
    rec = _mock(monkeypatch)
    from mac_network_b200.modules import MACModel
    t = _trainer(_cfg(variant), **kw)
    m = MACModel.from_trainer(t)
    k = B if index is None else max(index) + 1
    d = _data(k, index, nchw)
    rec.log.clear()
    t.full_forward_backward((B, S), d, global_batch=B)
    want = _launches(rec)
    at = want.index("mac_softmax_xent") + 1
    want = want[:at] + LOSS_LAUNCHES + want[at:]
    rec.log.clear()
    _model_step(m, d)
    assert _launches(rec) == want
    assert m.step == t.step_id + 1
    if "mac_read_bwd_tc" in want or "mac_read_bwd_tc32" in want:
        assert kw.get("bwd_tc")
    assert all(p.grad is not None for p in m.parameters())
    # the gradients are views of ONE flat buffer of this forward, not of a persistent one
    base = {p.grad.untyped_storage().data_ptr() for p in m.parameters()}
    assert len(base) == 1 and base != {m.params.flat.untyped_storage().data_ptr()}


def test_each_forward_owns_its_saved_state(monkeypatch):
    """Two forwards, then one backward through both: each unit's backward runs twice, on its own forward's state; a
    second backward through a freed graph and create_graph=True raise."""
    rec = _mock(monkeypatch)
    from mac_network_b200.modules import MACModel, answer_loss
    m = MACModel.from_trainer(_trainer(_cfg()))
    d = _data()
    la = answer_loss(m(d["questions"], d["questionLengths"], images_nchw=d["images_nchw"])[0], d["answers"])
    cell_a = m.cells._idle.get((True, B, S, E, H * W, None))
    assert cell_a is None                                     # held by graph a until its backward
    lb = answer_loss(m(d["questions"], d["questionLengths"], images_nchw=d["images_nchw"])[0], d["answers"])
    rec.log.clear()
    (la + lb).backward()
    names = _launches(rec)
    assert names.count("mac_lstm_bwd") == 2 and names.count("mac_softmax_xent") == 0
    with pytest.raises(RuntimeError, match="already run"):
        la.backward()
    lc = answer_loss(m(d["questions"], d["questionLengths"], images_nchw=d["images_nchw"])[0], d["answers"])
    with pytest.raises(RuntimeError, match="double backward"):
        torch.autograd.grad(lc, [next(m.parameters())], create_graph=True)
    ld = answer_loss(m(d["questions"], d["questionLengths"], images_nchw=d["images_nchw"])[0], d["answers"])
    with torch.no_grad():
        next(m.parameters()).add_(1.0)
    with pytest.raises(RuntimeError, match="modified in place"):
        ld.backward()


# ------------------------------------------------------------------------------------------------ inference
@pytest.mark.parametrize("how", ["eval", "no_grad", "nothing_requires_grad"])
def test_a_forward_without_gradients_runs_the_inference_form(monkeypatch, how):
    rec = _mock(monkeypatch)
    from mac_network_b200.modules import MACModel
    m = MACModel.from_trainer(_trainer(_cfg(), prec="bf16", stem_prec="bf16"))
    d = _data()
    if how == "eval":
        m.eval()
    elif how == "nothing_requires_grad":
        m.requires_grad_(False)
    rec.log.clear()
    with torch.no_grad() if how == "no_grad" else torch.enable_grad():
        logits, memory = m(d["questions"], d["questionLengths"], images_nchw=d["images_nchw"])
    names = _launches(rec)
    assert "mac_read_fwd_inv" in names and "mac_read_invariant" in names and "mac_read_fwd" not in names
    assert "mac_softmax_xent" not in names and not logits.requires_grad and m.step == 0
    assert len(m.attentions["kb"]) == L


def test_eval_fp8_with_shared_images(monkeypatch):
    rec = _mock(monkeypatch)
    from mac_network_b200.modules import MACNetwork
    from mac_network_b200.config import MACConfig
    cfg = MACConfig.args("args", netLength=L)                 # the e4m3 read step's d = 512
    net = MACNetwork(cfg, L, prec="bf16", eval_prec="fp8", device="cpu").eval()
    x = _cell_inputs(cfg, N=196)
    rec.log.clear()
    net(*x, kbIndex=torch.tensor([0, 1, 1, 0], dtype=torch.int32))
    names = _launches(rec)
    assert "mac_kb_gather" in names and "mac_read_fwd" not in names
    assert any(n.startswith("mac_pack_weight_fp8") for n in names)


def _cell_inputs(cfg, N=H * W, U=2):
    d = cfg.memDim
    return (torch.zeros(B, d), torch.zeros(B, S, E), torch.zeros(B, S, d), torch.full((B,), S, dtype=torch.int32),
            torch.zeros(U, N, d))


# ------------------------------------------------------------------------------------------------ refusals
def _refusals():
    from mac_network_b200.modules import MACModel, MACNetwork
    yield "fp8 training", lambda: MACNetwork(_cfg(), L, prec="fp8", device="cpu"), "inference form"
    yield "fp8 training (model)", lambda: MACModel(_cfg(), L, V, A, wrd_emb_dim=E, image_in_dim=C, classifier_dims=(16,),
                                                   prec="fp8", device="cpu"), "inference form"
    yield "tc32 on the tape", lambda: MACNetwork(_cfg("p2_read_add"), L, prec="tc32", device="cpu"), "fp32 kernels"
    yield "bwd_tc: (B*N) % 64", lambda: MACNetwork(_cfg(), L, prec="bf16", bwd_tc=True, device="cpu"), r"\(B\*N\) % 64"
    yield "bwd_tc on the tape", lambda: MACNetwork(_cfg("p2_read_add"), L, prec="fp32", bwd_tc=True, device="cpu"), \
        "fp32 kernels"


@pytest.mark.parametrize("case", ["fp8 training", "fp8 training (model)", "tc32 on the tape", "bwd_tc: (B*N) % 64",
                                  "bwd_tc on the tape"])
def test_refusals_come_before_any_launch(monkeypatch, case):
    rec = _mock(monkeypatch)
    build, match = {c: (b, m) for c, b, m in _refusals()}[case]
    mod = build()
    rec.log.clear()
    with pytest.raises(NotImplementedError, match=match):
        if hasattr(mod, "cells") and not hasattr(mod, "_enc"):
            x = _cell_inputs(mod.cfg, N=9, U=B)         # B * N = 36
            mod(*x)
        else:
            d = _data()
            mod(d["questions"], d["questionLengths"], images_nchw=d["images_nchw"])
    assert _launches(rec) == [] and mod.step == 0


def test_whole_model_refuses_raw_word_control_inputs(monkeypatch):
    rec = _mock(monkeypatch)
    from mac_network_b200.modules import MACModel
    cfg = _cfg()
    cfg.controlContextual = False
    with pytest.raises(NotImplementedError, match="controlContextual"):
        MACModel(cfg, L, V, A, wrd_emb_dim=E, image_in_dim=C, classifier_dims=(16,), device="cpu")
    assert _launches(rec) == []


# ------------------------------------------------------------------------------------------------ versions
def test_an_optimizer_step_drops_the_packs(monkeypatch):
    """The next forward after torch.optim's in-place update rebuilds every weight pack; one without an update does not."""
    rec = _mock(monkeypatch)
    from mac_network_b200.modules import MACModel
    m = MACModel.from_trainer(_trainer(_cfg(), prec="bf16", stem_prec="bf16"))
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    d = _data()
    packs = lambda: [n for n in _launches(rec) if n.startswith("mac_pack_weight")]
    _model_step(m, d)
    v = m.params.version
    rec.log.clear()
    _model_step(m, d)
    assert packs() == [] and m.params.version == v            # nothing moved: every pack is reused
    opt.step()
    rec.log.clear()
    _model_step(m, d)
    assert len(packs()) > 0 and m.params.version == v + 1
