"""Output unit + classifier + answer loss (SURVEY section 8(f) rank 2): oracle vs fixtures from the reference's own
MACnet.outputOp / classifier / addAnswerLossOp (CPU), product vs oracle and vs torch.autograd (GPU)."""
import json
import os

import numpy as np
import pytest

from oracle.model_torch_autograd import output_graph
from oracle.output_oracle import output_forward
from mac_network_b200.output_unit import output_specs, init_output_params
from tests._util import GOLDEN_DIR, max_rel


def _load(case):
    z = np.load(os.path.join(GOLDEN_DIR, case + ".npz"))
    meta = json.loads(bytes(z["meta_json"]).decode())
    return meta, {k: z[k] for k in z.files if k != "meta_json"}


@pytest.mark.parametrize("case", ["output_eval", "output_train"])
def test_output_oracle_matches_reference_fixture(case):
    meta, g = _load(case)
    specs = output_specs(meta["d"], meta["d"], meta["hidden"], meta["A"])
    assert {k: list(v[0]) for k, v in specs.items()} == meta["variables"]
    params = init_output_params(specs, seed=meta["param_seed"], dtype=np.float64)
    us = [g["uniform_%03d" % i] for i in range(meta["n_uniform"])]
    out = output_forward(meta["relu"], params, g["memory"], g["vecQuestions"], g["answers"], keep=meta["keep"], uniforms=us)
    assert np.max(np.abs(out["logits"] - g["logits"])) < 1e-12
    assert np.max(np.abs(out["losses"] - g["losses"])) < 1e-12
    assert abs(out["loss"] - g["loss"]) < 1e-12


@pytest.mark.gpu
@pytest.mark.parametrize("keep", [1.0, 0.85])
def test_output_unit_gpu_forward_backward(keep):
    import torch
    from mac_network_b200 import _lib as L
    from mac_network_b200.output_unit import OutputUnit, SITE_OUTPUT
    lib = L.load()
    B, d, A, hidden = 64, 512, 28, [512]
    specs = output_specs(d, d, hidden, A)
    pv = init_output_params(specs, seed=3, dtype=np.float64)
    rng = np.random.RandomState(4)
    memory, vecq = rng.standard_normal((B, d)), 0.5 * np.tanh(rng.standard_normal((B, d)))
    answers = rng.randint(0, A, size=(B,)).astype(np.int32)
    params = {k: torch.from_numpy(v.astype(np.float32)).cuda() for k, v in pv.items()}
    grads = {k: torch.zeros_like(v) for k, v in params.items()}
    ou = OutputUnit(params, relu="ELU", keep=keep, seed=99)
    tm, tq = torch.from_numpy(memory.astype(np.float32)).cuda(), torch.from_numpy(vecq.astype(np.float32)).cuda()
    logits, losses, _ = ou.forward(tm, tq, torch.from_numpy(answers).cuda(), step=5)
    dmem, dq = torch.zeros(B, d, device="cuda"), torch.zeros(B, d, device="cuda")
    ou.backward(grads, dmem, dq)
    torch.cuda.synchronize()
    us = []
    if keep < 1.0:
        for layer, n in ((0, (B, 2 * d)), (1, (B, hidden[0]))):
            u = torch.empty(n, device="cuda")
            L.check(lib.mac_dropout_uniform(99, SITE_OUTPUT + layer, 5, L.ptr(u), u.numel(), L.stream_ptr()))
            us.append(u.cpu().numpy().astype(np.float64))
    ref = output_forward("ELU", pv, memory, vecq, answers, keep=keep, uniforms=us)
    assert max_rel(logits.cpu().numpy(), ref["logits"]) < 1e-4
    assert max_rel(losses.cpu().numpy(), ref["losses"]) < 1e-4
    # gradients vs torch.autograd on the fp64 restatement with the same masks
    t = lambda a: torch.tensor(a, dtype=torch.float64, requires_grad=True)
    P = {k: t(v) for k, v in pv.items()}
    M_, Q_ = t(memory), t(vecq)
    _, ls = output_graph("ELU", P, M_, Q_, torch.from_numpy(answers).long(), keep=keep, uniforms=us)
    ls.mean().backward()
    assert max_rel(dmem.cpu().numpy(), M_.grad.numpy()) < 2e-4
    assert max_rel(dq.cpu().numpy(), Q_.grad.numpy()) < 2e-4
    for k in pv:
        assert max_rel(grads[k].cpu().numpy(), P[k].grad.numpy()) < 2e-4, k


@pytest.mark.gpu
def test_softmax_xent_out_of_range_label_is_nan_not_a_wild_read():
    """A label outside [0, A) (a data bug) must not index outside the logits row: that sample's loss is NaN, its gradient the
    plain softmax, and the other samples are untouched."""
    import torch
    from mac_network_b200 import _lib as L
    lib = L.load()
    B, A = 6, 28
    rng = np.random.RandomState(8)
    logits = torch.from_numpy(rng.standard_normal((B, A)).astype(np.float32)).cuda()
    labels = torch.tensor([3, -1, 27, 28, 0, 1 << 20], dtype=torch.int32).cuda()
    losses, dl = torch.empty(B, device="cuda"), torch.empty(B, A, device="cuda")
    L.check(lib.mac_softmax_xent(L.ptr(logits), L.ptr(labels), L.ptr(losses), L.ptr(dl), 1.0, B, A, L.stream_ptr()))
    torch.cuda.synchronize()
    ls, sm = losses.cpu().numpy(), torch.softmax(logits, 1).cpu().numpy()
    assert np.isnan(ls[[1, 3, 5]]).all() and np.isfinite(ls[[0, 2, 4]]).all()
    assert np.allclose(dl.cpu().numpy()[[1, 3, 5]], sm[[1, 3, 5]], atol=1e-6)
    ref = -np.log(sm[[0, 2, 4], [3, 27, 0]])
    assert np.allclose(ls[[0, 2, 4]], ref, atol=1e-5)
