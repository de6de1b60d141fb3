"""Mixed-precision TRAINING forms of the cell (DESIGN.md section 9, item 1): the tensor-core kernels they use are checked
against fp64 references of their own operation in tests/test_gpu_wgmma.py (the split-K weight gradient, the transposing
bf16 casts, the bf16 read chain with its dropout masks and saved I1); these tests check their COMPOSITION (`mac_read_bwd_tc`, the bf16 training forward with widened saved
activations).  Tolerances are mixed-precision ones (bf16 operands, fp32
accumulation), stated per test."""
import numpy as np
import pytest
import torch

from mac_network_b200.config import MACConfig
from mac_network_b200.params import init_params, perturb_biases
from mac_network_b200.synthetic import make_inputs
from tests._util import max_rel

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("prec,tc,tol", [("fp32", True, 3e-2), ("bf16", False, 3e-2), ("bf16", True, 5e-2)])
@pytest.mark.parametrize("variant,shape,dp", [("args", (8, 12, 64, 128, 3), (0.85, 0.85, 1.0)),
                                              ("gqa", (4, 7, 48, 128, 2), (1.0, 1.0, 1.0))])
def test_tensor_core_training_gradients(variant, shape, dp, prec, tc, tol):
    """Gradients against torch.autograd on the fp64 restatement with the same dropout masks; max-rel per tensor."""
    from mac_network_b200.autograd import mac_backward
    from mac_network_b200.mac_cell import MACCell, MACParams, mac_network
    from oracle import mac_torch_autograd as TA
    B, S, N, d, L = shape
    cfg = MACConfig.args(variant, netLength=L, memDim=d, ctrlDim=d, attDim=d)
    inputs = make_inputs(B, S, N, d, seed=61, dtype=np.float64)
    pv = perturb_biases(init_params(cfg, L, seed=62, dtype=np.float64), seed=63)
    rng = np.random.RandomState(64)
    gc, gm = rng.standard_normal((B, d)), rng.standard_normal((B, d))
    params = MACParams(cfg, L, values={k: v.astype(np.float32) for k, v in pv.items()})
    x = {k: torch.from_numpy(np.ascontiguousarray(v if v.dtype == np.int32 else v.astype(np.float32))).cuda()
         for k, v in inputs.items()}
    cell = MACCell(x["vecQuestions"], x["questionWords"], x["questionCntxWords"], x["questionLengths"],
                   x["knowledgeBase"], dp[0], dp[1], dp[2], B, True, config=cfg, params=params, seed=77, prec=prec,
                   save_for_backward=True)
    control, memory = mac_network(cell, L)
    grads = mac_backward(cell, torch.from_numpy(gc.astype(np.float32)).cuda(), torch.from_numpy(gm.astype(np.float32)).cuda(),
                         tc=tc)
    torch.cuda.synchronize()
    rc, rm, rg = TA.run(cfg, pv, inputs, L, dp, cell.dropout_uniforms(), gc, gm)
    assert max_rel(memory.cpu().numpy(), rm) < (1e-4 if prec == "fp32" else 3e-2)
    worst = {}
    for k, ref in rg.items():
        scale = np.max(np.abs(ref))
        if scale < 1e-12:
            continue
        worst[k] = float(np.max(np.abs(grads[k].cpu().numpy().reshape(ref.shape) - ref)) / scale)
    print({k: round(v, 5) for k, v in sorted(worst.items(), key=lambda kv: -kv[1])[:6]})
    bad = {k: v for k, v in worst.items() if v > tol}
    assert not bad, bad


def test_tensor_core_training_reduces_the_loss():
    """DP trainer (world 1) with bf16 forward + tensor-core backward on the reference loss: the loss goes down."""
    from mac_network_b200.dp import DPTrainer
    B, S, N, d, L, A = 16, 10, 64, 128, 3, 8
    cfg = MACConfig.args("args", netLength=L, memDim=d, ctrlDim=d, attDim=d)
    tr = DPTrainer(cfg, L, seed=3, lr=3e-3, classifier=(A, [64]), prec="bf16", bwd_tc=True)
    batch = {k: torch.from_numpy(v).cuda() for k, v in make_inputs(B, S, N, d, seed=4).items()}
    answers = torch.from_numpy(np.random.RandomState(5).randint(0, A, size=(B,)).astype(np.int32)).cuda()
    hist = []
    for _ in range(12):
        _, losses = tr.train_step_answers(0, batch, answers, B)
        hist.append(float(losses.mean().item()))
    assert np.all(np.isfinite(hist)) and min(hist[-3:]) < hist[0], hist
