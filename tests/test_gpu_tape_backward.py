"""Backward of the flag combinations outside the shipped flag files (SURVEY section 8(a) "P2": general read / write /
control units, wordsProj, controlWholeQ, controlContinuous, unsharedCells): `tape.py` on the CUDA backward kernels.

Two independent checks:
  * the tape machinery itself, forced onto the shipped flag files (tape_bwd=True), element-wise against torch.autograd
    on the fp64 restatement (`oracle/mac_torch_autograd.py`) -- the same bar as tests/test_gpu_backward.py;
  * every P2 fixture's flag set against central finite differences of the fp64 numpy oracle (`oracle/mac_oracle.py`, the
    restatement pinned to the reference's own outputs by tests/golden/): directional derivatives of
    sum(gc * control_L) + sum(gm * memory_L) along dense and sparse random directions of every parameter and input.
"""
import numpy as np
import pytest
import torch

from mac_network_b200.config import MACConfig
from mac_network_b200.params import init_params, perturb_biases
from mac_network_b200.synthetic import make_inputs
from tests._util import load_golden, max_rel, rebuild

pytestmark = pytest.mark.gpu

P2_CASES = ["p2_control", "p2_control_feed", "p2_ablations", "p2_wholeq", "p2_unshared", "p2_read_bl", "p2_read_add",
            "p2_read_plain", "p2_read_noproj", "p2_write_info", "p2_write_sum", "p2_write_mem", "p2_write_mul",
            "p2_read_add_train", "p2_read_plain_train", "p2_memory_bn", "p2_memory_bn_train"]


def _cell(cfg, pv32, inputs32, L, dp, seed=777, train=True, tape_bwd=False):
    from mac_network_b200.mac_cell import MACCell, MACParams, mac_network
    B = inputs32["knowledgeBase"].shape[0]
    params = MACParams(cfg, L, values=pv32)
    x = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in inputs32.items()}
    cell = MACCell(x["vecQuestions"], x["questionWords"], x["questionCntxWords"], x["questionLengths"],
                   x["knowledgeBase"], dp[0], dp[1], dp[2], B, train, config=cfg, params=params, seed=seed,
                   save_for_backward=True, tape_bwd=tape_bwd)
    control, memory = mac_network(cell, L)
    return cell, control, memory


@pytest.mark.parametrize("variant,shape,dp", [
    ("args", (6, 9, 50, 64, 3), (0.85, 0.85, 1.0)),
    ("gqa", (5, 7, 49, 128, 4), (0.9, 0.8, 0.9)),
    ("args4", (4, 6, 20, 64, 3), (1.0, 0.85, 1.0)),
    ("args1", (5, 7, 20, 64, 4), (0.85, 0.85, 1.0)),
])
def test_tape_bwd_on_the_shipped_flags_matches_autograd(variant, shape, dp):
    from mac_network_b200.autograd import mac_backward
    from oracle import mac_torch_autograd as TA
    B, S, N, d, L = shape
    over = dict(netLength=L, memDim=d, ctrlDim=d, attDim=d)
    if dp[2] < 1.0:
        over["writeDropout"] = dp[2]
    cfg = MACConfig.args(variant, **over)
    inputs = make_inputs(B, S, N, d, seed=51, dtype=np.float64)
    pv = perturb_biases(init_params(cfg, L, seed=52, dtype=np.float64), seed=53)
    rng = np.random.RandomState(54)
    gc, gm = rng.standard_normal((B, d)), rng.standard_normal((B, d))
    pv32 = {k: v.astype(np.float32) for k, v in pv.items()}
    in32 = {k: (v if v.dtype == np.int32 else v.astype(np.float32)) for k, v in inputs.items()}
    cell, control, memory = _cell(cfg, pv32, in32, L, dp, seed=4242, tape_bwd=True)
    assert cell._tape is not None
    grads = mac_backward(cell, torch.from_numpy(gc.astype(np.float32)).cuda(), torch.from_numpy(gm.astype(np.float32)).cuda())
    torch.cuda.synchronize()
    rc, rm, rg = TA.run(cfg, pv, inputs, L, dp, cell.dropout_uniforms(), gc, gm)
    assert max_rel(memory.cpu().numpy(), rm) < 1e-4 and max_rel(control.cpu().numpy(), rc) < 1e-4
    worst = {}
    for k, ref in rg.items():
        got = grads[k].cpu().numpy().reshape(ref.shape)
        scale = np.max(np.abs(ref))
        if scale < 1e-12:
            assert np.max(np.abs(got)) < 1e-4, k
            continue
        worst[k] = float(np.max(np.abs(got - ref)) / scale)
    bad = {k: v for k, v in worst.items() if v > 2e-4}
    assert not bad, (bad, {k: round(v, 7) for k, v in worst.items()})


def _oracle_loss(cfg, pv, inputs, L, dp, uniforms, gc, gm, train=False):
    from oracle.mac_oracle import MACOracle
    orc = MACOracle(cfg, pv, dtype=np.float64)
    orc.train = train                  # read by memoryBN only (batch vs stored statistics)
    st = orc.run(L, inputs["vecQuestions"], inputs["questionWords"], inputs["questionCntxWords"], inputs["questionLengths"],
                 inputs["knowledgeBase"], memoryDropout=dp[0], readDropout=dp[1], writeDropout=dp[2], uniforms=uniforms)
    return float(np.sum(st.control * gc) + np.sum(st.memory * gm))


@pytest.mark.parametrize("case", P2_CASES)
def test_tape_p2_gradients_match_finite_differences_of_the_oracle(case):
    from mac_network_b200.autograd import mac_backward
    meta, _ = load_golden(case)
    cfg, inputs, pv = rebuild(meta, dtype=np.float64)
    sh = meta["shape"]
    B, d, L = sh["B"], sh["d"], sh["L"]
    dpm = meta["dropouts"]
    dp = (dpm["memory"], dpm["read"], dpm["write"])
    # the function is evaluated where the fp32 product evaluates it
    pv = {k: v.astype(np.float32).astype(np.float64) for k, v in pv.items()}
    inputs = {k: (v if v.dtype == np.int32 else v.astype(np.float32).astype(np.float64)) for k, v in inputs.items()}
    pv32 = {k: v.astype(np.float32) for k, v in pv.items()}
    in32 = {k: (v if v.dtype == np.int32 else v.astype(np.float32)) for k, v in inputs.items()}
    rng = np.random.RandomState(2024)
    gc, gm = rng.standard_normal((B, d)), rng.standard_normal((B, d))
    cell, control, memory = _cell(cfg, pv32, in32, L, dp, train=bool(meta["train"]))
    assert cell._tape is not None, "this flag set is expected on the tape"
    grads = mac_backward(cell, torch.from_numpy(gc.astype(np.float32)).cuda(), torch.from_numpy(gm.astype(np.float32)).cuda())
    torch.cuda.synchronize()
    uniforms = cell.dropout_uniforms() if meta["train"] else None
    # forward agrees with the oracle (so the two sides differentiate the same function)
    from oracle.mac_oracle import MACOracle
    orc = MACOracle(cfg, pv, dtype=np.float64)
    orc.train = bool(meta["train"])
    st = orc.run(L, inputs["vecQuestions"], inputs["questionWords"], inputs["questionCntxWords"], inputs["questionLengths"],
                 inputs["knowledgeBase"], memoryDropout=dp[0], readDropout=dp[1], writeDropout=dp[2], uniforms=uniforms)
    assert max_rel(memory.cpu().numpy(), st.memory) < 1e-4 and max_rel(control.cpu().numpy(), st.control) < 1e-4

    def loss(p, x):
        return _oracle_loss(cfg, p, x, L, dp, uniforms, gc, gm, train=bool(meta["train"]))

    words_key = "questionCntxWords" if cfg.controlContextual else "questionWords"
    # (the stored batch-norm statistics are not trainable variables: TF gives them no gradient, neither does the tape)
    targets = ([("param", k) for k in pv if "/BatchNorm/moving_" not in k]
               + [("input", k) for k in ("knowledgeBase", words_key, "vecQuestions")])
    failures, checked, nonzero = {}, 0, 0
    for kind, k in targets:
        base = pv[k] if kind == "param" else inputs[k]
        g = grads[k].cpu().numpy().astype(np.float64).reshape(base.shape)
        gnorm = float(np.linalg.norm(g))
        for trial in range(4):
            v = rng.standard_normal(base.shape)
            if trial >= 2 and base.size > 8:            # sparse direction: close to an element-wise check
                keep = np.zeros(base.size, bool)
                keep[rng.choice(base.size, 8, replace=False)] = True
                v = v * keep.reshape(base.shape)
            h = 1e-6 * (1.0 + float(np.max(np.abs(base))))
            def at(t):
                if kind == "param":
                    p2 = dict(pv)
                    p2[k] = base + t * v
                    return loss(p2, inputs)
                x2 = dict(inputs)
                x2[k] = base + t * v
                return loss(pv, x2)
            fd = (at(h) - at(-h)) / (2 * h)
            ana = float(np.sum(g * v))
            # gradient error of the fp32 kernels ~1e-5 of the largest entry; the bound is relative to the Cauchy-Schwarz scale
            # of the direction restricted to its support
            support = v != 0
            scale = float(np.linalg.norm(g[support])) * float(np.linalg.norm(v)) if gnorm > 0 else 0.0
            # (+ an absolute floor: the softmax logit biases have an exactly zero gradient -- shift invariance -- of which the
            # fp32 kernels leave ~1e-7 of round-off)
            tol = 2e-3 * max(scale, 1e-3 * float(np.linalg.norm(v)) * max(gnorm, 1e-6)) + 2e-6 * float(np.linalg.norm(v))
            checked += 1
            nonzero += abs(fd) > 1e-9
            if abs(fd - ana) > tol:
                failures[(k, trial)] = (fd, ana, tol)
    assert not failures, failures
    # (writeInputs=MEM without a projection leaves the memory untouched: only the control path carries gradient there)
    assert nonzero >= checked // 4, "the directional derivatives should not all be trivial (%d of %d)" % (nonzero, checked)
