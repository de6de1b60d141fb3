"""GPU parity: the sm_90a kernels (through the C ABI / MACCell host mirror) against the fp64 oracle and
against the golden fixtures produced by the unmodified reference.  Tolerance (BASELINE.json north_star):
fp32 projections within 1e-4 relative (max |x - ref| / max |ref| per tensor), probabilities with a 1e-6
absolute floor."""
import numpy as np
import pytest
import torch

from oracle.mac_oracle import MACOracle
from mac_network_b200.config import MACConfig
from mac_network_b200.params import init_params, perturb_biases
from mac_network_b200.synthetic import make_inputs
from tests._util import golden_cases, load_golden, rebuild, max_rel

pytestmark = pytest.mark.gpu

TOL = 1e-4
FAST_FIXTURES = golden_cases()       # every fixture: the shipped flag files AND the P2 flag combinations


def _to_dev(inputs):
    out = {}
    for k, v in inputs.items():
        out[k] = torch.from_numpy(np.ascontiguousarray(v)).cuda()
    return out


def run_gpu(cfg, params_np, inputs_np, L, dropouts=(1.0, 1.0, 1.0), train=False, prec="fp32", seed=0, small_tc=None,
            save_for_backward=False):
    from mac_network_b200.mac_cell import MACCell, MACParams
    p32 = {k: np.asarray(v, np.float32) for k, v in params_np.items()}
    params = MACParams(cfg, L, values=p32)
    x = _to_dev({k: (np.asarray(v, np.float32) if v.dtype != np.int32 else v) for k, v in inputs_np.items()})
    cell = MACCell(x["vecQuestions"], x["questionWords"], x["questionCntxWords"], x["questionLengths"],
                   x["knowledgeBase"], dropouts[0], dropouts[1], dropouts[2], x["knowledgeBase"].shape[0], train,
                   config=cfg, params=params, prec=prec, seed=seed, small_tc=small_tc,
                   save_for_backward=save_for_backward)
    state = cell.zero_state(cell.batchSize)
    trace = []
    for i in range(L):
        cell.iteration = i
        _, state = cell(cell.none, state)
        trace.append((state.control, state.memory, cell.contControl))
    torch.cuda.synchronize()
    out = {
        "control": np.stack([t[0].cpu().numpy() for t in trace]),
        "memory": np.stack([t[1].cpu().numpy() for t in trace]),
        "contControl": np.stack([t[2].cpu().numpy() for t in trace]),
        "info": cell.infos.permute(1, 0, 2)[1:].cpu().numpy(),
        "att_question": np.stack([a.cpu().numpy() for a in cell.attentions["question"]]),
        "att_kb": np.stack([a.cpu().numpy() for a in cell.attentions["kb"]]),
    }
    if cell.attentions["gate"]:
        out["att_gate"] = np.stack([a.cpu().numpy() for a in cell.attentions["gate"]])
    for i, a in enumerate(cell.attentions["self"]):
        out["att_self_%d" % i] = a.cpu().numpy()
    return out, cell


def run_oracle(cfg, params_np, inputs_np, L, dropouts=(1.0, 1.0, 1.0), uniforms=None, train=False, keep=None):
    orc = MACOracle(cfg, params_np, dtype=np.float64)
    orc.train = train                   # read by memoryBN only
    if keep is not None:
        keep.append(orc)
    orc.run(L, inputs_np["vecQuestions"], inputs_np["questionWords"], inputs_np["questionCntxWords"],
            inputs_np["questionLengths"], inputs_np["knowledgeBase"], memoryDropout=dropouts[0],
            readDropout=dropouts[1], writeDropout=dropouts[2], uniforms=uniforms)
    return orc.outputs()


def compare(got, ref, tol=TOL, what=""):
    assert set(got) == set(ref), (sorted(got), sorted(ref))
    worst = {}
    for k in ref:
        err = max_rel(got[k], ref[k])
        worst[k] = err
        if k.startswith("att_") and k != "att_gate":
            assert np.max(np.abs(got[k] - ref[k])) < max(tol * np.max(np.abs(ref[k])), 1e-6), (what, k, err)
        else:
            assert err < tol, (what, k, err)
    return worst


def test_library_is_native_and_device_ok():
    from mac_network_b200 import _lib
    lib = _lib.load()
    assert lib.mac_b200_device_ok() == 1


@pytest.mark.parametrize("case", [c for c in FAST_FIXTURES if "train" not in c])
def test_eval_matches_reference_fixture(case):
    """Kernels vs the outputs of the unmodified reference cell (fixture) -- eval mode."""
    meta, gold = load_golden(case)
    cfg, inputs, params = rebuild(meta, np.float64)
    L = meta["shape"]["L"]
    got, _ = run_gpu(cfg, params, inputs, L)
    ref = {k: v.astype(np.float64) for k, v in gold.items() if not k.startswith(("uniform_", "final_"))}
    compare(got, ref, what=case)


@pytest.mark.parametrize("variant,shape", [
    ("args", (32, 20, 196, 512, 4)),      # BASELINE configs[1]
    ("args3", (16, 20, 196, 512, 4)),
    ("args4", (16, 20, 196, 512, 4)),
    ("args1", (16, 20, 196, 512, 4)),
    ("gqa", (64, 30, 49, 512, 6)),        # BASELINE configs[4]
    ("args", (5, 9, 50, 64, 3)),          # ragged: B*N not a tile multiple, d = 64
    ("gqa", (3, 1, 1, 128, 2)),           # degenerate: one word, one KB cell
])
def test_eval_matches_oracle(variant, shape):
    B, S, N, d, L = shape
    cfg = MACConfig.args(variant, netLength=L, memDim=d, ctrlDim=d, attDim=d)
    inputs = make_inputs(B, S, N, d, seed=11, dtype=np.float64)
    params = perturb_biases(init_params(cfg, L, seed=12, dtype=np.float64), seed=13)
    got, _ = run_gpu(cfg, params, inputs, L)
    ref = run_oracle(cfg, params, inputs, L)
    compare(got, ref, what="%s%s" % (variant, shape))
    # properties the domain offers, at full size
    qa = got["att_question"]
    assert np.allclose(qa.sum(-1), 1.0, atol=1e-5)
    for b, n in enumerate(inputs["questionLengths"]):
        assert np.all(qa[:, b, n:] == 0.0)
    assert np.allclose(got["att_kb"].sum(-1), 1.0, atol=1e-5)


@pytest.mark.parametrize("variant,shape,dp", [
    ("args", (8, 12, 196, 512, 3), (0.85, 0.85, 1.0)),
    ("gqa", (8, 10, 49, 128, 4), (0.85, 0.85, 0.9)),
    ("args1", (4, 6, 20, 64, 3), (0.7, 0.6, 1.0)),
])
def test_train_mode_matches_oracle_with_same_masks(variant, shape, dp):
    """Training-mode forward: the kernels draw Philox masks in-kernel; the oracle is fed the same uniforms
    (materialised by mac_dropout_uniform) in the reference's call order."""
    B, S, N, d, L = shape
    over = dict(netLength=L, memDim=d, ctrlDim=d, attDim=d)
    if dp[2] < 1.0:
        over["writeDropout"] = dp[2]
    cfg = MACConfig.args(variant, **over)
    inputs = make_inputs(B, S, N, d, seed=21, dtype=np.float64)
    params = perturb_biases(init_params(cfg, L, seed=22, dtype=np.float64), seed=23)
    got, cell = run_gpu(cfg, params, inputs, L, dropouts=dp, train=True, seed=1234567)
    ref = run_oracle(cfg, params, inputs, L, dropouts=dp, uniforms=cell.dropout_uniforms())
    compare(got, ref, what="train-%s" % variant)


def test_novardp_fixture_train_semantics():
    """Non-variational memory dropout draws a fresh [B,d] mask every step (mac_cell.py:217)."""
    B, S, N, d, L = 4, 6, 20, 64, 3
    flags = ["--relu=ELU", "--controlContextual", "--readProjInputs", "--readMemConcatKB", "--readMemConcatProj",
             "--readMemProj", "--readCtrl", "--writeMemProj", "--initCtrl=Q", "--controlInputUnshared"]
    cfg = MACConfig.from_flags(flags, netLength=L, memDim=d, ctrlDim=d, attDim=d)
    inputs = make_inputs(B, S, N, d, seed=31, dtype=np.float64)
    params = perturb_biases(init_params(cfg, L, seed=32, dtype=np.float64), seed=33)
    dp = (0.8, 0.9, 1.0)
    got, cell = run_gpu(cfg, params, inputs, L, dropouts=dp, train=True, seed=99)
    ref = run_oracle(cfg, params, inputs, L, dropouts=dp, uniforms=cell.dropout_uniforms())
    compare(got, ref, what="novardp")


def test_inputs_are_not_modified():
    B, S, N, d, L = 4, 6, 20, 64, 2
    cfg = MACConfig.args("gqa", netLength=L, memDim=d, ctrlDim=d, attDim=d)
    inputs = make_inputs(B, S, N, d, seed=5, dtype=np.float64)
    params = init_params(cfg, L, seed=6, dtype=np.float64)
    _, cell = run_gpu(cfg, params, inputs, L)
    assert np.array_equal(cell.knowledgeBase.cpu().numpy(), inputs["knowledgeBase"].astype(np.float32))
    assert np.array_equal(cell.questionCntxWords.cpu().numpy(), inputs["questionCntxWords"].astype(np.float32))
    assert np.array_equal(cell.vecQuestions.cpu().numpy(), inputs["vecQuestions"].astype(np.float32))


@pytest.mark.parametrize("variant,shape", [("args", (8, 12, 196, 512, 4)), ("gqa", (64, 30, 49, 512, 6))])
def test_bf16_tensor_core_path(variant, shape):
    """Headline precision (bf16 operands on wgmma, fp32 accumulate, bf16 knowledge base): error against the fp64
    oracle is REPORTED and bounded loosely -- the 1e-4 bar applies to the fp32 path only (DESIGN.md section 5)."""
    B, S, N, d, L = shape
    cfg = MACConfig.args(variant, netLength=L, memDim=d, ctrlDim=d, attDim=d)
    inputs = make_inputs(B, S, N, d, seed=41, dtype=np.float64)
    params = perturb_biases(init_params(cfg, L, seed=42, dtype=np.float64), seed=43)
    got, _ = run_gpu(cfg, params, inputs, L, prec="bf16")
    ref = run_oracle(cfg, params, inputs, L)
    errs = {k: max_rel(got[k], ref[k]) for k in ("control", "memory", "info", "att_kb")}
    print("bf16 path max-rel errors:", errs)
    assert errs["control"] < 1e-4            # the control chain stays fp32
    assert errs["memory"] < 3e-2 and errs["info"] < 3e-2


def test_bf16_train_mode_forward():
    """Tensor-core path with training dropouts: same Philox masks as the fp32 path, so the oracle fed the kernels'
    uniforms bounds the error the same way as in eval."""
    B, S, N, d, L = 8, 10, 196, 512, 3
    cfg = MACConfig.args("args", netLength=L, memDim=d, ctrlDim=d, attDim=d)
    inputs = make_inputs(B, S, N, d, seed=81, dtype=np.float64)
    params = perturb_biases(init_params(cfg, L, seed=82, dtype=np.float64), seed=83)
    dp = (0.85, 0.85, 1.0)
    got, cell = run_gpu(cfg, params, inputs, L, dropouts=dp, train=True, prec="bf16", seed=777)
    ref = run_oracle(cfg, params, inputs, L, dropouts=dp, uniforms=cell.dropout_uniforms())
    errs = {k: max_rel(got[k], ref[k]) for k in ("control", "memory", "info")}
    print("bf16 train-mode max-rel errors:", errs)
    assert errs["control"] < 1e-4 and errs["memory"] < 3e-2 and errs["info"] < 3e-2


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_full_size_properties(prec):
    """BASELINE.json's full headline shape (B=64, S=40, N=196, d=512, netLength=12) through size-independent properties:
    run-to-run determinism (bit-identical), attention rows are distributions with exact zeros behind the question
    length, batch independence (a sample's trajectory does not depend on its batch mates), and state boundedness."""
    from mac_network_b200.synthetic import SHAPES
    B, S, N, d, L = SHAPES["headline"]
    cfg = MACConfig.args("args", netLength=L)
    inputs = make_inputs(B, S, N, d, seed=1234)
    params = perturb_biases(init_params(cfg, L, seed=100), seed=101)
    a, _ = run_gpu(cfg, params, inputs, L, prec=prec)
    b, _ = run_gpu(cfg, params, inputs, L, prec=prec)
    for k in a:
        assert np.array_equal(a[k], b[k]), k                                  # deterministic: no atomics anywhere
    assert np.allclose(a["att_question"].sum(-1), 1.0, atol=1e-5)
    assert np.allclose(a["att_kb"].sum(-1), 1.0, atol=1e-5)
    for bi, n in enumerate(inputs["questionLengths"]):
        assert np.all(a["att_question"][:, bi, n:] == 0.0)
    assert np.isfinite(a["memory"]).all() and np.isfinite(a["control"]).all()
    # batch independence: samples 0..7 alone give the same trajectories as inside the batch of 64
    sub = {k: np.ascontiguousarray(v[:8]) for k, v in inputs.items()}
    c, _ = run_gpu(cfg, params, sub, L, prec=prec)
    tol = 1e-5 if prec == "fp32" else 2e-3       # different tile -> row mapping changes only the bf16 rounding pattern
    assert max_rel(c["memory"], a["memory"][:, :8]) < tol
    assert max_rel(c["att_kb"], a["att_kb"][:, :8]) < max(tol, 1e-5)


def test_checkpoint_roundtrip_and_attention_export(tmp_path):
    """Weights travel under the reference's TF variable names; attention maps come out as attMap[key][step][sample]."""
    from mac_network_b200.checkpoint import save_checkpoint, load_checkpoint, write_preds, MODEL_SCOPE, EMA_SUFFIX
    from mac_network_b200.mac_cell import MACParams
    B, S, N, d, L = 4, 6, 196, 64, 2
    cfg = MACConfig.args("gqa", netLength=L, memDim=d, ctrlDim=d, attDim=d)
    pv = perturb_biases(init_params(cfg, L, seed=7), seed=8)
    params = MACParams(cfg, L, values=pv)
    ema = params.flat * 0.5
    names = save_checkpoint(str(tmp_path / "w.npz"), params, ema_flat=ema)
    assert (MODEL_SCOPE + "MACnetwork/MACCell/read/linearLayermemKbProj/linearLayermemKbProj_2/weights/weight") in names
    assert any(n.endswith(EMA_SUFFIX) for n in names)
    back = load_checkpoint(str(tmp_path / "w.npz"))
    for k, v in pv.items():
        assert np.array_equal(back[k].reshape(v.shape), v), k
    half = load_checkpoint(str(tmp_path / "w.npz"), use_ema=True)
    k0 = "MACnetwork/MACCell/linearLayerqInput/weights/weight"
    assert np.allclose(half[k0], 0.5 * pv[k0])
    inputs = make_inputs(B, S, N, d, seed=9)
    got, cell = run_gpu(cfg, back, inputs, L)
    recs = write_preds(str(tmp_path / "preds.json"), cell)
    assert len(recs) == B and len(recs[0]["attentions"]["kb"]) == L
    assert np.asarray(recs[0]["attentions"]["kb"][0]).shape == (14, 14)       # visualization.py:121 reshapes to the grid
    assert abs(np.asarray(recs[1]["attentions"]["kb"][1]).sum() - 1.0) < 1e-5
    assert len(recs[0]["attentions"]["self"]) == L and len(recs[0]["attentions"]["gate"]) == L


@pytest.mark.parametrize("prec,variant,shape", [
    ("fp32", "args", (16, 20, 196, 512, 4)),
    ("fp32", "gqa", (5, 7, 49, 128, 3)),
    ("bf16", "args", (8, 12, 196, 512, 4)),
    ("bf16", "gqa", (64, 30, 49, 512, 6)),
])
def test_step_invariant_read_hoist_is_the_same_function(prec, variant, shape):
    """Eval mode computes P = KB@Wx+bx and Q = P@Wm[d:2d]+bm once per forward (mac_read_invariant / mac_read_fwd_inv).
    The per-step form (mac_read_fwd, what training uses; here selected by save_for_backward with eval dropouts) must stay
    the same function: both against the oracle, and against each other."""
    B, S, N, d, L = shape
    cfg = MACConfig.args(variant, netLength=L, memDim=d, ctrlDim=d, attDim=d)
    inputs = make_inputs(B, S, N, d, seed=61, dtype=np.float64)
    params = perturb_biases(init_params(cfg, L, seed=62, dtype=np.float64), seed=63)
    hoisted, cell = run_gpu(cfg, params, inputs, L, prec=prec)
    assert cell._read_hoist
    stepwise, cell = run_gpu(cfg, params, inputs, L, prec=prec, save_for_backward=True)
    assert not cell._read_hoist
    ref = run_oracle(cfg, params, inputs, L)
    tol = 1e-4 if prec == "fp32" else 3e-2
    for k in ("memory", "info", "att_kb"):
        assert max_rel(hoisted[k], ref[k]) < tol, (k, "hoisted")
        assert max_rel(stepwise[k], ref[k]) < tol, (k, "stepwise")
        assert max_rel(hoisted[k], stepwise[k]) < (2e-5 if prec == "fp32" else 2e-2), k
    print(prec, variant, {k: (max_rel(hoisted[k], ref[k]), max_rel(stepwise[k], ref[k])) for k in ("memory", "info")})


@pytest.mark.parametrize("prec,host_cast", [("bf16", None), ("bf16", True), ("fp32", None)])
def test_host_pipeline_matches_direct_small_tc_cell(prec, host_cast):
    """serving.HostPipeline (host fp32 in -> [host bf16 cast through the staging ring] -> H2D -> graph -> D2H) returns
    bit for bit what a small_tc cell computes from device-resident inputs; in-flight slots and staging buffers do not mix
    batches up.  host_cast=True casts whatever the timing rule would decide (it switches the cast off at this small shape)."""
    from mac_network_b200.mac_cell import MACParams
    from mac_network_b200.serving import HostPipeline
    B, S, N, d, L = 8, 6, 49, 128, 3
    cfg = MACConfig.args("args", netLength=L, memDim=d, ctrlDim=d, attDim=d)
    pv = perturb_biases(init_params(cfg, L, seed=82), seed=83)
    params = MACParams(cfg, L, values=pv)
    pipe = HostPipeline(cfg, params, (B, S, N, d, L), prec=prec, slots=2, cast_threads=3, host_cast=host_cast)
    if host_cast:
        assert pipe.host_kb_bf16 and len(pipe._stages) == 3
    batches = [make_inputs(B, S, N, d, seed=90 + i) for i in range(5)]
    host = [{k: torch.from_numpy(v).pin_memory() for k, v in b.items() if k != "questionWords"} for b in batches]
    got = []
    for i, hb in enumerate(host):
        t = pipe.submit(hb, next_batch=host[(i + 1) % len(host)])
        got.append({k: v.clone() for k, v in pipe.result(t).items()})
    for b, g in zip(batches, got):
        # the pipeline's cells use the throughput form (small_tc): same form for the direct cell
        ref, _ = run_gpu(cfg, pv, b, L, prec=prec, small_tc=True)
        assert np.array_equal(g["memory"].numpy(), ref["memory"][-1]), prec       # same kernels, same bits
        assert np.array_equal(g["control"].numpy(), ref["control"][-1])
        assert np.array_equal(g["att_kb"].numpy(), ref["att_kb"])
