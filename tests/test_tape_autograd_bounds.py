"""CPU checks of the fp64 autograd restatement (`oracle/mac_torch_autograd.py`) over the whole flag space, and of the
comparison tests/test_gpu_tape_autograd.py makes between it and the tape backward (`mac_network_b200/tape.py`).

1. Forward pin: the restatement equals the numpy oracle (`oracle/mac_oracle.py`, fp64) to 1e-12 on every cell fixture in
   tests/golden/, eval and train (fed their stored uniforms), and each step's control / memory / info equals the fixture's
   own arrays at the parity bar of tests/test_oracle_golden.py.
2. Gradient pin: for every P2 flag set (the flags outside the shipped args*.txt files, SURVEY section 8(a)) its gradients
   equal central differences of the numpy oracle along sparse directions of every parameter and input, both in fp64.
3. The comparison (`grad_errs`, `bad`, the bars) is defined here and imported by the GPU test: a per-tensor max-norm bar, a
   per-sample bar on the input gradients, exact zeros in the gradient of the padded words, and a "null" bar for the
   gradients that are exactly zero (the softmax logit biases: shift invariance).  Each planted fault below, applied to the
   restatement's own gradients, fails the fp32 bars by at least 10x: one sample's dKB scaled by 1 + 1e-3, one step's
   contribution to a weight gradient dropped, two concat segments of a weight gradient swapped, a non-zero value in a
   padded word's gradient, one sample missing from a bias gradient."""
import numpy as np
import pytest

from mac_network_b200.config import MACConfig
from oracle import mac_torch_autograd as TA
from oracle.mac_oracle import MACOracle
from tests._util import golden_cases, load_golden, rebuild, uniforms_of

P2_CASES = ["p2_control", "p2_control_feed", "p2_ablations", "p2_wholeq", "p2_unshared", "p2_read_bl", "p2_read_add",
            "p2_read_plain", "p2_read_noproj", "p2_write_info", "p2_write_sum", "p2_write_mem", "p2_write_mul",
            "p2_read_add_train", "p2_read_plain_train", "p2_memory_bn", "p2_memory_bn_train"]

# ------------------------------------------------------------------------------------------------ the comparison
# Bars of the tape against the fp64 restatement (tests/test_gpu_tape_autograd.py), each about three times the worst value
# measured over that file's cases on an H100 80GB HBM3 at a 700 W power limit, written beside it.  memoryBN normalises
# with the statistics of batches of 1-16 rows (1 / sqrt(var + 1e-3) up to ~30): its flag sets get their own fp32 bars.
#                                                                                                   measured
TOL_FP32 = {"tensor": 1e-5,   # max |tape - ref| / max |ref| per gradient tensor                    3.3e-6
            "sample": 1e-5,   # max |tape - ref| / max |ref| per sample of dKB, dwords, dvecQ       2.7e-6
            "null": 4e-5}     # max |tape| / median of the tensors' maxima, exactly-zero gradients  1.2e-5
TOL_FP32_BN = {"tensor": 2e-4, "sample": 6e-5, "null": 1e-3}   # memoryBN:                         8.5e-5, 2.1e-5, 3.3e-4
TOL_BF16 = {"tensor": 4e-2, "sample": 6e-2, "null": 6e-5}      # the bf16 tape (tc=True):          1.3e-2, 2.0e-2, 1.9e-5
# a reference gradient whose maximum is below this fraction of the median maximum is zero in exact arithmetic (fp64
# round-off of a sum that cancels, e.g. the softmax logit biases)
NULL_REL = 1e-9
INPUTS = ("knowledgeBase", "questionWords", "questionCntxWords", "vecQuestions")
MARGIN = 10


def grad_errs(got, ref, lengths, words_key):
    """got, ref: {name: array}.  Returns {"tensor:<k>", "sample:<k>[b]", "null:<k>", "pad:<words>": value}:
    tensor / sample -- max |got - ref| over max |ref| of the tensor / of its b-th sample (input gradients only);
    null -- max |got| over the median of the reference maxima, for a gradient that is exactly zero;
    pad -- max |got| over the words past each question's length (must be exactly 0)."""
    ref = {k: np.asarray(v, np.float64) for k, v in ref.items()}
    got = {k: np.asarray(got[k], np.float64).reshape(r.shape) for k, r in ref.items()}
    scales = {k: float(np.max(np.abs(r))) if r.size else 0.0 for k, r in ref.items()}
    med = float(np.median([v for v in scales.values() if v > 0]))
    out = {}
    for k, r in ref.items():
        if scales[k] <= NULL_REL * med:
            out["null:" + k] = float(np.max(np.abs(got[k]))) / med if r.size else 0.0
            continue
        out["tensor:" + k] = float(np.max(np.abs(got[k] - r))) / scales[k]
        if k in INPUTS:
            for b in range(r.shape[0]):
                s = float(np.max(np.abs(r[b])))
                if s > NULL_REL * med:
                    out["sample:%s[%d]" % (k, b)] = float(np.max(np.abs(got[k][b] - r[b]))) / s
    w = got[words_key]
    pad = [np.abs(w[b, int(n):]) for b, n in enumerate(lengths)]
    out["pad:" + words_key] = max(float(np.max(p)) if p.size else 0.0 for p in pad)
    return out


def over_bar(errs, tol):
    """{key: value / bar}; the padded words' bar is exact zero (any non-zero value -> inf)."""
    out = {}
    for k, v in errs.items():
        kind = k.split(":", 1)[0]
        out[k] = (np.inf if v > 0 else 0.0) if kind == "pad" else v / tol[kind]
    return out


def bad(errs, tol):
    return {k: v for k, v in over_bar(errs, tol).items() if not v <= 1.0}


def worst(errs, kind):
    return max([v for k, v in errs.items() if k.startswith(kind + ":")] + [0.0])


# ------------------------------------------------------------------------------------------------ helpers
def _fixture(case):
    meta, gold = load_golden(case)
    cfg, inputs, pv = rebuild(meta, np.float64)
    dm = meta["dropouts"]
    return meta, gold, cfg, inputs, pv, (dm["memory"], dm["read"], dm["write"])


def _oracle(cfg, pv, inputs, L, dp, uniforms, train):
    orc = MACOracle(cfg, pv, dtype=np.float64)
    orc.train = train
    return orc.run(L, inputs["vecQuestions"], inputs["questionWords"], inputs["questionCntxWords"], inputs["questionLengths"],
                   inputs["knowledgeBase"], memoryDropout=dp[0], readDropout=dp[1], writeDropout=dp[2], uniforms=uniforms)


def _words_key(cfg):
    return "questionCntxWords" if cfg.controlContextual else "questionWords"


def _restated(case, seed=5):
    meta, gold, cfg, inputs, pv, dp = _fixture(case)
    sh = meta["shape"]
    rng = np.random.RandomState(seed)
    gc, gm = rng.standard_normal((sh["B"], sh["d"])), rng.standard_normal((sh["B"], sh["d"]))
    us = uniforms_of(meta, gold)
    _, _, g = TA.run(cfg, pv, inputs, sh["L"], dp, us, gc, gm, train=bool(meta["train"]))
    return meta, cfg, inputs, pv, dp, us, gc, gm, g


# ------------------------------------------------------------------------------------------------ 1. forward pin
@pytest.mark.parametrize("case", golden_cases())
def test_forward_equals_the_numpy_oracle_and_the_fixture(case):
    meta, gold, cfg, inputs, pv, dp = _fixture(case)
    L, train = meta["shape"]["L"], bool(meta["train"])
    us = uniforms_of(meta, gold)
    st = _oracle(cfg, pv, inputs, L, dp, us, train)
    trace = []
    c, m, _ = TA.run(cfg, pv, inputs, L, dp, us, train=train, trace=trace)
    for got, want in ((c, st.control), (m, st.memory)):
        assert np.max(np.abs(got - want)) <= 1e-12 * np.max(np.abs(want)), case
    tol = 2e-6 if gold["control"].dtype == np.float32 else 1e-12          # tests/test_oracle_golden.py
    for k in ("control", "memory", "info"):
        g = gold[k].astype(np.float64)
        got = np.stack([t[k] for t in trace])
        assert np.max(np.abs(got - g)) / np.max(np.abs(g)) < tol, (case, k)


# ------------------------------------------------------------------------------------------------ 2. gradient pin
TOL_FD = 1e-6      # |fd - analytic| over the Cauchy-Schwarz scale of the direction on its support (+ round-off)


@pytest.mark.parametrize("case", P2_CASES)
def test_gradients_equal_central_differences_of_the_numpy_oracle(case):
    meta, cfg, inputs, pv, dp, us, gc, gm, g = _restated(case)
    L, train = meta["shape"]["L"], bool(meta["train"])
    wk = _words_key(cfg)

    def loss(p, x):
        st = _oracle(cfg, p, x, L, dp, us, train)
        return float(np.sum(st.control * gc) + np.sum(st.memory * gm))

    rng = np.random.RandomState(11)
    targets = [("param", k) for k in pv if "/BatchNorm/moving_" not in k] + [("input", k) for k in
                                                                            ("knowledgeBase", wk, "vecQuestions")]
    worst_seen, failures = 0.0, {}
    for kind, k in targets:
        base = pv[k] if kind == "param" else inputs[k]
        gk = g[k]
        for trial in range(2):
            v = np.zeros(base.size)
            v[rng.choice(base.size, min(3, base.size), replace=False)] = rng.standard_normal(min(3, base.size))
            v = v.reshape(base.shape) / np.linalg.norm(v)
            h = 1e-5 * (1.0 + float(np.max(np.abs(base))))

            def at(t):
                if kind == "param":
                    return loss(dict(pv, **{k: base + t * v}), inputs)
                return loss(pv, dict(inputs, **{k: base + t * v}))
            fd = (at(h) - at(-h)) / (2 * h)
            ana = float(np.sum(gk * v))
            # TOL_FD of the Cauchy-Schwarz scale of the direction on its support, plus 100 fp64 ulps over h: the round-off
            # of the difference quotient, all that is left of a gradient that is exactly zero (seen up to 2.2e-10 at h = 1e-5)
            allowed = TOL_FD * float(np.linalg.norm(gk[v != 0])) + 100 * np.finfo(np.float64).eps / h       # |v| = 1
            r = abs(fd - ana) / allowed
            worst_seen = max(worst_seen, r)
            if not r < 1.0:
                failures[(k, trial)] = (fd, ana, r)
    print("%s: worst |fd - analytic| / allowed %.2f over %d tensors" % (case, worst_seen, len(targets)))     # <= 0.15
    assert not failures, failures


# ------------------------------------------------------------------------------------------------ 3. planted faults
def _assert_caught(errs, what):
    r = over_bar(errs, TOL_FP32)
    k = max(r, key=lambda q: r[q])
    print("%s: worst %s at %.3g x its fp32 bar" % (what, k, r[k]))
    assert r[k] >= MARGIN, (what, k, r[k])
    return r[k]


def test_the_restatement_passes_its_own_comparison_with_exact_zeros():
    """The unfaulted restatement against itself passes; its padded-word gradients are exactly zero; a logit bias is null."""
    for case in ("p2_control", "p2_read_plain_train", "p2_memory_bn_train"):
        meta, cfg, inputs, pv, dp, us, gc, gm, g = _restated(case)
        errs = grad_errs(g, g, inputs["questionLengths"], _words_key(cfg))
        assert not bad(errs, TOL_FP32), (case, bad(errs, TOL_FP32))
        assert errs["pad:" + _words_key(cfg)] == 0.0
        assert "null:MACnetwork/MACCell/control/inter2logits/linearLayerlogits/biases/bias" in errs, case


def test_fault_one_sample_of_dkb_scaled():
    meta, cfg, inputs, pv, dp, us, gc, gm, g = _restated("p2_read_add_train")
    r = g["knowledgeBase"]
    b = int(np.argmin([np.max(np.abs(r[i])) for i in range(r.shape[0])]))     # the sample the tensor bar sees least
    bad_g = dict(g, knowledgeBase=r.copy())
    bad_g["knowledgeBase"][b] *= 1 + 1e-3
    _assert_caught(grad_errs(bad_g, g, inputs["questionLengths"], _words_key(cfg)), "dKB[%d] x (1 + 1e-3)" % b)


@pytest.mark.parametrize("step", [0, 2])
def test_fault_one_step_dropped_from_a_weight_gradient(step):
    """qInputU is shared by the steps.  The same function with controlInputUnshared and every qInput<i> equal to qInputU has
    one weight per step: their gradients are the steps' contributions, and they sum to the shared gradient."""
    meta, cfg, inputs, pv, dp, us, gc, gm, g = _restated("p2_read_plain_train")
    L = meta["shape"]["L"]
    assert not cfg.controlInputUnshared
    cfg_u = MACConfig(**dict(meta["cell_flags"], controlInputUnshared=True)).validate()
    tail = "MACCell/linearLayerqInput%s/weights/weight"
    name = TA.PREFIX + tail % "U"
    pv_u = {k: v for k, v in pv.items() if "qInputU" not in k}
    for i in range(L):
        for part in ("weights/weight", "biases/bias"):
            pv_u[TA.PREFIX + "MACCell/linearLayerqInput%d/" % i + part] = pv[TA.PREFIX + "MACCell/linearLayerqInputU/" + part]
    _, _, gu = TA.run(cfg_u, pv_u, inputs, L, dp, us, gc, gm, train=bool(meta["train"]))
    per_step = [gu[TA.PREFIX + tail % str(i)] for i in range(L)]
    assert np.max(np.abs(sum(per_step) - g[name])) <= 1e-12 * np.max(np.abs(g[name]))
    bad_g = dict(g, **{name: g[name] - per_step[step]})
    _assert_caught(grad_errs(bad_g, g, inputs["questionLengths"], _words_key(cfg)), "step %d dropped from qInputU" % step)


def test_fault_two_concat_segments_swapped():
    """newMemory of p2_write_mul reads [memory, info, memory * info, selfSmry]: swap the rows of the first two segments."""
    meta, cfg, inputs, pv, dp, us, gc, gm, g = _restated("p2_write_mul")
    d = meta["shape"]["d"]
    name = TA.PREFIX + "MACCell/write/linearLayernewMemory/weights/weight"
    assert g[name].shape[0] == 4 * d
    w = g[name].copy()
    w[:d], w[d:2 * d] = g[name][d:2 * d], g[name][:d]
    _assert_caught(grad_errs(dict(g, **{name: w}), g, inputs["questionLengths"], _words_key(cfg)), "segments 0 and 1 swapped")


def test_fault_nonzero_padded_word_gradient():
    meta, cfg, inputs, pv, dp, us, gc, gm, g = _restated("p2_control")
    wk, lengths = _words_key(cfg), inputs["questionLengths"]
    b = int(np.argmin(lengths))
    assert lengths[b] < meta["shape"]["S"]
    w = g[wk].copy()
    w[b, lengths[b], 0] = 1e-7 * np.max(np.abs(w))
    errs = grad_errs(dict(g, **{wk: w}), g, lengths, wk)
    assert errs["tensor:" + wk] < TOL_FP32["tensor"]           # invisible to the tensor bar
    _assert_caught(errs, "padded word gradient")


def test_fault_one_sample_missing_from_a_bias_gradient():
    """The samples are independent without memoryBN: the loss restricted to sample b gives its contribution."""
    meta, cfg, inputs, pv, dp, us, gc, gm, g = _restated("p2_write_info")
    L, B = meta["shape"]["L"], meta["shape"]["B"]
    name = TA.PREFIX + "MACCell/write/linearLayernewMemory/biases/bias"
    parts = []
    for b in range(B):
        keep = (np.arange(B) == b)[:, None]
        parts.append(TA.run(cfg, pv, inputs, L, dp, us, gc * keep, gm * keep, train=bool(meta["train"]))[2][name])
    assert np.max(np.abs(sum(parts) - g[name])) <= 1e-12 * np.max(np.abs(g[name]))
    b = int(np.argmin([np.max(np.abs(p)) for p in parts]))
    bad_g = dict(g, **{name: g[name] - parts[b]})
    _assert_caught(grad_errs(bad_g, g, inputs["questionLengths"], _words_key(cfg)), "sample %d missing from a bias" % b)


def test_the_oracle_gets_the_kernels_fp32_keep():
    """The kernels take keep as a float and keep an element iff its 24-bit uniform u >= 1 - keep, i.e. floor(keep + u) for
    float32(keep).  For keep = 0.85 the fp64 rule drops the element with u = 1 - float32(0.85), which the kernels keep:
    tests/test_gpu_tape_autograd.py therefore hands the restatement float32(keep)."""
    keep = 0.85
    k32 = float(np.float32(keep))
    u = 2516582 / 2.0 ** 24                 # the 24-bit uniform on the boundary
    assert u == 1.0 - k32
    assert np.floor(k32 + u) == 1.0 and np.floor(keep + u) == 0.0
