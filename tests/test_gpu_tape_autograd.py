"""The tape backward (`mac_network_b200/tape.py`) of every flag set outside the shipped flag files, element by element
against torch.autograd on the fp64 restatement (`oracle/mac_torch_autograd.py`, run in fp64 on the GPU), with the
comparison and bars of tests/test_tape_autograd_bounds.py: every gradient tensor at a max-norm bar, each sample of dKB,
dwords and dvecQ at a bar relative to its own maximum, exact zeros in the gradient of the padded words, and the exactly-zero
gradients (softmax logit biases) at a null bar.

The flag sets: the 17 P2 fixtures of tests/golden/ and two variants of args1 that the scheduled sweep refuses and the tape
takes (controlFeedPrev without controlFeedPrevAtt; controlFeedPrev with writeSelfAtt=CONT).  Every case sets the question
lengths so that its batch holds a question of length 1, one of length S and one in between (a batch of one: length 1), and
also checks the forward (control_L, memory_L) against the restatement and that two backward sweeps of the same forward give
the same bits.

    shape      (B, S, N, d, L)          what it reaches                               sets                  dropouts
    fixture    (3, 5, 7, 16, 3)         the golden fixtures' shape                    all 19                fixture's, train
    ragged     (5, 9, 50, 20, 4)        d % 32 != 0; B*N = 250, not a multiple of 64   all 19                train
    tiles      (3, 40, 257, 64, 3)      N > 256: the knowledge base past one box; S=40 all 19                train
    one        (1, 6, 49, 64, 3)        a batch of one                                without memoryBN      train
    headline   (16, 40, 196, 512, 3)    the headline width, 14 x 14 grid              NINE                  train
    bf16       (4, 7, 16, 128, 3),      the bf16 tape (prec="bf16", tc=True):          NINE                  train
               (16, 40, 196, 512, 3)    d = 128 with B*N = 64, and d = 512
"train" is (memory, read, write) keeps (0.85, 0.85, 0.9) with the cell's train flag set."""
import numpy as np
import pytest
import torch

from mac_network_b200.config import MACConfig
from mac_network_b200.params import init_params, perturb_biases
from mac_network_b200.synthetic import make_inputs
from oracle import mac_torch_autograd as TA
from tests._util import load_golden, max_rel
from tests.test_tape_autograd_bounds import P2_CASES, TOL_BF16, TOL_FP32, TOL_FP32_BN, bad, grad_errs, worst

pytestmark = pytest.mark.gpu

ARGS1_TAPE = ["args1_feed_cont", "args1_selfatt_cont"]
SETS = P2_CASES + ARGS1_TAPE
NO_BN = [s for s in SETS if not s.startswith("p2_memory_bn")]
NINE = ["p2_read_add", "p2_read_bl", "p2_read_plain", "p2_control", "p2_control_feed", "p2_write_info", "p2_write_mul",
        "p2_memory_bn_train", "p2_unshared"]
TRAIN = (0.85, 0.85, 0.9)
SHAPES = {"fixture": (3, 5, 7, 16, 3), "ragged": (5, 9, 50, 20, 4), "tiles": (3, 40, 257, 64, 3), "one": (1, 6, 49, 64, 3),
          "headline": (16, 40, 196, 512, 3), "bf16_128": (4, 7, 16, 128, 3), "bf16_512": (16, 40, 196, 512, 3)}
#                                                                                                   measured
TOL_FWD = 1e-4            # control_L / memory_L max-rel against the restatement, the fp32 parity bar     6.8e-6
TOL_FWD_BF16 = 2.5e-2     # the bf16 cell's forward bar (tests/test_gpu_tape_tc.py)                       8.9e-3
WORST = {}


def _flags(name):
    """(cell flags, fixture dropouts, fixture train flag)"""
    if name in ARGS1_TAPE:
        meta, _ = load_golden("args1_small")
        flags = dict(meta["cell_flags"])
        if name == "args1_feed_cont":
            flags["controlFeedPrevAtt"] = False
        else:
            flags.update(writeSelfAtt=True, writeSelfAttMod="CONT")
    else:
        meta, _ = load_golden(name)
        flags = dict(meta["cell_flags"])
    dm = meta["dropouts"]
    return flags, (dm["memory"], dm["read"], dm["write"]), bool(meta["train"])


def _lengths(B, S, rng):
    """1, S, then lengths strictly in between (a batch of one: 1)."""
    out = np.concatenate([[1, S], rng.randint(2, S, size=max(B - 2, 0))])[:B] if S > 2 else np.ones(B)
    return out.astype(np.int32)


def _fp32(a):
    """the value the fp32 product sees, in fp64: both sides differentiate the same function"""
    return a if a.dtype == np.int32 else a.astype(np.float32).astype(np.float64)


def _case(name, shape, dropouts, prec="fp32", seed=31):
    from mac_network_b200.autograd import mac_backward
    from mac_network_b200.mac_cell import MACCell, MACParams, mac_network
    B, S, N, d, L = shape
    flags, dp_fixture, train_fixture = _flags(name)
    dp, train = (dp_fixture, train_fixture) if dropouts == "fixture" else (TRAIN, True)
    # the kernels take each keep as a float and keep an element iff u >= 1 - keep (fp32): floor(keep + u) for the fp32 keep.
    # The fp64 keep 0.85 drops the element with u = 1 - float32(0.85) that the kernels keep; with one chance in 2^24 per
    # element it turned up at the headline shape (a whole step's read dropout at 1e-2 of the gradients)
    dp = tuple(float(np.float32(k)) for k in dp)
    flags.update(memDim=d, ctrlDim=d, attDim=d, netLength=L)
    if dp[2] < 1.0:
        flags["writeDropout"] = dp[2]
    cfg = MACConfig(**flags).validate()
    rng = np.random.RandomState(seed)
    inputs = {k: _fp32(v) for k, v in make_inputs(B, S, N, d, seed=seed, dtype=np.float64).items()}
    inputs["questionLengths"] = _lengths(B, S, rng)
    pv = {k: _fp32(v) for k, v in perturb_biases(init_params(cfg, L, seed=seed + 1, dtype=np.float64), seed=seed + 2).items()}
    gc, gm = (_fp32(rng.standard_normal((B, d))) for _ in range(2))

    params = MACParams(cfg, L, values={k: v.astype(np.float32) for k, v in pv.items()})
    x = {k: torch.from_numpy(np.ascontiguousarray(v if v.dtype == np.int32 else v.astype(np.float32))).cuda()
         for k, v in inputs.items()}
    cell = MACCell(x["vecQuestions"], x["questionWords"], x["questionCntxWords"], x["questionLengths"], x["knowledgeBase"],
                   dp[0], dp[1], dp[2], B, train, config=cfg, params=params, prec=prec, seed=4242, save_for_backward=True)
    control, memory = mac_network(cell, L)
    tape = cell._tape
    assert tape is not None, "this flag set is expected on the tape"
    tc = prec == "bf16"
    dc, dm = (torch.from_numpy(a.astype(np.float32)).cuda() for a in (gc, gm))
    # two sweeps of the same forward: the tape releases its nodes after a sweep and accumulates into its buffers, so the
    # second sweep gets the recorded nodes back and zeroed buffers
    nodes, finalizers = list(tape.nodes), list(tape.finalizers)
    g1 = {k: v.clone() for k, v in mac_backward(cell, dc, dm, tc=tc).items()}
    for buf in tape.grads.values():
        buf.zero_()
    tape.nodes, tape.finalizers = nodes, finalizers
    g2 = mac_backward(cell, dc, dm, tc=tc)
    torch.cuda.synchronize()
    same = [k for k in g1 if not torch.equal(g1[k], g2[k])]

    rc, rm, rg = TA.run(cfg, pv, inputs, L, dp, cell.dropout_uniforms(), gc, gm, train=train, device="cuda")
    fwd = max(max_rel(control.cpu().numpy(), rc), max_rel(memory.cpu().numpy(), rm))
    words_key = "questionCntxWords" if cfg.controlContextual else "questionWords"
    errs = grad_errs({k: g1[k].cpu().numpy() for k in rg}, rg, inputs["questionLengths"], words_key)
    tol, tol_fwd = (TOL_BF16, TOL_FWD_BF16) if tc else (TOL_FP32_BN if cfg.memoryBN else TOL_FP32, TOL_FWD)
    key = "bf16" if tc else "fp32 BN" if cfg.memoryBN else "fp32"
    WORST[key + " fwd"] = max(WORST.get(key + " fwd", 0.0), fwd)
    for kind in ("tensor", "sample", "null"):
        WORST["%s %s" % (key, kind)] = max(WORST.get("%s %s" % (key, kind), 0.0), worst(errs, kind))
    top = sorted(((k, v) for k, v in errs.items() if not k.startswith("pad:")), key=lambda kv: -kv[1] / tol[kv[0].split(":")[0]])
    print("%s %s %s %s: fwd %.2e, tensor %.2e, sample %.2e, null %.2e, pad %g; worst %s" % (
        name, shape, dropouts, prec, fwd, worst(errs, "tensor"), worst(errs, "sample"), worst(errs, "null"),
        errs["pad:" + words_key], ", ".join("%s %.2e" % (k.replace("MACnetwork/MACCell/", ""), v) for k, v in top[:2])))
    assert fwd < tol_fwd, fwd
    assert not same, ("second sweep differs", same)
    failing = bad(errs, tol)
    assert not failing, failing


def _params():
    out = []
    for s in SETS:
        out += [(s, "fixture", "fixture"), (s, "fixture", "train"), (s, "ragged", "train"), (s, "tiles", "train")]
    out += [(s, "one", "train") for s in NO_BN]
    out += [(s, "headline", "train") for s in NINE]
    return out


@pytest.mark.parametrize("name,shape,dropouts", _params())
def test_tape_matches_fp64_autograd(name, shape, dropouts):
    _case(name, SHAPES[shape], dropouts)


@pytest.mark.parametrize("shape", ["bf16_128", "bf16_512"])
@pytest.mark.parametrize("name", NINE)
def test_bf16_tape_matches_fp64_autograd(name, shape):
    _case(name, SHAPES[shape], "train", prec="bf16")


def test_zz_print_worst():
    print("worst measured:", {k: "%.2e" % v for k, v in sorted(WORST.items())})
