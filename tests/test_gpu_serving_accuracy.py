"""What `ModelPipeline` serves, in every precision it ships, against one exact reference of the whole model: the fp64 graph
`oracle/model_torch_autograd.run` (encoder -> stem -> optional imageIndex gather -> L MAC steps -> output unit; pinned to
the reference by tests/test_model_autograd_oracle.py and tests/golden), every keep at 1.0, on the `MACnet`'s own
parameters, at the CLEVR (B=64, S=40, 1024x14x14, d=512, L=12) and GQA (B=64, S=30, 2048x7x7, d=512, L=6) serving shapes.

The other pipeline tests compare the pipeline with `runBatch` or with another arm of itself, bit for bit, so an error every
arm shares cancels there; here it does not.  Each arm is compared by max-norm relative error (`tests._util.max_rel`):
the logits, the final memory, the question and knowledge-base attention maps of every step, and the top-k probabilities
against the fp64 softmax at the served ids; and, so that a failed bar points at a unit, the stem's output
(`net._stem.forward_nchw`) and the encoder's question vectors and contextual words (`net._enc`).  The answers: column 0
is the argmax of the served logits, and every question whose fp64 top-two margin exceeds twice the logits bar (as a
fraction of max |logits|) gets the fp64 answer.

Arms: fp32; split parity (`prec="tc32"`, `eval_stem_prec="bf16x3"`: the tc32 cell has an inference form, so `MACnet`
takes it); bf16; fp8 (e4m3 stem and read step, bf16 encoder); fp8 with fp16-stored features (its reference is the fp64
graph of the fp16-rounded features, so the storage rounding is not counted); bf16 and fp8 with 16 distinct images for the
64 questions through the knowledge-base cache (`images=16, cache=64`; the fp64 graph gets imageIndex).  The served question
attention is also checked to be exactly 0 beyond each question's length.

`test_bars_tell_a_wrong_kernel_from_a_right_one` evaluates the fp64 graph with perturbations that imitate plausible kernel
bugs and asserts each moves the metric it would show in by more than twice that metric's loosest bar."""
import numpy as np
import pytest
import torch

from oracle import mac_torch_autograd as TA
from oracle import model_torch_autograd as MA
from tests._util import max_rel

pytestmark = pytest.mark.gpu

V, E, A, TOPK, SEED = 90, 300, 28, 5, 3
SHAPES = {"clevr": dict(variant="args", B=64, S=40, C=1024, H=14, W=14, L=12, seed=11),
          "gqa": dict(variant="gqa", B=64, S=30, C=2048, H=7, W=7, L=6, seed=12)}
U = 16                      # distinct images of the shared-image arms
FP8 = dict(prec="fp8", eval_stem_prec="fp8", eval_enc_prec="bf16")
ARMS = {"fp32": dict(model=dict(prec="fp32")),
        "split": dict(model=dict(prec="tc32", eval_stem_prec="bf16x3")),
        "bf16": dict(model=dict(prec="bf16")),
        "fp8": dict(model=FP8),
        "fp8_f16": dict(model=FP8, image_dtype=torch.float16),
        "bf16_shared": dict(model=dict(prec="bf16"), shared=True),
        "fp8_shared": dict(model=FP8, shared=True)}
METRICS = ("logits", "memory", "att_kb", "att_question", "probs", "stem", "vecq", "words")
KEEPS = {"encoder": (1.0, 1.0), "stem": 1.0, "cell": (1.0, 1.0, 1.0), "output": 1.0}

# Bars: max_rel against the fp64 graph, the worst of the two shapes.  fp32 and split parity: the project's 1e-4 parity bar
# on everything.  The others: about three times the worst error measured on an H100 80GB HBM3 (700 W power limit) over the
# two shapes and the arms that share the bar (the fp16-storage and shared-image arms take their precision's), written beside
# each bar.  In the bf16 arm the encoder and the control unit stay fp32.
PARITY = {m: 1e-4 for m in METRICS}
BARS = {"fp32": PARITY, "split": PARITY,
        "bf16": dict(logits=2.2e-2,                 # 7.2e-3
                     memory=6.5e-3,                 # 2.1e-3
                     att_kb=3e-3,                   # 9.6e-4
                     att_question=3e-7,             # 9.4e-8
                     probs=7.5e-3,                  # 2.4e-3
                     stem=1.1e-2,                   # 3.6e-3
                     vecq=1.5e-6,                   # 4.4e-7
                     words=1.7e-6),                 # 5.6e-7
        "fp8": dict(logits=0.26,                    # 8.7e-2
                    memory=9e-2,                    # 3.1e-2
                    att_kb=4e-2,                    # 1.4e-2
                    att_question=1.5e-4,            # 5.1e-5
                    probs=0.1,                      # 3.2e-2
                    stem=0.17,                      # 5.8e-2
                    vecq=9e-3,                      # 2.9e-3
                    words=1.05e-2)}                 # 3.5e-3
BARS.update(fp8_f16=BARS["fp8"], bf16_shared=BARS["bf16"], fp8_shared=BARS["fp8"])
# The margin rule must decide at least half of the questions, or its check would say nothing.  Not in the fp8 arms: their
# logits move by 7-9 % of max |logits| (2.0-2.1e-2 of the uncentred logits' maximum, which is 3.6-3.9 times the centred
# one: in line with the 2.8e-2 measured against the fp32 model), so 2 x the bar is 0.52 of max |logits|, above nearly every
# top-two margin of this model (median 0.07-0.12), and the rule decides almost nothing.  Their answers are reported as the
# agreement with fp64 (0.83-0.92 measured), and the questions the rule does decide are still checked.
DECIDE_HALF = {a: not a.startswith("fp8") for a in ARMS}

_REF = {}
_CENTRE = {}


def _batch(sh, shared):
    """One host batch: ReLU-of-normal NCHW features, random question ids with ragged lengths (one question of length S),
    0-padded to S; `shared`: U distinct images, question b about image imageIndex[b], every image asked about."""
    rng = np.random.RandomState(sh["seed"] + (1000 if shared else 0))
    B, S = sh["B"], sh["S"]
    lengths = rng.randint(1, S + 1, size=(B,)).astype(np.int32)
    lengths[rng.randint(B)] = S
    q = rng.randint(1, V + 1, size=(B, S)).astype(np.int32)
    q[np.arange(S)[None, :] >= lengths[:, None]] = 0
    k = U if shared else B
    out = {"questions": q, "questionLengths": lengths,
           "images": np.maximum(rng.standard_normal((k, sh["C"], sh["H"], sh["W"])), 0).astype(np.float32)}
    if shared:
        index = rng.randint(U, size=(B,))
        index[rng.choice(B, U, replace=False)] = np.arange(U)
        out["imageIndex"] = index.astype(np.int32)
    return out


def _net(shape, arm):
    """The arm's `MACnet`, the same parameters in every arm: every bias moved off TF's zero initialisation, then the last
    classifier bias lowered by each answer's mean fp64 logit over the shape's batch.  At initialisation the logits hardly
    depend on the question and the image, and every question gets the same answer; centred, the answers vary and the
    margin rule below decides something."""
    from mac_network_b200.config import MACConfig
    from mac_network_b200.model import MACnet
    sh = SHAPES[shape]
    cfg = MACConfig.args(sh["variant"], netLength=sh["L"])
    assert not cfg.memoryBN             # the fp64 graph's cell runs its training-mode batch norm
    net = MACnet(cfg, sh["L"], V, A, wrd_emb_dim=E, image_in_dim=sh["C"], classifier_dims=(512,), seed=SEED,
                 **ARMS[arm]["model"])
    p = net.trainer.params
    g = torch.Generator(device="cuda").manual_seed(SEED)
    with torch.no_grad():
        for name, v in p.t.items():
            if name.endswith("bias"):
                v.add_(0.1 * torch.randn(v.shape, device=v.device, generator=g))
    if shape not in _CENTRE:
        batch = _batch(sh, False)
        _CENTRE[shape] = _fp64(cfg, sh["L"], p.numpy(), batch, batch["images"].astype(np.float64))["logits"].mean(0)
    nfc = len([k for k in p.t if k.startswith("classifier/linearLayerfc_") and k.endswith("weights/weight")])
    with torch.no_grad():
        p.t["classifier/linearLayerfc_%d/biases/bias" % (nfc - 1)].sub_(torch.from_numpy(_CENTRE[shape]).float().cuda())
    p.touch()
    return net


def _fp64(cfg, L, values, batch, images):
    """The fp64 graph on the batch trimmed to its longest question, as runBatch does: the logits, the final memory and the
    stacked attention maps as numpy, and the units' outputs the cell reads as fp64 device tensors."""
    S = int(batch["questionLengths"].max())
    data = {"questions": batch["questions"][:, :S], "questionLengths": batch["questionLengths"],
            "answers": np.zeros(len(batch["questionLengths"]), np.int32), "images_nchw": images}
    if "imageIndex" in batch:
        data["imageIndex"] = batch["imageIndex"]
    trace = []
    out = MA.run(cfg, L, values, data, KEEPS, grad=False, device="cuda", trace=trace)
    return {"logits": out["logits"].cpu().numpy(), "memory": trace[-1]["memory"],
            "att_kb": np.stack([t["att_kb"] for t in trace]), "att_question": np.stack([t["att_question"] for t in trace]),
            "stem": out["knowledgeBase"], "vecq": out["vecQuestions"], "words": out["questionCntxWords"],
            "questionWords": out["questionWords"]}


def _reference(shape, kind, net):
    """The fp64 result of one (shape, batch kind), computed once per module; the net's parameters must be the cached ones."""
    values = net.trainer.params.numpy()
    key = (shape, kind)
    if key not in _REF:
        sh = SHAPES[shape]
        batch = _batch(sh, kind == "shared")
        images = batch["images"].astype(np.float16) if kind == "f16" else batch["images"]
        _REF[key] = (values, batch, images, _fp64(net.cfg, sh["L"], values, batch, images.astype(np.float64)))
    cached = _REF[key][0]
    assert all(np.array_equal(values[k], cached[k]) for k in cached)
    return _REF[key][1:]


def _serve(net, shape, arm, batch, images):
    """The pipeline's outputs for one batch, as numpy; the shared arms go through the knowledge-base cache twice (all
    misses, then all hits), and the two results must agree bit for bit."""
    from mac_network_b200.serving import ModelPipeline
    sh = SHAPES[shape]
    dims = (sh["B"], sh["S"], sh["H"], sh["W"])
    a = ARMS[arm]
    if not a.get("shared"):
        pipe = ModelPipeline(net, dims, slots=1, topk=TOPK, host_cast=False,
                             image_dtype=a.get("image_dtype", torch.float32))
        out = {k: v.numpy().copy() for k, v in pipe.result(pipe.submit(dict(batch, images=images))).items()}
        pipe.drain()
        return out
    pipe = ModelPipeline(net, dims, slots=2, topk=TOPK, images=U, cache=sh["B"])
    ids = 100 + batch["imageIndex"].astype(np.int64)
    req = {"questions": batch["questions"], "questionLengths": batch["questionLengths"], "imageIds": ids,
           "images": lambda miss: images[miss - 100]}
    first = {k: v.numpy().copy() for k, v in pipe.result(pipe.submit(req)).items()}
    second = {k: v.numpy().copy() for k, v in pipe.result(pipe.submit(req)).items()}
    stats = pipe.cache_stats()
    assert stats["misses"] == U and stats["hits"] == U, stats
    for k in first:
        assert np.array_equal(first[k], second[k]), k
    pipe.drain()
    return first


def _units(net, batch, images):
    """The stem's and the encoder's outputs on their own."""
    x = torch.from_numpy(np.ascontiguousarray(images)).cuda()
    kb = net._stem.forward_nchw(x)
    q = torch.from_numpy(batch["questions"]).cuda()
    ln = torch.from_numpy(batch["questionLengths"]).cuda()
    words, cntx, vecq = net._enc.forward(q, ln)
    torch.cuda.synchronize()
    return {"stem": kb.cpu().numpy(), "vecq": vecq.cpu().numpy(), "words": cntx.cpu().numpy()}


def _errors(out, units, ref, lengths):
    beyond = np.arange(out["att_question"].shape[-1])[None, :] >= lengths[:, None]
    assert not out["att_question"][:, beyond].any(), "question attention beyond a question's length"
    errs = {k: max(max_rel(out[k][i], ref[k][i]) for i in range(len(ref[k]))) for k in ("att_kb", "att_question")}
    errs["logits"] = max_rel(out["logits"], ref["logits"])
    errs["memory"] = max_rel(out["memory"], ref["memory"])
    z = torch.from_numpy(ref["logits"])
    p64 = torch.softmax(z, -1).gather(1, torch.from_numpy(out["answers"]).long()).numpy()
    errs["probs"] = max_rel(out["probs"], p64)
    for k in ("stem", "vecq", "words"):
        errs[k] = max_rel(units[k], ref[k].cpu().numpy())
    return errs


def _answers(out, ref, bar):
    """(decided, agreement): the questions whose fp64 top-two margin exceeds 2 * bar * max |logits| must get the fp64
    answer; column 0 of the answers is the argmax of the served logits (ties to the lower id)."""
    served = out["answers"][:, 0]
    assert np.array_equal(served, np.argmax(out["logits"], axis=1))
    z = ref["logits"]
    want = np.argmax(z, axis=1)
    top2 = np.sort(z, axis=1)[:, -2:]
    decided = (top2[:, 1] - top2[:, 0]) > 2 * bar * np.abs(z).max()
    wrong = np.nonzero(decided & (served != want))[0]
    assert not len(wrong), ("decided questions answered differently", wrong, served[wrong], want[wrong])
    return int(decided.sum()), float((served == want).mean())


@pytest.mark.parametrize("arm", list(ARMS))
@pytest.mark.parametrize("shape", list(SHAPES))
def test_served_outputs_against_the_fp64_graph(shape, arm):
    net = _net(shape, arm)
    a = ARMS[arm]
    kind = "shared" if a.get("shared") else "f16" if a.get("image_dtype") == torch.float16 else "plain"
    batch, images, ref = _reference(shape, kind, net)
    out = _serve(net, shape, arm, batch, images)
    errs = _errors(out, _units(net, batch, images), ref, batch["questionLengths"])
    bars = BARS[arm]
    print("%s %s: %s" % (shape, arm, ", ".join("%s %.2e" % kv for kv in errs.items())))
    decided, agree = _answers(out, ref, bars["logits"])
    B = len(batch["questionLengths"])
    print("%s %s: answers decided by the margin %d / %d%s, agreement with fp64 %.3f"
          % (shape, arm, decided, B, "" if DECIDE_HALF[arm] else " (no floor: see DECIDE_HALF)", agree))
    bad = {k: v for k, v in errs.items() if not v < bars[k]}
    assert not bad, bad
    if DECIDE_HALF[arm]:
        assert decided >= B / 2, ("the logits bar decides too few answers", decided)


def _cell_and_output(cfg, L, values, x, lengths):
    """The fp64 graph from the cell on: the cell over `x` (vecQuestions, questionWords, questionCntxWords and the
    per-question knowledge base, fp64 device tensors) and the output unit, as `_fp64` returns them."""
    p = {k: torch.as_tensor(v, dtype=torch.float64).cuda() for k, v in values.items()}
    ln = torch.as_tensor(lengths).long().cuda()
    trace = []
    _, memory = TA.graph(cfg, p, x, ln, L, trace=trace)
    logits, _ = MA.output_graph(cfg.relu, p, memory, x["vecQuestions"], torch.zeros_like(ln), 1.0)
    return {"logits": logits.cpu().numpy(), "memory": trace[-1]["memory"],
            "att_kb": np.stack([t["att_kb"] for t in trace]), "att_question": np.stack([t["att_question"] for t in trace])}


def _np(a):
    return a.cpu().numpy() if torch.is_tensor(a) else a


def _moved(got, ref, metrics):
    """max_rel of `got` against `ref` per metric, per step for the attention maps."""
    return {k: max(max_rel(got[k][i], ref[k][i]) for i in range(len(ref[k]))) if k.startswith("att_")
            else max_rel(_np(got[k]), _np(ref[k])) for k in metrics}


@pytest.mark.parametrize("shape", list(SHAPES))
def test_bars_tell_a_wrong_kernel_from_a_right_one(shape):
    """Each perturbation of the fp64 graph imitates a plausible kernel bug and must move the metric it would show in by
    more than twice the loosest bar of that metric over the arms:
    - the features shifted by one pixel along W, column 0 zero (an im2col or ingest off-by-one): the stem's output and the
      knowledge-base attention;
    - the full-length question's length reduced by one in the cell (a mask off-by-one): the question attention;
    - the knowledge bases of questions 0 and 1 swapped (a tile-ownership or gather bug): the knowledge-base attention;
    - the last knowledge-base position left out of the read attention (a tail-tile bug): the knowledge-base attention.
    The swap also moves the final memory and the logits (measured 8.8e-2 / 2.0e-1 and 3.0e-1 / 5.2e-1, CLEVR / GQA), but by
    no more than the fp8 bars of those metrics: in the fp8 arms the attention maps, not the memory or the logits, are what
    would catch it.  It is printed, not asserted, for those two metrics."""
    net = _net(shape, "fp32")
    sh = SHAPES[shape]
    cfg, L = net.cfg, sh["L"]
    batch, images, ref = _reference(shape, "plain", net)
    values = net.trainer.params.numpy()
    x = {"vecQuestions": ref["vecq"], "questionWords": ref["questionWords"], "questionCntxWords": ref["words"],
         "knowledgeBase": ref["stem"]}
    lengths = batch["questionLengths"]
    clean = _cell_and_output(cfg, L, values, x, lengths)
    assert max(_moved(clean, ref, ("logits", "memory", "att_kb", "att_question")).values()) < 1e-12
    loosest = {m: max(BARS[a][m] for a in ARMS) for m in METRICS}
    moved = {}
    shifted = np.zeros_like(images, dtype=np.float64)
    shifted[..., 1:] = images[..., :-1]
    moved["shift"] = _moved(_fp64(cfg, L, values, batch, shifted), ref, ("stem", "att_kb"))
    short = lengths.copy()
    short[int(np.argmax(lengths))] -= 1
    moved["mask"] = _moved(_cell_and_output(cfg, L, values, x, short), ref, ("att_question",))
    swap = torch.arange(len(lengths), device="cuda")
    swap[[0, 1]] = swap[[1, 0]]
    moved["swap"] = _moved(_cell_and_output(cfg, L, values, dict(x, knowledgeBase=x["knowledgeBase"][swap]), lengths),
                           ref, ("att_kb", "memory", "logits"))
    tail = _cell_and_output(cfg, L, values, dict(x, knowledgeBase=x["knowledgeBase"][:, :-1]), lengths)
    tail["att_kb"] = np.concatenate([tail["att_kb"], np.zeros_like(tail["att_kb"][..., :1])], -1)
    moved["tail"] = _moved(tail, ref, ("att_kb",))
    print("%s: perturbed fp64 against clean, over the loosest bar: %s" % (shape, {
        b: {m: "%.2e (%.1fx)" % (v, v / loosest[m]) for m, v in ms.items()} for b, ms in moved.items()}))
    asserted = {"shift": ("stem", "att_kb"), "mask": ("att_question",), "swap": ("att_kb",), "tail": ("att_kb",)}
    weak = {(b, m): v / loosest[m] for b, ms in moved.items() for m, v in ms.items()
            if m in asserted[b] and not v > 2 * loosest[m]}
    assert not weak, weak
