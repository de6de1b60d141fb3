"""The reference's stem, location, output-unit and batch-norm options in the whole model, in every precision that ships them,
against one exact reference: the fp64 graph `oracle/model_torch_autograd.run` with the same options (`stem=`, `output=`,
and `train=False` for the stored batch-norm statistics; pinned to the reference by tests/test_model_options_oracle.py).

The other tests of these options compare the pipelines with `runBatch` bit for bit, which run the same kernels, or train
in fp32 and split bf16 only; here an error every arm shares does not cancel.

Serving (`ModelPipeline`), as tests/test_gpu_serving_accuracy.py does it and with its helpers and metrics: the logits, the
final memory, both attention maps of every step, the top-k probabilities, the stem's output, the question vectors and
contextual words, each by max-norm relative error; the classifier bias centred the same way; the margin rule for the
answers.  Option sets, each a `MACnet` with the same parameters in every arm (every bias and stored statistic moved off
its initial value):

    stride2   stem_strides=[2, 1]                                  CLEVR 1024x14x14 -> 7x7, N = 49
    k53_s21   stem_kernel_sizes=[5, 3], stem_strides=[2, 1]        CLEVR -> 7x7
    linear    stem_linear=True                                     GQA 2048x7x7
    loc_L     stem_location="L"                                    CLEVR
    loc_PE    stem_location="PE", dim 8, bias 0.5                  GQA
    q0        out_question=False                                   GQA
    qmul_bn   out_question_mul=True, output_bn=True                CLEVR
    memory_bn the p2_memory_bn cell flags at d = 512 (memoryBN)    GQA
    all       loc_PE + stride2 + qmul_bn                           CLEVR

Arms: fp32 and split (tc32 cell, bf16x3 stem) at the 1e-4 parity bar; bf16; fp8 (e4m3 read step, bf16 encoder; the e4m3
stem where it runs the option, else the bf16 stem, so the e4m3 read step still reads the new grid); and for stride2 and
loc_L 16 distinct images for the 64 questions through the knowledge-base cache in bf16 and fp8.  Every set runs in every
arm: memory_bn's flag set keeps the fused read unit, so the split and e4m3 cells take it.  The one refusal is the e4m3
stem's, of every stem option (`eval_stem_prec="fp8"`), at `MACnet` construction before any launch.

Training: the `DPTrainer` step against the fp64 graph with the library's own dropout masks (tests/test_gpu_model_gradients.py's
machinery and per-precision bars) for the stem sets and `all` in the bf16 and all-tensor-core configurations, `all` also in
fp32; and `MACModel` on `all` in bf16 with fp16 NCHW images that require grad and an imageIndex."""
import numpy as np
import pytest
import torch

from oracle import model_torch_autograd as MA
from oracle import output_options as OO
from oracle import stem_geometry as SG
from oracle.stem_location import grid_torch
from tests import test_gpu_model_gradients as MG
from tests import test_gpu_serving_accuracy as SA

pytestmark = pytest.mark.gpu

LOC_PE = dict(stem_location="PE", stem_location_dim=8, stem_location_bias=0.5)
QMUL_BN = dict(out_question_mul=True, output_bn=True)
SETS = {"stride2": dict(shape="clevr", net=dict(stem_strides=[2, 1])),
        "k53_s21": dict(shape="clevr", net=dict(stem_kernel_sizes=[5, 3], stem_strides=[2, 1])),
        "linear": dict(shape="gqa", net=dict(stem_linear=True)),
        "loc_L": dict(shape="clevr", net=dict(stem_location="L")),
        "loc_PE": dict(shape="gqa", net=LOC_PE),
        "q0": dict(shape="gqa", net=dict(out_question=False)),
        "qmul_bn": dict(shape="clevr", net=QMUL_BN),
        "memory_bn": dict(shape="gqa", net={}, flags="p2_memory_bn"),
        "all": dict(shape="clevr", net=dict(LOC_PE, stem_strides=[2, 1], **QMUL_BN))}
SHARED = ("stride2", "loc_L")
PRECS = ("fp32", "split", "bf16", "fp8")
CASES = [(s, a) for s in SETS for a in PRECS] + [(s, a) for s in SHARED for a in ("bf16_shared", "fp8_shared")]

# Bars: max_rel against the fp64 graph, by arm; the shared-image arms take their precision's.  fp32 and split: the 1e-4
# parity bar (measured worst 3.9e-6 and 1.1e-5).  The others: about three times the worst error measured on an H100 80GB
# HBM3 (700 W power limit) over the sets of the arm, written beside each bar, and never above the arm's bar in
# tests/test_gpu_serving_accuracy.py (where three times the worst would be, the bar is that one: marked "cap").  The fp8
# arm of a stem option runs the bf16 stem, whose error dominates the e4m3 arm's elsewhere: its bars are "fp8_bf16_stem".
BARS = {"fp32": SA.PARITY, "split": SA.PARITY,
        "bf16": dict(logits=2e-2,                   # 6.8e-3  q0
                     memory=6.5e-3,                 # 2.4e-3  k53_s21, cap
                     att_kb=3e-3,                   # 1.2e-3  linear, cap
                     att_question=1.5e-7,           # 5.1e-8
                     probs=6.7e-3,                  # 2.2e-3
                     stem=1.1e-2,                   # 3.6e-3  stride2, cap
                     vecq=1.3e-6,                   # 4.4e-7
                     words=1.7e-6),                 # 5.6e-7  cap
        "fp8": dict(logits=0.26,                    # 1.2e-1  q0, cap
                    memory=9e-2,                    # 3.1e-2  qmul_bn, cap
                    att_kb=4e-2,                    # 1.3e-2  q0
                    att_question=1e-4,              # 3.2e-5
                    probs=8.5e-2,                   # 2.8e-2  qmul_bn
                    stem=0.15,                      # 5.0e-2  qmul_bn
                    vecq=9e-3,                      # 3.0e-3  cap
                    words=1.05e-2),                 # 3.5e-3  cap
        "fp8_bf16_stem": dict(logits=2e-2,          # 6.5e-3  stride2
                              memory=7e-3,          # 2.4e-3  k53_s21
                              att_kb=3.3e-2,        # 1.1e-2  linear
                              att_question=8e-5,    # 2.7e-5
                              probs=7.5e-3,         # 2.5e-3
                              stem=1.1e-2,          # 3.6e-3  stride2
                              vecq=9e-3,            # 2.9e-3
                              words=1.05e-2)}       # 3.5e-3


def _bars(name, arm):
    base = arm.replace("_shared", "")
    return BARS["fp8_bf16_stem" if base == "fp8" and _stem_options(SETS[name]["net"]) else base]


_REF, _CENTRE = {}, {}


def _stem_options(net_kw):
    """The set's stem options in the form `run(stem=)` and `DPTrainer(stem=(C, layers, geometry))` take; None: the 3x3
    stride-1 stem."""
    g = {}
    if net_kw.get("stem_kernel_sizes"):
        g["ksizes"] = net_kw["stem_kernel_sizes"]
    if net_kw.get("stem_strides"):
        g["strides"] = net_kw["stem_strides"]
    if net_kw.get("stem_linear"):
        g["linear"] = True
    if net_kw.get("stem_location"):
        g.update(location=net_kw["stem_location"], location_bias=net_kw.get("stem_location_bias", 1.0),
                 location_dim=net_kw.get("stem_location_dim", 32))
    return g or None


def _output_options(net_kw):
    o = dict(question=net_kw.get("out_question", True), mul=net_kw.get("out_question_mul", False),
             bn=net_kw.get("output_bn", False))
    return None if o == dict(question=True, mul=False, bn=False) else o


def _arm_model(name, arm):
    """The `MACnet` precision keywords of one arm of one set."""
    base = arm.replace("_shared", "")
    if base == "fp32":
        return dict(prec="fp32")
    if base == "split":
        return dict(prec="tc32", eval_stem_prec="bf16x3")
    if base == "bf16":
        return dict(prec="bf16")
    # the e4m3 stem runs the 3x3 stride-1 stem without location features; elsewhere the fp8 arm's stem is bf16's
    return dict(prec="fp8", eval_enc_prec="bf16", eval_stem_prec=None if _stem_options(SETS[name]["net"]) else "fp8")


def _cfg(name):
    from mac_network_b200.config import MACConfig
    from tests.test_model_autograd_oracle import model_config
    s, sh = SETS[name], SA.SHAPES[SETS[name]["shape"]]
    if s.get("flags"):
        return model_config(s["flags"], 512, sh["L"])[0]
    return MACConfig.args(sh["variant"], netLength=sh["L"])


def _build(name, arm):
    from mac_network_b200.model import MACnet
    sh = SA.SHAPES[SETS[name]["shape"]]
    return MACnet(_cfg(name), sh["L"], SA.V, SA.A, wrd_emb_dim=SA.E, image_in_dim=sh["C"], classifier_dims=(512,),
                  seed=SA.SEED, **_arm_model(name, arm), **SETS[name]["net"])


def _net(name, arm):
    """The arm's `MACnet`: every bias moved off zero and every stored batch-norm statistic off (0, 1) by one generator, so
    every arm holds the same values; then the last classifier bias centred as tests/test_gpu_serving_accuracy.py does."""
    net = _build(name, arm)
    p = net.trainer.params
    g = torch.Generator(device="cuda").manual_seed(SA.SEED)
    with torch.no_grad():
        for k, v in p.t.items():
            if k.endswith("bias"):
                v.add_(0.1 * torch.randn(v.shape, device=v.device, generator=g))
            elif k.endswith("/moving_mean"):
                v.copy_(0.2 * torch.randn(v.shape, device=v.device, generator=g))
            elif k.endswith("/moving_variance"):
                v.copy_(torch.exp(0.5 * torch.randn(v.shape, device=v.device, generator=g)))
    sh = SA.SHAPES[SETS[name]["shape"]]
    if name not in _CENTRE:
        batch = SA._batch(sh, False)
        _CENTRE[name] = _fp64(name, net.cfg, p.numpy(), batch, batch["images"].astype(np.float64))["logits"].mean(0)
    nfc = len([k for k in p.t if k.startswith("classifier/linearLayerfc_") and k.endswith("weights/weight")])
    with torch.no_grad():
        p.t["classifier/linearLayerfc_%d/biases/bias" % (nfc - 1)].sub_(torch.from_numpy(_CENTRE[name]).float().cuda())
    p.touch()
    return net


def _fp64(name, cfg, values, batch, images, **over):
    """SA._fp64 with the set's options and the evaluation batch norms; `over` replaces run's keywords (perturbations)."""
    net_kw = SETS[name]["net"]
    S = int(batch["questionLengths"].max())
    data = {"questions": batch["questions"][:, :S], "questionLengths": batch["questionLengths"],
            "answers": np.zeros(len(batch["questionLengths"]), np.int32), "images_nchw": images}
    if "imageIndex" in batch:
        data["imageIndex"] = batch["imageIndex"]
    trace = []
    kw = dict(stem=_stem_options(net_kw), output=_output_options(net_kw), train=False)
    kw.update(over)
    out = MA.run(cfg, SA.SHAPES[SETS[name]["shape"]]["L"], values, data, SA.KEEPS, grad=False, device="cuda",
                 trace=trace, **kw)
    return {"logits": out["logits"].cpu().numpy(), "memory": trace[-1]["memory"],
            "att_kb": np.stack([t["att_kb"] for t in trace]), "att_question": np.stack([t["att_question"] for t in trace]),
            "stem": out["knowledgeBase"], "vecq": out["vecQuestions"], "words": out["questionCntxWords"],
            "questionWords": out["questionWords"]}


def _reference(name, shared, net):
    values = net.trainer.params.numpy()
    key = (name, shared)
    if key not in _REF:
        batch = SA._batch(SA.SHAPES[SETS[name]["shape"]], shared)
        _REF[key] = (values, batch, _fp64(name, net.cfg, values, batch, batch["images"].astype(np.float64)))
    cached = _REF[key][0]
    assert all(np.array_equal(values[k], cached[k]) for k in cached)
    return _REF[key][1:]


def _serve(net, name, shared, batch):
    """SA._serve for the set's shape: one batch, or with `shared` two passes through the knowledge-base cache (all misses,
    then all hits) that must agree bit for bit."""
    from mac_network_b200.serving import ModelPipeline
    sh = SA.SHAPES[SETS[name]["shape"]]
    dims = (sh["B"], sh["S"], sh["H"], sh["W"])
    images = batch["images"]
    if not shared:
        pipe = ModelPipeline(net, dims, slots=1, topk=SA.TOPK, host_cast=False)
        out = {k: v.numpy().copy() for k, v in pipe.result(pipe.submit(dict(batch, images=images))).items()}
        pipe.drain()
        return out
    pipe = ModelPipeline(net, dims, slots=2, topk=SA.TOPK, images=SA.U, cache=sh["B"])
    assert tuple(pipe.pool.shape[:2]) == (sh["B"], int(np.prod(net._stem.grid(sh["H"], sh["W"]))))
    req = {"questions": batch["questions"], "questionLengths": batch["questionLengths"],
           "imageIds": 100 + batch["imageIndex"].astype(np.int64), "images": lambda miss: images[miss - 100]}
    first = {k: v.numpy().copy() for k, v in pipe.result(pipe.submit(req)).items()}
    second = {k: v.numpy().copy() for k, v in pipe.result(pipe.submit(req)).items()}
    stats = pipe.cache_stats()
    assert stats["misses"] == SA.U and stats["hits"] == SA.U, stats
    for k in first:
        assert np.array_equal(first[k], second[k]), k
    pipe.drain()
    return first


@pytest.mark.parametrize("name,arm", CASES)
def test_served_outputs_with_options_against_the_fp64_graph(name, arm):
    net = _net(name, arm)
    shared = arm.endswith("_shared")
    batch, ref = _reference(name, shared, net)
    sh = SA.SHAPES[SETS[name]["shape"]]
    assert ref["stem"].shape[1] == int(np.prod(net._stem.grid(sh["H"], sh["W"])))
    out = _serve(net, name, shared, batch)
    errs = SA._errors(out, SA._units(net, batch, batch["images"]), ref, batch["questionLengths"])
    bars = _bars(name, arm)
    print("%s %s: %s" % (name, arm, ", ".join("%s %.2e" % kv for kv in errs.items())))
    decided, agree = SA._answers(out, ref, bars["logits"])
    B = len(batch["questionLengths"])
    fp8 = arm.startswith("fp8")
    print("%s %s: answers decided by the margin %d / %d%s, agreement with fp64 %.3f"
          % (name, arm, decided, B, " (no floor: see SA.DECIDE_HALF)" if fp8 else "", agree))
    bad = {k: v for k, v in errs.items() if not v < bars[k]}
    assert not bad, bad
    if not fp8:
        assert decided >= B / 2, ("the logits bar decides too few answers", decided)


@pytest.mark.parametrize("name", [s for s in SETS if _stem_options(SETS[s]["net"])])
def test_e4m3_stem_refuses_the_stem_options_at_construction(name):
    """The e4m3 stem runs the 3x3 stride-1 stem without location features: `eval_stem_prec="fp8"` with any stem option
    raises before anything is launched (the fp8 arm above runs the bf16 stem instead)."""
    from mac_network_b200._lib import load
    from mac_network_b200.model import MACnet
    lib = load()
    sh = SA.SHAPES[SETS[name]["shape"]]
    torch.cuda.synchronize()
    launches = lib.mac_b200_launch_count()
    with pytest.raises(NotImplementedError):
        MACnet(_cfg(name), sh["L"], SA.V, SA.A, wrd_emb_dim=SA.E, image_in_dim=sh["C"], classifier_dims=(512,),
               seed=SA.SEED, prec="fp8", eval_stem_prec="fp8", **SETS[name]["net"])
    torch.cuda.synchronize()
    assert lib.mac_b200_launch_count() == launches


# ------------------------------------------------------------------------------------------------ the bars' power
def _loosest(name):
    arms = [a for s, a in CASES if s == name]
    return {m: max(_bars(name, a)[m] for a in arms) for m in SA.METRICS}


# The metrics each perturbation must move by more than twice their loosest bar.  location_xy moves the knowledge-base
# attention by 1.5e-2 (CLEVR, loc_L), 0.47 times the fp8 arm's bar of that metric (the e4m3 read step's error): the
# stem's output, which every arm checks at its stem's own bar, is what catches a transposed location channel.  It is
# printed, not asserted, for the attention.
ASSERTED = {"location_xy": ("stem",), "pad_side": ("stem", "att_kb"), "output_bn_batch": ("logits",),
            "memory_bn_batch": ("memory", "logits"), "mul_dropped": ("logits",), "kb_grid": ("att_kb", "memory", "logits")}


@pytest.mark.parametrize("what", ["location_xy", "pad_side", "output_bn_batch", "memory_bn_batch", "mul_dropped",
                                  "kb_grid"])
def test_bars_tell_a_wrong_kernel_from_a_right_one(what, monkeypatch):
    """Each perturbation of the fp64 graph imitates a plausible bug of the new pieces and must move the metric it would
    show in by more than twice that metric's loosest bar over the set's arms:
    - location_xy (loc_L): the location grid's x and y channels swapped (a transposed location channel in layer 0's
      product): the stem's output and the knowledge-base attention;
    - pad_side (stride2): SAME padding's odd row and column before the image instead of after it (14 -> 7 at stride 2
      pads one): the stem's output and the knowledge-base attention;
    - output_bn_batch (qmul_bn): the output unit's batch norm on the batch's statistics instead of the stored ones: the
      logits;
    - memory_bn_batch (memory_bn): the cell's memoryBN on the batch's statistics: the memory and the logits;
    - mul_dropped (qmul_bn): outQuestionMul's product left out of the classifier's input: the logits;
    - kb_grid (stride2): the knowledge base laid out on the 14x14 input grid and read as the 7x7 one (the first 49 rows of
      the stride-1 stem's output): the knowledge-base attention, the memory and the logits."""
    name = {"location_xy": "loc_L", "pad_side": "stride2", "output_bn_batch": "qmul_bn", "memory_bn_batch": "memory_bn",
            "mul_dropped": "qmul_bn", "kb_grid": "stride2"}[what]
    net = _net(name, "fp32")
    cfg, L = net.cfg, SA.SHAPES[SETS[name]["shape"]]["L"]
    batch, ref = _reference(name, False, net)
    values = net.trainer.params.numpy()
    images = batch["images"].astype(np.float64)
    if what == "location_xy":
        def stem(relu, p, x, keep=1.0, uniforms=None):
            B, H, W, _ = x.shape
            g = grid_torch("L", 1.0, 32, H, W, device=x.device)[..., [1, 0]]
            x = torch.cat([x, g[None].expand(B, H, W, 2)], -1)
            return SG.stem_torch(relu, {k: v for k, v in p.items() if k.startswith("stem/")}, x)
        monkeypatch.setattr(MA, "stem_graph", stem)
        got, metrics = _fp64(name, cfg, values, batch, images, stem=None), ("stem", "att_kb")
    elif what == "pad_side":
        same = SG.same_pads
        monkeypatch.setattr(SG, "same_pads", lambda n, k, s: same(n, k, s)[::-1])
        got, metrics = _fp64(name, cfg, values, batch, images), ("stem", "att_kb")
    elif what in ("output_bn_batch", "memory_bn_batch"):
        got = _fp64(name, cfg, values, batch, images, train=True)
        metrics = ("logits",) if what == "output_bn_batch" else ("memory", "logits")
    elif what == "mul_dropped":
        p = {k: torch.as_tensor(v, dtype=torch.float64).cuda() for k, v in values.items()}
        w = p["classifier/linearLayerfc_0/weights/weight"].clone()
        d = cfg.memDim
        w[2 * d:3 * d] = 0                       # the rows that read memory * q'
        p["classifier/linearLayerfc_0/weights/weight"] = w
        memory = torch.as_tensor(ref["memory"]).cuda()
        logits, _ = OO.output_graph(cfg.relu, p, memory, ref["vecq"], torch.zeros(len(memory), dtype=torch.long).cuda(),
                                    question=True, mul=True, bn=True, train=False)
        got, metrics = {"logits": logits.cpu().numpy()}, ("logits",)
    else:
        full = SG.stem_torch(cfg.relu, {k: torch.as_tensor(v, dtype=torch.float64).cuda() for k, v in values.items()
                                        if k.startswith("stem/")},
                             torch.as_tensor(images).cuda().permute(0, 2, 3, 1))
        N = ref["stem"].shape[1]
        assert full.shape[1] == 4 * N
        x = {"vecQuestions": ref["vecq"], "questionWords": ref["questionWords"], "questionCntxWords": ref["words"],
             "knowledgeBase": full[:, :N].contiguous()}
        got = SA._cell_and_output(cfg, L, values, x, batch["questionLengths"])
        metrics = ("att_kb", "memory", "logits")
    loosest = _loosest(name)
    moved = SA._moved(got, ref, metrics)
    print("%s (%s): perturbed fp64 against clean, over the loosest bar: %s" % (what, name, {
        m: "%.2e (%.1fx)" % (v, v / loosest[m]) for m, v in moved.items()}))
    weak = {m: v / loosest[m] for m, v in moved.items() if m in ASSERTED[what] and not v > 2 * loosest[m]}
    assert not weak, weak


# ------------------------------------------------------------------------------------------------ training
GEOMS = {"stride2": dict(geom=dict(strides=[2, 1]), HW=(7, 8)),
         "k53_s21": dict(geom=dict(ksizes=[5, 3], strides=[2, 1]), HW=(7, 8)),
         "linear": dict(geom=dict(linear=True), HW=(4, 4)),
         "loc_L": dict(geom=dict(location="L"), HW=(4, 4)),
         "loc_PE": dict(geom=dict(location="PE", location_bias=0.5, location_dim=8), HW=(4, 4)),
         "all": dict(geom=dict(location="PE", location_bias=0.5, location_dim=8, strides=[2, 1]), HW=(7, 8),
                     out=dict(question=True, mul=True, bn=True))}
# the bf16 configuration, and the all-tensor-core one (tc32 cell, bf16x3 stem, bf16 encoder); fp32 at its own d and C.
# The knowledge bases are 4 x 4: B * N = 128, whole tiles of the tensor-core read backward.
CONFIGS = {"bf16": dict(d=512, C=128, prec="bf16", bwd_tc=True, stem_prec="bf16", enc_prec="bf16"),
           "all_tc": dict(d=512, C=128, prec="tc32", bwd_tc=True, stem_prec="bf16x3", enc_prec="bf16"),
           "fp32": dict()}
TRAIN_CASES = [(g, c) for g in GEOMS for c in ("bf16", "all_tc")] + [("all", "fp32")]
# Bars: test_gpu_model_gradients.py's for each precision (MG.BARS), with two exceptions, measured on an H100 80GB HBM3
# (700 W power limit):
# - the null gradients (a softmax logit bias, exactly 0 in exact arithmetic: the rounding of a sum over the batch and the
#   knowledge base, against the model's largest gradient) take the fp32 path's bar, 3e-7: measured 1.1e-8 (loc_PE,
#   all_tc), above that configuration's 1e-8, and 1.6e-7 (all, all_tc; 9.7e-8 in fp32);
# - `all` in bf16 and all_tc trains the output unit's batch norm on the statistics of B = 8 rows, which divide the error
#   the bf16 encoder and cell bring into the classifier's input by a small batch's deviation: every part takes the bar
#   tests/test_gpu_output_options.py sets for that unit's whole-model bf16 step, 5e-2 (its qmul_bn_bf16 case measures
#   1.2e-2).  Measured worst: bf16 1.7e-2 (cell; logits and losses 1.2e-2, output 9.2e-3, stem 6.7e-3), all_tc 6.1e-3
#   (cell; logits 1.9e-3, stem 2.4e-3), MACModel 1.8e-2 (cell; encoder and output 1.4e-2, the image gradient 1.0e-2).
#   The same options without the batch norm (the stride2 and loc_PE sets) stay inside MG.BARS, and `all` in fp32 inside
#   the fp32 bars (logits 1.4e-6), so the options' arithmetic is right and what grows is the batch norm's conditioning.
NULL_BAR = MG.BARS["fp32"]["null"]
OUTPUT_BN_STEP = 5e-2


def _report(monkeypatch, name, gname, errs, null, kind):
    """MG._report at this file's bars for the case (see above)."""
    bars = dict(MG.BARS[kind], null=max(MG.BARS[kind]["null"], NULL_BAR))
    if gname == "all" and kind != "fp32":
        bars = dict({p: OUTPUT_BN_STEP for p in ("cell", "encoder", "stem", "output", "logits", "d_images")},
                    null=NULL_BAR)
        kind = kind + ", output batch norm"
    monkeypatch.setitem(MG.BARS, kind, bars)
    MG._report(name, errs, null, kind)


def _trainer(gname, config, data_seed=61, index=None):
    from mac_network_b200.dp import DPTrainer
    from tests.test_model_autograd_oracle import make_data, model_config
    g = GEOMS[gname]
    c = dict(MG.DEFAULT, flags="args", HW=g["HW"], **CONFIGS[config])
    cfg, cell_dp = model_config(c["flags"], c["d"], MG.L)
    H, W = c["HW"]
    classifier = (MG.A, MG.HIDDEN) + ((g["out"],) if g.get("out") else ())
    tr = DPTrainer(cfg, MG.L, seed=MG.BASE_SEED, lr=1e-3, dropouts=cell_dp, classifier=classifier, encoder=(MG.V, MG.E),
                   stem=(c["C"], 2, g["geom"]), prec=c["prec"], bwd_tc=c["bwd_tc"], stem_prec=c["stem_prec"],
                   enc_prec=c["enc_prec"])
    first = make_data(MG.B, MG.S, MG.V, MG.B, H, W, c["C"], MG.A, seed=60)
    tr.train_step_full("step0", {k: torch.from_numpy(v).cuda() for k, v in first.items()}, global_batch=MG.B)
    k = MG.B if index is None else int(index.max()) + 1
    data = make_data(MG.B, MG.S, MG.V, k, H, W, c["C"], MG.A, seed=data_seed, index=index)
    return c, cfg, cell_dp, tr, data


def _masks(gname, cfg, values, keeps, k, c, step):
    """The library's dropout masks of one step in the fp64 graph's order: the stem's planned on each layer's own grid, and
    with location features the image and location draws of layer 0 joined into the one draw over its whole input."""
    from tests import test_gpu_stem_geometry_training as GT
    from tests import test_gpu_stem_location as SL
    geom = GEOMS[gname]["geom"]
    H, W = c["HW"]
    plan = (SL._plan if geom.get("location") else GT._plan)(cfg, values, keeps, k, H, W, c["C"], geom, step)
    masks = MG.kernel_masks(plan, MG.draws(plan, MG.philox_seed(MG.BASE_SEED, step, 0)), keeps)
    if geom.get("location") and masks["stem"]:
        masks["stem"] = [torch.cat([masks["stem"][0], masks["stem"][1]], -1)] + masks["stem"][2:]
    return masks


@pytest.mark.parametrize("gname,config", TRAIN_CASES)
def test_trainer_step_with_options_against_the_fp64_graph(gname, config, monkeypatch):
    from tests.test_model_autograd_oracle import training_keeps
    c, cfg, cell_dp, tr, data = _trainer(gname, config)
    keeps = training_keeps(cell_dp)
    H, W = c["HW"]
    dev = MG._device(data, "nhwc")
    values = tr.params.numpy()
    logits, losses = tr.full_forward_backward("t", dev, global_batch=MG.B)
    torch.cuda.synchronize()
    cell = tr._cells["t"][0]
    assert cell.N == int(np.prod(tr.stem.grid(H, W)))
    masks = _masks(gname, cfg, values, keeps, MG.B, c, tr.step_id)
    ref = MA.run(cfg, MG.L, values, MG._oracle_data(data, dev), keeps, masks, global_batch=MG.B, device="cuda",
                 stem=GEOMS[gname]["geom"], output=GEOMS[gname].get("out"), moving={})
    p = tr.params
    got = {n: tr.bucket[p.offsets[n]:p.offsets[n] + max(1, int(np.prod(p.specs[n][0])))] for n in p.specs}
    errs, null = MG._compare(got, ref, logits, losses)
    _report(monkeypatch, "%s %s" % (gname, config), gname, errs, null, MG._kind(c))


def test_mac_model_with_every_option_in_bf16_against_the_fp64_graph(monkeypatch):
    """`MACModel.from_trainer` of the bf16 trainer with location features, a stride-2 stem, outQuestionMul and outputBN:
    fp16 NCHW images that require grad, five images for eight questions (image 1 unused): the parameter gradients at the
    bf16 bars, each used image's gradient (less its fp16 rounding) and exactly 0 for the unused one."""
    from mac_network_b200.modules import MACModel, answer_loss
    from tests.test_model_autograd_oracle import training_keeps
    c, cfg, cell_dp, tr, data = _trainer("all", "bf16", index=MG.INDEX)
    keeps = training_keeps(cell_dp)
    model = MACModel.from_trainer(tr)
    model.train()
    dev = MG._device(data, "nchw16")
    x = dev["images_nchw"].clone().requires_grad_(True)
    values = {n: v.detach().cpu().numpy().astype(np.float64) for n, v in model.named_parameters()}
    values.update({n: v.detach().cpu().numpy().astype(np.float64) for n, v in model.named_buffers()})
    step = model.step
    logits, _ = model(dev["questions"], dev["questionLengths"], images_nchw=x, imageIndex=dev["imageIndex"])
    answer_loss(logits, dev["answers"]).backward()
    torch.cuda.synchronize()
    k = data["images"].shape[0]
    masks = _masks("all", cfg, values, keeps, k, c, step)
    ref = MA.run(cfg, MG.L, values, MG._oracle_data(data, dict(dev, images_nchw=x.detach())), keeps, masks,
                 device="cuda", stem=GEOMS["all"]["geom"], output=GEOMS["all"]["out"], moving={})
    errs, null = MG._compare({n: v.grad for n, v in model.named_parameters()}, ref, logits, None)
    dimg = x.grad.double()
    used = sorted(set(MG.INDEX.tolist()))
    for u in range(k):
        if u not in used:
            assert not bool(dimg[u].any()), u
            continue
        r = ref["d_images"][u]
        excess = (dimg[u] - r).abs() - torch.clamp(2.0 ** -11 * r.abs(), min=2.0 ** -25)     # less the fp16 rounding
        errs["d_images[%d]" % u] = float(excess.max()) / float(r.abs().max())
    assert len(used) < k
    _report(monkeypatch, "MACModel all bf16", "all", errs, null, "bf16")
