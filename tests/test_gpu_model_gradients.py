"""The whole model's training step on the GPU element by element against one fp64 autograd graph of the reference's loss
(`oracle/model_torch_autograd.py`, pinned on the CPU by tests/test_model_autograd_oracle.py), built on the GPU with every
dropout mask drawn independently of the library: `oracle/philox.py` at the library's Philox sites, with the per-(step,
rank) seed restated here.

Every case trains at the reference's dropouts (encoder 0.85 / 0.92, stem 0.82, the cell's from its flag set, output unit
0.85), at weights moved by one optimizer step (every bias off zero, step counter 1) and with questions of lengths 1 and S
beside padded ones.  It compares:
- the logits and the loss of each question, row by row, so that one wrong row cannot hide behind a larger one;
- every parameter tensor's gradient, max |got - ref| / max |ref|; a softmax logit bias, whose true gradient is 0, against
  the largest gradient of the model;
- for `MACModel`, the image gradient of each image, and an image no question asks about gets exactly 0.

Matrix: `DPTrainer` in fp32 over the shipped flag sets and the tape's (`p2_*`), one shard of rank 1 of 2 with the global
batch 2B, fp16 NCHW features, k < B images with `imageIndex` (one unused) on the fp32, tc32 / bf16x3 and bf16 paths, the
bf16 and all-tensor-core configurations at d = 512; `MACModel` with images that require grad, NHWC and NCHW fp32 and NCHW
fp16, with and without `imageIndex`.  Each bar is about three times the worst error measured on an H100 80GB HBM3 (700 W
power limit, 1980 MHz max SM clock), written beside it, and no higher than the suite's bar for that precision."""
import numpy as np
import pytest
import torch

from oracle import model_torch_autograd as MA
from oracle.philox import philox_uniform
from tests.test_gpu_tc32_training import NULL_GRADIENTS
from tests.test_gpu_wgmma import keep_threshold
from tests.test_model_autograd_oracle import dropout_plan, make_data, model_config, training_keeps

pytestmark = pytest.mark.gpu

V, E, A, HIDDEN, L = 13, 16, 8, [32], 3
BASE_SEED = 7

# case -> flag set, widths, shape, precisions, data layout and sharding
CASES = {
    "args": dict(flags="args"),
    "gqa": dict(flags="gqa"),
    "args1": dict(flags="args1"),
    "args3": dict(flags="args3"),
    "args4": dict(flags="args4"),
    "tape_memory_bn": dict(flags="p2_memory_bn_train", d=16),
    "tape_read_add": dict(flags="p2_read_add_train", d=16),
    "rank1_of_2": dict(flags="args", rank=1, world=2),
    "fp16_nchw": dict(flags="args", C=64, layout="nchw16"),         # forward_nchw: channels a multiple of 64
    "indexed_fp32": dict(flags="args", indexed=True),
    "indexed_tc32_bf16x3": dict(flags="args", d=128, C=128, HW=(4, 4), indexed=True, prec="tc32", bwd_tc=True,
                                stem_prec="bf16x3"),
    "indexed_tc32_fp32bwd_bf16x3": dict(flags="args", d=128, C=128, HW=(4, 4), indexed=True, prec="tc32", bwd_tc=False,
                                        stem_prec="bf16x3"),
    "indexed_bf16": dict(flags="args", d=128, C=128, HW=(4, 4), indexed=True, prec="bf16", bwd_tc=True, stem_prec="bf16"),
    "bf16_enc_bf16": dict(flags="args", d=512, C=128, HW=(4, 4), prec="bf16", bwd_tc=True, stem_prec="bf16",
                          enc_prec="bf16"),
    "all_tc": dict(flags="args", d=512, C=128, HW=(4, 4), prec="tc32", bwd_tc=True, stem_prec="bf16x3", enc_prec="bf16"),
}
B, S = 8, 6
# N = 3 x 5 = 15 (not a multiple of 64) for the fp32 paths; 4 x 4 with B * N % 64 == 0 for the tensor-core ones
DEFAULT = dict(d=64, C=32, HW=(3, 5), rank=0, world=1, layout="nhwc", indexed=False, prec="fp32", bwd_tc=False,
               stem_prec="fp32", enc_prec="fp32")
INDEX = np.array([3, 0, 3, 4, 0, 2, 3, 4])          # 5 images, image 1 unused

# Bars by configuration and part of the model: max |got - ref| / max |ref| of each tensor of that part; the logits and the
# losses row by row; each used image's gradient; the null gradients of the model's largest.  Ceilings: the suite's gradient
# bar 2e-4 for fp32, tc32 and bf16x3; for the bf16 paths the unit bars (TOL_STEM_BF16 1.2e-2 for the stem, 9e-3 for the
# bf16 encoder's gradients, 5e-2 for the bf16 cell backward).                                          measured worst
BARS = {
    "fp32": dict(cell=2.5e-5,           # the memoryBN tape's initMem; the other flag sets 2.0e-6              7.7e-6
                 encoder=5e-6,                                                                             # 1.7e-6
                 stem=8e-6,                                                                                # 2.6e-6
                 output=4e-6,                                                                              # 1.3e-6
                 logits=1e-5,                                                                              # 3.4e-6
                 d_images=1.5e-6,                                                                          # 4.9e-7
                 null=3e-7),                                                                               # 8.8e-8
    "tc32": dict(cell=8e-5,             # tc32 cell, bwd_tc on or off, bf16x3 stem                            2.6e-5
                 encoder=1.5e-5,                                                                           # 4.5e-6
                 stem=2e-5,                                                                                # 6.3e-6
                 output=2e-5,                                                                              # 6.0e-6
                 logits=1.5e-5,                                                                            # 4.1e-6
                 null=1e-7),                                                                               # 2.7e-8
    "bf16": dict(cell=4.5e-2,           # bf16 cell and stem, d = 128 and d = 512 with the bf16 encoder       1.4e-2
                 encoder=8e-3,                                                                             # 2.6e-3
                 stem=7e-3,                                                                                # 2.2e-3
                 output=7e-3,                                                                              # 2.3e-3
                 logits=2.5e-3,                                                                            # 7.9e-4
                 null=3e-8),                                                                               # 9.8e-9
    "all_tc": dict(cell=2.1e-2,         # tc32 cell and bf16x3 stem, the bf16 encoder's error through the cell  7.0e-3
                   encoder=7e-3,                                                                           # 2.2e-3
                   stem=8e-5,                                                                              # 2.7e-5
                   output=7e-3,                                                                            # 2.3e-3
                   logits=8e-5,                                                                            # 2.7e-5
                   null=1e-8),                                                                             # 2.1e-9
}
PARTS = {"encoder": ("encoder/", "qEmbeddings/"), "stem": ("stem/",), "cell": ("MACnetwork/",),
         "output": ("outputUnit/", "classifier/")}


def _case(name):
    return dict(DEFAULT, **(CASES[name] if isinstance(name, str) else name))


def _kind(c):
    if c["prec"] == "tc32" and c["enc_prec"] == "bf16":
        return "all_tc"
    if "bf16" in (c["prec"], c["stem_prec"], c["enc_prec"]):
        return "bf16"
    return "tc32" if c["prec"] == "tc32" or c["stem_prec"] == "bf16x3" else "fp32"


def philox_seed(base, step, rank):
    """The Philox key of one training forward: one stream per (step, rank)."""
    return (base * 1000003 + step * 7919 + rank * 104729 + 1) & 0x7FFFFFFFFFFFFFFF


def _unit_keep(unit, site, keeps):
    from mac_network_b200 import _lib
    from mac_network_b200.encoder import SITE_ENC_INPUT
    if unit == "encoder":
        return keeps["encoder"][0 if site == SITE_ENC_INPUT else 1]
    if unit == "cell":
        km, kr, kw = keeps["cell"]
        return km if site in (_lib.SITE_MEM_VAR, _lib.SITE_MEM_PLAIN) else kw if site == _lib.SITE_WRITE_INFO else kr
    return keeps[unit]


def draws(plan, seed):
    """The raw uniforms of each unit's draws, from oracle/philox.py."""
    return {u: [philox_uniform(seed, site, step, int(np.prod(shape))).reshape(shape) for site, step, shape in d]
            for u, d in plan.items()}


def kernel_masks(plan, raw, keeps):
    """Each draw as the kernels' exact keep-mask, [u >= 1 - float32(keep)] on the 24-bit integer, in uniforms the oracle's
    floor(keep + U) turns into that mask."""
    out = {}
    for u, d in plan.items():
        out[u] = [MA.mask_uniforms(r * 16777216.0 >= keep_threshold(_unit_keep(u, site, keeps)))
                  for (site, _, _), r in zip(d, raw[u])]
    return out


def _setup(name):
    """A trainer one optimizer step past its initialisation, and the batch of the step under test."""
    from mac_network_b200.dp import DPTrainer
    c = _case(name)
    cfg, cell_dp = model_config(c["flags"], c["d"], L)
    H, W = c["HW"]
    tr = DPTrainer(cfg, L, seed=BASE_SEED, rank=c["rank"], world=c["world"], lr=1e-3, dropouts=cell_dp,
                   classifier=(A, HIDDEN), encoder=(V, E), stem=(c["C"], 2), prec=c["prec"], bwd_tc=c["bwd_tc"],
                   stem_prec=c["stem_prec"], enc_prec=c["enc_prec"])
    gb = B * c["world"]
    first = make_data(B, S, V, B, H, W, c["C"], A, seed=60)
    tr.train_step_full("step0", {k: torch.from_numpy(v).cuda() for k, v in first.items()}, global_batch=gb)
    data = make_data(B, S, V, INDEX.max() + 1 if c["indexed"] else B, H, W, c["C"], A, seed=61,
                     index=INDEX if c["indexed"] else None)
    return c, cfg, cell_dp, tr, data, gb


def _device(data, layout):
    dev = {k: torch.from_numpy(v).cuda() for k, v in data.items() if k != "images"}
    x = torch.from_numpy(data["images"]).cuda()
    if layout == "nhwc":
        dev["images"] = x
    else:
        dev["images_nchw"] = x.permute(0, 3, 1, 2).contiguous().to(torch.float16 if layout == "nchw16" else torch.float32)
    return dev


def _oracle_data(data, dev):
    """What the fp64 graph is fed: the images exactly as the library reads them (fp16 features widened)."""
    out = {k: v for k, v in data.items() if k != "images"}
    if "images" in dev:
        out["images"] = dev["images"].double()
    else:
        out["images_nchw"] = dev["images_nchw"].float().double()
    return out


def _rowwise(got, ref):
    """max over rows of max |got_b - ref_b| / max |ref_b|."""
    got, ref = got.double().reshape(got.shape[0], -1), ref.reshape(ref.shape[0], -1)
    return float(((got - ref).abs().max(1)[0] / ref.abs().max(1)[0]).max())


def _compare(got_grads, ref, logits, losses):
    """Errors per checked quantity: logits and losses (when given) row by row, each gradient tensor; and the null
    gradients against the model's largest gradient."""
    errs = {"logits": _rowwise(logits, ref["logits"])}
    if losses is not None:
        errs["losses"] = _rowwise(losses.view(-1, 1), ref["losses"].view(-1, 1))
    gmax = max(float(g.abs().max()) for g in ref["grads"].values())
    null = {}
    for n, g in ref["grads"].items():
        if "/BatchNorm/moving_" in n:
            continue
        got = got_grads[n].double().reshape(-1)
        want = g.reshape(-1)
        if n.endswith(NULL_GRADIENTS):
            null[n] = float(got.abs().max()) / gmax
            continue
        errs[n] = float((got - want).abs().max()) / float(want.abs().max())
    return errs, null


def _part(key):
    if key in ("logits", "losses"):
        return "logits"
    if key.startswith("d_images"):
        return "d_images"
    return next(p for p, prefixes in PARTS.items() if key.startswith(prefixes))


def _report(name, errs, null, kind):
    worst = {}
    for k, v in errs.items():
        part = _part(k)
        if v >= worst.get(part, (-1.0, ""))[0]:
            worst[part] = (v, k)
    worst["null"] = (max(null.values()), "") if null else (0.0, "")
    where = lambda k: " (%s)" % k.replace("MACnetwork/MACCell/", "") if "/" in k else ""
    print("%s [%s]: %s" % (name, kind, ", ".join("%s %.2e%s" % (p, v, where(k)) for p, (v, k) in sorted(worst.items()))))
    bars = BARS[kind]
    bad = {k: v for k, v in errs.items() if not v < bars[_part(k)]}
    bad.update({k: v for k, v in null.items() if not v < bars["null"]})
    assert not bad, (name, bad)


@pytest.mark.parametrize("name", list(CASES))
def test_trainer_step_against_the_fp64_graph(name):
    c, cfg, cell_dp, tr, data, gb = _setup(name)
    keeps = training_keeps(cell_dp)
    H, W = c["HW"]
    dev = _device(data, c["layout"])
    values = tr.params.numpy()          # before the forward: memoryBN's training forward writes its moving statistics
    assert tr.step_id == 1
    logits, losses = tr.full_forward_backward("t", dev, global_batch=gb)
    torch.cuda.synchronize()
    k = data["images"].shape[0]
    seed = philox_seed(BASE_SEED, tr.step_id, c["rank"])
    plan = dropout_plan(cfg, L, values, keeps, B, S, k, H, W, step=tr.step_id)
    raw = draws(plan, seed)
    cell = tr._cells["t"][0]
    assert cell.seed == seed
    lib_cell = cell.dropout_uniforms()
    assert len(lib_cell) == len(raw["cell"]) and all(np.array_equal(a, b) for a, b in zip(lib_cell, raw["cell"]))
    lib_enc = tr.enc.dropout_uniforms(B, S, step=tr.step_id)
    assert len(lib_enc) == 2 and all(np.array_equal(a, b) for a, b in zip(lib_enc, raw["encoder"]))
    ref = MA.run(cfg, L, values, _oracle_data(data, dev), keeps, kernel_masks(plan, raw, keeps), global_batch=gb,
                 device="cuda")
    p = tr.params
    got = {n: tr.bucket[p.offsets[n]:p.offsets[n] + max(1, int(np.prod(p.specs[n][0])))] for n in p.specs}
    if c["indexed"]:
        assert float(ref["grads"]["stem/cnnLayercnn_0/kernels/kernel"].abs().max()) > 0
    errs, null = _compare(got, ref, logits, losses)
    _report(name, errs, null, _kind(c))


MODULE_CASES = [(layout, indexed) for layout in ("nhwc", "nchw", "nchw16") for indexed in (False, True)]


@pytest.mark.parametrize("layout,indexed", MODULE_CASES)
def test_mac_model_backward_against_the_fp64_graph(layout, indexed):
    """`MACModel` from a trainer one step on, images that require grad: `answer_loss(...).backward()` against the graph,
    the parameter gradients and each image's gradient (fp16 images: the gradient comes back in fp16, so the bar adds its
    rounding to each entry)."""
    from mac_network_b200.modules import MACModel, answer_loss
    c, cfg, cell_dp, tr, data, _ = _setup(dict(flags="args", C=64, indexed=indexed))
    keeps = training_keeps(cell_dp)
    H, W = c["HW"]
    model = MACModel.from_trainer(tr)
    model.train()
    dev = _device(data, layout)
    key = "images" if layout == "nhwc" else "images_nchw"
    x = dev[key].clone().requires_grad_(True)
    values = {n: v.detach().cpu().numpy().astype(np.float64) for n, v in model.named_parameters()}
    step = model.step
    logits, _ = model(dev["questions"], dev["questionLengths"], imageIndex=dev.get("imageIndex"), **{key: x})
    answer_loss(logits, dev["answers"]).backward()
    torch.cuda.synchronize()
    k = data["images"].shape[0]
    plan = dropout_plan(cfg, L, values, keeps, B, S, k, H, W, step=step)
    raw = draws(plan, philox_seed(BASE_SEED, step, 0))
    odata = _oracle_data(data, dict(dev, **{key: x.detach()}))
    ref = MA.run(cfg, L, values, odata, keeps, kernel_masks(plan, raw, keeps), device="cuda")
    errs, null = _compare({n: v.grad for n, v in model.named_parameters()}, ref, logits, None)
    assert x.grad.dtype == x.dtype
    dimg = x.grad.double()
    used = sorted(set(INDEX.tolist())) if indexed else list(range(k))
    for u in range(k):
        if u not in used:
            assert not bool(dimg[u].any()), u
            continue
        r = ref["d_images"][u]
        excess = (dimg[u] - r).abs()
        if layout == "nchw16":          # less the rounding to fp16: half an ulp, 2^-25 below its normal range
            excess = excess - torch.clamp(2.0 ** -11 * r.abs(), min=2.0 ** -25)
        errs["d_images[%d]" % u] = float(excess.max()) / float(r.abs().max())
    assert indexed == (len(used) < k)
    _report("MACModel %s%s" % (layout, " indexed" if indexed else ""), errs, null, "fp32")
