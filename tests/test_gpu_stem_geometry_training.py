"""Whole-model training with the stem's other geometries (--stemKernelSizes, --stemStrideSizes, --stemLinear), on the GPU.

- `DPTrainer.full_forward_backward` element by element against the fp64 autograd graph of tests/test_gpu_model_gradients.py,
  its stem replaced by `oracle/stem_geometry.py`'s (strides, even kernels, the linear stem) and the stem's dropout draws
  planned on each layer's own grid: stride 2 and 5x3 / stride 2-1 stems in fp32, NHWC and fp16 NCHW features (the NHWC
  ingest, then the general patch pass), the linear stem, and the tc32 cell with the bf16x3 stem; `MACModel.from_trainer`
  with a stride-2 stem and images that require grad.  Same bars as that file.
- `TrainPipeline` bit for bit a twin `MACnet` looping over `runBatch(train=True)`, stride-2 and linear stems.
- A reference-named TensorFlow checkpoint of a linear and of a 5x3 stride-2 stem loads into `MACModel` with strict=True;
  `ImageStem` with a geometry equals `Stem`; `write_preds` maps on the stem's grid; refusals at construction."""
import numpy as np
import pytest
import torch

from oracle import model_torch_autograd as MA
from oracle.stem_geometry import stem_torch
from mac_network_b200.stem import SITE_STEM, stem_grid
from tests import test_gpu_model_gradients as MG
from tests import test_gpu_train_pipeline as TP
from tests.test_model_autograd_oracle import dropout_plan, make_data, model_config, training_keeps

pytestmark = pytest.mark.gpu

B, S, L = MG.B, MG.S, MG.L
STRIDE2 = {"ksizes": [3, 3], "strides": [2, 1]}
CASES = {
    "stride2_fp32": dict(geom=STRIDE2, HW=(7, 6)),
    "k53_s21_fp32": dict(geom={"ksizes": [5, 3], "strides": [2, 1]}, HW=(5, 4)),
    "k42_fp32_nchw16": dict(geom={"ksizes": [4, 2]}, HW=(3, 5), C=64, layout="nchw16"),
    "stride2_fp32_nchw": dict(geom=STRIDE2, HW=(7, 6), C=64, layout="nchw"),
    "linear_fp32": dict(geom={"linear": True}, HW=(3, 5)),
    "stride2_tc32_bf16x3": dict(geom=STRIDE2, d=128, C=128, HW=(7, 8), prec="tc32", bwd_tc=True, stem_prec="bf16x3"),
}


def _case(name):
    c = dict(MG.DEFAULT, flags="args", **CASES[name])
    c.pop("geom")
    return c, CASES[name]["geom"]


def _stem_oracle(monkeypatch, geom):
    """The fp64 graph's stem with this geometry (the linear stem: no dropout, no activation)."""
    strides, linear = geom.get("strides"), geom.get("linear", False)

    def graph(relu, p, images, keep=1.0, uniforms=None):
        return stem_torch(relu, {k: v for k, v in p.items() if k.startswith("stem/")}, images, keep, uniforms, strides,
                          linear)
    monkeypatch.setattr(MA, "stem_graph", graph)


def _plan(cfg, values, keeps, k, H, W, C, geom, step):
    """dropout_plan with the cell's draws over the knowledge base's grid and the stem's over each layer's input grid."""
    strides = geom.get("strides") or [1] * len(geom.get("ksizes", [3, 3]))
    Ho, Wo = stem_grid(H, W, strides)
    plan = dropout_plan(cfg, L, values, keeps, B, S, k, Ho, Wo, step)
    plan["stem"] = []
    if not geom.get("linear") and keeps["stem"] < 1.0:
        h, w, c = H, W, C
        for i, s in enumerate(strides):
            plan["stem"].append((SITE_STEM + i, step, (k, h, w, c)))
            h, w = stem_grid(h, w, [s])
            c = values["stem/cnnLayercnn_%d/kernels/kernel" % i].shape[3]
    return plan


def _trainer(c, geom):
    from mac_network_b200.dp import DPTrainer
    cfg, cell_dp = model_config(c["flags"], c["d"], L)
    H, W = c["HW"]
    tr = DPTrainer(cfg, L, seed=MG.BASE_SEED, lr=1e-3, dropouts=cell_dp, classifier=(MG.A, MG.HIDDEN), encoder=(MG.V, MG.E),
                   stem=(c["C"], 2, geom), prec=c["prec"], bwd_tc=c["bwd_tc"], stem_prec=c["stem_prec"],
                   enc_prec=c["enc_prec"])
    first = make_data(B, S, MG.V, B, H, W, c["C"], MG.A, seed=60)
    tr.train_step_full("step0", {k: torch.from_numpy(v).cuda() for k, v in first.items()}, global_batch=B)
    data = make_data(B, S, MG.V, B, H, W, c["C"], MG.A, seed=61)
    return cfg, cell_dp, tr, data


@pytest.mark.parametrize("name", list(CASES))
def test_trainer_step_with_the_stem_geometry_against_the_fp64_graph(name, monkeypatch):
    c, geom = _case(name)
    _stem_oracle(monkeypatch, geom)
    cfg, cell_dp, tr, data = _trainer(c, geom)
    keeps = training_keeps(cell_dp)
    H, W = c["HW"]
    dev = MG._device(data, c["layout"])
    values = tr.params.numpy()
    logits, losses = tr.full_forward_backward("t", dev, global_batch=B)
    torch.cuda.synchronize()
    cell = tr._cells["t"][0]
    assert cell.N == int(np.prod(tr.stem.grid(H, W)))
    seed = MG.philox_seed(MG.BASE_SEED, tr.step_id, 0)
    assert cell.seed == seed
    plan = _plan(cfg, values, keeps, B, H, W, c["C"], geom, tr.step_id)
    raw = MG.draws(plan, seed)
    lib_cell = cell.dropout_uniforms()
    assert len(lib_cell) == len(raw["cell"]) and all(np.array_equal(a, b) for a, b in zip(lib_cell, raw["cell"]))
    ref = MA.run(cfg, L, values, MG._oracle_data(data, dev), keeps, MG.kernel_masks(plan, raw, keeps), global_batch=B,
                 device="cuda")
    p = tr.params
    got = {n: tr.bucket[p.offsets[n]:p.offsets[n] + max(1, int(np.prod(p.specs[n][0])))] for n in p.specs}
    errs, null = MG._compare(got, ref, logits, losses)
    MG._report(name, errs, null, MG._kind(c))


def test_mac_model_with_a_stride2_stem_against_the_fp64_graph(monkeypatch):
    """`MACModel.from_trainer` of a stride-2 trainer: parameter and image gradients of `answer_loss(...).backward()`."""
    from mac_network_b200.modules import MACModel, answer_loss
    c, geom = _case("stride2_fp32_nchw")
    _stem_oracle(monkeypatch, geom)
    cfg, cell_dp, tr, data = _trainer(c, geom)
    keeps = training_keeps(cell_dp)
    H, W = c["HW"]
    model = MACModel.from_trainer(tr)
    model.train()
    dev = MG._device(data, "nchw")
    x = dev["images_nchw"].clone().requires_grad_(True)
    values = {n: v.detach().cpu().numpy().astype(np.float64) for n, v in model.named_parameters()}
    step = model.step
    logits, _ = model(dev["questions"], dev["questionLengths"], images_nchw=x)
    answer_loss(logits, dev["answers"]).backward()
    torch.cuda.synchronize()
    plan = _plan(cfg, values, keeps, B, H, W, c["C"], geom, step)
    raw = MG.draws(plan, MG.philox_seed(MG.BASE_SEED, step, 0))
    ref = MA.run(cfg, L, values, MG._oracle_data(data, dict(dev, images_nchw=x.detach())), keeps,
                 MG.kernel_masks(plan, raw, keeps), device="cuda")
    errs, null = MG._compare({n: v.grad for n, v in model.named_parameters()}, ref, logits, None)
    errs["d_images"] = float((x.grad.double() - ref["d_images"]).abs().max()) / float(ref["d_images"].abs().max())
    MG._report("MACModel stride2", errs, null, "fp32")


# ------------------------------------------------------------------------------------------------ the training pipeline
PIPE_GEOMS = {"stride2": dict(stem_kernel_sizes=[3, 3], stem_strides=[2, 1]), "linear": dict(stem_linear=True)}


def _pipe_net(geom, config):
    from mac_network_b200.config import MACConfig
    from mac_network_b200.model import MACnet
    cfg = MACConfig.args("args", netLength=TP.L)
    return MACnet(cfg, TP.L, TP.V, TP.A, wrd_emb_dim=TP.E, image_in_dim=TP.C, classifier_dims=(512,), seed=3, prec="bf16",
                  **TP.HP, **TP.CONFIGS[config], **PIPE_GEOMS[geom])


@pytest.mark.parametrize("config", ["fp32", "tc32"])
@pytest.mark.parametrize("geom", sorted(PIPE_GEOMS))
def test_train_pipeline_equals_run_batch_training_with_the_stem_geometry(geom, config):
    from mac_network_b200.serving import TrainPipeline
    net, twin = _pipe_net(geom, config), _pipe_net(geom, config)
    assert net._stem.grid(TP.HW, TP.HW) == ((4, 4) if geom == "stride2" else (TP.HW, TP.HW))
    batches = TP._batches(4)
    pipe = TrainPipeline(net, (TP.BS, TP.SMAX, TP.HW, TP.HW), depth=2)
    tickets, wants = [], []
    for i, b in enumerate(batches):
        tickets.append(pipe.submit(TP._pinned(b) if i % 2 else b))
        wants.append(TP._twin_step(twin, b))
        if i >= 1:
            TP._check(pipe.result(tickets[i - 1]), wants[i - 1], pipe, i - 1)
    TP._check(pipe.result(tickets[-1]), wants[-1], pipe, len(batches) - 1)
    pipe.drain()
    TP._same_state(net, twin)


# ------------------------------------------------------------------------------------------------ entry points
@pytest.mark.parametrize("geom", [{"linear": True}, {"ksizes": [5, 3], "strides": [2, 1]}])
def test_reference_checkpoint_loads_strictly(geom, tmp_path, monkeypatch):
    """A TensorFlow checkpoint under the reference's names (stem/linearLayer/... or 5x5 and 3x3 kernels) loads into a
    `DPTrainer` and a `MACModel` of that geometry with strict=True, and the model computes what the trainer's values do."""
    from mac_network_b200.checkpoint import load_tf_checkpoint, save_tf_checkpoint
    from mac_network_b200.modules import MACModel
    c, _ = _case("stride2_fp32")
    _stem_oracle(monkeypatch, geom)
    cfg, cell_dp, tr, data = _trainer(c, geom)
    values = {k: v.reshape(tr.params.specs[k][0]) for k, v in tr.params.numpy().items()}
    stem_names = [k for k in values if k.startswith("stem/")]
    assert stem_names == (["stem/linearLayer/weights/weight", "stem/linearLayer/biases/bias"] if geom.get("linear") else
                          ["stem/cnnLayercnn_%d/%s" % (i, n) for i in range(2) for n in ("kernels/kernel", "biases/bias")])
    if not geom.get("linear"):
        assert values["stem/cnnLayercnn_0/kernels/kernel"].shape == (5, 5, c["C"], c["d"])
    prefix = str(tmp_path / "weights.ckpt")
    save_tf_checkpoint(prefix, values)
    back = load_tf_checkpoint(prefix)
    assert set(back) == set(values)
    model = MACModel(cfg, L, MG.V, MG.A, wrd_emb_dim=MG.E, image_in_dim=c["C"], classifier_dims=MG.HIDDEN, seed=1,
                     stem_geometry=geom)
    missing, unexpected = model.load_state_dict({k: torch.from_numpy(v) for k, v in back.items()}, strict=True)
    assert not missing and not unexpected
    model.eval()
    dev = MG._device(data, "nhwc")
    with torch.no_grad():
        logits, _ = model(dev["questions"], dev["questionLengths"], images=dev["images"])
    ref = MA.run(cfg, L, {k: v.astype(np.float64) for k, v in back.items()}, data,
                 {"encoder": (1.0, 1.0), "stem": 1.0, "cell": (1.0, 1.0, 1.0), "output": 1.0}, device="cuda", grad=False)
    assert MG._rowwise(logits, ref["logits"]) < 1e-4


def test_stem_modules_and_preds_follow_the_geometry(tmp_path, monkeypatch):
    from mac_network_b200.checkpoint import write_preds
    from mac_network_b200.modules import ImageStem
    from mac_network_b200.stem import Stem
    x = torch.rand(3, 128, 7, 6, device="cuda")
    for kw in (dict(ksizes=[5, 3], strides=[2, 1]), dict(linear=True)):
        m = ImageStem(128, 128, prec="bf16", **kw).eval()
        st = Stem({k: v.detach() for k, v in m.named_parameters()}, prec="bf16", strides=kw.get("strides"),
                  linear=kw.get("linear", False))
        with torch.no_grad():
            kb = m(images_nchw=x)
        assert kb.shape == (3, int(np.prod(st.grid(7, 6))), 128)
        assert torch.equal(kb, st.forward_nchw(x))
    # runBatch's maps and write_preds on a stride-2 knowledge base
    net = _pipe_net("stride2", "fp32")
    b = TP._batches(1)[0]
    res = net.runBatch(None, {k: b[k] for k in ("questions", "questionLengths", "answers")}, {"images": b["images"]},
                       train=False, getAtt=True)
    assert np.asarray(res["preds"][0]["attentions"]["kb"][0]).shape == (4, 4)
    recs = write_preds(str(tmp_path / "p.json"), net.macCell, image_dims=net._stem.grid(TP.HW, TP.HW))
    assert np.asarray(recs[0]["attentions"]["kb"][0]).shape == (4, 4)
    recs = write_preds(str(tmp_path / "p.json"), net.macCell)
    assert np.asarray(recs[0]["attentions"]["kb"][0]).shape == (16,)
    with pytest.raises(ValueError):
        write_preds(str(tmp_path / "p.json"), net.macCell, image_dims=(8, 8))


def test_model_refusals_at_construction():
    from mac_network_b200.config import MACConfig
    from mac_network_b200.dp import check_model_precisions, stem_geometry
    from mac_network_b200.model import MACnet
    from mac_network_b200._lib import load
    lib = load()
    cfg = MACConfig.args("args", netLength=2)
    launches = lib.mac_b200_launch_count()
    for kw in (dict(stem_strides=[2, 1]), dict(stem_linear=True), dict(stem_kernel_sizes=[1, 1])):
        with pytest.raises(NotImplementedError):
            MACnet(cfg, 2, 10, 5, image_in_dim=128, eval_stem_prec="fp8", **kw)
    with pytest.raises(NotImplementedError):
        check_model_precisions(cfg, (10, 300), (128, 2, {"stem_dim": 200}), "bf16", "fp32")
    for bad in ({"linear": True, "ksizes": [3]}, {"linear": True, "strides": [2]}, {"linear": True, "stem_dim": 256},
                {"kernel": 3}):
        with pytest.raises(ValueError):
            stem_geometry((128, 2, bad))
    torch.cuda.synchronize()
    assert lib.mac_b200_launch_count() == launches
