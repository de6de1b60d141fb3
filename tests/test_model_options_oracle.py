"""The fp64 graph of the whole model (`oracle/model_torch_autograd.run`) with the reference's stem, location, output-unit and
batch-norm options, and its evaluation form (`train=False`: both batch norms on the stored statistics), pinned on the CPU
before tests/test_gpu_model_options_accuracy.py trusts it:

- each unit the options change, taken out of the composed graph, against the reference's own fixtures in tests/golden:
  the knowledge base of the stem geometries and location grids (`stem_geom_*_eval`, `stem_loc_*_eval`); the logits of
  every output layout with batch norm on its stored statistics (`output_*_bn_*_eval`, statistics off 0 and 1) through the
  numpy restatement pinned to those fixtures; the cell's memoryBN on its stored statistics (`p2_memory_bn`);
- the evaluation form differs from the training form where it should, and only there;
- the default keywords are the graph the rest of the suite uses: `train=True` and the shipped options bit for bit the
  defaults, and the option keywords bit for bit the monkeypatched units the older tests install."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import mac_torch_autograd as TA
from oracle import model_torch_autograd as MA
from oracle import output_options as OO
from tests._util import GOLDEN_DIR, load_golden, rebuild, uniforms_of
from tests.test_model_autograd_oracle import (dropout_plan, make_data, model_config, model_values, random_uniforms,
                                              training_keeps)

EVAL = {"encoder": (1.0, 1.0), "stem": 1.0, "cell": (1.0, 1.0, 1.0), "output": 1.0}
V, E, S, L = 11, 8, 6, 2
GEOM_CASES = ["stem_geom_%s_eval" % c for c in ("k1", "k53_s21", "k42", "linear")]
LOC_CASES = ["stem_loc_%s_eval" % c for c in ("L", "PE_d4_b05", "PE_k53_s21")]
OUT_LAYOUTS = {"q0": dict(question=False, mul=False), "q1": dict(question=True, mul=False),
               "qmul": dict(question=True, mul=True)}
OUT_CASES = [(l, w) for l in OUT_LAYOUTS for w in ("h0", "h8", "h8_6")]


def _fixture(case):
    z = np.load(os.path.join(GOLDEN_DIR, case + ".npz"))
    return json.loads(bytes(z["meta_json"]).decode()), {k: z[k] for k in z.files if k != "meta_json"}


def _geometry(meta):
    """The fixture's stem options in the form `run(stem=)` and `DPTrainer(stem=(C, layers, geometry))` take."""
    g = {"strides": meta["strides"], "linear": meta.get("linear", False)}
    if meta.get("location"):
        kind, bias, dim = meta["location"]
        g.update(location=kind, location_bias=bias, location_dim=dim)
    return g


def _stem_params(meta):
    from mac_network_b200.stem import init_stem_params, stem_specs
    _, _, _, cin, cout = meta["shape"]
    loc = tuple(meta["location"]) if meta.get("location") else None
    specs = stem_specs(cin, cout, meta["layers"], meta["ksize"], ksizes=meta["ksizes"], linear=meta.get("linear", False),
                       location=loc)
    return init_stem_params(specs, seed=meta["param_seed"], dtype=np.float64)


@pytest.mark.parametrize("case", GEOM_CASES + LOC_CASES)
def test_stem_of_the_composed_graph_matches_the_reference_fixture(case):
    """The stem's fixture parameters and images in a whole model of the fixture's width: the knowledge base the composed
    graph's cell reads is the reference's, and the stem's output grid is what the cell attends over."""
    meta, g = _fixture(case)
    B, H, W, cin, d = meta["shape"]
    cfg, _ = model_config("args", d, L)
    values = {k: v for k, v in model_values(cfg, L, V, E, cin, 7, [9], seed=3).items() if not k.startswith("stem/")}
    values.update(_stem_params(meta))
    data = make_data(B, S, V, B, H, W, cin, 7, seed=4)
    data["images"] = g["images"]
    trace = []
    out = MA.run(cfg, L, values, data, EVAL, grad=False, trace=trace, stem=_geometry(meta), train=False)
    kb = out["knowledgeBase"].numpy()
    assert kb.shape == g["kb"].shape
    assert np.max(np.abs(kb - g["kb"])) < 1e-12
    assert trace[0]["att_kb"].shape == (B, g["kb"].shape[1])


def _output_fixture(layout, widths):
    from mac_network_b200.output_unit import init_output_params, output_specs
    meta, z = _fixture("output_%s_bn_%s_eval" % (layout, widths))
    specs = output_specs(meta["d"], meta["d"], meta["hidden"], meta["A"], bn=True, **OUT_LAYOUTS[layout])
    return meta, z, init_output_params(specs, seed=meta["param_seed"], dtype=np.float64)


@pytest.mark.parametrize("layout,widths", OUT_CASES)
def test_output_unit_of_the_composed_graph_on_stored_statistics(layout, widths):
    """The layout's fixture parameters (stored statistics off 0 and 1) as the output unit of a whole model: the logits of
    `run(train=False)` are the numpy restatement's on the memory and question vectors the composed graph computed, and that
    restatement reproduces the reference's fixture; `train=True` normalises by the batch instead and moves them."""
    meta, z, params = _output_fixture(layout, widths)
    opts = dict(OUT_LAYOUTS[layout], bn=True)
    stats = {k: v for k, v in params.items() if "/moving_" in k}
    assert all(np.abs(v - (1.0 if k.endswith("variance") else 0.0)).max() > 1e-2 for k, v in stats.items())
    fixed = OO.output_forward(meta["relu"], params, z["memory"], z["vecQuestions"], z["answers"], train=False, **opts)
    assert np.max(np.abs(fixed["logits"] - z["logits"])) <= 1e-12 * max(1.0, np.abs(z["logits"]).max())
    d, B = meta["d"], meta["B"]
    cfg, _ = model_config("args", d, L)
    assert cfg.relu == meta["relu"]
    base = model_values(cfg, L, V, E, 6, meta["A"], meta["hidden"], seed=5)
    values = {k: v for k, v in base.items() if not k.startswith(("outputUnit/", "classifier/"))}
    values.update(params)
    data = make_data(B, S, V, B, 3, 2, 6, meta["A"], seed=6)
    trace = []
    out = MA.run(cfg, L, values, data, EVAL, grad=False, trace=trace, output=opts, train=False)
    want = OO.output_forward(meta["relu"], params, trace[-1]["memory"], out["vecQuestions"].numpy(), data["answers"],
                             train=False, **opts)
    for k in ("logits", "losses"):
        assert np.max(np.abs(out[k].numpy() - want[k])) <= 1e-12 * max(1.0, np.abs(want[k]).max()), k
    moving = {}
    batch = MA.run(cfg, L, values, data, EVAL, grad=False, output=opts, train=True, moving=moving)
    assert np.abs(batch["logits"].numpy() - want["logits"]).max() > 1e-3
    assert set(moving) == set(stats) and all(not np.array_equal(moving[k].numpy(), stats[k]) for k in stats)


def test_cell_memory_bn_on_stored_statistics():
    """The `p2_memory_bn` fixture (the reference's cell at evaluation, memoryBN on the stored statistics): the cell graph
    with train=False reproduces it; in the composed graph `train=False` reaches the cell, whose memory is then the cell
    graph's on stored statistics (moved off 0 and 1 here) over the inputs the composed graph computed, and not the
    batch-statistics one."""
    meta, gold = load_golden("p2_memory_bn")
    assert not meta["train"]
    cfg, inputs, params = rebuild(meta, np.float64)
    dp = meta["dropouts"]
    _, m, _ = TA.run(cfg, params, inputs, meta["shape"]["L"], (dp["memory"], dp["read"], dp["write"]),
                     uniforms_of(meta, gold), train=False)
    assert np.max(np.abs(m - gold["final_memory"])) < 1e-11
    d = meta["shape"]["d"]
    cfg, _ = model_config("p2_memory_bn", d, L)
    assert cfg.memoryBN
    values = model_values(cfg, L, V, E, 6, 7, [9], seed=7)
    rng = np.random.RandomState(8)
    for k in [k for k in values if "/BatchNorm/moving_" in k]:
        values[k] = (0.3 * rng.standard_normal(values[k].shape) if k.endswith("mean")
                     else np.exp(0.5 * rng.standard_normal(values[k].shape)))
    data = make_data(5, S, V, 5, 3, 2, 6, 7, seed=9)
    trace = []
    out = MA.run(cfg, L, values, data, EVAL, grad=False, trace=trace, train=False)
    p = {k: torch.as_tensor(v, dtype=torch.float64) for k, v in values.items()}
    x = {k: out[k] for k in ("vecQuestions", "questionWords", "questionCntxWords", "knowledgeBase")}
    ln = torch.as_tensor(data["questionLengths"]).long()
    for train in (False, True):
        _, memory = TA.graph(cfg, p, x, ln, L, train=train)
        same = np.array_equal(memory.numpy(), trace[-1]["memory"])
        assert same == (not train), train


def _training_case(flags="args", seed=20):
    cfg, cell_dp = model_config(flags, 16, L)
    values = model_values(cfg, L, V, E, 6, 7, [9], seed=seed)
    keeps = training_keeps(cell_dp)
    data = make_data(5, S, V, 5, 3, 2, 6, 7, seed=seed + 1)
    us = random_uniforms(dropout_plan(cfg, L, values, keeps, 5, S, 5, 3, 2, step=0), seed=seed + 2)
    return cfg, values, keeps, data, us


def _same(a, b):
    assert all(torch.equal(a[k], b[k]) for k in ("logits", "losses", "loss", "d_images"))
    assert set(a["grads"]) == set(b["grads"]) and all(torch.equal(a["grads"][k], b["grads"][k]) for k in a["grads"])


def test_defaults_are_the_training_graph_bit_for_bit():
    """`train=True` is the default, and the training graph of the shipped model is unchanged by the new keywords: the
    defaults, `train=True` and the memoryBN flag set's training cell give the same bits."""
    for flags in ("args", "p2_memory_bn_train"):
        cfg, values, keeps, data, us = _training_case(flags)
        _same(MA.run(cfg, L, values, data, keeps, us), MA.run(cfg, L, values, data, keeps, us, train=True))


@pytest.mark.parametrize("geometry", [dict(strides=[2, 1]), dict(linear=True), dict(location="PE", location_bias=0.5,
                                                                                    location_dim=4)],
                         ids=["stride2", "linear", "loc_PE"])
def test_option_keywords_equal_the_monkeypatched_units(geometry, monkeypatch):
    """With training dropouts and gradients, `run(stem=, output=)` computes bit for bit what the older tests get by
    replacing `stem_graph` and `output_graph` (tests/test_gpu_stem_geometry_training.py, tests/test_gpu_stem_location.py,
    tests/test_gpu_output_options.py), the output unit's stored statistics included."""
    from oracle.stem_geometry import stem_torch
    from oracle.stem_location import stem_loc_torch
    from mac_network_b200.output_unit import init_output_params, output_specs
    from mac_network_b200.stem import init_stem_params, location_channels, stem_grid, stem_specs
    cfg, values, keeps, data, _ = _training_case()
    opts = dict(question=True, mul=True, bn=True)
    loc = geometry.get("location")
    loc = None if loc is None else (loc, geometry["location_bias"], geometry["location_dim"])
    C, d = 6, cfg.memDim
    specs = stem_specs(C, d, linear=geometry.get("linear", False), location=loc)
    values = {k: v for k, v in values.items() if not k.startswith(("stem/", "outputUnit/", "classifier/"))}
    values.update(init_stem_params(specs, seed=21, dtype=np.float64))
    values.update(init_output_params(output_specs(d, d, [9], 7, bn=True, question=True, mul=True), seed=22,
                                     dtype=np.float64))
    B, H, W = 5, 5, 4
    data = make_data(B, S, V, B, H, W, C, 7, seed=23)
    strides = geometry.get("strides") or [1, 1]
    plan = dropout_plan(cfg, L, values, keeps, B, S, B, *stem_grid(H, W, strides), step=0)
    # the reference's stem draws: each layer's whole input, layer 0's with the location channels
    plan["stem"] = [] if geometry.get("linear") else [(0, 0, (B, H, W, C + location_channels(loc))),
                                                      (0, 0, (B,) + tuple(stem_grid(H, W, strides[:1])) + (d,))]
    us = random_uniforms(plan, seed=25)
    moving_kw = {}
    got = MA.run(cfg, L, values, data, keeps, us, stem=geometry, output=opts, moving=moving_kw)

    def stem(relu, p, images, keep=1.0, uniforms=None):
        ps = {k: v for k, v in p.items() if k.startswith("stem/")}
        if loc is not None:
            return stem_loc_torch(relu, ps, images, loc, keep, uniforms, geometry.get("strides"))
        return stem_torch(relu, ps, images, keep, uniforms, geometry.get("strides"), geometry.get("linear", False))
    moving_mp = {}
    monkeypatch.setattr(MA, "stem_graph", stem)
    monkeypatch.setattr(MA, "output_graph", OO.output_graph_for(opts, cfg.bnDecay, moving_mp))
    _same(got, MA.run(cfg, L, values, data, keeps, us))
    assert set(moving_kw) == set(moving_mp) and all(torch.equal(moving_kw[k], moving_mp[k]) for k in moving_kw)
