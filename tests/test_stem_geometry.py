"""The stem's geometry flags (--stemKernelSize(s), --stemStrideSizes, --stemLinear): the fp64 oracle against fixtures from the
reference's own `MACnet.stem` on the TF1 shim, and `stem_specs` against the variables the reference created (CPU)."""
import json
import os

import numpy as np
import pytest

from oracle.stem_geometry import same_pads, stem_forward
from mac_network_b200.stem import init_stem_params, stem_grid, stem_specs
from tests._util import GOLDEN_DIR

CASES = ["stem_geom_%s_%s" % (c, m) for c in ("k1", "k53_s21", "k42", "linear") for m in ("eval", "train")]


def load_case(case):
    z = np.load(os.path.join(GOLDEN_DIR, case + ".npz"))
    meta = json.loads(bytes(z["meta_json"]).decode())
    return meta, {k: z[k] for k in z.files if k != "meta_json"}


def case_specs(meta):
    _, _, _, cin, cout = meta["shape"]
    return stem_specs(cin, cout, meta["layers"], meta["ksize"], ksizes=meta["ksizes"], linear=meta["linear"])


@pytest.mark.parametrize("case", CASES)
def test_stem_specs_match_reference_variables(case):
    meta, _ = load_case(case)
    assert {k: list(v[0]) for k, v in case_specs(meta).items()} == meta["variables"]


@pytest.mark.parametrize("case", CASES)
def test_geometry_oracle_matches_reference_fixture(case):
    meta, g = load_case(case)
    B, H, W, _, cout = meta["shape"]
    params = init_stem_params(case_specs(meta), seed=meta["param_seed"], dtype=np.float64)
    us = [g["uniform_%03d" % i] for i in range(meta["n_uniform"])]
    kb = stem_forward(meta["relu"], params, g["images"], keep=meta["keep"], uniforms=us, strides=meta["strides"],
                      linear=meta["linear"])
    Ho, Wo = stem_grid(H, W, meta["strides"])
    assert g["kb"].shape == (B, Ho * Wo, cout) == kb.shape
    assert np.max(np.abs(kb - g["kb"])) < 1e-12


def test_training_fixtures_draw_one_mask_per_layer_input():
    """The linear stem has no dropout (ops.linear, dropout = 1.0); a CNN stem draws each layer's input once."""
    for case in CASES:
        meta, g = load_case(case)
        if not meta["train"] or meta["linear"]:
            assert meta["n_uniform"] == 0, case
            continue
        B, H, W, cin, cout = meta["shape"]
        grids = [(H, W)]
        for s in meta["strides"][:-1]:
            grids.append(stem_grid(*grids[-1], [s]))
        want = [(B, h, w, c) for (h, w), c in zip(grids, [cin] + [cout] * (meta["layers"] - 1))]
        assert [g["uniform_%03d" % i].shape for i in range(meta["n_uniform"])] == want, case


@pytest.mark.parametrize("n,k,s,want", [(14, 3, 1, (1, 1)), (14, 3, 2, (0, 1)), (5, 5, 2, (2, 2)), (4, 5, 2, (1, 2)),
                                        (7, 4, 1, (1, 2)), (7, 1, 2, (0, 0)), (14, 1, 1, (0, 0)), (3, 2, 1, (0, 1))])
def test_same_padding(n, k, s, want):
    """TF SAME: pad_total = max((ceil(n / s) - 1) s + k - n, 0), the odd row after."""
    assert same_pads(n, k, s) == want
