"""The location-aware stem (--locationAware, --locationType L / PE, --locationBias, --locationDim) without a GPU: the fp64
oracle and the product's grid against fixtures from the reference's own `MACnet.stem` on the TF1 shim, `stem_specs` against
the variables the reference created, the call sequence of `Stem` in every precision against the dry-run library, the
Python-level refusals, and the new entry points' status codes (each returned before any CUDA call)."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from oracle.stem_location import grid_torch, stem_loc_forward
from mac_network_b200 import _lib as L_
from mac_network_b200.stem import (SITE_LOCATION, SITE_STEM, init_stem_params, location_channels, location_grid,
                                   location_width, stem_grid, stem_specs)
from tests import _mocklib
from tests._util import GOLDEN_DIR
from tests.test_stem_tc_training import _cpu_params, _fake_ptr, _recorder

CASES = ["stem_loc_%s_%s" % (c, m) for c in ("L", "PE_d4_b05", "PE_k53_s21") for m in ("eval", "train")]
INVALID, ALIGN, UNSUPPORTED = -1, -2, -3
ACT_ELU, ACT_NON = L_.ACT["ELU"], L_.ACT["NON"]


def load_case(case):
    z = np.load(os.path.join(GOLDEN_DIR, case + ".npz"))
    meta = json.loads(bytes(z["meta_json"]).decode())
    return meta, {k: z[k] for k in z.files if k != "meta_json"}


def case_specs(meta):
    _, _, _, cin, cout = meta["shape"]
    return stem_specs(cin, cout, meta["layers"], meta["ksize"], ksizes=meta["ksizes"], location=tuple(meta["location"]))


@pytest.mark.parametrize("case", CASES)
def test_stem_specs_match_reference_variables(case):
    meta, _ = load_case(case)
    assert {k: list(v[0]) for k, v in case_specs(meta).items()} == meta["variables"]
    assert location_channels(tuple(meta["location"])) == meta["l"]


@pytest.mark.parametrize("case", CASES)
def test_grid_matches_reference(case):
    meta, g = load_case(case)
    _, H, W, _, _ = meta["shape"]
    loc = tuple(meta["location"])
    assert g["grid"].shape == (H, W, meta["l"])
    assert np.max(np.abs(location_grid(loc, H, W) - g["grid"])) < 1e-12
    assert np.max(np.abs(grid_torch(*loc, H, W).numpy() - g["grid"])) < 1e-12


@pytest.mark.parametrize("case", CASES)
def test_location_oracle_matches_reference_fixture(case):
    meta, g = load_case(case)
    B, H, W, cin, cout = meta["shape"]
    params = init_stem_params(case_specs(meta), seed=meta["param_seed"], dtype=np.float64)
    us = [g["uniform_%03d" % i] for i in range(meta["n_uniform"])]
    if meta["train"]:                      # the dropout covers layer 0's whole input, location channels included
        assert us[0].shape == (B, H, W, cin + meta["l"])
    kb = stem_loc_forward(meta["relu"], params, g["images"], tuple(meta["location"]), keep=meta["keep"], uniforms=us,
                          strides=meta["strides"])
    Ho, Wo = stem_grid(H, W, meta["strides"])
    assert g["kb"].shape == (B, Ho * Wo, cout) == kb.shape
    assert np.max(np.abs(kb - g["kb"])) < 1e-12


def test_grid_axis_order_and_single_point():
    """Channel 0 follows the width, channel 1 the height; TF's linspace of one point is [start]."""
    g = location_grid(("L", 2.0, 32), 3, 5)
    assert np.allclose(g[0, :, 0], np.linspace(-2, 2, 5)) and np.allclose(g[:, 0, 1], np.linspace(-2, 2, 3))
    assert np.all(location_grid(("L", 1.5, 32), 1, 1) == -1.5)
    assert location_grid("PE", 2, 3).shape == (2, 3, 128)
    assert location_width(2, 3) == 128 and location_width(128, 3) == 1152 and location_width(12, 5) == 384


# ------------------------------------------------------------------------------------------------ the stem's calls
def _stem(prec, location, cin=128, cout=256, ksizes=None, strides=None):
    from mac_network_b200.stem import Stem
    p = _cpu_params(init_stem_params(stem_specs(cin, cout, ksizes=ksizes, location=location), seed=1))
    return Stem(p, relu="ELU", prec=prec, seed=1, strides=strides, location=location), p


@pytest.mark.parametrize("location,l", [("L", 2), (("PE", 0.5, 32), 128)])
@pytest.mark.parametrize("prec", ["fp32", "bf16", "bf16x3"])
def test_forward_and_backward_calls(monkeypatch, prec, location, l):
    rec = _recorder(monkeypatch)
    st, p = _stem(prec, location)
    assert st.in_dim == 128 and st.nloc == l
    Kq = location_width(l, 3)
    kb = st.forward(torch.zeros(2, 5, 7, 128), keep=0.82, step=3, save_for_backward=True)
    assert kb.shape == (2, 35, 256)
    (loc,) = rec.args_of("mac_loc_cols")
    form = {"fp32": 0, "bf16": 1, "bf16x3": 2}[prec]
    assert loc[2] == form and loc[3] == pytest.approx(0.82) and loc[5:7] == (SITE_LOCATION, 3)
    assert loc[7:13] == (2, 5, 7, l, 3, 1)
    names = [n for n, _ in rec.log]
    if prec == "fp32":
        (l0, l1) = rec.args_of("mac_linear_fwd")
        assert l0[3] == 2 and list(l0[1]) == [9 * 128, Kq] and l1[3] == 1
        assert not rec.args_of("mac_linear_tc_fwd_acc")
    else:
        acc = "mac_linear_tc_fwd_acc" if prec == "bf16" else "mac_linear_tc32_fwd_acc"
        gemm = "mac_linear_tc_fwd" if prec == "bf16" else "mac_linear_tc32_fwd"
        z, l1 = rec.args_of(gemm)
        (a,) = rec.args_of(acc)
        assert names.index("mac_loc_cols") < names.index(gemm) < names.index(acc)
        assert z[3] == ACT_NON and (z[-4:-1] == (70, Kq, 256))
        assert a[2] == ACT_ELU and a[-4:-1] == (70, 9 * 128, 256)
    grads = {k: torch.zeros_like(v) for k, v in p.items()}
    rec.log.clear()
    assert st.backward(torch.zeros_like(kb), grads, need_d_images=True).shape == (2, 5, 7, 128)
    if prec == "fp32":
        assert len(rec.args_of("mac_loc_cols")) == 1 and len(rec.args_of("mac_linear_bwd")) == 2
        l0 = rec.args_of("mac_linear_bwd")[1]
        assert l0[3] == 2 and list(l0[1]) == [9 * 128, Kq]
    else:
        name = "mac_conv_bwd_loc_tc" if prec == "bf16" else "mac_conv_bwd_loc_tc32"
        (b,) = rec.args_of(name)
        assert b[10:12] == (l, SITE_LOCATION) and b[7] == SITE_STEM and b[-8:-1] == (2, 5, 7, 128, 256, 3, 1)
        assert rec.args_of(name + "_workspace_bytes") == [(2, 5, 7, 128, 256, l, 3, 1, 1)]
        assert len(rec.args_of(name.replace("_loc", "").replace("conv_", "conv3x3_"))) == 1          # layer 1 only


def test_weight_split_and_gradient_scatter(monkeypatch):
    """W_img and W_loc are the interleaved kernel's rows (W_loc padded with zero rows to Kq), and the two gradients go back
    to the rows they came from."""
    _mocklib.install(monkeypatch)
    st, p = _stem("fp32", "L", ksizes=[5, 3], strides=[2, 1])
    K = p["stem/cnnLayercnn_0/kernels/kernel"]
    cat, W_img, W_loc = st._loc_weights()
    assert W_img.shape == (25 * 128, 256) and W_loc.shape == (128, 256)
    assert torch.equal(W_img.view(25, 128, 256), K.view(25, 130, 256)[:, :128])
    assert torch.equal(W_loc[:50].view(25, 2, 256), K.view(25, 130, 256)[:, 128:]) and not W_loc[50:].any()
    grads = {k: torch.zeros_like(v) for k, v in p.items()}
    st._loc_scatter(grads, W_img, W_loc)
    assert torch.equal(grads["stem/cnnLayercnn_0/kernels/kernel"], K)


def test_refusals():
    from mac_network_b200 import dp
    from mac_network_b200.stem import Stem, location_spec
    for bad in (("X", 1.0, 32), ("PE", 1.0, 0), ("PE", float("nan"), 4), ("L", float("inf"), 32), ("PE", 1.0, 2.5)):
        with pytest.raises(ValueError):
            location_spec(bad)
    with pytest.raises(ValueError, match="linear"):
        stem_specs(128, 128, linear=True, location="L")
    lin = _cpu_params(init_stem_params(stem_specs(128, 128, linear=True), seed=1))
    with pytest.raises(ValueError, match="linear"):
        Stem(lin, linear=True, location="L")
    conv = _cpu_params(init_stem_params(stem_specs(128, 128, location="L"), seed=1))
    with pytest.raises(NotImplementedError, match="fp8"):
        Stem(conv, prec="fp8", location="L")
    with pytest.raises(ValueError, match="linear"):
        dp.stem_geometry((128, 1, {"linear": True, "location": "L"}))
    with pytest.raises(ValueError):
        dp.stem_geometry((128, 2, {"location": "PE", "location_dim": 0}))
    with pytest.raises(ValueError):
        dp.stem_geometry((128, 2, {"location": "Q"}))
    assert dp.stem_location(dp.stem_geometry((128, 2, {"location": "PE", "location_bias": 0.5, "location_dim": 4}))) == \
        ("PE", 0.5, 4)


def test_macnet_refuses_fp8_stem_with_location(monkeypatch):
    from tests.test_stem_fp8_host import _macnet
    with pytest.raises(NotImplementedError, match="location"):
        _macnet(monkeypatch, 128, "bf16", eval_stem_prec="fp8", stem_location="L")


def test_trainer_and_model_carry_location(monkeypatch):
    from tests.test_stem_fp8_host import _macnet
    _, net, _, _ = _macnet(monkeypatch, 128, "bf16", stem_location="PE", stem_location_bias=0.5, stem_location_dim=4)
    assert net.trainer.stem.location == ("PE", 0.5, 4) and net._stem.location == ("PE", 0.5, 4)
    assert net.trainer.params.t["stem/cnnLayercnn_0/kernels/kernel"].shape == (3, 3, 128 + 16, 128)
    assert net._stem.in_dim == 128


# ------------------------------------------------------------------------------------------------ entry points
def test_entry_point_status_codes():
    lib = L_.load()
    buf = (ctypes.c_float * 4096)()
    p = _fake_ptr(buf)
    assert lib.mac_loc_cols_width(2, 3) == 128 and lib.mac_loc_cols_width(128, 3) == 1152 and lib.mac_loc_cols_width(0, 3) == 0

    def cols(grid=p, out=p, form=0, keep=0.82, B=2, H=5, W=4, l=2, k=3, s=1):
        return lib.mac_loc_cols(grid, out, form, keep, 7, SITE_LOCATION, 1, B, H, W, l, k, s, None)
    assert cols(grid=None) == INVALID and cols(out=None) == INVALID
    assert cols(l=0) == INVALID and cols(k=0) == INVALID and cols(s=0) == INVALID and cols(B=0) == INVALID
    assert cols(keep=0.0) == INVALID and cols(keep=1.5) == INVALID
    assert cols(form=3) == UNSUPPORTED and cols(k=17) == UNSUPPORTED
    assert cols(out=p + 4) == ALIGN and cols(grid=p + 8) == ALIGN
    assert lib.mac_loc_cols_t(p, p, 2, 1.0, 7, 50, 1, 2, 5, 4, 2, 3, 1, None) == UNSUPPORTED
    assert lib.mac_loc_cols_t(p, None, 0, 1.0, 7, 50, 1, 2, 5, 4, 2, 3, 1, None) == INVALID
    assert lib.mac_loc_cols_t(p, p + 4, 0, 1.0, 7, 50, 1, 2, 5, 4, 2, 3, 1, None) == ALIGN
    for acc in (lib.mac_linear_tc_fwd_acc, lib.mac_linear_tc32_fwd_acc):
        assert acc(None, p, ACT_ELU, p, 64, 128, 128, None) == INVALID
        assert acc(p, p, ACT_ELU, p, 0, 128, 128, None) == INVALID
        assert acc(p, p, ACT_ELU, p, 64, 96, 128, None) == UNSUPPORTED
        assert acc(p, p, ACT_ELU, p, 64, 128, 96, None) == UNSUPPORTED
        assert acc(p, p, L_.ACT["TANH"], p, 64, 128, 128, None) == UNSUPPORTED
        assert acc(p, p, ACT_ELU, p + 4, 64, 128, 128, None) == ALIGN
    for name in ("mac_conv_bwd_loc_tc", "mac_conv_bwd_loc_tc32"):
        fn = getattr(lib, name)

        def bwd(grid=p, l=2, dwloc=p, C=128, Cout=128, keep=0.82, ws=1 << 40):
            return fn(p, p, p, p, ACT_ELU, keep, 7, SITE_STEM, 1, grid, l, SITE_LOCATION, p, dwloc, p, p, p, ws, 2, 5, 4,
                      C, Cout, 3, 1, None)
        assert bwd(grid=None) == INVALID and bwd(dwloc=None) == INVALID and bwd(l=0) == INVALID
        assert bwd(keep=0.0) == INVALID
        assert bwd(C=64) == UNSUPPORTED and bwd(Cout=96) == UNSUPPORTED
        assert bwd(grid=p + 4) == ALIGN and bwd(dwloc=p + 8) == ALIGN
        assert bwd(ws=16) == -4                                                # MAC_ERR_WORKSPACE
        q = getattr(lib, name + "_workspace_bytes")
        assert q(2, 5, 4, 128, 128, 0, 3, 1, 1) == 0
        plain = getattr(lib, name.replace("_loc", "") + "_workspace_bytes")(2, 5, 4, 128, 128, 3, 1, 1)
        assert q(2, 5, 4, 128, 128, 2, 3, 1, 1) > plain > 0
