"""CPU checks for the stem's general and location-aware tensor-core backward (tests/test_gpu_conv_bwd.py).

1. With that file's own fp64 reference code and its bars: the exact answer, accumulated in fp32 as the kernels do, passes,
   and each of the mistakes a general patch pass or a padded GEMM could make is rejected -- one tap dropped from col2im, the
   odd SAME padding row of an even kernel on the top / left instead of the bottom / right, one location tap missing from
   dW_loc, the bias gradient added twice, the last partial 64-row block dropped from dKernel -- in both precisions.
2. The six conv backward entry points refuse, before any launch, a dZ grid of more than 65 535 64-row blocks (M above
   4 194 240), and their workspace queries return 0 for it (fake pointers: nothing is dereferenced)."""
import ctypes

import numpy as np
import pytest
import torch

from mac_network_b200 import _lib as L_
from oracle.stem_geometry import same_pads
from tests.test_gpu_conv_bwd import TOL, col2im, conv_bwd_reference, grid_out, patches, unread_pixels
from tests.test_gpu_wgmma import bf16_round, excess
from tests.test_stem_tc_training import _fake_ptr

UNSUPPORTED = -3


def _case(shape, act, keep, l=0, seed=1):
    """fp32 inputs, keep-masks (random draws) and non-zero starting gradients on the CPU"""
    B, H, W, C, Cout, k, s = shape
    M = B * int(np.prod(grid_out(H, W, s)))
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, H, W, C, generator=g)
    kernel = torch.randn(k, k, C, Cout, generator=g) * (2.0 / (k * k * (C + Cout))) ** 0.5
    z = torch.randn(M, Cout, generator=g)
    y = {"ELU": torch.nn.functional.elu(z), "RELU_STD": torch.relu(z), "NON": z}[act]
    dy = torch.randn(M, Cout, generator=g)
    mask = torch.rand(B, H, W, C, generator=g) < keep if keep < 1 else None
    c = dict(x=x, kernel=kernel, y=y, dy=dy, mask=mask, pre_k=torch.randn(k * k * C, Cout, generator=g) * 0.1,
             pre_b=torch.randn(Cout, generator=g))
    if l:
        from mac_network_b200.stem import location_grid, location_width
        c["grid"] = torch.from_numpy(np.ascontiguousarray(location_grid(("PE", 0.5, l // 4) if l > 2 else "L", H, W),
                                                          dtype=np.float32))
        c["qmask"] = torch.rand(B, H, W, l, generator=g) < keep
        c["Kq"] = location_width(l, k)
        c["pre_q"] = torch.randn(c["Kq"], Cout, generator=g) * 0.1
    return c


def _operands(c, keep, k, s, split, pads=same_pads):
    """What the kernels multiply: dZ and the patch matrices, bf16-rounded or fp32, as fp32 tensors"""
    from tests.test_gpu_conv_bwd import act_grad
    act = c["act"]
    scale = np.float32(1.0) / np.float32(keep)
    rnd = (lambda t: t) if split else (lambda t: bf16_round(t).float())
    dz32 = c["dy"] * act_grad(act, c["y"])
    m = 1.0 if c["mask"] is None else c["mask"].float()
    cols = patches(rnd(c["x"] * scale) * m, k, s, pads)
    out = dict(dz32=dz32, dz=rnd(dz32), cols=cols, kr=rnd(c["kernel"].reshape(-1, c["kernel"].shape[-1])), f=m * scale)
    if "grid" in c:
        B, H, W, _ = c["x"].shape
        l = c["grid"].shape[-1]
        q = patches(rnd(c["grid"].expand(B, H, W, l) * scale) * c["qmask"].float(), k, s, pads)
        out["q"] = torch.nn.functional.pad(q, (0, c["Kq"] - q.shape[1]))
    return out


def _fp32(o, c, shape, pads=same_pads):
    """the kernels' result computed in fp32: dkernel, dbias, dx and dW_loc"""
    B, H, W, C, Cout, k, s = shape
    r = {"dkernel": c["pre_k"] + o["cols"].t() @ o["dz"], "dbias": c["pre_b"] + o["dz32"].sum(0),
         "dx": col2im(o["dz"] @ o["kr"].t(), (B, H, W, C), k, s, pads) * o["f"]}
    if "q" in o:
        r["dwloc"] = c["pre_q"] + o["q"].t() @ o["dz"]
    return r


def _fractions(got, ref, c, split, l=0, k=0):
    """each output's excess over the reference as a fraction of its bar"""
    out = {}
    for name, (r, a) in ref.items():
        pre = {"dkernel": c["pre_k"], "dbias": c["pre_b"], "dwloc": c.get("pre_q")}.get(name)
        if pre is not None:
            r, a = r + pre.double(), a + pre.double().abs()
        g = got[name]
        if name == "dwloc":
            n = k * k * l
            g, r, a = g[:n], r[:n], a[:n]
        out[name] = excess(g, r, a) / TOL[split]["dkernel" if name == "dwloc" else name]
    return out


def _reference(c, shape, keep, split, with_dx=True):
    B, H, W, C, Cout, k, s = shape
    return conv_bwd_reference(c["x"], c["y"], c["dy"], c["kernel"], c["act"], keep, c["mask"], k, s, split, with_dx,
                              grid=c.get("grid"), qmask=c.get("qmask"), Kq=c.get("Kq", 0))


def _setup(shape, act, keep, split, l=0):
    c = _case(shape, act, keep, l)
    c["act"] = act
    k, s = shape[5], shape[6]
    o = _operands(c, keep, k, s, split)
    ref = _reference(c, shape, keep, split)
    exact = _fractions(_fp32(o, c, shape), ref, c, split, l, k)
    print("exact answer, fraction of each bar:", {n: "%.3f" % v for n, v in exact.items()})
    assert all(v <= 1.0 for v in exact.values()), exact
    return c, o, ref


@pytest.mark.parametrize("split", [False, True])
def test_a_tap_dropped_from_col2im_is_rejected(split):
    shape = (2, 7, 6, 128, 128, 5, 2)
    B, H, W, C, Cout, k, s = shape
    c, o, ref = _setup(shape, "RELU_STD", 0.82, split)
    dcols = o["dz"] @ o["kr"].t()
    worst = []
    for tap in range(k * k):
        d = dcols.clone()
        d[:, tap * C:(tap + 1) * C] = 0
        bad = col2im(d, (B, H, W, C), k, s) * o["f"]
        worst.append(excess(bad, *ref["dx"]) / TOL[split]["dx"])
    print("dx with one col2im tap dropped: smallest fraction of the bar %.0f" % min(worst))
    assert min(worst) > 100


@pytest.mark.parametrize("split", [False, True])
def test_the_odd_padding_row_on_the_wrong_side_is_rejected(split):
    """k = 4 on 5 x 3: pad_total 3 on both axes, (1, 2) in TF's SAME; (2, 1) must fail dkernel and dx"""
    shape = (3, 5, 3, 128, 256, 4, 1)
    k, s = 4, 1
    assert same_pads(5, k, s) == (1, 2) and same_pads(3, k, s) == (1, 2)
    c, _, ref = _setup(shape, "ELU", 0.82, split)
    flipped = lambda n, k_, s_: same_pads(n, k_, s_)[::-1]
    bad = _fractions(_fp32(_operands(c, 0.82, k, s, split, flipped), c, shape, pads=flipped), ref, c, split)
    print("odd padding row on the top / left:", {n: "%.0f" % v for n, v in bad.items()})
    assert bad["dkernel"] > 100 and bad["dx"] > 100


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("l,shape", [(2, (1, 7, 5, 128, 128, 3, 2)), (12, (2, 7, 6, 128, 128, 5, 2))])
def test_a_missing_location_tap_is_rejected(l, shape, split):
    k = shape[5]
    c, o, ref = _setup(shape, "ELU", 0.82, split, l=l)
    worst = []
    for tap in range(k * k):
        q = o["q"].clone()
        q[:, tap * l:(tap + 1) * l] = 0
        bad = dict(_fp32(o, c, shape), dwloc=c["pre_q"] + q.t() @ o["dz"])
        worst.append(_fractions(bad, {"dwloc": ref["dwloc"]}, c, split, l, k)["dwloc"])
    print("dW_loc with one location tap missing: smallest fraction of the bar %.0f" % min(worst))
    assert min(worst) > 100


@pytest.mark.parametrize("split", [False, True])
def test_the_bias_gradient_added_twice_is_rejected(split):
    """the location path's schedule adds dbias once; twice is rejected"""
    shape = (1, 7, 5, 128, 128, 3, 2)
    c, o, ref = _setup(shape, "ELU", 0.82, split, l=2)
    bad = _fractions({"dbias": c["pre_b"] + 2 * o["dz32"].sum(0)}, {"dbias": ref["dbias"]}, c, split)["dbias"]
    print("dbias added twice: %.0f of the bar" % bad)
    assert bad > 100


@pytest.mark.parametrize("split", [False, True])
def test_a_dropped_partial_row_block_is_rejected(split):
    """M = 98: rows 64..97 are the partly filled second 64-row block of the weight gradient's contraction"""
    shape = (2, 14, 14, 128, 128, 3, 2)
    c, o, ref = _setup(shape, "RELU_STD", 0.82, split)
    assert o["dz"].shape[0] == 98
    cols = o["cols"].clone()
    cols[64:] = 0
    bad = _fractions({"dkernel": c["pre_k"] + cols.t() @ o["dz"]}, {"dkernel": ref["dkernel"]}, c, split)["dkernel"]
    print("dkernel without the partial 64-row block: %.0f of the bar" % bad)
    assert bad > 100


def test_unread_pixels_of_a_stride_larger_than_the_kernel():
    """k = 1, s = 2 on 7 x 5 reads rows 0, 2, 4, 6 and columns 0, 2, 4; k = 2, s = 3 on 7 rows (padding 0 / 1) rows 0, 1,
    3, 4, 6"""
    u = unread_pixels(1, 7, 5, 1, 2)[0, :, :, 0]
    assert torch.equal(~u, torch.from_numpy(np.logical_and.outer(np.arange(7) % 2 == 0, np.arange(5) % 2 == 0)))
    u = unread_pixels(1, 7, 7, 2, 3)[0, :, 0, 0]
    assert [int(v) for v in ~u] == [1, 1, 0, 1, 1, 0, 1]


# ------------------------------------------------------------------------------------------------ the row-grid refusal
def test_dz_grids_beyond_65535_row_blocks_are_refused():
    lib = L_.load()
    buf = (ctypes.c_float * 4096)()
    p = _fake_ptr(buf)
    C = Cout = 128
    big, edge = (1, 2048, 2049), (1, 64, 65535)              # M = 4 196 352 (Mp / 64 = 65 568) and M = 4 194 240 (65 535)
    # the queries first: they call nothing on the device
    for name in ("mac_conv_bwd_tc", "mac_conv_bwd_tc32"):
        q = getattr(lib, name + "_workspace_bytes")
        assert q(*big, C, Cout, 1, 1, 1) == 0 and q(*big, C, Cout, 1, 1, 0) == 0
        assert q(*edge, C, Cout, 1, 1, 0) > 0
    for name in ("mac_conv_bwd_loc_tc", "mac_conv_bwd_loc_tc32"):
        q = getattr(lib, name + "_workspace_bytes")
        assert q(*big, C, Cout, 2, 1, 1, 1) == 0
        assert q(*edge, C, Cout, 2, 1, 1, 0) > 0
    for name in ("mac_conv3x3_bwd_tc", "mac_conv3x3_bwd_tc32"):
        q = getattr(lib, name + "_workspace_bytes")
        assert q(*big, C, Cout, 1) == 0
        assert q(*edge, C, Cout, 0) > 0
    launches = lib.mac_b200_launch_count()
    ws = 1 << 62
    head = (p, p, p, p, L_.ACT["ELU"], 0.82, 7, 32, 1)
    for dx in (p, None):
        for name in ("mac_conv_bwd_tc", "mac_conv_bwd_tc32"):
            assert getattr(lib, name)(*head, p, p, dx, p, ws, *big, C, Cout, 1, 1, None) == UNSUPPORTED, name
        for name in ("mac_conv_bwd_loc_tc", "mac_conv_bwd_loc_tc32"):
            assert getattr(lib, name)(*head, p, 2, 50, p, p, p, dx, p, ws, *big, C, Cout, 1, 1, None) == UNSUPPORTED, name
        for name in ("mac_conv3x3_bwd_tc", "mac_conv3x3_bwd_tc32"):
            assert getattr(lib, name)(*head, p, p, dx, p, ws, *big, C, Cout, None) == UNSUPPORTED, name
    assert lib.mac_b200_launch_count() == launches
