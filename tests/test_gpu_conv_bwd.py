"""The stem's general and location-aware backward on tensor cores -- `mac_conv_bwd_tc`, `mac_conv_bwd_tc32`,
`mac_conv_bwd_loc_tc`, `mac_conv_bwd_loc_tc32` -- against fp64 references of their OWN operation, at the shapes where a
patch pass or a padded GEMM goes wrong: a partly filled last 64-row block (zero padding columns in dZ^T, the patches^T and
Q^T), strides larger than the kernel (input pixels no tap reads), even kernels (TF's SAME padding puts the odd row at the
bottom / right), kernels larger than the image, the linear stem's NON activation, several split-K slices, and location
patch matrices spanning one to 25 128-row tiles with zero rows after the k^2 l real ones.

The reference follows tests/test_stem_tc_training.py and tests/test_gpu_stem_bf16x3.py: computed on exactly the operands
the kernels see -- dZ = dy * act'(y) in fp32, the SAME patches of dropout(x) with the keep-mask `mac_dropout_uniform` draws
at the layer's site, and for the location forms the SAME patches of the fp32 grid broadcast over the batch with the
SITE_LOCATION mask over [B, H, W, l], zero-padded to Kq -- rounded to bf16 for the bf16 form and kept in fp32 for the split
form (the bias sums in both forms from the fp32 dZ).  Each output must satisfy |got - ref| <= tol * absref element by
element (`excess`, absref the same products on absolute values) under each precision's TOL_CONV, unchanged but for the
split form's dx (see TOL); dW_loc is held to that precision's dkernel bar, since the general pass changes only which patch
enters the same GEMMs.

Every case also checks: the workspace filled with 0xFF and passed at byte offsets 0, 16 and 1008 from a 1 KB boundary,
with the bytes before it and a 4 KB sentinel after its reported size untouched and the results bit-identical at all three
offsets; `+=` onto random non-zero gradients, with dW_loc's rows k^2 l..Kq-1 back bit for bit; dx NaN-filled before the
call, finite after, and exactly 0 at the pixels no tap reads; the location entry points' image outputs bit for bit those of
the plain ones; and at k = 3, s = 1 the general entry points bit for bit the 3x3 ones.  tests/test_conv_bwd_bounds.py
shows on the CPU, with this file's reference code, that these bars reject a dropped col2im tap, the odd SAME padding row on
the wrong side, a missing location tap, the bias gradient added twice and a dropped partial 64-row block.

The stem-level tests run Stem(prec="bf16" | "bf16x3") forward(save) + backward with location features away from 3x3
stride 1, and the location-free geometries at an M that is not a multiple of 64, against the fp64 autograd oracles with the
bars of tests/test_gpu_stem_location.py and tests/test_gpu_stem_geometry.py."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from mac_network_b200 import _lib as L_
from oracle.stem_geometry import same_pads
from tests.test_gpu_stem_bf16x3 import TOL_CONV as TOL_CONV_TC32
from tests.test_gpu_stem_geometry import BIG
from tests.test_gpu_wgmma import align1k, bf16_round, excess, pick_ksplit
from tests.test_stem_tc_training import TOL_CONV as TOL_CONV_BF16

pytestmark = pytest.mark.gpu

# split -> bars (fraction of absref); dW_loc under "dkernel".  Every bar is the 3x3 tests' except the split form's dx: a
# pixel read by one tap only (s >= k, k = 1, the image border at s = 2) takes a contraction over Cout alone -- 64 non-zero
# terms when ReLU zeroes half of dZ -- where the 3x3 stride-1 pixels sum four to nine taps, so the dropped lo * lo products
# (up to 2^-18 of each term, 3 * 2^-18 = 1.1e-5 with the lo roundings) average out far less.  Measured on an H100 80GB
# HBM3 (700 W power limit): worst 4.7e-6 over four seeds at (2, 14, 14, 128, 128, 3, 2) with ReLU (3x3 stride 1: 1.7e-6),
# and there the kernel is within 2.0e-7 of an fp64 emulation of its three split products, so the rest is the split itself.
TOL = {False: TOL_CONV_BF16, True: dict(TOL_CONV_TC32, dx=1.2e-5)}
OFFSETS = (0, 16, 1008)                                  # workspace byte offsets from a 1 KB boundary
SENTINEL, GUARD = 4096, 0x5A
LOCS = {"L": ("L", 1.0, 32), "PE3": ("PE", 0.5, 3), "PE": ("PE", 1.0, 32)}     # l = 2, 12, 128


# ------------------------------------------------------------------------------------------------ fp64 reference
def act_grad(act, y):
    """act'(.) from the activation's fp32 output, as csrc/common.cuh's act_grad_from_output forms it"""
    one = torch.ones_like(y)
    if act == "ELU":
        return torch.where(y > 0, one, y + 1)
    if act == "RELU_STD":
        return torch.where(y > 0, one, torch.zeros_like(y))
    assert act == "NON", act
    return one


def grid_out(H, W, s):
    return -(-H // s), -(-W // s)


def patches(x, k, s, pads=same_pads):
    """[B, H, W, C] -> the patch matrix [B Ho Wo, k^2 C], tap-major (kh k + kw), channel fastest, padded by `pads`"""
    B, H, W, C = x.shape
    Ho, Wo = grid_out(H, W, s)
    (pt, pb), (pl, pr) = pads(H, k, s), pads(W, k, s)
    xp = F.pad(x, (0, 0, pl, pr, pt, pb))
    return torch.cat([xp[:, i:i + (Ho - 1) * s + 1:s, j:j + (Wo - 1) * s + 1:s].reshape(-1, C)
                      for i in range(k) for j in range(k)], 1)


def col2im(dcols, shape, k, s, pads=same_pads):
    """patches' adjoint: each entry of dcols [B Ho Wo, k^2 C] added back to the input pixel it copied"""
    B, H, W, C = shape
    Ho, Wo = grid_out(H, W, s)
    (pt, pb), (pl, pr) = pads(H, k, s), pads(W, k, s)
    acc = dcols.new_zeros(B, H + pt + pb, W + pl + pr, C)
    d = dcols.reshape(B, Ho, Wo, k * k, C)
    for tap in range(k * k):
        i, j = divmod(tap, k)
        acc[:, i:i + (Ho - 1) * s + 1:s, j:j + (Wo - 1) * s + 1:s] += d[:, :, :, tap]
    return acc[:, pt:pt + H, pl:pl + W]


def unread_pixels(B, H, W, k, s):
    """[B, H, W, 1] True where no tap of any output pixel reads the input pixel"""
    Ho, Wo = grid_out(H, W, s)
    return col2im(torch.ones(B * Ho * Wo, k * k, dtype=torch.float64), (B, H, W, 1), k, s) == 0


def conv_bwd_reference(x, y, dy, kernel, act, keep, mask, k, s, split, with_dx, grid=None, qmask=None, Kq=0,
                       pads=same_pads):
    """{output: (ref, absref)} in fp64 of what one call adds (dkernel [k^2 C, Cout], dbias, dwloc [Kq, Cout]) or writes
    (dx [B, H, W, C]), on the operands the kernels see.  x [B,H,W,C], y and dy [M, Cout], kernel [k,k,C,Cout] and grid
    [H,W,l] fp32; mask / qmask the keep-masks (bool, [B,H,W,C] / [B,H,W,l]) or None at keep 1.  `split`: the tc32 form (fp32
    operands), else bf16-rounded operands."""
    B, H, W, C = x.shape
    Cout = y.shape[1]
    scale = np.float32(1.0) / np.float32(keep)
    rnd = (lambda t: t.double()) if split else bf16_round
    dz32 = dy * act_grad(act, y)
    dz = rnd(dz32)
    m = 1.0 if mask is None else mask.double()
    cols = patches(rnd(x * scale) * m, k, s, pads)
    out = {"dkernel": (cols.t() @ dz, cols.abs().t() @ dz.abs())}
    del cols
    out["dbias"] = (dz32.double().sum(0), dz32.double().abs().sum(0))
    if with_dx:
        kr = rnd(kernel.reshape(-1, Cout))
        f = m * float(scale)
        out["dx"] = (col2im(dz @ kr.t(), (B, H, W, C), k, s, pads) * f,
                     col2im(dz.abs() @ kr.abs().t(), (B, H, W, C), k, s, pads) * f)
    if grid is not None:
        l = grid.shape[-1]
        qm = 1.0 if qmask is None else qmask.double()
        q = patches(rnd(grid.expand(B, H, W, l) * scale) * qm, k, s, pads)
        q = F.pad(q, (0, Kq - q.shape[1]))
        out["dwloc"] = (q.t() @ dz, q.abs().t() @ dz.abs())
    return out


# ------------------------------------------------------------------------------------------------ the entry points
def _lib():
    return L_.load()


def _entry(split, loc):
    return "mac_conv_bwd_%stc%s" % ("loc_" if loc else "", "32" if split else "")


def _workspace(nbytes, off):
    """(buffer, start): nbytes of 0xFF at 1 KB boundary + off, GUARD bytes before and at least SENTINEL bytes after"""
    buf = torch.full((nbytes + 2048 + SENTINEL,), GUARD, dtype=torch.uint8, device="cuda")
    start = align1k(buf) + off
    buf[start:start + nbytes] = 0xFF                    # NaN everywhere: the workspace is not assumed zero
    return buf, start


def _call(split, shape, act, keep, ins, outs, off, grid=None, k3x3=False):
    """One call of the entry point at workspace offset `off`; returns (buffer, start, nbytes) for the guard checks."""
    lib = _lib()
    B, H, W, C, Cout, k, s = shape
    x, y, dy, kernel = ins
    dkernel, dbias, dx, dwloc = outs
    seed, site, step, loc_site = 4321, 33, 5, 50
    head = (L_.ptr(x), L_.ptr(y), L_.ptr(dy), L_.ptr(kernel), L_.ACT[act], keep, seed, site, step)
    wdx = int(dx is not None)
    if k3x3:
        name = "mac_conv3x3_bwd_tc%s" % ("32" if split else "")
        nbytes = int(getattr(lib, name + "_workspace_bytes")(B, H, W, C, Cout, wdx))
    elif grid is not None:
        name = _entry(split, True)
        nbytes = int(getattr(lib, name + "_workspace_bytes")(B, H, W, C, Cout, grid.shape[-1], k, s, wdx))
    else:
        name = _entry(split, False)
        nbytes = int(getattr(lib, name + "_workspace_bytes")(B, H, W, C, Cout, k, s, wdx))
    assert nbytes > 0
    buf, start = _workspace(nbytes, off)
    ws = buf.data_ptr() + start
    if grid is not None:
        args = head + (L_.ptr(grid), grid.shape[-1], loc_site, L_.ptr(dkernel), L_.ptr(dwloc), L_.ptr(dbias), L_.ptr(dx), ws,
                       nbytes, B, H, W, C, Cout, k, s)
    else:
        args = head + (L_.ptr(dkernel), L_.ptr(dbias), L_.ptr(dx), ws, nbytes, B, H, W, C, Cout) + (() if k3x3 else (k, s))
    L_.check(getattr(lib, name)(*args, L_.stream_ptr()), name)
    return buf, start, nbytes


def _inputs(shape, act, seed):
    B, H, W, C, Cout, k, s = shape
    Ho, Wo = grid_out(H, W, s)
    M = B * Ho * Wo
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, H, W, C, device="cuda", generator=g)
    kernel = torch.randn(k, k, C, Cout, device="cuda", generator=g) * (2.0 / (k * k * (C + Cout))) ** 0.5
    z = torch.randn(M, Cout, device="cuda", generator=g)
    y = {"ELU": F.elu(z), "RELU_STD": torch.relu(z), "NON": z}[act]          # RELU_STD: about half of y exactly 0
    dy = torch.randn(M, Cout, device="cuda", generator=g)
    pre_k = torch.randn(k, k, C, Cout, device="cuda", generator=g) * 0.1
    pre_b = torch.randn(Cout, device="cuda", generator=g)
    return (x, y, dy, kernel), pre_k, pre_b, g


def _mask(seed, site, step, shape, keep):
    from tests.test_stem_tc_training import _uniform_mask
    return None if keep == 1.0 else _uniform_mask(_lib(), seed, site, step, shape, keep)


def _same(a, b):
    if a is None or b is None:
        return a is None and b is None
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _slices(split, Mp, rows, Cout):
    """tc_pick_ksplit's slice count for a weight gradient of `rows` x Cout contracting over Mp (3 Mp split)"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return pick_ksplit((3 if split else 1) * Mp, (rows // 128) * (Cout // 128), sms)


def _run_case(split, shape, act, keep, with_dx, loc=None):
    B, H, W, C, Cout, k, s = shape
    Ho, Wo = grid_out(H, W, s)
    M = B * Ho * Wo
    Mp = (M + 63) // 64 * 64
    ins, pre_k, pre_b, g = _inputs(shape, act, seed=sum(shape) + 7 * int(split) + (len(loc) if loc else 0))
    x, y, dy, kernel = ins
    grid = l = Kq = pre_q = None
    if loc is not None:
        from mac_network_b200.stem import location_grid
        grid = torch.from_numpy(np.ascontiguousarray(location_grid(LOCS[loc], H, W), dtype=np.float32)).cuda()
        l = grid.shape[-1]
        Kq = int(_lib().mac_loc_cols_width(l, k))
        pre_q = torch.randn(Kq, Cout, device="cuda", generator=g) * 0.1
    runs = []
    for off in OFFSETS:
        dkernel, dbias = pre_k.clone(), pre_b.clone()
        dx = torch.full((B, H, W, C), float("nan"), device="cuda") if with_dx else None
        dwloc = None if loc is None else pre_q.clone()
        buf, start, nbytes = _call(split, shape, act, keep, ins, (dkernel, dbias, dx, dwloc), off, grid=grid)
        runs.append((dkernel, dbias, dx, dwloc, buf, start, nbytes))
    torch.cuda.synchronize()
    for _, _, _, _, buf, start, nbytes in runs:
        assert bool((buf[:start] == GUARD).all()), "bytes before the workspace written"
        assert bool((buf[start + nbytes:] == GUARD).all()), "bytes after the reported workspace size written"
    dkernel, dbias, dx, dwloc = runs[0][:4]
    for r in runs[1:]:
        assert all(_same(a, b) for a, b in zip(runs[0][:4], r[:4])), "results differ between workspace offsets"
    if loc is not None:                          # the image half is the plain entry point's, bit for bit
        plain = (pre_k.clone(), pre_b.clone(), torch.full((B, H, W, C), float("nan"), device="cuda") if with_dx else None,
                 None)
        _call(split, shape, act, keep, ins, plain, 16)
        torch.cuda.synchronize()
        assert _same(plain[0], dkernel) and _same(plain[1], dbias) and _same(plain[2], dx)
        assert _same(dwloc[k * k * l:], pre_q[k * k * l:]), "dW_loc's zero rows k^2 l..Kq-1 changed"
    seed, site, step = 4321, 33, 5
    mask = _mask(seed, site, step, (B, H, W, C), keep)
    qmask = None if loc is None else _mask(seed, 50, step, (B, H, W, l), keep)
    ref = conv_bwd_reference(x, y, dy, kernel, act, keep, mask, k, s, split, with_dx, grid=grid, qmask=qmask, Kq=Kq or 0)
    rows = {}
    r, a = ref.pop("dkernel")
    pk = pre_k.double().view(-1, Cout)
    rows["dkernel"] = excess(dkernel.view(-1, Cout), pk + r, a + pk.abs()) / TOL[split]["dkernel"]
    r, a = ref.pop("dbias")
    rows["dbias"] = excess(dbias, pre_b.double() + r, a + pre_b.double().abs()) / TOL[split]["dbias"]
    if with_dx:
        r, a = ref.pop("dx")
        assert bool(torch.isfinite(dx).all()), "dx not written everywhere"
        unread = unread_pixels(B, H, W, k, s).cuda().expand(B, H, W, C)
        assert bool((dx[unread] == 0).all()), "a pixel no tap reads has a non-zero gradient"
        rows["dx"] = excess(dx, r, a) / TOL[split]["dx"]
    if loc is not None:
        r, a = ref.pop("dwloc")
        n = k * k * l
        pq = pre_q.double()[:n]
        rows["dW_loc"] = excess(dwloc[:n], pq + r[:n], a[:n] + pq.abs()) / TOL[split]["dkernel"]
    S = _slices(split, Mp, k * k * C, Cout)
    Sq = "" if loc is None else ", dW_loc %d" % _slices(split, Mp, Kq, Cout)
    print("%s %s %s keep %s dx=%s M=%d: split-K slices %d%s; fraction of the bar: %s" % (
        _entry(split, loc is not None), shape if loc is None else "%s %s" % (loc, shape), act, keep, with_dx, M, S, Sq,
        ", ".join("%s %.3f" % kv for kv in rows.items())))
    bad = {kk: v for kk, v in rows.items() if not v <= 1.0}
    assert not bad, bad


# (B, H, W, C, Cout, k, s), activation, keep, with_dx options
CASES = [
    ((1, 7, 5, 128, 128, 1, 2), "ELU", 0.82, (True, False)),           # M = 12 < 64; s > k: pixels no tap reads
    ((2, 7, 6, 128, 128, 5, 2), "RELU_STD", 0.82, (True, False)),      # W padding 1 / 2; M = 24
    ((3, 5, 3, 128, 256, 4, 1), "ELU", 0.82, (True, False)),           # even k: the odd row at the bottom / right; M = 45
    ((1, 3, 5, 128, 128, 7, 1), "RELU_STD", 0.82, (True, False)),      # k larger than the image; M = 15
    ((5, 7, 7, 256, 128, 2, 3), "ELU", 0.82, (True, False)),           # s > k with even k; M = 45
    ((2, 14, 14, 128, 128, 3, 2), "RELU_STD", 0.82, (True, False)),    # M = 98: one full and one partial 64-row block
    ((3, 5, 7, 256, 128, 1, 1), "NON", 1.0, (True, False)),            # the linear stem's call; M = 105
    ((3, 14, 14, 256, 128, 1, 1), "ELU", 0.82, (True, False)),         # M = 588: split-K over 5 (bf16) / 15 (split) slices
    ((64, 14, 14, 1024, 512, 5, 2), "ELU", 0.82, (False,)),            # a layer 0 at serving scale
    ((64, 14, 14, 512, 512, 2, 1), "RELU_STD", 0.82, (True,)),         # a layer 1 at serving scale
]
LOC_CASES = [
    ("L", (1, 7, 5, 128, 128, 3, 2), "ELU", (True, False)),           # M = 12; Kq = 128: 18 rows and 110 zero rows
    ("L", (2, 14, 14, 128, 128, 3, 1), "RELU_STD", (True, False)),    # the 3x3 passes under the location product; M = 392
    ("PE3", (2, 7, 6, 128, 128, 5, 2), "ELU", (True, False)),         # l = 12: Kq = 384, three tiles, 84 zero rows; M = 24
    ("PE", (64, 14, 14, 1024, 512, 5, 2), "ELU", (False,)),           # default PE, l = 128: Kq = 3200 at serving scale
]


def _params(cases):
    """(case..., with_dx, split) for every dx option of each case, in both precisions"""
    out = []
    for c in cases:
        for dx in c[-1]:
            for split in (False, True):
                out.append(c[:-1] + (dx, split))
    return out


@pytest.mark.parametrize("shape,act,keep,with_dx,split", _params(CASES))
def test_conv_bwd_against_fp64(shape, act, keep, with_dx, split):
    _run_case(split, shape, act, keep, with_dx)


@pytest.mark.parametrize("loc,shape,act,with_dx,split", _params(LOC_CASES))
def test_conv_bwd_loc_against_fp64(loc, shape, act, with_dx, split):
    _run_case(split, shape, act, 0.82, with_dx, loc=loc)


def test_cases_run_one_and_several_split_k_slices():
    counts = set()
    for shape, _, _, _ in CASES:
        B, H, W, C, Cout, k, s = shape
        Mp = (B * int(np.prod(grid_out(H, W, s))) + 63) // 64 * 64
        counts |= {_slices(split, Mp, k * k * C, Cout) for split in (False, True)}
    assert 1 in counts and max(counts) > 1, counts


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("shape,with_dx", [((2, 5, 7, 128, 128, 3, 1), True), ((1, 7, 7, 128, 256, 3, 1), False)])
def test_general_entry_point_at_3x3_stride_1_is_the_3x3_one(shape, with_dx, split):
    B, H, W, C, Cout, k, s = shape
    ins, pre_k, pre_b, _ = _inputs(shape, "ELU", seed=3)
    got = []
    for k3x3 in (False, True):
        outs = (pre_k.clone(), pre_b.clone(), torch.full((B, H, W, C), float("nan"), device="cuda") if with_dx else None,
                None)
        _call(split, shape, "ELU", 0.82, ins, outs, 0, k3x3=k3x3)
        got.append(outs[:3])
    torch.cuda.synchronize()
    assert all(_same(a, b) for a, b in zip(*got))
    lib = _lib()
    q, q3 = _entry(split, False) + "_workspace_bytes", "mac_conv3x3_bwd_tc%s_workspace_bytes" % ("32" if split else "")
    assert getattr(lib, q)(B, H, W, C, Cout, 3, 1, int(with_dx)) == getattr(lib, q3)(B, H, W, C, Cout, int(with_dx))


# ------------------------------------------------------------------------------------------------ the stem
STEM_LOC_GEOMS = [dict(ksizes=[5, 3], strides=[2, 1]), dict(ksizes=[4, 2], strides=[1, 1])]
STEM_SHAPES = [(64, 14, 14, 1024, 512), (5, 7, 6, 128, 128)]    # M = 12 544 / 3 136, and 210 / 60: not multiples of 64


def _bars(prec):
    return (1e-4, 2e-4) if prec == "bf16x3" else (2e-2, 1.2e-2)


@pytest.mark.parametrize("prec", ["bf16", "bf16x3"])
@pytest.mark.parametrize("loc", ["L", "PE"])
@pytest.mark.parametrize("geom", range(len(STEM_LOC_GEOMS)))
@pytest.mark.parametrize("shape", STEM_SHAPES)
def test_location_stem_at_other_geometries_against_fp64(shape, geom, loc, prec):
    """Layer 0 with location features away from 3x3 stride 1: `_loc_weights`' gather, mac_conv_bwd_loc_tc(32) and
    `_loc_scatter`, against the fp64 autograd oracle with the bars of tests/test_gpu_stem_location.py."""
    from mac_network_b200.stem import Stem, init_stem_params, stem_specs
    from tests.test_gpu_stem_location import LOCS as STEM_LOCS, _check_stem
    B, H, W, C, Cout = shape
    gm = STEM_LOC_GEOMS[geom]
    pv = init_stem_params(stem_specs(C, Cout, ksizes=gm["ksizes"], location=STEM_LOCS[loc]), seed=19 + geom,
                          dtype=np.float64)
    params = {k: torch.from_numpy(v.astype(np.float32)).cuda() for k, v in pv.items()}
    st = Stem(params, relu="ELU", prec=prec, seed=23, strides=gm["strides"], location=STEM_LOCS[loc])
    g = torch.Generator(device="cuda").manual_seed(29)
    images = torch.randn(B, H, W, C, device="cuda", generator=g, dtype=torch.float64).clamp_(min=0)
    _check_stem(st, pv, images, 0.82, gm["strides"], *_bars(prec), seed=31)


@pytest.mark.parametrize("prec", ["bf16", "bf16x3"])
@pytest.mark.parametrize("geom", range(len(BIG)))
def test_geometry_stem_at_a_partial_row_block_against_fp64(geom, prec):
    """tests/test_gpu_stem_geometry.py's BIG geometries at B = 5 on 7 x 6, 128 channels: M = 210 or 60."""
    from mac_network_b200.stem import Stem, init_stem_params, stem_specs
    from tests.test_gpu_stem_geometry import _check_stem
    gm = BIG[geom]
    linear = gm.get("linear", False)
    strides = gm.get("strides", [1] if linear else [1, 1])
    pv = init_stem_params(stem_specs(128, 128, ksizes=gm.get("ksizes"), linear=linear), seed=19 + geom, dtype=np.float64)
    params = {k: torch.from_numpy(v.astype(np.float32)).cuda() for k, v in pv.items()}
    st = Stem(params, relu="ELU", prec=prec, seed=23, strides=strides, linear=linear)
    g = torch.Generator(device="cuda").manual_seed(29)
    images = torch.randn(5, 7, 6, 128, device="cuda", generator=g, dtype=torch.float64).clamp_(min=0)
    _check_stem(st, pv, images, 0.82, strides, linear, "ELU", *_bars(prec), seed=31)
