"""`mac_linear_tc_seg_fwd` and `mac_linear_bwd_tc` (csrc/linear_tc.cuh) against fp64 products of their OWN operands: the
bf16-rounded (round to nearest even) segments, weights and output gradients the kernels multiply.  The bound is the one of
tests/test_gpu_backward_kernels.py, |got - ref| <= tol * absref, absref being the same product on absolute values (what
fp32 accumulation error scales with).  Each `tol` is about three times the worst value measured on an H100 80GB HBM3,
written beside it."""
import ctypes

import numpy as np
import pytest
import torch

from mac_network_b200 import _lib as L_

pytestmark = pytest.mark.gpu

#                                                                                           measured
TOL_FWD = 1.5e-6        # y against fp64 of bf16(x) @ bf16(W) + b + bias_const, after act    4.9e-7
TOL_DX = 1e-6           # dx against fp64 of bf16(dy) @ bf16(W_s)^T                          2.9e-7
TOL_DW = 6e-7           # dW against fp64 of bf16(x)^T @ bf16(dy) (split-K, fp32 partials)   1.8e-7
TOL_DB = 2.5e-7         # db against fp64 column sums of the fp32 dy                         7.4e-8

MS = [1, 63, 64, 65, 3136, 12544]
SEGS = [(128,), (256, 128), (512, 128, 256), (128, 256, 384, 1024), (1024,)]
ACTS = ["NON", "TANH", "SIGMOID", "ELU", "RELU_STD"]
WORST = {}


def lib():
    return L_.load()


def bf(t):
    return t.to(torch.bfloat16).to(torch.float64)


def ints(v):
    return (ctypes.c_int * len(v))(*v)


def ptrs(ts):
    return (ctypes.c_void_p * len(ts))(*[None if t is None else t.data_ptr() for t in ts])


def _segs(M, ks, seed):
    """Segments as column blocks of wider buffers: every segment has its own leading dimension."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    xs = []
    for i, k in enumerate(ks):
        buf = torch.randn(M, k + 4 * (i + 1), device="cuda", generator=g)
        xs.append(buf[:, :k])
    return xs


def _act64(x, act):
    if act == "TANH":
        return torch.tanh(x)
    if act == "SIGMOID":
        return torch.sigmoid(x)
    if act == "ELU":
        return torch.where(x > 0, x, torch.expm1(x))
    if act == "RELU_STD":
        return torch.clamp(x, min=0)
    return x


def _note(key, v):
    WORST[key] = max(WORST.get(key, 0.0), v)
    return v


def _rel(got, ref, absref, floor=0.0):
    return float(((got.double() - ref).abs() / (absref + floor + 1e-30)).max())


def _fwd(xs, Wt16, b, bc, act, y, M, n_out):
    ks = [x.shape[1] for x in xs]
    K = sum(ks)
    ws = torch.empty(lib().mac_linear_tc_seg_workspace_bytes(M, K), dtype=torch.uint8, device="cuda")
    L_.check(lib().mac_linear_tc_seg_fwd(ptrs(xs), ints(ks), ints([x.stride(0) for x in xs]), len(xs), L_.ptr(Wt16),
                                         L_.ptr(b), float(bc), L_.ACT[act], L_.ptr(y), y.stride(0), M, n_out, L_.ptr(ws),
                                         ws.numel(), L_.stream_ptr()), "mac_linear_tc_seg_fwd")


@pytest.mark.parametrize("M", MS)
@pytest.mark.parametrize("act", ACTS)
def test_linear_tc_seg_fwd(M, act):
    ks = SEGS[(MS.index(M) + ACTS.index(act)) % len(SEGS)]
    n_out = 512 if act in ("NON", "ELU") else 128
    K = sum(ks)
    xs = _segs(M, ks, seed=M + 7)
    W = torch.randn(K, n_out, device="cuda") / np.sqrt(K)
    Wt16 = torch.empty(n_out, K, dtype=torch.bfloat16, device="cuda")
    L_.check(lib().mac_pack_weight_bf16(L_.ptr(W), L_.ptr(Wt16), K, n_out, L_.stream_ptr()))
    with_bias = ACTS.index(act) % 2 == 0
    b = 0.1 * torch.randn(n_out, device="cuda") if with_bias else None
    bc = -0.5 if act == "SIGMOID" else (0.25 if act == "TANH" else 0.0)
    ypad = torch.full((M, n_out + 8), 7.0, device="cuda")
    y = ypad[:, :n_out]
    _fwd(xs, Wt16, b, bc, act, y, M, n_out)
    x64 = torch.cat([bf(x) for x in xs], dim=1)
    w64 = bf(W)
    pre = x64 @ w64 + (b.double() if b is not None else 0.0) + bc
    ref = _act64(pre, act)
    absref = x64.abs() @ w64.abs() + (b.double().abs() if b is not None else 0.0) + abs(bc)
    err = _note("fwd", _rel(y, ref, absref, floor=1e-3 if act == "ELU" else 0.0))
    print("mac_linear_tc_seg_fwd M=%d segs=%s n_out=%d act=%s bias=%s bc=%g: %.2e" % (M, ks, n_out, act, with_bias, bc, err))
    assert err < TOL_FWD
    assert bool((ypad[:, n_out:] == 7.0).all()), "wrote outside ldy"
    # a rerun gives the same bits
    y2 = torch.empty_like(y)
    _fwd(xs, Wt16, b, bc, act, y2, M, n_out)
    assert torch.equal(y, y2)


def _bwd(xs, W, dy, dxs, accum, dW, db, M, n_out):
    ks = [x.shape[1] for x in xs]
    need = lib().mac_linear_bwd_tc_workspace_bytes(M, ints(ks), len(ks), n_out)
    ws = torch.full((need,), 0x5A, dtype=torch.uint8, device="cuda")          # not zero: the padding must be rewritten
    st = lib().mac_linear_bwd_tc(ptrs(xs), ints(ks), ints([x.stride(0) for x in xs]), len(xs), L_.ptr(W), L_.ptr(dy),
                                 dy.stride(0), ptrs(dxs), ints([d.stride(0) if d is not None else 0 for d in dxs]),
                                 ints(accum), L_.ptr(dW), L_.ptr(db), M, n_out, L_.ptr(ws), ws.numel(), L_.stream_ptr())
    L_.check(st, "mac_linear_bwd_tc")


@pytest.mark.parametrize("M", MS)
@pytest.mark.parametrize("si", range(len(SEGS) - 1))
def test_linear_bwd_tc(M, si):
    ks = SEGS[si]
    n_out = 128 if si % 2 else 512
    K = sum(ks)
    xs = _segs(M, ks, seed=3 * M + si)
    W = torch.randn(K, n_out, device="cuda") / np.sqrt(K)
    dy = torch.randn(M, n_out, device="cuda")
    accum = [(i + si) % 2 for i in range(len(ks))]                           # dx_accum on and off
    dx0 = [torch.randn(M, k + 8, device="cuda")[:, :k] for k in ks]
    dxs = [d.clone() for d in dx0]
    dW0 = torch.randn(K, n_out, device="cuda")
    db0 = torch.randn(n_out, device="cuda")
    dW, db = dW0.clone(), db0.clone()
    with_db = si != 1
    _bwd(xs, W, dy, dxs, accum, dW, db if with_db else None, M, n_out)
    dy64, w64 = bf(dy), bf(W)
    errs = {}
    koff = 0
    for i, k in enumerate(ks):
        ws_ = w64[koff:koff + k]
        ref = dy64 @ ws_.T + (dx0[i].double() if accum[i] else 0.0)
        absref = dy64.abs() @ ws_.abs().T + (dx0[i].double().abs() if accum[i] else 0.0)
        errs["dx%d" % i] = _note("dx", _rel(dxs[i], ref, absref))
        x64 = bf(xs[i])
        ref = dW0[koff:koff + k].double() + x64.T @ dy64
        absref = dW0[koff:koff + k].double().abs() + x64.abs().T @ dy64.abs()
        errs["dW%d" % i] = _note("dW", _rel(dW[koff:koff + k], ref, absref))
        koff += k
    if with_db:
        ref = db0.double() + dy.double().sum(0)
        absref = db0.double().abs() + dy.double().abs().sum(0)
        errs["db"] = _note("db", _rel(db, ref, absref))
    else:
        assert torch.equal(db, db0)
    print("mac_linear_bwd_tc M=%d segs=%s n_out=%d accum=%s: %s" % (M, ks, n_out, accum,
                                                                    ", ".join("%s %.2e" % kv for kv in errs.items())))
    tol = {"dx": TOL_DX, "dW": TOL_DW, "db": TOL_DB}
    bad = {k: v for k, v in errs.items() if not v < tol[k.rstrip("0123456789")]}
    assert not bad, bad
    # a rerun from the same state gives the same bits
    dxs2 = [d.clone() for d in dx0]
    dW2, db2 = dW0.clone(), db0.clone()
    _bwd(xs, W, dy, dxs2, accum, dW2, db2 if with_db else None, M, n_out)
    assert torch.equal(dW, dW2) and torch.equal(db, db2) and all(torch.equal(a, b) for a, b in zip(dxs, dxs2))


def test_linear_tc_weight_gradient_only():
    """dx_segs NULL: only the weight and bias gradients (no weight needed)."""
    M, ks, n_out = 65, (256,), 128
    xs = _segs(M, ks, seed=5)
    dy = torch.randn(M, n_out, device="cuda")
    dW, db = torch.zeros(256, n_out, device="cuda"), torch.zeros(n_out, device="cuda")
    need = lib().mac_linear_bwd_tc_workspace_bytes(M, ints(ks), 1, n_out)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    L_.check(lib().mac_linear_bwd_tc(ptrs(xs), ints(ks), ints([xs[0].stride(0)]), 1, None, L_.ptr(dy), n_out, None, None,
                                     None, L_.ptr(dW), L_.ptr(db), M, n_out, L_.ptr(ws), need, L_.stream_ptr()))
    ref = bf(xs[0]).T @ bf(dy)
    assert _rel(dW, ref, bf(xs[0]).abs().T @ bf(dy).abs()) < TOL_DW


def test_unsupported_shapes_launch_nothing():
    lb = lib()
    M = 64
    x = torch.randn(M, 192, device="cuda")
    Wt16 = torch.zeros(192, 192, dtype=torch.bfloat16, device="cuda")
    y = torch.empty(M, 192, device="cuda")
    ws = torch.empty(1 << 22, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    n0 = lb.mac_b200_launch_count()
    for k, n_out in ((192, 128), (128, 192), (64, 128)):
        st = lb.mac_linear_tc_seg_fwd(ptrs([x]), ints([k]), ints([192]), 1, L_.ptr(Wt16), None, 0.0, 0, L_.ptr(y), 192, M,
                                      n_out, L_.ptr(ws), ws.numel(), L_.stream_ptr())
        assert st == -3, (k, n_out, st)
        st = lb.mac_linear_bwd_tc(ptrs([x]), ints([k]), ints([192]), 1, L_.ptr(y), L_.ptr(y), 192, ptrs([y]), ints([192]),
                                  ints([0]), L_.ptr(y), None, M, n_out, L_.ptr(ws), ws.numel(), L_.stream_ptr())
        assert st == -3, (k, n_out, st)
    assert lb.mac_b200_launch_count() == n0


def test_zz_print_worst():
    print("worst measured (fraction of absref):", {k: "%.2e" % v for k, v in sorted(WORST.items())})
