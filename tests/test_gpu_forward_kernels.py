"""The fp32 forward kernels against fp64 references of their OWN operation, called through the C ABI.

The method of tests/test_gpu_backward_kernels.py: each reference is computed on exactly the operands the kernel sees (in a
chain, every stage from the kernel's own previous stage, so rounding does not compound), and evaluated a second time on
absolute values.  The bound is element-wise:

    |got - ref| <= tol * absref + tiny

The five activations have |act'| <= 1, so the pre-activation absref bounds the activated output too.  A dropped skinny
K-slice, split-K slice or logit part, a segment read at the wrong offset or a batch row off by one moves a result by a
sizeable fraction of its absref and fails (tests/test_forward_bounds.py shows that on the CPU with this file's code).

Every case also checks the output contracts: "=" outputs are NaN-filled, so an unwritten element fails, and padding
columns (ldy > n_out) are still NaN afterwards; two runs from the same state agree bit for bit; the split-K counters (the
first 4 096 bytes of every workspace) are zero afterwards.

Each `tol` is about three times the worst value measured on an H100 80GB HBM3 (SXM, 132 SMs) at a 700 W power limit,
written beside it."""
import ctypes

import numpy as np
import pytest
import torch

from mac_network_b200 import _lib as L_
from tests.test_gpu_backward_kernels import (COUNTER_BYTES, READ_CASES, Report, gen, ints, lib, ptrs, randn, read_masks,
                                             run_twice, same_bits, strided)
from tests.test_gpu_wgmma import act_ref, attention_bound_check, elu

pytestmark = pytest.mark.gpu

MAC_OK, ERR_UNSUPPORTED = 0, -3
PREC_FP32 = 0

# ---- bounds (fraction of absref); measured worst value on the H100 beside each
TOL_LINEAR = 1e-6        # mac_linear_fwd (sgemm 64/128 tiles, split-K, skinny cluster kernel)     measured 3.5e-7
TOL_WRITE = 8e-7         # mac_write_fwd, mac_write_fwd_next_y                                     measured 2.6e-7
TOL_READ = 1.5e-6        # fp32 read unit stages y, P, Q, H, I1                                    measured 5.0e-7
TOL_ATT = 1.2e-6         # softmax + weighted sum (kb_attend, control_attend, attend)              measured 4.0e-7
TOL_ROWDOT = 1.5e-7      # mac_rowdot_fwd                                                          measured 4.1e-8
TOL_ELEM = 5e-7          # mac_bcast_op, mac_bcast_mul, mac_activation                             measured 1.7e-7
TOL_NORM = 2e-7          # mac_clip_adam_ema_step global norm                                      measured 5.8e-8
TOL_ADAM = 6e-7          # mac_clip_adam_ema_step clip factor, m, v, p, ema                        measured 2.2e-7
TOL_XENT = 3e-7          # mac_softmax_xent losses and dlogits                                     measured 9.6e-8
# (the read unit's att and info are checked through attention_bound_check: measured at most 8.7e-3 of that bound)
TINY_ACT = 5e-7          # relative fp32 evaluation error of tanhf / expf / expm1f in the epilogues


def nanfill(*shape):
    return torch.full(shape, float("nan"), device="cuda")


def counters_zero(ws):
    return ws is None or not bool(ws[:COUNTER_BYTES].any())


def add_attention(rep, fractions):
    """att and info of the read unit: the fraction of attention_bound_check's bound each uses (at most 1)"""
    rep.rows.append(("att (of its bound)", fractions[0], 1.0))
    rep.rows.append(("info (of its bound)", fractions[1], 1.0))


# ================================================================================================ references
def linear_reference(xs, W, b, bias_const):
    """z = concat(x_s) @ W + b + bias_const in fp64 and |concat(x_s)| @ |W| + |b| + |bias_const| (pre-activation)"""
    X = torch.cat([x.double() for x in xs], 1)
    Wd = W.double()
    z = X @ Wd + bias_const
    az = X.abs() @ Wd.abs() + abs(bias_const)
    if b is not None:
        z = z + b.double()
        az = az + b.double().abs()
    return z, az


def softmax_bound(logits, abs_logits, valid=None):
    """softmax over the last dim in fp64 and the scale of its fp32 error: att * (1 + max |logit terms| of the row).  The
    logits reach the kernel as fp32 sums whose rounding is a fraction of abs_logits; exp(l - max) turns an absolute logit
    error into a relative error of att.  `valid` masks the terms that enter (the rest are -inf in both)."""
    if valid is not None:
        logits = logits.masked_fill(~valid, float("-inf"))
        abs_logits = abs_logits.masked_fill(~valid, 0.0)
    att = torch.softmax(logits, -1)
    lmax = abs_logits.amax(-1, keepdim=True)
    return att, att * (1.0 + lmax)


def kb_attend_reference(parts, br, kb):
    """att = softmax_n(sum_p parts + br), info = sum_n att * kb with their bounds (parts [B, N, P], kb [B, N, d])"""
    pd = parts.double()
    att, aatt = softmax_bound(pd.sum(-1) + br, pd.abs().sum(-1) + abs(br))
    kbd = kb.double()
    return att, aatt, torch.einsum("bn,bnd->bd", att, kbd), torch.einsum("bn,bnd->bd", aatt, kbd.abs())


def read_forward_stages(kb, mem, W, masks, P, y, H):
    """the stages of the fp32 read unit (include/mac_b200.h), each from the kernel's own previous stage: name -> (ref,
    absref).  P, y and H are the kernel's; y and P come from the inputs and the Philox masks."""
    B, N, d = kb.shape
    M = B * N
    mkb, mmem, _ = masks
    D = lambda t: t.double()
    Wx, Wy, Wm, Wm2 = D(W["Wx"]), D(W["Wy"]), D(W["Wm"]), D(W["Wm2"])
    bx, by, bm, bm2 = D(W["bx"]), D(W["by"]), D(W["bm"]), D(W["bm2"])
    r = {}
    md = D(mem) * mmem
    r["y"] = (md @ Wy + by, md.abs() @ Wy.abs() + by.abs())
    kbd = D(kb).view(M, d) * mkb
    r["P"] = (kbd @ Wx + bx, kbd.abs() @ Wx.abs() + bx.abs())
    yb = D(y).repeat_interleave(N, 0)
    I0 = torch.cat([D(P) * yb, D(P)], 1)
    z = I0 @ Wm + bm
    r["H"] = (elu(z), I0.abs() @ Wm.abs() + bm.abs())
    Hd = D(H)
    r["I1"] = (Hd @ Wm2 + bm2, Hd.abs() @ Wm2.abs() + bm2.abs())
    return r


def adam_reference(p, g, m, v, ema, clip, grad_scale, lr, b1, b2, eps, step, decay, m_got, v_got, p_got):
    """one clip + Adam + EMA step in fp64 from the kernel's own inputs, with fp32-rounded hyperparameters and the kernel's
    own clip factor; m, v from the inputs, p from the kernel's m and v, ema from the kernel's p: name -> (ref, absref, tiny)"""
    f = lambda x: float(np.float32(x))
    gs, lr, b1, b2, eps, decay = f(grad_scale), f(lr), f(b1), f(b2), f(eps), f(decay)
    D = lambda t: t.double()
    gi = D(g) * gs * float(clip)
    agi = gi.abs()
    r = {"m": (b1 * D(m) + (1 - b1) * gi, b1 * D(m).abs() + (1 - b1) * agi, 0.0),
         "v": (b2 * D(v) + (1 - b2) * gi * gi, b2 * D(v).abs() + (1 - b2) * gi * gi, 0.0)}
    # the bias corrections: 1 - b^step is computed in fp32 from powf, which may be 2 ulps off b^step
    pw1, pw2 = b1 ** step, b2 ** step
    bc1, bc2 = 1 - pw1, 1 - pw2
    lr_t = lr * np.sqrt(bc2) / bc1
    upd = lr_t * D(m_got) / (torch.sqrt(D(v_got)) + eps)
    rel_bc = 2 * 2.0 ** -23 * (pw1 / bc1 + 0.5 * pw2 / bc2)
    r["p"] = (D(p) - upd, D(p).abs() + upd.abs(), upd.abs() * rel_bc)
    if ema is not None:
        r["ema"] = (decay * D(ema) + (1 - decay) * D(p_got), decay * D(ema).abs() + (1 - decay) * D(p_got).abs(), 0.0)
    return r


def adam_inputs(g, n, device):
    """parameters, gradients and Adam state of the scales a trained model has after a while: |update| ~ lr, well above the
    rounding of p, so that an EMA of the pre-update parameters is visible"""
    r = lambda *s, scale=1.0: torch.randn(*s, generator=g, device=device) * scale
    p, grads = r(n, scale=0.01), r(n)
    m, v, ema = r(n, scale=0.1), r(n).abs() * 0.01 + 1e-4, r(n, scale=0.01)
    return p, grads, m, v, ema


ADAM_HYPER = dict(lr=1e-3, b1=0.9, b2=0.999, eps=1e-8, decay=0.99)


# ================================================================================================ 1. mac_linear_fwd
# (M, segments as (k, ldx pad), n_out, ldy pad, bias vector, bias_const, act, workspace)
# workspace: "full" (mac_linear_workspace_bytes), "fit2" (room for exactly two split-K slices), None (no split-K).
# M = 1..64 with K % 32 == 0 and K / 8 <= 256 runs the 8-CTA cluster kernel; K = 2080 (slice 260) and K % 32 != 0 fall back
# to the sgemm; M >= 512 (with K >= 256) takes 128-wide tiles.  Segments of width 4 and 20 end inside a 16-wide k-block and
# inside a skinny K-slice.
LINEAR_CASES = [
    (1, [(512, 0)], 512, 0, True, 0.0, "NON", "full"),
    (37, [(4, 4), (20, 12), (488, 0)], 20, 4, True, 0.25, "SIGMOID", "full"),
    (64, [(2048, 0)], 36, 0, False, -0.5, "TANH", "full"),
    (64, [(2080, 0)], 512, 0, True, 0.0, "ELU", "full"),
    (65, [(1028, 0)], 512, 8, True, 0.1, "RELU_STD", "full"),
    (64, [(1028, 4)], 6144, 0, True, 0.0, "NON", None),
    (128, [(20, 4), (4, 0), (512, 0), (500, 12)], 512, 0, True, 0.0, "NON", "fit2"),
    (511, [(512, 0)], 512, 0, True, 0.0, "TANH", "full"),
    (512, [(512, 0)], 512, 4, False, 0.5, "SIGMOID", "fit2"),
    (700, [(256, 8), (256, 0)], 4, 0, True, 0.0, "ELU", "full"),
    (700, [(512, 0), (16, 0)], 36, 12, True, -0.3, "RELU_STD", None),
    (1, [(4, 0)], 4, 0, True, 0.0, "TANH", "full"),
    (12544, [(512, 0), (512, 0)], 512, 0, True, 0.0, "NON", "full"),
    (12544, [(1024, 4)], 20, 0, True, 0.0, "ELU", "full"),
    (12544, [(9216, 0)], 512, 0, True, 0.0, "ELU", "full"),
]


@pytest.mark.parametrize("M,segs,n_out,ldy_pad,with_b,bias_const,act,wsmode", LINEAR_CASES)
def test_linear_fwd_matches_fp64(M, segs, n_out, ldy_pad, with_b, bias_const, act, wsmode):
    lb = lib()
    g = gen(M * 7 + n_out + len(segs))
    xs = [strided(g, M, k, pad) for k, pad in segs]
    K = sum(k for k, _ in segs)
    W = randn(g, K, n_out, scale=K ** -0.5)
    b = randn(g, n_out) if with_b else None
    ldy = n_out + ldy_pad
    y = nanfill(M, ldy)
    if wsmode == "full":
        wsb = lb.mac_linear_workspace_bytes(M, K, n_out)
    elif wsmode == "fit2":
        wsb = COUNTER_BYTES + 2 * M * n_out * 4 + 64
    else:
        wsb = 0
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda") if wsb else None

    def call():
        L_.check(lb.mac_linear_fwd(ptrs(xs), ints([k for k, _ in segs]), ints([x.stride(0) for x in xs]), len(segs), L_.ptr(W),
                                   L_.ptr(b), bias_const, L_.ACT[act], L_.ptr(y), ldy, M, n_out, L_.ptr(ws), wsb,
                                   L_.stream_ptr()), "mac_linear_fwd")

    got, same = run_twice(call, {"y": y})
    z, az = linear_reference(xs, W, b, bias_const)
    ref = act_ref(act, z)
    rep = Report("mac_linear_fwd M=%d K=%s n_out=%d ldy=%d %s ws=%s" % (M, [k for k, _ in segs], n_out, ldy, act, wsmode))
    rep.add("y", got["y"][:, :n_out], ref, az, TOL_LINEAR, tiny=TINY_ACT * ref.abs())
    if ldy_pad:
        rep.check(bool(got["y"][:, n_out:].isnan().all()), "padding columns untouched")
    rep.check(same, "bit-identical rerun")
    rep.check(counters_zero(ws), "split-K counters zero")
    rep.done()


# ================================================================================================ 2. write unit
def write_setup(B, d, seed):
    g = gen(seed)
    W = {"Ww": randn(g, 3 * d, d, scale=(3 * d) ** -0.5), "bw": randn(g, d, scale=0.1), "Wg": randn(g, d, d, scale=d ** -0.5),
         "bg": randn(g, d, scale=0.1), "Wy": randn(g, d, d, scale=d ** -0.5), "by": randn(g, d, scale=0.1)}
    mem, info, ss, c = randn(g, B, d), randn(g, B, d), randn(g, B, d), randn(g, B, d)
    return g, W, mem, info, ss, c


# (B, d, self_smry, gate): B = 65 runs both products (and the gate's EPI_GATE epilogue) through the split-K sgemm instead of
# the cluster kernel; d = 20 is not a multiple of 32, so even B <= 64 takes the sgemm
WRITE_CASES = [(1, 20, False, True), (1, 64, True, False), (1, 512, True, True),
               (64, 20, True, True), (64, 64, False, True), (64, 512, True, False),
               (65, 20, False, True), (65, 64, True, True), (65, 512, False, True),
               (128, 20, True, False), (128, 64, False, True), (128, 512, True, True)]


@pytest.mark.parametrize("B,d,self_smry,gate", WRITE_CASES)
def test_write_fwd_matches_fp64(B, d, self_smry, gate):
    """m' = [memory, info(, self_smry)] @ Ww + bw, then the gate z = sigmoid(control @ Wg + bg + gate_bias) and
    m' z + memory (1 - z) from the kernel's own m' (left in the workspace) and z; without gate_out the same bits"""
    lb = lib()
    g, W, mem, info, ss, c = write_setup(B, d, B * 10 + d)
    gate_bias = -0.75
    nseg = 3 if self_smry else 2
    Ww = W["Ww"][:nseg * d].contiguous()
    wsb = lb.mac_write_workspace_bytes(B, d)
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    new_m, z = nanfill(B, d), nanfill(B, d)

    def call(out, gate_out):
        L_.check(lb.mac_write_fwd(L_.ptr(mem), L_.ptr(info), L_.ptr(ss) if self_smry else None, L_.ptr(c), L_.ptr(Ww),
                                  L_.ptr(W["bw"]), L_.ptr(W["Wg"]) if gate else None, L_.ptr(W["bg"]) if gate else None,
                                  gate_bias, L_.ptr(out), L_.ptr(gate_out), L_.ptr(ws), wsb, B, d, L_.stream_ptr()),
                 "mac_write_fwd")

    got, same = run_twice(lambda: call(new_m, z if gate else None), {"m": new_m, "z": z})
    rep = Report("mac_write_fwd B=%d d=%d%s%s" % (B, d, " self_smry" if self_smry else "", " gate" if gate else ""))
    xs = [mem, info] + ([ss] if self_smry else [])
    m1, am1 = linear_reference(xs, Ww, W["bw"], 0.0)
    if not gate:
        rep.add("new_memory", got["m"], m1, am1, TOL_WRITE)
        rep.check(bool(got["z"].isnan().all()), "gate_out untouched without a gate")
    else:
        tmp = ws[COUNTER_BYTES:COUNTER_BYTES + B * d * 4].view(torch.float32).view(B, d)
        rep.add("m' (workspace)", tmp, m1, am1, TOL_WRITE)
        pre, apre = linear_reference([c], W["Wg"], W["bg"], gate_bias)
        zr = torch.sigmoid(pre)
        rep.add("z", got["z"], zr, apre, TOL_WRITE, tiny=TINY_ACT * zr)
        zk, tk, md = got["z"].double(), tmp.double(), mem.double()
        rep.add("new_memory", got["m"], tk * zk + md * (1 - zk), tk.abs() * zk + md.abs() * (1 - zk) + md.abs() * zk,
                TOL_WRITE)
        again = nanfill(B, d)
        call(again, None)
        torch.cuda.synchronize()
        rep.check(same_bits(again, got["m"]), "gate_out NULL gives the same new_memory")
    rep.check(same, "bit-identical rerun")
    rep.check(counters_zero(ws), "split-K counters zero")
    rep.done()


@pytest.mark.parametrize("B,d", [(B, d) for B in (1, 64, 65, 128) for d in (20, 64, 512)])
def test_write_fwd_next_y_matches_fp64(B, d):
    """[memory, info] @ Wf + bf with Wf = [Ww | Ww @ Wy], bf = [bw | bw @ Wy + by] (built as the header describes): columns
    [0, d) to new_memory and [d, 2d) to y_next"""
    lb = lib()
    g, W, mem, info, _, _ = write_setup(B, d, B * 10 + d + 1)
    Ww = W["Ww"][:2 * d]
    Wf = torch.cat([Ww, Ww @ W["Wy"]], 1).contiguous()
    bf = torch.cat([W["bw"], W["bw"] @ W["Wy"] + W["by"]]).contiguous()
    wsb = lb.mac_write_workspace_bytes(B, d)
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    new_m, y_next = nanfill(B, d), nanfill(B, d)

    def call():
        L_.check(lb.mac_write_fwd_next_y(L_.ptr(mem), L_.ptr(info), L_.ptr(Wf), L_.ptr(bf), L_.ptr(new_m), L_.ptr(y_next),
                                         L_.ptr(ws), wsb, B, d, L_.stream_ptr()), "mac_write_fwd_next_y")

    got, same = run_twice(call, {"m": new_m, "y": y_next})
    z, az = linear_reference([mem, info], Wf, bf, 0.0)
    rep = Report("mac_write_fwd_next_y B=%d d=%d" % (B, d))
    rep.add("new_memory", got["m"], z[:, :d], az[:, :d], TOL_WRITE)
    rep.add("y_next", got["y"], z[:, d:], az[:, d:], TOL_WRITE)
    rep.check(same, "bit-identical rerun")
    rep.check(counters_zero(ws), "split-K counters zero")
    rep.done()


# ================================================================================================ 3. read unit (fp32)
def read_weights(g, d):
    W = {"Wx": randn(g, d, d, scale=d ** -0.5), "bx": randn(g, d, scale=0.1), "Wy": randn(g, d, d, scale=d ** -0.5),
         "by": randn(g, d, scale=0.1), "Wm": randn(g, 2 * d, d, scale=(2 * d) ** -0.5), "bm": randn(g, d, scale=0.1),
         "Wm2": randn(g, d, d, scale=d ** -0.5), "bm2": randn(g, d, scale=0.1), "wr": randn(g, d, scale=4 * d ** -0.5)}
    v = lambda t: t.data_ptr()
    rw = L_.ReadWeights(v(W["Wx"]), v(W["bx"]), v(W["Wy"]), v(W["by"]), v(W["Wm"]), v(W["bm"]), v(W["Wm2"]), v(W["bm2"]),
                        v(W["wr"]), 0.25, None, None, None, None, None, None, None)
    return W, rw


def read_ws_offsets(B, N, d):
    """byte offsets of md, y, P, H in the fp32 read workspace (read_ws_layout in csrc/units.cu)"""
    o, offs = COUNTER_BYTES, {}
    for name, n in (("md", B * d), ("y", B * d), ("P", B * N * d), ("H", B * N * d)):
        offs[name] = o
        o += (n * 4 + 255) & ~255
    return offs


def ws_floats(ws, off, *shape):
    n = int(np.prod(shape))
    return ws[off:off + n * 4].view(torch.float32).view(*shape)


# READ_CASES of the backward tests, plus: B*N >= 512 at d = 512 (128-wide tiles, 4 logit parts) and below it (64-wide, 8
# parts); N = 1; and the widths d % 16 != 0 of the fp32 path (4- and 8-column knowledge-base slices)
READ_FWD_CASES = READ_CASES + [
    (3, 49, 512, 1.0),
    (4, 1, 128, 0.85),
    (3, 49, 4, 0.85),
    (5, 33, 20, 1.0),
    (2, 300, 36, 0.85),
]


@pytest.mark.parametrize("B,N,d,keep", READ_FWD_CASES)
def test_read_fwd_fp32_matches_fp64(B, N, d, keep):
    """mac_read_fwd(MAC_PREC_FP32) with `save`: y, P, H, I1 stage by stage with the Philox masks, then att and info
    through the attention bound"""
    lb = lib()
    g = gen(B * 1000 + N * 10 + d + 5)
    W, rw = read_weights(g, d)
    kb = elu(randn(g, B, N, d))
    mem, c = randn(g, B, d), randn(g, B, d)
    seed, step, M = 4242, 5, B * N
    wsb = lb.mac_read_workspace_bytes(B, N, d, PREC_FP32)
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    save, info, att = nanfill(3 * M * d + B * d), nanfill(B, d), nanfill(B, N)

    def call():
        L_.check(lb.mac_read_fwd(L_.ptr(kb), None, L_.ptr(mem), L_.ptr(c), ctypes.byref(rw), keep, seed, step, PREC_FP32,
                                 L_.ptr(info), L_.ptr(att), L_.ptr(save), L_.ptr(ws), wsb, B, N, d, L_.stream_ptr()),
                 "mac_read_fwd")

    got, same = run_twice(call, {"save": save, "info": info, "att": att})
    sv = got["save"]
    P, H, I1 = (sv[i * M * d:(i + 1) * M * d].view(M, d) for i in range(3))
    y = sv[3 * M * d:].view(B, d)
    masks = read_masks(keep, seed, step, B, N, d, "cuda")
    r = read_forward_stages(kb, mem, W, masks, P, y, H)
    rep = Report("mac_read_fwd fp32 %s keep %.2f" % ((B, N, d), keep))
    for name, t in (("y", y), ("P", P), ("H", H), ("I1", I1)):
        rep.add(name, t, *r[name], TOL_READ)
    add_attention(rep, attention_bound_check(got["att"], got["info"], *r["I1"], c, W["wr"], 0.25, kb, B, N, TOL_READ,
                                             ms=masks[2]))
    rep.check(same, "bit-identical rerun")
    rep.check(counters_zero(ws), "split-K counters zero")
    rep.done()


@pytest.mark.parametrize("B,N,d", [(3, 49, 512), (64, 196, 512), (5, 33, 20), (2, 300, 36), (1, 1, 64)])
@pytest.mark.parametrize("with_y_pre", [False, True])
def test_read_inv_fp32_matches_fp64(B, N, d, with_y_pre):
    """mac_read_invariant at fp32 (P, Q read back from inv), then mac_read_fwd_inv: y (workspace, or the caller's y_pre),
    H = ELU((P*y) @ Wm[0:d] + Q) (workspace), att and info"""
    lb = lib()
    g = gen(B * 100 + N + d + with_y_pre)
    W, rw = read_weights(g, d)
    kb = elu(randn(g, B, N, d))
    mem, c, y_pre = randn(g, B, d), randn(g, B, d), randn(g, B, d)
    M = B * N
    nb = lb.mac_read_invariant_bytes(B, N, d, PREC_FP32)
    inv = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    inv[:2 * M * d * 4].view(torch.float32).fill_(float("nan"))
    L_.check(lb.mac_read_invariant(L_.ptr(kb), None, ctypes.byref(rw), PREC_FP32, L_.ptr(inv), nb, B, N, d, L_.stream_ptr()),
             "mac_read_invariant")
    wsb = lb.mac_read_workspace_bytes(B, N, d, PREC_FP32)
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    offs = read_ws_offsets(B, N, d)
    ws_floats(ws, offs["y"], B, d).fill_(float("nan"))
    ws_floats(ws, offs["H"], M, d).fill_(float("nan"))
    info, att = nanfill(B, d), nanfill(B, N)

    def call():
        L_.check(lb.mac_read_fwd_inv(L_.ptr(kb), None, L_.ptr(inv), L_.ptr(y_pre) if with_y_pre else None, L_.ptr(mem),
                                     L_.ptr(c), ctypes.byref(rw), PREC_FP32, L_.ptr(info), L_.ptr(att), L_.ptr(ws), wsb, B, N,
                                     d, L_.stream_ptr()), "mac_read_fwd_inv")

    got, same = run_twice(call, {"info": info, "att": att, "ws": ws})
    wk = got["ws"]
    P, Q = ws_floats(inv, 0, M, d), ws_floats(inv, M * d * 4, M, d)
    y = y_pre if with_y_pre else ws_floats(wk, offs["y"], B, d)
    H = ws_floats(wk, offs["H"], M, d)
    ones = read_masks(1.0, 0, 0, B, N, d, "cuda")
    r = read_forward_stages(kb, mem, W, ones, P, y, H)
    D = lambda t: t.double()
    Wm, bm = D(W["Wm"]), D(W["bm"])
    Pd, Qd = D(P), D(Q)
    PY = Pd * D(y).repeat_interleave(N, 0)
    rep = Report("mac_read_fwd_inv fp32 %s%s" % ((B, N, d), " y_pre" if with_y_pre else ""))
    rep.add("P", P, *r["P"], TOL_READ)
    rep.add("Q", Q, Pd @ Wm[d:] + bm, Pd.abs() @ Wm[d:].abs() + bm.abs(), TOL_READ)
    if not with_y_pre:
        rep.add("y", y, *r["y"], TOL_READ)
    rep.add("H", H, elu(PY @ Wm[:d] + Qd), PY.abs() @ Wm[:d].abs() + Qd.abs(), TOL_READ)
    add_attention(rep, attention_bound_check(got["att"], got["info"], *r["I1"], c, W["wr"], 0.25, kb, B, N, TOL_READ))
    rep.check(same, "bit-identical rerun")
    rep.check(counters_zero(wk), "split-K counters zero")
    rep.done()


@pytest.mark.parametrize("B,N,d", [(1, 4, 2112), (1, 512, 4224)])
@pytest.mark.parametrize("with_inv", [False, True])
def test_read_fp32_refuses_too_many_logit_parts(B, N, d, with_inv):
    """d = 2112 below 512 knowledge-base rows (64-wide tiles) and d = 4224 at B*N = 512 (128-wide tiles) need 33 partial
    logits per row: MAC_ERR_UNSUPPORTED before anything is launched or written"""
    lb = lib()
    g = gen(B + N + d)
    W, rw = read_weights(g, d)
    kb, mem, c = randn(g, B, N, d), randn(g, B, d), randn(g, B, d)
    M = B * N
    wsb = lb.mac_read_workspace_bytes(B, N, d, PREC_FP32)
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    save, info, att = nanfill(3 * M * d + B * d), nanfill(B, d), nanfill(B, N)
    inv = torch.zeros(lb.mac_read_invariant_bytes(B, N, d, PREC_FP32), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    before = lb.mac_b200_launch_count()
    if with_inv:
        st = lb.mac_read_fwd_inv(L_.ptr(kb), None, L_.ptr(inv), None, L_.ptr(mem), L_.ptr(c), ctypes.byref(rw), PREC_FP32,
                                 L_.ptr(info), L_.ptr(att), L_.ptr(ws), wsb, B, N, d, L_.stream_ptr())
    else:
        st = lb.mac_read_fwd(L_.ptr(kb), None, L_.ptr(mem), L_.ptr(c), ctypes.byref(rw), 0.85, 1, 0, PREC_FP32, L_.ptr(info),
                             L_.ptr(att), L_.ptr(save), L_.ptr(ws), wsb, B, N, d, L_.stream_ptr())
    torch.cuda.synchronize()
    assert st == ERR_UNSUPPORTED, st
    assert lb.mac_b200_launch_count() == before
    assert bool(save.isnan().all()) and bool(info.isnan().all()) and bool(att.isnan().all())
    assert not bool(ws.any())


def test_cell_fp32_at_d20_matches_oracle():
    """MACCell(prec="fp32") with the shipped flags at d = 20 (4-column knowledge-base slices) against the fp64 oracle"""
    from mac_network_b200.config import MACConfig
    from mac_network_b200.params import init_params, perturb_biases
    from mac_network_b200.synthetic import make_inputs
    from tests.test_gpu_parity import compare, run_gpu, run_oracle
    B, S, N, d, L = 5, 9, 50, 20, 3
    cfg = MACConfig.args("args", netLength=L, memDim=d, ctrlDim=d, attDim=d)
    inputs = make_inputs(B, S, N, d, seed=31, dtype=np.float64)
    params = perturb_biases(init_params(cfg, L, seed=32, dtype=np.float64), seed=33)
    got, _ = run_gpu(cfg, params, inputs, L)
    ref = run_oracle(cfg, params, inputs, L)
    worst = compare(got, ref, what="args d=20")
    print("MACCell fp32 d=20: %s" % ", ".join("%s %.1e" % kv for kv in sorted(worst.items())))


# ================================================================================================ 4. general-path primitives
ATTEND_CASES = [
    # (B, M, d, lengths or None, feature row padding)
    (2, 1, 3, None, 0),
    (3, 129, 129, [0, 129, 57], 3),
    (3, 129, 128, None, 0),
    (2, 129, 512, [200, 1], 8),
    (2, 12545, 512, [12545, 0], 0),
    (4, 12545, 3, [0, 12545, 100, -5], 1),
]


@pytest.mark.parametrize("B,M,d,lens,pad", ATTEND_CASES)
def test_attend_fwd_matches_fp64(B, M, d, lens, pad):
    """att = softmax(logits - 1e30 [m >= len]), out = sum_m att * feats: d not a multiple of the 128-column block, M = 12 545
    (more than 48 KB of logits in shared memory), lengths 0 (uniform) and >= M, feature rows step-major
    (bstride = d + pad, rstride = B (d + pad) != d), so feat_bstride != M * feat_rstride"""
    lb = lib()
    g = gen(B * 7 + M + d + pad)
    logits = randn(g, B, M, scale=3.0)
    ld = d + pad
    fbuf = randn(g, M, B, ld)
    feats = fbuf[:, :, :d].permute(1, 0, 2)                   # [B, M, d] view: bstride ld, rstride B * ld
    lengths = torch.tensor(lens, dtype=torch.int32, device="cuda") if lens is not None else None
    att, out = nanfill(B, M), nanfill(B, d)

    def call():
        L_.check(lb.mac_attend_fwd(L_.ptr(logits), L_.ptr(lengths), L_.ptr(fbuf), ld, B * ld, L_.ptr(att), L_.ptr(out), B, M,
                                   d, L_.stream_ptr()), "mac_attend_fwd")

    got, same = run_twice(call, {"att": att, "out": out})
    ln = torch.full((B,), M, device="cuda") if lengths is None else lengths.long().clamp(0, M)
    valid = torch.arange(M, device="cuda")[None, :] < ln[:, None]
    valid = valid | (ln[:, None] == 0)           # length 0: every logit is -1e30 in both, so the softmax is uniform
    ld_ = logits.double()
    a, aa = softmax_bound(ld_.masked_fill(ln[:, None] == 0, 0.0), ld_.abs().masked_fill(ln[:, None] == 0, 0.0), valid)
    F = feats.double()
    rep = Report("mac_attend_fwd B=%d M=%d d=%d lengths=%s pad=%d" % (B, M, d, lens, pad))
    rep.add("att", got["att"], a, aa, TOL_ATT)
    rep.add("out", got["out"], torch.einsum("bm,bmd->bd", a, F), torch.einsum("bm,bmd->bd", aa, F.abs()), TOL_ATT)
    rep.check(bool((got["att"][~valid] == 0).all()), "masked attention exactly zero")
    rep.check(same, "bit-identical rerun")
    rep.done()


ROWDOT_FWD_CASES = [
    (1, [(64, 4), (31, 1), (20, 0)]),
    (7, [(100, 0)]),
    (8, [(33, 3), (64, 0)]),
    (9, [(4, 4), (127, 1), (1, 7)]),
    (12544, [(64, 4), (36, 0), (97, 3)]),
    (12544, [(512, 0)]),
]


@pytest.mark.parametrize("R,segs", ROWDOT_FWD_CASES)
def test_rowdot_fwd_matches_fp64(R, segs):
    lb = lib()
    g = gen(R + sum(k for k, _ in segs))
    xs = [strided(g, R, k, pad) for k, pad in segs]
    Kt = sum(k for k, _ in segs)
    w = randn(g, Kt)
    b = -0.625
    out = nanfill(R)

    def call():
        L_.check(lb.mac_rowdot_fwd(ptrs(xs), ints([k for k, _ in segs]), ints([x.stride(0) for x in xs]), len(segs), L_.ptr(w),
                                   b, L_.ptr(out), R, L_.stream_ptr()), "mac_rowdot_fwd")

    got, same = run_twice(call, {"out": out})
    z, az = linear_reference(xs, w.view(-1, 1), None, b)
    rep = Report("mac_rowdot_fwd R=%d segs=%s" % (R, segs))
    rep.add("out", got["out"], z.view(-1), az.view(-1), TOL_ROWDOT)
    rep.check(same, "bit-identical rerun")
    rep.done()


def bcast_op_reference(x, v, mode, mb, bias):
    X, V = x.double(), v.double()[:, None, :]
    if mode == 0:
        return (X + mb) * (V + mb), (X.abs() + abs(mb)) * (V.abs() + abs(mb)), 0.0
    if mode == 1:
        bb = bias.double() if bias is not None else 0.0
        ab = bias.double().abs() if bias is not None else 0.0
        return X * V + bb, X.abs() * V.abs() + ab, 0.0
    r = torch.tanh(X + V)
    return r, X.abs() + V.abs(), TINY_ACT * r.abs()


@pytest.mark.parametrize("mode,with_bias", [(0, False), (1, True), (1, False), (2, False)])
@pytest.mark.parametrize("N,d", [(1, 7), (49, 130), (196, 512)])
def test_bcast_op_matches_fp64(mode, with_bias, N, d):
    lb = lib()
    B, mb = 3, 0.375
    g = gen(mode * 10 + N + d + with_bias)
    x, v = randn(g, B, N, d), randn(g, B, d)
    bias = randn(g, d) if with_bias else None
    out = nanfill(B, N, d)
    got, same = run_twice(lambda: L_.check(lb.mac_bcast_op(L_.ptr(x), L_.ptr(v), mode, mb, L_.ptr(bias), L_.ptr(out), B, N, d,
                                                           L_.stream_ptr()), "mac_bcast_op"), {"out": out})
    ref, absref, tiny = bcast_op_reference(x, v, mode, mb, bias)
    rep = Report("mac_bcast_op mode %d N=%d d=%d%s" % (mode, N, d, " bias" if with_bias else ""))
    rep.add("out", got["out"], ref, absref, TOL_ELEM, tiny=tiny)
    rep.check(same, "bit-identical rerun")
    rep.done()


@pytest.mark.parametrize("N,d", [(1, 4), (49, 20), (196, 512)])
def test_bcast_mul_in_place_matches_fp64(N, d):
    """out = (x + mb) * (v + mb) with out == x"""
    lb = lib()
    B, mb = 5, -0.25
    g = gen(N + d)
    x, v = randn(g, B, N, d), randn(g, B, d)
    ref, absref, _ = bcast_op_reference(x, v, 0, mb, None)
    L_.check(lb.mac_bcast_mul(L_.ptr(x), L_.ptr(v), mb, L_.ptr(x), B, N, d, L_.stream_ptr()), "mac_bcast_mul")
    torch.cuda.synchronize()
    rep = Report("mac_bcast_mul in place N=%d d=%d" % (N, d))
    rep.add("out", x, ref, absref, TOL_ELEM)
    rep.done()


@pytest.mark.parametrize("act", ["NON", "TANH", "SIGMOID", "ELU", "RELU_STD"])
def test_activation_matches_fp64(act):
    """|x| up to 100 (saturated tanh / sigmoid, ELU at -1), n not a multiple of the 256-thread block"""
    lb = lib()
    g = gen(L_.ACT[act] + 60)
    n = 256 * 41 + 77
    x = (torch.rand(n, device="cuda", generator=g) * 200 - 100).contiguous()
    x[:6] = torch.tensor([0.0, -0.0, 100.0, -100.0, 1e-30, -1e-30], device="cuda")
    out = nanfill(n)
    L_.check(lb.mac_activation(L_.ptr(x), L_.ACT[act], L_.ptr(out), n, L_.stream_ptr()), "mac_activation")
    torch.cuda.synchronize()
    ref = act_ref(act, x.double())
    rep = Report("mac_activation %s" % act)
    rep.add("out", out, ref, ref.abs(), TOL_ELEM, tiny=1e-37)
    rep.done()


# ================================================================================================ 5. bf16 casts
def cast_inputs(g, n):
    """random values over many binades, then the edge cases: ties to even (both directions), signed zeros, subnormals,
    infinities, the largest finite value (rounds to inf), NaN"""
    x = torch.randn(n, device="cuda", generator=g) * torch.pow(10.0, torch.randint(-30, 30, (n,), device="cuda",
                                                                                  generator=g).float())
    special = torch.tensor([0.0, -0.0, float("inf"), float("-inf"), 1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, -(1.0 + 2 ** -8),
                            1e-40, -1e-40, 1.4e-45, 3.4028235e38, -3.4028235e38, 1.17549435e-38, float("nan")],
                           device="cuda")
    x[:special.numel()] = special
    return x.contiguous()


def check_bf16_bits(got16, x, what):
    ref = x.to(torch.bfloat16).view(torch.int16)
    fin = ~x.isnan()
    assert torch.equal(got16.view(torch.int16)[fin], ref[fin]), what
    nb = got16.view(torch.int16)[~fin].int() & 0xffff
    assert bool(((nb & 0x7f80) == 0x7f80).all()) and bool(((nb & 0x007f) != 0).all()), what + ": NaN not kept"


@pytest.mark.parametrize("n", [4, 1 << 12, 64 * 196 * 512])
def test_cast_bf16_bit_exact(n):
    """mac_cast_bf16 against torch's round-to-nearest-even, and mac_host_cast_bf16 on the same finite inputs"""
    lb = lib()
    g = gen(n)
    x = cast_inputs(g, n) if n > 16 else torch.tensor([1.0 + 2 ** -8, -0.0, 1e-40, float("nan")], device="cuda")
    out = torch.empty(n, dtype=torch.bfloat16, device="cuda")
    L_.check(lb.mac_cast_bf16(L_.ptr(x), L_.ptr(out), n, L_.stream_ptr()), "mac_cast_bf16")
    torch.cuda.synchronize()
    check_bf16_bits(out, x, "mac_cast_bf16")
    xh = x.cpu().numpy()
    host = np.empty(n, np.int16)
    assert lb.mac_host_cast_bf16(xh.ctypes.data_as(ctypes.c_void_p), host.ctypes.data_as(ctypes.c_void_p), n, 4) == 0
    fin = ~np.isnan(xh)
    assert np.array_equal(host[fin], out.view(torch.int16).cpu().numpy()[fin]), "host and device casts differ"


@pytest.mark.parametrize("nslab", [1, 2, 3])
def test_widen_bf16_bit_exact(nslab):
    """n = 64 * 196 * 512: the grid-stride loop runs more than one pass over each slab"""
    lb = lib()
    n = 64 * 196 * 512
    g = gen(nslab)
    srcs = [cast_inputs(g, n).to(torch.bfloat16) for _ in range(nslab)]
    dsts = [nanfill(n) for _ in range(nslab)]
    L_.check(lb.mac_widen_bf16(ptrs(srcs), ptrs(dsts), nslab, n, L_.stream_ptr()), "mac_widen_bf16")
    torch.cuda.synchronize()
    for i, (s, dd) in enumerate(zip(srcs, dsts)):
        ref = s.float()
        fin = ~ref.isnan()
        assert same_bits(dd[fin], ref[fin]), "slab %d" % i
        assert bool(dd[~fin].isnan().all()), "slab %d NaN" % i


# ================================================================================================ 6. optimizer step
# (n, step, clip, ema): n = 592 * 256 + 1 and 5e6 run the norm reduction's grid-stride loop more than once
ADAM_CASES = [
    (1, 1, "active", True),
    (255, 2, "inactive", False),
    (255, 1000, "active", True),
    (592 * 256 + 1, 1000, "off", True),
    (592 * 256 + 1, 1, "inactive", True),
    (5_000_000, 2, "active", True),
    (5_000_000, 1, "off", False),
]


@pytest.mark.parametrize("n,step,clip,with_ema", ADAM_CASES)
def test_clip_adam_ema_step_matches_fp64(n, step, clip, with_ema):
    """from nonzero m, v and ema, grad_scale != 1, clipping active / inactive / off: the global norm against fp64, then
    m, v, p, ema element-wise against fp64 of the kernel's own inputs with the kernel's clip factor"""
    lb = lib()
    g = gen(n + step)
    p, grads, m, v, ema = adam_inputs(g, n, "cuda")
    if not with_ema:
        ema = None
    gs = 0.37
    true_norm = float(grads.double().norm()) * float(np.float32(gs))
    max_norm = {"active": 0.5 * true_norm, "inactive": 2.0 * true_norm, "off": 0.0}[clip]
    h = ADAM_HYPER
    norm_out = nanfill(2)
    wsb = lb.mac_optimizer_workspace_bytes()
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    pre = {"p": p.clone(), "m": m.clone(), "v": v.clone(), "ema": ema.clone() if ema is not None else None}

    def call():
        L_.check(lb.mac_clip_adam_ema_step(L_.ptr(p), L_.ptr(grads), L_.ptr(m), L_.ptr(v), L_.ptr(ema), n, gs, max_norm,
                                           h["lr"], h["b1"], h["b2"], h["eps"], step, h["decay"], L_.ptr(norm_out),
                                           L_.ptr(ws), wsb, L_.stream_ptr()), "mac_clip_adam_ema_step")

    got, same = run_twice(call, {"p": p, "m": m, "v": v, "ema": ema, "norm": norm_out})
    rep = Report("mac_clip_adam_ema_step n=%d step=%d clip %s%s" % (n, step, clip, "" if with_ema else " ema NULL"))
    norm = got["norm"].double()
    gsd = float(np.float32(gs))
    nref = grads.double().norm() * gsd
    rep.add("norm", norm[0:1], nref.view(1), nref.view(1), TOL_NORM)
    mn = float(np.float32(max_norm))
    cf_ref = mn / max(float(norm[0]), mn) if max_norm > 0 else 1.0
    rep.add("clip factor", norm[1:2], torch.tensor([cf_ref], dtype=torch.float64, device="cuda"),
            torch.tensor([cf_ref], dtype=torch.float64, device="cuda"), TOL_ADAM)
    r = adam_reference(pre["p"], grads, pre["m"], pre["v"], pre["ema"], float(norm[1]), gs, h["lr"], h["b1"], h["b2"],
                       h["eps"], step, h["decay"], got["m"], got["v"], got["p"])
    for k in ("m", "v", "p", "ema"):
        if k in r:
            ref, ab, tiny = r[k]
            rep.add(k, got[k], ref, ab, TOL_ADAM, tiny=tiny)
    rep.check(same, "bit-identical rerun")
    rep.done()


# ================================================================================================ 7. answer loss
def xent_reference(logits, labels, scale):
    """losses = logsumexp - l[label] and dlogits = (softmax - onehot) * scale with their bounds; a label outside [0, A)
    gives NaN and no one-hot"""
    Ld = logits.double()
    B, A = Ld.shape
    lab = labels.long()
    ok = (lab >= 0) & (lab < A)
    mx = Ld.amax(1)
    lse = mx + torch.log(torch.exp(Ld - mx[:, None]).sum(1))
    ll = Ld.gather(1, lab.clamp(0, A - 1)[:, None])[:, 0]
    loss = torch.where(ok, lse - ll, torch.full_like(lse, float("nan")))
    aloss = mx.abs() + (lse - mx).abs() + ll.abs()
    # expf(l - max) with l - max rounded to fp32: a relative error of the size of eps |l - max|
    p, ap = softmax_bound(Ld, (Ld - mx[:, None]).abs())
    onehot = torch.zeros_like(p)
    onehot[ok] = torch.nn.functional.one_hot(lab[ok], A).double()
    return loss, aloss, (p - onehot) * scale, (ap + onehot) * abs(scale)


@pytest.mark.parametrize("B", [1, 7, 8, 9, 300])
@pytest.mark.parametrize("A", [1, 31, 32, 33, 2000])
def test_softmax_xent_matches_fp64(B, A):
    """logits offset by 0, +1000 and -1000, scale != 1; for B >= 7 one label out of range (NaN loss, no one-hot)"""
    lb = lib()
    g = gen(B * 10 + A)
    scale = 1.0 / 48
    for off in (0.0, 1000.0, -1000.0):
        logits = (randn(g, B, A, scale=4.0) + off).contiguous()
        labels = torch.randint(0, A, (B,), device="cuda", generator=g, dtype=torch.int32)
        if B >= 7:
            labels[3] = A
        losses, dl = nanfill(B), nanfill(B, A)
        got, same = run_twice(lambda: L_.check(lb.mac_softmax_xent(L_.ptr(logits), L_.ptr(labels), L_.ptr(losses), L_.ptr(dl),
                                                                   scale, B, A, L_.stream_ptr()), "mac_softmax_xent"),
                              {"loss": losses, "dl": dl})
        loss, aloss, dref, adref = xent_reference(logits, labels, scale)
        ok = ~loss.isnan()
        rep = Report("mac_softmax_xent B=%d A=%d offset %g" % (B, A, off))
        rep.add("losses", got["loss"][ok], loss[ok], aloss[ok], TOL_XENT)
        rep.check(bool(got["loss"][~ok].isnan().all()), "out-of-range label gives NaN")
        rep.add("dlogits", got["dl"], dref, adref, TOL_XENT, tiny=1e-30)
        rep.check(same, "bit-identical rerun")
        rep.done()
