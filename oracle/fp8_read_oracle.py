"""fp64 restatement of the e4m3 (FP8) read step: MAC_PREC_FP8, mac_network_b200/csrc/read_step_fp8.cuh.

Every rounding the library makes on that path is restated here: e4m3 through torch.float8_e4m3fn (round to nearest even,
saturating at +-448), bf16 through torch.bfloat16; all other arithmetic is fp64.  It is the reference the kernel is tested
against (tests/test_gpu_read_step_fp8.py); the model-level error of the scheme is measured against the plain fp64 oracle
(oracle/mac_oracle.py).

    P8  = e4m3(P / sP_r),  sP_r = max|P_r| / 448                 P = bf16(bf16(KB) @ bf16(Wx) + bx), per row
    W8  = e4m3(W / sW_c),  sW_c = max_k |W[k, c]| / 448          Wm[0:d] and Wm2, per output column
    A8  = e4m3(P8 * (y_b / ay_b)),  ay_b = max|y_b|              per sample
    H   = ELU((A8 @ W1_8) * sP_r * ay_b * sW1_c + Q)             Q = bf16(P @ bf16(Wm[d:2d]) + bm)
    H8  = e4m3(H / sH_r),  sH_r = max|H_r| / 448                 per row
    I1  = (H8 @ W2_8) * sH_r * sW2_c + bm2;  logits = ELU(I1 * control_b) . wr + br
    att = softmax_n(logits);  info = sum_n att * bf16(KB)

An all-zero row or column has scale 0 and quantises to zeros.

quant_rows_f32, pack_weight_f32 and a8_f32 restate the three quantisers with the kernels' own fp32 operations instead, so
the library's bytes and scales are checked against them bit for bit (tests/test_gpu_read_step_fp8.py,
tests/test_gpu_fp8_kernels.py); the fp64 functions above them stay the model of the scheme.
"""
import torch

E4M3_MAX = 448.0


def e4m3(x):
    """x rounded to the nearest e4m3 value (ties to even), saturating at +-448; returned as fp64."""
    return torch.as_tensor(x).float().clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn).to(torch.float64)


def bf16(x):
    return torch.as_tensor(x).to(torch.bfloat16).to(torch.float64)


def _quantise(x, amax):
    """(e4m3(x / s), s) with s = amax / 448, amax broadcast against x; zeros and s = 0 where amax == 0."""
    s = amax / E4M3_MAX
    nz = amax > 0
    return e4m3(torch.where(nz, x / torch.where(nz, s, torch.ones_like(s)), torch.zeros_like(x))), s


def quant_rows(X):
    """Per-row scaling of X [M, K]: (X8 [M, K], s [M, 1])."""
    return _quantise(X, X.abs().amax(1, keepdim=True))


def pack_weight(W):
    """Per-output-column scaling of W [K, n_out] ([in, out], the reference's layout): (W8 [K, n_out], s [1, n_out]).
    The library stores W8 transposed ([out, in], K-major); the values are the same."""
    return _quantise(W, W.abs().amax(0, keepdim=True))


# ---- fp32 restatements of the quantisers: the kernels' own fp32 operations, so their bytes and scales compare bit for bit.
# Every division runs on full tensors (torch divides by a 0-d tensor as a product with its reciprocal).
def _quantise_f32(X, amax):
    """(e4m3(X / fp32(amax / 448)), fp32 amax / 448) with IEEE fp32 division, amax broadcast against X; zeros where
    amax == 0 (quant_rows_e4m3_kernel, pack_weight_fp8_kernel)."""
    s = amax / torch.full_like(amax, E4M3_MAX)
    sx, nz = s.expand_as(X).contiguous(), (amax > 0).expand_as(X)
    return e4m3(torch.where(nz, X / torch.where(nz, sx, torch.ones_like(sx)), torch.zeros_like(X))), s


def quant_rows_f32(X):
    """P8 and sP as mac_read_invariant computes them from the bf16 P (fp32 X [M, K]): (X8 [M, K] fp64, s [M] fp32)."""
    X = torch.as_tensor(X).float()
    X8, s = _quantise_f32(X, X.abs().amax(1, keepdim=True))
    return X8, s.reshape(-1)


def pack_weight_f32(W):
    """mac_pack_weight_fp8 of fp32 W [K, n_out] ([in, out]): (W8 [K, n_out] fp64 e4m3 values, sW [n_out] fp32)."""
    W = torch.as_tensor(W).float()
    W8, s = _quantise_f32(W, W.abs().amax(0, keepdim=True))
    return W8, s.reshape(-1)


def a8_f32(P8, y, N):
    """The read step's GEMM 1 operand, A8 = e4m3(P8 * fp32(y_b * fp32(1 / ay_b))), ay_b = max|y_b| (1 / ay_b = 0 for an
    all-zero y_b), from the e4m3 values P8 [B*N, d] and fp32 y [B, d]: fp64 [B*N, d]."""
    y = torch.as_tensor(y).float()
    ay = y.abs().amax(1, keepdim=True)
    nz = ay > 0
    iay = torch.where(nz, torch.ones_like(ay) / torch.where(nz, ay, torch.ones_like(ay)), torch.zeros_like(ay))
    ys = (y * iay.expand_as(y).contiguous()).repeat_interleave(N, 0)
    return e4m3(torch.as_tensor(P8).float() * ys)


def invariant(KB, Wx, bx, Wm, bm):
    """Step-invariant part, as mac_read_invariant computes it: (P, Q, P8, sP) for KB [M, d] and the fp32 weights."""
    d = Wx.shape[0]
    P = bf16(bf16(KB) @ bf16(Wx) + bx)
    Q = bf16(P @ bf16(Wm[d:]) + bm)
    P8, sP = quant_rows(P)
    return P, Q, P8, sP


def _elu(x):
    return torch.nn.functional.elu(x)


def read_step(P8, sP, Q, y, control, W1, s1, W2, s2, bm2, wr, br, KB, N):
    """One read step from the quantised operands: P8, Q [B*N, d], sP [B*N, 1]; y, control [B, d]; W1, W2 [d, d] ([in, out]
    e4m3 values) with their column scales s1, s2 [1, d]; bm2, wr [d]; br scalar; KB [B*N, d] (rounded to bf16 here, as
    kb_attend reads it).  Returns (att [B, N], info [B, d])."""
    f64 = lambda t: torch.as_tensor(t, dtype=torch.float64)
    P8, sP, Q, y, control = f64(P8), f64(sP).reshape(-1, 1), f64(Q), f64(y), f64(control)
    W1, s1, W2, s2 = f64(W1), f64(s1).reshape(1, -1), f64(W2), f64(s2).reshape(1, -1)
    bm2, wr, KB = f64(bm2), f64(wr), f64(KB)
    B, d = y.shape
    rows = lambda v: v.repeat_interleave(N, 0)
    ay = y.abs().amax(1, keepdim=True)
    yn = torch.where(ay > 0, y / torch.where(ay > 0, ay, torch.ones_like(ay)), torch.zeros_like(y))
    A8 = e4m3(P8 * rows(yn))
    H = _elu((A8 @ W1) * sP * rows(ay) * s1 + Q)
    H8, sH = quant_rows(H)
    I1 = (H8 @ W2) * sH * s2 + bm2
    logits = (_elu(I1 * rows(control)) @ wr + float(br)).reshape(B, N)
    att = torch.softmax(logits, 1)
    info = torch.einsum("bn,bnd->bd", att, bf16(KB).reshape(B, N, d))
    return att, info


def read_step_from_weights(KB, y, control, Wx, bx, Wm, bm, Wm2, bm2, wr, br, N):
    """The whole step from the fp32 weights ([in, out]) and the fp32 knowledge base [B*N, d]."""
    f64 = lambda t: torch.as_tensor(t, dtype=torch.float64)
    KB, Wx, bx, Wm, bm, Wm2 = f64(KB), f64(Wx), f64(bx), f64(Wm), f64(bm), f64(Wm2)
    d = Wx.shape[0]
    _, Q, P8, sP = invariant(KB, Wx, bx, Wm, bm)
    W1, s1 = pack_weight(Wm[:d])
    W2, s2 = pack_weight(Wm2)
    return read_step(P8, sP, Q, y, control, W1, s1, W2, s2, bm2, wr, br, KB, N)
