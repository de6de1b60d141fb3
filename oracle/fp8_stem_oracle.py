"""Restatement of the e4m3 (FP8) inference stem: Stem(prec="fp8"), mac_network_b200/csrc/tc_gemm_fp8.cuh.

The row scales and the patch quantisation use the kernels' own fp32 operations (so bytes and scales compare bit for bit);
e4m3 rounding goes through torch.float8_e4m3fn (round to nearest even, saturating at +-448); the products are fp64.

    amax_m = max |x| over the in-image pixels of output pixel m's 3x3 window          fp32
    sA_m   = amax_m / 448;   cols8[m, k] = e4m3(patch[m, k] * (448 / amax_m))         fp32 division and product
    W8     = e4m3(W / sW_n), sW_n = max_k |W[k, n]| / 448                             per output column (fp32 pack)
    y      = act((cols8 @ W8) * sA_m * sW_n + b_n)                                    fp64, stored as fp32

A window that is all zero has sA = 0, zero bytes and y = act(b).
"""
import numpy as np
import torch

from oracle.fp8_read_oracle import E4M3_MAX, e4m3, pack_weight_f32


def im2col3x3(x):
    """x [B, H, W, C] -> patch matrix [B*H*W, 9*C] (tap-major, channel fastest; zero outside the image), same dtype."""
    x = torch.as_tensor(x)
    B, H, W, C = x.shape
    xp = torch.nn.functional.pad(x, (0, 0, 1, 1, 1, 1))
    return torch.cat([xp[:, i:i + H, j:j + W, :] for i in range(3) for j in range(3)], dim=-1).reshape(B * H * W, 9 * C)


def window_amax(x):
    """fp32 [B*H*W]: max |x| over each output pixel's 3x3 window (the padding contributes 0)."""
    x = torch.as_tensor(x, dtype=torch.float32)
    pa = x.abs().amax(-1)                                          # per input pixel
    B, H, W = pa.shape
    pp = torch.nn.functional.pad(pa, (1, 1, 1, 1))
    win = torch.stack([pp[:, i:i + H, j:j + W] for i in range(3) for j in range(3)], 0)
    return win.amax(0).reshape(B * H * W)


def quant_patches(x):
    """(cols8 [M, 9C] fp64 e4m3 values, sA [M] fp32) exactly as mac_im2col3x3_fp8 computes them from fp32 x [B, H, W, C]."""
    x = torch.as_tensor(x, dtype=torch.float32)
    am = window_amax(x)
    c448 = torch.full_like(am, E4M3_MAX)        # a full tensor: torch divides by a scalar as a product with its reciprocal
    sA = am / c448
    inv = torch.where(am > 0, c448 / torch.where(am > 0, am, torch.ones_like(am)), torch.zeros_like(am))
    return e4m3(im2col3x3(x) * inv[:, None]), sA


def pack_weight(W):
    """(W8 [K, n_out] fp64 e4m3 values, sW [n_out] fp32) as mac_pack_weight_fp8 computes them from fp32 W [K, n_out]."""
    return pack_weight_f32(W)


def _act(y, relu):
    return torch.nn.functional.elu(y) if relu == "ELU" else torch.relu(y)


def linear(cols8, sA, W8, sW, b, relu="ELU"):
    """fp64 y = act((cols8 @ W8) * sA * sW + b) from the quantised operands (W8 [K, n_out] in the [in, out] layout)."""
    f64 = lambda t: torch.as_tensor(t).to(torch.float64)
    y = (f64(cols8) @ f64(W8)) * f64(sA).reshape(-1, 1) * f64(sW).reshape(1, -1)
    if b is not None:
        y = y + f64(b)
    return y if relu is None else _act(y, relu)


def _f32(v, device):
    return torch.as_tensor(v if torch.is_tensor(v) else np.asarray(v), dtype=torch.float32, device=device)


def stem_forward(relu, params, images, device=None):
    """The whole e4m3 stem on fp32 images [B, H, W, C] and the fp32 HWIO kernels / biases (numpy arrays or tensors): the
    knowledge base [B, H*W, outDim] in fp64 (each layer's output is rounded to fp32 before the next quantisation, as the
    kernels store it).  `device`: where to compute (default: the images' device, or the CPU)."""
    device = device or (images.device if torch.is_tensor(images) else "cpu")
    x = _f32(images, device)
    nlayers = len([k for k in params if k.endswith("kernels/kernel")])
    B, H, W, _ = x.shape
    for i in range(nlayers):
        K = _f32(params["stem/cnnLayercnn_%d/kernels/kernel" % i], device)
        b = _f32(params["stem/cnnLayercnn_%d/biases/bias" % i], device)
        cols8, sA = quant_patches(x)
        W8, sW = pack_weight(K.reshape(-1, K.shape[3]))
        y = linear(cols8, sA, W8, sW, b, relu)
        x = y.to(torch.float32).reshape(B, H, W, -1)
    return y.reshape(B, H * W, -1)
