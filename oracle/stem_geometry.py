"""ORACLE (test infrastructure only): fp64 restatement of the reference's image stem for every geometry its flags allow.

  * `model.py:165-204`  stem: `--stemLinear` -> `ops.linear(images, inDim, outDim)` (no dropout, no activation); else
                        `ops.CNNLayer(images, dims, dropout, kernelSizes=--stemKernelSizes, strides=--stemStrideSizes)`;
                        then reshape to the knowledge base `[B, Ho*Wo, outDim]`
  * `ops.py:380-405`    cnn: dropout on the layer INPUT, `tf.nn.conv2d(strides=[1, s, s, 1], padding="SAME")` with an HWIO
                        kernel of size `--stemKernelSize` (or the layer's entry of `--stemKernelSizes`), + bias, activation
  * TF's SAME padding:  Ho = ceil(H / s), pad_total = max((Ho - 1) s + k - H, 0), pad_top = pad_total // 2 (the odd row on
                        the bottom); the same for the width

Written with torch.nn.functional.conv2d on explicitly padded fp64 tensors, so it shares nothing with the product's
patch passes and differentiates with torch.autograd.  Pinned by `tests/golden/stem_geom_*.npz` (the reference's own stem
on the TF1 shim, `oracle/gen_stem_geometry.py`)."""
import numpy as np
import torch
import torch.nn.functional as F

LINEAR_W, LINEAR_B = "stem/linearLayer/weights/weight", "stem/linearLayer/biases/bias"


def same_pads(n, k, s):
    """(before, after) SAME padding of one spatial extent."""
    no = -(-n // s)
    total = max((no - 1) * s + k - n, 0)
    return total // 2, total - total // 2


def _act(relu, y):
    return F.elu(y) if relu == "ELU" else torch.clamp(y, min=0)


def stem_torch(relu, params, images, keep=1.0, uniforms=None, strides=None, linear=False):
    """The knowledge base [B, Ho*Wo, outDim] from torch fp64 tensors (params: name -> tensor, images [B,H,W,C]), in the
    autograd graph.  `uniforms[i]` [B, H_i, W_i, C_i]: the uniform draws of layer i's input dropout."""
    x = images
    if linear:
        y = x.reshape(-1, x.shape[-1]) @ params[LINEAR_W] + params[LINEAR_B]
        return y.reshape(x.shape[0], -1, y.shape[-1])
    n = len([k for k in params if k.endswith("kernels/kernel")])
    strides = [1] * n if strides is None else list(strides)
    us = iter(uniforms or [])
    for i in range(n):
        K = params["stem/cnnLayercnn_%d/kernels/kernel" % i]
        b = params["stem/cnnLayercnn_%d/biases/bias" % i]
        if float(keep) != 1.0:
            u = next(us)
            u = u.to(x) if torch.is_tensor(u) else torch.as_tensor(np.asarray(u), dtype=x.dtype, device=x.device)
            x = x / keep * torch.floor(keep + u)
        k, s = int(K.shape[0]), strides[i]
        ph, pw = same_pads(x.shape[1], k, s), same_pads(x.shape[2], k, s)
        xn = F.pad(x.permute(0, 3, 1, 2), (pw[0], pw[1], ph[0], ph[1]))
        y = F.conv2d(xn, K.permute(3, 2, 0, 1), bias=b, stride=s)
        x = _act(relu, y).permute(0, 2, 3, 1)
    return x.reshape(x.shape[0], -1, x.shape[-1])


def stem_forward(relu, params, images, keep=1.0, uniforms=None, strides=None, linear=False):
    """`stem_torch` on numpy inputs; returns the fp64 knowledge base as numpy."""
    p = {k: torch.as_tensor(np.asarray(v, np.float64)) for k, v in params.items()}
    x = torch.as_tensor(np.asarray(images, np.float64))
    return stem_torch(relu, p, x, keep, uniforms, strides, linear).numpy()


def _f64(v, device=None):
    if torch.is_tensor(v):
        return v.detach().to(dtype=torch.float64, device=device or v.device).clone()
    return torch.as_tensor(np.asarray(v, np.float64), device=device)


def stem_grads(relu, params, images, keep, uniforms, d_kb, strides=None, linear=False):
    """(kb, {name: gradient}, d_images) of sum(kb * d_kb), all fp64 numpy.  Inputs are numpy arrays or tensors; the graph
    runs on the images' device."""
    x = _f64(images).requires_grad_(True)
    p = {k: _f64(v, x.device).requires_grad_(True) for k, v in params.items()}
    kb = stem_torch(relu, p, x, keep, uniforms, strides, linear)
    (kb * _f64(d_kb, x.device)).sum().backward()
    return kb.detach().cpu().numpy(), {k: v.grad.cpu().numpy() for k, v in p.items()}, x.grad.cpu().numpy()
