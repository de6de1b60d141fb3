"""ORACLE (test infrastructure only): fp64 restatement of the reference's location-aware image stem (--locationAware).

  * `model.py:165-204`  stem: in the CNN branch only, `ops.addLocation(images, inDim, locationDim, locType=...)` on the
                        NHWC features before `ops.CNNLayer`; layer 0 then has Cin = inDim + l
  * `ops.py:514-559`    addLocation, mod CNCT, outDim -1: the grid is tiled over the batch and concatenated AFTER the image
                        channels; no variable is created
  * `ops.py:448-464`    L: l = 2, [x, y] with x = linspace(-b, b, W)[w], y = linspace(-b, b, H)[h] (tf.meshgrid's "xy")
  * `ops.py:466-488`    PE: l = 4 dim, [sin x_i | cos x_i | sin y_i | cos y_i], x_i = x / 10000^(i / dim)
  * `ops.py:380-405`    cnn: the dropout covers layer 0's whole input, location channels included

The grid is written here in torch fp64 on its own; the convolutions are `oracle.stem_geometry.stem_torch` on the
concatenated input, so the gradients come from torch.autograd.  Pinned by `tests/golden/stem_loc_*.npz` (the reference's
own stem on the TF1 shim, `oracle/gen_stem_location.py`)."""
import numpy as np
import torch

from oracle.stem_geometry import _f64, stem_torch


def grid_torch(kind, bias, dim, H, W, dtype=torch.float64, device=None):
    """The location grid [H, W, l]."""
    def lin(n):
        if n == 1:
            return torch.full((1,), -float(bias), dtype=dtype, device=device)
        return -float(bias) + 2.0 * float(bias) * torch.arange(n, dtype=dtype, device=device) / (n - 1)
    x = lin(W)[None, :, None].expand(H, W, 1)
    y = lin(H)[:, None, None].expand(H, W, 1)
    if kind == "L":
        return torch.cat([x, y], dim=-1)
    f = torch.pow(torch.tensor(10000.0, dtype=dtype, device=device), torch.arange(dim, dtype=dtype, device=device) / dim)
    return torch.cat([torch.sin(x / f), torch.cos(x / f), torch.sin(y / f), torch.cos(y / f)], dim=-1)


def with_location(images, location):
    """concat(images, grid) on the channel axis, the grid broadcast over the batch."""
    kind, bias, dim = location
    B, H, W, _ = images.shape
    g = grid_torch(kind, bias, dim, H, W, dtype=images.dtype, device=images.device)
    return torch.cat([images, g[None].expand(B, H, W, g.shape[-1])], dim=-1)


def stem_loc_torch(relu, params, images, location, keep=1.0, uniforms=None, strides=None):
    """The knowledge base [B, Ho*Wo, outDim]; `uniforms[0]` covers layer 0's whole input [B, H, W, C + l]."""
    return stem_torch(relu, params, with_location(images, location), keep, uniforms, strides)


def stem_loc_grads(relu, params, images, location, keep, uniforms, d_kb, strides=None):
    """(kb, {name: gradient}, d_images) of sum(kb * d_kb), fp64 numpy; the graph runs on the images' device."""
    x = _f64(images).requires_grad_(True)
    p = {k: _f64(v, x.device).requires_grad_(True) for k, v in params.items()}
    kb = stem_loc_torch(relu, p, x, location, keep, uniforms, strides)
    (kb * _f64(d_kb, x.device)).sum().backward()
    return kb.detach().cpu().numpy(), {k: v.grad.cpu().numpy() for k, v in p.items()}, x.grad.cpu().numpy()


def stem_loc_forward(relu, params, images, location, keep=1.0, uniforms=None, strides=None):
    p = {k: torch.as_tensor(np.asarray(v, np.float64)) for k, v in params.items()}
    x = torch.as_tensor(np.asarray(images, np.float64))
    return stem_loc_torch(relu, p, x, location, keep, uniforms, strides).numpy()
