"""Weight-derived tensors -- bf16, split-bf16, e4m3 and transposed copies of fp32 weights, and structures of pointers into
them -- and the one cache that keeps them until the weights they were built from change.

The pack builders take an fp32 [in, out] weight and return what the kernels read; each is the only host-side spelling of
its layout (include/mac_b200.h).  Those that launch a kernel take the caller's stream, as every entry point does.
"""
import torch

from . import _lib
from ._lib import check, ptr


class Cache(object):
    """Entries built on first use and kept until `clear()`, or until `version()` (optional callable, e.g.
    `lambda: params.version`) returns another value than it did when they were built: whoever moved the weights (optimizer
    step, EMA swap, checkpoint restore), the next lookup rebuilds from the new values."""

    def __init__(self, version=None):
        self._version_fn, self._version = version, None
        self._entries = {}

    def clear(self):
        self._entries.clear()

    def get(self, key, build):
        if self._version_fn is not None:
            v = self._version_fn()
            if v != self._version:
                self._entries.clear()
                self._version = v
        if key not in self._entries:
            self._entries[key] = build()
        return self._entries[key]

    def pack(self, builder, W, *args, **kw):
        """builder(W, *args, **kw), keyed by the builder, W's address and shape and `args`; `kw` (the stream) is not part
        of the key.  `Wm[:d]` and `Wm` share an address.  Only for tensors that live as long as the entry -- parameter
        views, or entries of this cache -- so an address is never reused meanwhile."""
        return self.get((builder, W.data_ptr(), W.shape, args), lambda: builder(W, *args, **kw))


def bf16(W, stream):
    """bf16 [out, in]: the K-major B operand of wgmma (mac_pack_weight_bf16)."""
    o = torch.empty((W.shape[1], W.shape[0]), dtype=torch.bfloat16, device=W.device)
    check(_lib.load().mac_pack_weight_bf16(ptr(W), ptr(o), W.shape[0], W.shape[1], stream), "mac_pack_weight_bf16")
    return o


def bf16_kpad(W, Kp, stream):
    """bf16 [out, Kp] with zero columns in..Kp-1 (mac_pack_weight_bf16_kpad)."""
    o = torch.empty((W.shape[1], Kp), dtype=torch.bfloat16, device=W.device)
    check(_lib.load().mac_pack_weight_bf16_kpad(ptr(W), ptr(o), W.shape[0], Kp, W.shape[1], stream),
          "mac_pack_weight_bf16_kpad")
    return o


def bf16_split(W, stream):
    """(hi, lo): the bf16 halves [out, in] of W, hi + lo ~ W (mac_pack_weight_bf16_split)."""
    hi = torch.empty((W.shape[1], W.shape[0]), dtype=torch.bfloat16, device=W.device)
    lo = torch.empty_like(hi)
    check(_lib.load().mac_pack_weight_bf16_split(ptr(W), ptr(hi), ptr(lo), W.shape[0], W.shape[1], stream),
          "mac_pack_weight_bf16_split")
    return hi, lo


def split3(W, stream):
    """bf16 [out, 3*in] = [hi | hi | lo] (mac_pack_weight_split3)."""
    o = torch.empty((W.shape[1], 3 * W.shape[0]), dtype=torch.bfloat16, device=W.device)
    check(_lib.load().mac_pack_weight_split3(ptr(W), ptr(o), W.shape[0], W.shape[1], stream),
          "mac_pack_weight_split3")
    return o


def fp8(W, stream):
    """(Wt, scale): e4m3 [out, in] and the fp32 scale of each output column (mac_pack_weight_fp8)."""
    o = torch.empty((W.shape[1], W.shape[0]), dtype=torch.uint8, device=W.device)
    s = torch.empty(W.shape[1], dtype=torch.float32, device=W.device)
    check(_lib.load().mac_pack_weight_fp8(ptr(W), ptr(o), ptr(s), W.shape[0], W.shape[1], stream),
          "mac_pack_weight_fp8")
    return o, s


def transposed(W):
    """fp32 [out, in]: the weight operand of mac_linear_bwd's data gradients."""
    return W.t().contiguous()
