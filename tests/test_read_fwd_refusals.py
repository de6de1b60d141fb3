"""Refusals of the read unit's forward entry points (mac_read_fwd, mac_read_fwd_inv, mac_read_invariant): every MAC_ERR_*
a form can return comes back before any launch and before any write (include/mac_b200.h, csrc/read_fwd.cuh).

Each case names the call, the precision and shape that pick the form, and one defect: a missing pack or knowledge base, a d
the form's tiles do not take, more than 32 partial logits per row, a workspace or `inv` one byte short, or a pointer 8 bytes
off its 16-byte alignment.  The CPU test hands the library aligned host buffers that it never dereferences: a CUDA call
before the refusal comes back as a CUDA error (35 without a driver) instead of the expected code.  Its GPU twin hands it
device buffers (NaN-filled info, att and save, a zeroed workspace and inv) and checks that they stay untouched."""
import ctypes

import pytest
import torch

from mac_network_b200 import _lib as L_

INVALID, ALIGN, UNSUPPORTED, WORKSPACE = -1, -2, -3, -4
FP32, BF16, TC32, FP8 = 0, 1, 2, 3
PACKS = ["Wx_bf16", "Wm_bf16", "Wm2_bf16", "Wx_s3", "Wma_s3", "Wmb_s3", "Wm2_s3", "Wm_fp8", "Wm_fp8_scale", "Wm2_fp8",
         "Wm2_fp8_scale", "Wm_s3"]
SMALL, STEP = (2, 9), (2, 49)           # (B, N): any form; the fused read step's shapes (with d = 512)


def case(call, prec, d, expect, BN=SMALL, keep=1.0, drop=(), odd=(), short=False):
    return pytest.param(dict(call=call, prec=prec, d=d, B=BN[0], N=BN[1], keep=keep, drop=drop, odd=odd, short=short),
                        expect, id="%s-%s-d%d%s%s%s%s" % (call, ["fp32", "bf16", "tc32", "fp8"][prec], d,
                                                           "-keep%g" % keep if keep < 1 else "",
                                                           "".join("-no_" + k for k in drop), "".join("-odd_" + k for k in odd),
                                                           "-short" if short else ""))


CASES = [
    # d the tensor-core forms' 128-wide tiles do not take
    case("fwd", BF16, 192, UNSUPPORTED),
    case("fwd", BF16, 192, UNSUPPORTED, keep=0.5),
    case("fwd", TC32, 192, UNSUPPORTED),
    case("fwd_inv", BF16, 192, UNSUPPORTED),
    case("fwd_inv", TC32, 192, UNSUPPORTED),
    case("invariant", BF16, 192, UNSUPPORTED),
    case("invariant", TC32, 192, UNSUPPORTED),
    # more than 32 partial logits per row (the fused steps take d = 512 only: one logit per row)
    case("fwd", FP32, 4100, UNSUPPORTED),
    case("fwd", FP32, 2112, UNSUPPORTED),
    case("fwd_inv", FP32, 2112, UNSUPPORTED),
    case("fwd", BF16, 8192, UNSUPPORTED),
    case("fwd", BF16, 4224, UNSUPPORTED),
    case("fwd_inv", BF16, 4224, UNSUPPORTED),
    case("fwd", TC32, 4224, UNSUPPORTED),
    case("fwd_inv", TC32, 4224, UNSUPPORTED),
    # the packs and the bf16 knowledge base each form reads
    *[case("fwd", BF16, 128, INVALID, drop=(k,)) for k in ("kb_bf16", "Wx_bf16", "Wm_bf16", "Wm2_bf16")],
    *[case("fwd_inv", BF16, 128, INVALID, drop=(k,)) for k in ("Wm_bf16", "Wm2_bf16")],
    *[case("fwd_inv", BF16, 512, INVALID, BN=STEP, drop=(k,)) for k in ("Wm_bf16", "Wm2_bf16")],
    *[case("fwd", TC32, 128, INVALID, drop=(k,)) for k in ("Wx_s3", "Wm_s3", "Wm2_s3")],
    *[case("fwd_inv", TC32, 128, INVALID, drop=(k,)) for k in ("Wma_s3", "Wm2_s3")],
    *[case("fwd_inv", FP8, 512, INVALID, BN=STEP, drop=(k,)) for k in ("Wm_fp8", "Wm_fp8_scale", "Wm2_fp8", "Wm2_fp8_scale")],
    *[case("invariant", BF16, 128, INVALID, drop=(k,)) for k in ("kb_bf16", "Wx_bf16", "Wm_bf16")],
    *[case("invariant", TC32, 128, INVALID, drop=(k,)) for k in ("kb", "Wx_s3", "Wmb_s3")],
    *[case("invariant", FP8, 512, INVALID, BN=STEP, drop=(k,)) for k in ("Wx_bf16", "Wm_bf16")],
    # a workspace or inv one byte short
    *[case("fwd", p, 128, WORKSPACE, short=True) for p in (FP32, BF16, TC32)],
    *[case("fwd_inv", p, 128, WORKSPACE, short=True) for p in (FP32, BF16, TC32)],
    *[case("fwd_inv", p, 512, WORKSPACE, BN=STEP, short=True) for p in (BF16, FP8)],
    *[case("invariant", p, 128, WORKSPACE, short=True) for p in (FP32, BF16, TC32)],
    case("invariant", FP8, 512, WORKSPACE, BN=STEP, short=True),
    # misalignment
    case("fwd", FP32, 128, ALIGN, odd=("ws",)),
    case("fwd", BF16, 128, ALIGN, odd=("kb_bf16",)),
    case("fwd", BF16, 128, ALIGN, odd=("save",)),
    case("fwd", TC32, 128, ALIGN, odd=("Wm_s3",)),
    case("fwd_inv", BF16, 128, ALIGN, odd=("Wm_bf16",)),
    case("fwd_inv", BF16, 512, ALIGN, BN=STEP, odd=("kb_bf16",)),
    case("fwd_inv", FP8, 512, ALIGN, BN=STEP, odd=("Wm2_fp8",)),
    case("invariant", BF16, 128, ALIGN, odd=("kb_bf16",)),
    case("invariant", TC32, 128, ALIGN, odd=("Wx_s3",)),
    case("invariant", FP8, 512, ALIGN, BN=STEP, odd=("inv",)),
]


def call(lib, c, ops, info, att, save, ws, inv):
    """Run case c with every operand (knowledge bases, memory, control, weights and packs) at address `ops`."""
    prec, B, N, d = c["prec"], c["B"], c["N"], c["d"]
    ptr = lambda name, base: None if name in c["drop"] else base + (8 if name in c["odd"] else 0)
    rw = L_.ReadWeights()
    for f, _ in L_.ReadWeights._fields_:
        if f != "br":
            setattr(rw, f, ptr(f, ops))
    kb, kb16, save, ws, inv = ptr("kb", ops), ptr("kb_bf16", ops), ptr("save", save), ptr("ws", ws), ptr("inv", inv)
    if c["call"] == "invariant":
        nb = lib.mac_read_invariant_bytes(B, N, d, prec) - (1 if c["short"] else 0)
        return lib.mac_read_invariant(kb, kb16, ctypes.byref(rw), prec, inv, nb, B, N, d, None)
    wsb = lib.mac_read_workspace_bytes(B, N, d, prec) - (1 if c["short"] else 0)
    if c["call"] == "fwd_inv":
        return lib.mac_read_fwd_inv(kb, kb16, inv, None, ops, ops, ctypes.byref(rw), prec, info, att, ws, wsb, B, N, d, None)
    return lib.mac_read_fwd(kb, kb16, ops, ops, ctypes.byref(rw), c["keep"], 1, 0, prec, info, att, save, ws, wsb, B, N, d,
                            None)


@pytest.mark.parametrize("c,expect", CASES)
def test_read_fwd_refuses_before_any_cuda_call(c, expect):
    if torch.cuda.is_available():
        pytest.skip("host pointers stand in for device buffers: the GPU twin below covers this device")
    lib = L_.load()
    buf = (ctypes.c_char * 4096)()
    p = (ctypes.addressof(buf) + 15) & ~15              # 16-byte aligned, never dereferenced
    before = lib.mac_b200_launch_count()
    st = call(lib, c, p, p, p, p, p, p)
    assert st == expect, st
    assert lib.mac_b200_launch_count() == before


@pytest.mark.gpu
@pytest.mark.parametrize("c,expect", CASES)
def test_read_fwd_refuses_before_any_launch_or_write(c, expect):
    lib = L_.load()
    prec, B, N, d = c["prec"], c["B"], c["N"], c["d"]
    M = B * N
    # every operand at one zeroed buffer as large as the largest of them (the [d, 6d] bf16 Wm_s3 pack, inv, the knowledge base)
    ops = torch.zeros(max(12 * d * d, 8 * d * d + 64, M * d * 4 + 64), dtype=torch.uint8, device="cuda")
    nan = lambda n: torch.full((n,), float("nan"), device="cuda")
    info, att, save = nan(B * d), nan(M), nan(3 * M * d + B * d + 4)
    ws = torch.zeros(lib.mac_read_workspace_bytes(B, N, d, prec) + 64, dtype=torch.uint8, device="cuda")
    inv = torch.zeros(lib.mac_read_invariant_bytes(B, N, d, prec) + 64, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    before = lib.mac_b200_launch_count()
    st = call(lib, c, ops.data_ptr(), info.data_ptr(), att.data_ptr(), save.data_ptr(), ws.data_ptr(), inv.data_ptr())
    torch.cuda.synchronize()
    assert st == expect, st
    assert lib.mac_b200_launch_count() == before
    assert bool(info.isnan().all()) and bool(att.isnan().all()) and bool(save.isnan().all())
    assert not bool(ws.any()) and not bool(inv.any()) and not bool(ops.any())
