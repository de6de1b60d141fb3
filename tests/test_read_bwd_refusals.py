"""Refusals of the read unit's backward entry points (mac_read_bwd, mac_read_bwd_tc, mac_read_bwd_tc32): every MAC_ERR_* a
form can return comes back before any launch and before any write (include/mac_b200.h, csrc/backward.cu).  Most outputs of
these calls accumulate into the caller's buffers, so a refusal after a launch would leave gradients half added.

Each case names the form, the shape and one defect: a required pointer missing, a d or B*N the form's kernels do not take,
keep_read outside (0, 1], a workspace one byte short, or a pointer that a kernel of the form reads or writes with 16-byte
accesses, 8 bytes off that alignment.  The CPU test hands the library aligned host buffers that it never dereferences: a
CUDA call before the refusal comes back as a CUDA error (35 without a driver) instead of the expected code.  Its GPU twin
hands it device buffers (NaN-filled outputs, a zeroed workspace and zeroed inputs) and checks that they stay untouched."""
import ctypes

import pytest
import torch

from mac_network_b200 import _lib as L_

INVALID, ALIGN, UNSUPPORTED, WORKSPACE = -1, -2, -3, -4
FORMS = ("fp32", "tc", "tc32")
OUTS = ["dkb", "dmem_in", "dcontrol", "dWx", "dbx_part", "dWy", "dby", "dWm", "dbm_part", "dWm2", "dbm2_part", "dwr_part",
        "dbr_part"]
# what every form reads or writes unconditionally, then per form the weights of its data gradients (fp32: transposed
# arguments; tensor-core forms: mac_read_weights fields) and the weight gradients it cannot skip
REQUIRED = ["kb", "memory_in", "control", "w", "wr", "att", "save", "dinfo", "dmem_in", "dcontrol", "Wy_t", "dbx_part",
            "dbm_part", "dbm2_part", "dwr_part", "ws"]
REQUIRED_FORM = {"fp32": ["Wx_t", "Wm_t", "Wm2_t"], "tc": ["Wx", "Wm", "Wm2", "dWx", "dWm", "dWm2"]}
REQUIRED_FORM["tc32"] = REQUIRED_FORM["tc"]
# read or written with 16-byte accesses (float4 loads and stores, cp.async, the split-K accumulation into dW)
ALIGNED = ["kb", "memory_in", "control", "wr", "save", "dinfo", "dmem_in", "Wy_t", "ws", "dkb", "dWx", "dWy", "dWm", "dWm2"]
ALIGNED_FORM = {"fp32": ["Wx_t", "Wm_t", "Wm2_t"], "tc": ["Wx", "Wm", "Wm2"], "tc32": ["Wx", "Wm", "Wm2"]}
SHAPE = (2, 32, 128)                    # (B, N, d): every form takes it


def case(form, expect, shape=SHAPE, keep=1.0, drop=(), odd=(), short=False):
    B, N, d = shape
    return pytest.param(dict(form=form, B=B, N=N, d=d, keep=keep, drop=drop, odd=odd, short=short), expect,
                        id="%s-%d_%d_%d%s%s%s%s" % (form, B, N, d, "-keep%g" % keep if keep != 1 else "",
                                                 "".join("-no_" + k for k in drop), "".join("-odd_" + k for k in odd),
                                                 "-short" if short else ""))


CASES = [
    # each required pointer missing
    *[case(f, INVALID, drop=(k,)) for f in FORMS for k in REQUIRED + REQUIRED_FORM[f]],
    # d not a multiple of 4 (fp32) or of 128 (the tensor-core forms); B*N not a multiple of 64 for tc
    case("fp32", INVALID, shape=(2, 32, 130)),
    *[case(f, UNSUPPORTED, shape=s) for f in ("tc", "tc32") for s in ((2, 32, 130), (1, 64, 192))],
    case("tc", UNSUPPORTED, shape=(5, 13, 128)),
    case("tc32", UNSUPPORTED, shape=(5, 13, 64)),
    # keep_read outside (0, 1]
    *[case(f, INVALID, keep=k) for f in FORMS for k in (0.0, -0.5, 1.5)],
    # a workspace one byte short
    *[case(f, WORKSPACE, short=True) for f in FORMS],
    # misalignment
    *[case(f, ALIGN, odd=(k,)) for f in FORMS for k in ALIGNED + ALIGNED_FORM[f]],
]


def call(lib, c, ops, outs, ws):
    """Run case c with every input (knowledge base, memory, control, save, weights) at address `ops`, the outputs at
    outs[name] and the workspace at `ws`."""
    B, N, d = c["B"], c["N"], c["d"]
    ptr = lambda name, base: None if name in c["drop"] else base + (8 if name in c["odd"] else 0)
    rw = L_.ReadWeights()
    for f, _ in L_.ReadWeights._fields_:
        if f != "br":
            setattr(rw, f, ptr(f, ops))
    w = None if "w" in c["drop"] else ctypes.byref(rw)
    head = [ptr(k, ops) for k in ("kb", "memory_in", "control")] + [w]
    wt = [ptr(k, ops) for k in (("Wx_t", "Wy_t", "Wm_t", "Wm2_t") if c["form"] == "fp32" else ("Wy_t",))]
    mid = [ptr(k, ops) for k in ("att", "save", "dinfo")] + [c["keep"], 1, 0]
    o = [ptr(k, outs[k]) for k in OUTS]
    name = {"fp32": "mac_read_bwd", "tc": "mac_read_bwd_tc", "tc32": "mac_read_bwd_tc32"}[c["form"]]
    wsb = getattr(lib, name + "_workspace_bytes")(B, N, d) - (1 if c["short"] else 0)
    return getattr(lib, name)(*head, *wt, *mid, *o, ptr("ws", ws), wsb, B, N, d, None)


@pytest.mark.parametrize("c,expect", CASES)
def test_read_bwd_refuses_before_any_cuda_call(c, expect):
    if torch.cuda.is_available():
        pytest.skip("host pointers stand in for device buffers: the GPU twin below covers this device")
    lib = L_.load()
    buf = (ctypes.c_char * 4096)()
    p = (ctypes.addressof(buf) + 15) & ~15              # 16-byte aligned, never dereferenced
    before = lib.mac_b200_launch_count()
    st = call(lib, c, p, {k: p for k in OUTS}, p)
    assert st == expect, st
    assert lib.mac_b200_launch_count() == before


@pytest.mark.gpu
@pytest.mark.parametrize("c,expect", CASES)
def test_read_bwd_refuses_before_any_launch_or_write(c, expect):
    lib = L_.load()
    B, N, d = c["B"], c["N"], c["d"]
    M = B * N
    # every input at one zeroed buffer as large as the largest of them (`save`, the knowledge base, Wm), 16 bytes of slack
    ops = torch.zeros(max(3 * M * d + B * d, 2 * d * d) + 4, device="cuda")
    size = {"dkb": M * d, "dWx": d * d, "dWy": d * d, "dby": d, "dWm": 2 * d * d, "dWm2": d * d, "dbr_part": B}
    outs = {k: torch.full((size.get(k, B * d) + 4,), float("nan"), device="cuda") for k in OUTS}
    wsb = max(getattr(lib, n)(B, N, d) for n in ("mac_read_bwd_workspace_bytes", "mac_read_bwd_tc_workspace_bytes",
                                                 "mac_read_bwd_tc32_workspace_bytes"))
    ws = torch.zeros(wsb + 16, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    before = lib.mac_b200_launch_count()
    st = call(lib, c, ops.data_ptr(), {k: v.data_ptr() for k, v in outs.items()}, ws.data_ptr())
    torch.cuda.synchronize()
    assert st == expect, st
    assert lib.mac_b200_launch_count() == before
    assert all(bool(v.isnan().all()) for v in outs.values())
    assert not bool(ws.any()) and not bool(ops.any())
