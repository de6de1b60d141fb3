"""CPU checks of tests/test_gpu_skinny_tc.py with that file's own cases and reference code.

Its cases launch all 8 kernel instances and every ring remainder; the kernel's arithmetic restated in fp32 passes its bars
at every form case, and five faults planted in that restatement -- the two warpgroups' column halves swapped, n_split off
by 32, the A_lo B_hi pass dropped, rows shifted by one in the column form, a k-block taken from the wrong segment -- are
rejected by at least 100 times the bar.  Outputs a fault leaves unwritten hold stale finite values (zeros), as reused
buffers do.  Then its refusals with host pointers the library never dereferences: every one comes back before any CUDA
call (without a driver, a CUDA call first would return a CUDA error instead), and a valid call gets as far as the device
check."""
import ctypes
import itertools

import pytest
import torch

from mac_network_b200 import _lib as L_
from tests.test_gpu_skinny_tc import (ALL_FORMS, FORM_CASES, REFUSALS, RING_CASES, RING_SEGS, call_refused, check_call,
                                      launch_form, operands)
from tests.test_gpu_wgmma import split_hi_lo

ERR_ARCH = -5
FORMS = [p.values[0] for p in FORM_CASES]
HEADLINE = next(c for c in FORMS if (c["M"], c["segs"], c["n_out"], c["n_split"], c["ldy"]) == (64, (512, 512), 1024, 512, 512))
COLS37 = next(c for c in FORMS if c["M"] == 37)


def test_form_cases_launch_every_instance_and_epilogue():
    assert {launch_form(c["M"], c["n_out"], c["split"]) for c in FORMS} == ALL_FORMS
    assert {c["act"] for c in FORMS} == {"NON", "TANH", "SIGMOID", "ELU", "RELU_STD"}
    assert {c["bias"] for c in FORMS} == {"vec", "const", "none"}
    assert {(c["M"], c["gate"]) for c in FORMS if c["gate"]} >= {(64, "z"), (100, "no_z")}
    # n_split at an odd multiple of 32 under BN 64, in the column form: between the two warpgroups' halves of one CTA
    assert any(c["n_split"] % 64 == 32 and launch_form(c["M"], c["n_out"], c["split"])[0] == 64 and c["M"] <= 64
               for c in FORMS)
    assert HEADLINE["split"] and HEADLINE["wide"] is None


def test_ring_cases_cover_every_remainder():
    assert {n % 12 for n in RING_SEGS} == set(range(12)) and max(RING_SEGS) > 24
    for n, blocks in RING_SEGS.items():
        assert sum(blocks) == n and len(blocks) <= 4
        assert all(b % 2 and b % 3 for b in itertools.accumulate(blocks[:-1])), (n, "a boundary on a ring boundary")
    rings = [p.values[0] for p in RING_CASES]
    assert {c["M"] for c in rings} == {64, 128}
    assert any(c["M"] <= 64 and len(c["segs"]) == 4 and c["wide"] is not None for c in rings)


# ------------------------------------------------------------------------------------------------ the kernel restated
def act32(name, t):
    return {"NON": lambda x: x, "TANH": torch.tanh, "SIGMOID": torch.sigmoid, "ELU": torch.nn.functional.elu,
            "RELU_STD": lambda x: x.clamp_min(0)}[name](t)


def kernel_fp32(c, ops, X=None, drop_lo_hi=False):
    """[M, n_out] before the column split: the products accumulated in fp32, the bias, then the activation or the gate
    (returned as (y, z))"""
    X = torch.cat([x.contiguous() for x in ops["xs"]], 1) if X is None else X
    xh, xl = (t.float() for t in split_hi_lo(X))
    wh, wl = ops["hi"].float().t(), ops["lo"].float().t()
    acc = xh @ wh
    if c["split"]:
        acc = (acc if drop_lo_hi else acc + xl @ wh) + xh @ wl
    t = acc + ops["bias_const"] + (ops["b"] if ops["b"] is not None else 0.0)
    if c["gate"]:
        n = c["n_out"]
        z = torch.sigmoid(t)
        return ops["gnew"][:, :n] * z + ops["gold"][:, :n] * (1 - z), z
    return act32(c["act"], t)


def use(c, ops, full, n_split=None):
    """The largest fraction of its bar any output of `full` uses, as the kernel would store it (y2 from column n_split)."""
    if c["gate"]:
        y, z = full
        res = check_call(c, ops, y, z=z if c["gate"] == "z" else None)
    elif c["n_split"]:
        ns, n = c["n_split"], c["n_out"]
        s = ns if n_split is None else n_split
        y, y2 = torch.zeros(c["M"], ns), torch.zeros(c["M"], n - ns)
        y[:, :min(s, ns)] = full[:, :min(s, ns)]
        w = min(n - s, n - ns)
        y2[:, :w] = full[:, s:s + w]
        res = check_call(c, ops, y, y2)
    else:
        res = check_call(c, ops, full)
    return max(e / bar for e, bar in res.values())


@pytest.mark.parametrize("c", FORM_CASES)
def test_restated_kernel_passes_the_bars(c):
    ops = operands(c, 11, device="cpu")
    u = use(c, ops, kernel_fp32(c, ops))
    print("restated kernel, %s: %.2f of the bar" % (c, u))
    assert u <= 1, u


def rejected(what, u):
    print("%s: %.0f x the bar" % (what, u))
    assert u >= 100, (what, u)


def test_swapped_column_halves_are_rejected():
    c = HEADLINE
    assert launch_form(c["M"], c["n_out"], c["split"]) == (64, True, True)
    ops = operands(c, 21, device="cpu")
    full = kernel_fp32(c, ops)
    swapped = full.view(c["M"], c["n_out"] // 64, 2, 32).flip(2).reshape(c["M"], c["n_out"])
    rejected("warpgroup column halves swapped", use(c, ops, swapped))


@pytest.mark.parametrize("off", [32, -32])
def test_n_split_off_by_32_is_rejected(off):
    c = HEADLINE
    ops = operands(c, 22, device="cpu")
    rejected("n_split off by %d" % off, use(c, ops, kernel_fp32(c, ops), n_split=c["n_split"] + off))


def test_dropped_lo_hi_pass_is_rejected():
    c = HEADLINE
    ops = operands(c, 23, device="cpu")
    rejected("A_lo B_hi pass dropped", use(c, ops, kernel_fp32(c, ops, drop_lo_hi=True)))


def test_rows_shifted_by_one_are_rejected():
    c = COLS37
    assert launch_form(c["M"], c["n_out"], c["split"])[2]
    ops = operands(c, 24, device="cpu")
    full = kernel_fp32(c, ops)
    shifted = torch.zeros_like(full)
    shifted[1:] = full[:-1]
    rejected("rows shifted by one", use(c, ops, shifted))


def test_k_block_from_the_wrong_segment_is_rejected():
    c = HEADLINE
    ops = operands(c, 25, device="cpu")
    X = torch.cat([x.contiguous() for x in ops["xs"]], 1)
    k0 = c["segs"][0]
    wrong = X.clone()
    wrong[:, k0:k0 + 64] = X[:, :64]                    # segment 1's first k-block read from segment 0
    rejected("k-block from the wrong segment", use(c, ops, kernel_fp32(c, ops, X=wrong)))


# ------------------------------------------------------------------------------------------------ refusals
def host_call(r):
    """r with aligned host buffers the library never dereferences; returns (status, launches counted)"""
    lib = L_.load()
    buf = (ctypes.c_char * 4096)()
    p = (ctypes.addressof(buf) + 15) & ~15
    before = lib.mac_b200_launch_count()
    st = call_refused(lib, r, p, p)
    return st, lib.mac_b200_launch_count() - before


@pytest.mark.parametrize("r,expect", REFUSALS)
def test_refused_before_any_cuda_call(r, expect):
    if torch.cuda.is_available():
        pytest.skip("host pointers stand in for device buffers: tests/test_gpu_skinny_tc.py covers this device")
    assert host_call(r) == (expect, 0)


@pytest.mark.parametrize("n_split,gate", [(None, None), (32, None), (None, "z")])
def test_valid_call_reaches_the_device_check(n_split, gate):
    if torch.cuda.is_available():
        pytest.skip("a valid call would launch on this device")
    r = dict(M=8, segs=((64, 64),), n_out=64, ldy=64, n_split=n_split, gate=gate, odd=())
    assert host_call(r) == (ERR_ARCH, 0)
