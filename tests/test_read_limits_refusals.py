"""Batch and row limits of the read unit's forward (include/mac_b200.h, csrc/read_fwd.cuh): a launch grid's y extent is at
most 65535, so the forms refuse, before any launch, a call whose [B*N, d] products would need more row tiles -- 128-row
tiles for tc_gemm and tc3_gemm (MAC_PREC_BF16, TC32 and mac_read_invariant's tensor-core parts, FP8 included), the tiles
sgemm picks for MAC_PREC_FP32 -- and a kb_attend of more than 2^31 - 1 CTAs (B * d / its column slice).  Uses the harness
of tests/test_read_fwd_refusals.py: on the CPU aligned host buffers that the library never dereferences, so a refusal that
comes too late shows up as a CUDA error (35 without a driver) instead of MAC_ERR_UNSUPPORTED; on the GPU device buffers as
large as the form reads (the cases small enough to allocate), NaN-filled outputs and a zeroed workspace that stay as they
were.  One tile under each limit the call passes the checks (on the CPU its first launch or tensor-map encode then fails).  tests/test_gpu_read_step_bounds.py runs the forms at B = 65535, 65536 and 200 003, past kb_attend's old limit."""
import ctypes

import pytest
import torch

from mac_network_b200 import _lib as L_
from tests.test_read_fwd_refusals import (BF16, FP8, FP32, TC32, UNSUPPORTED, call, case, check_device_refusal,
                                          check_host_refusal)

TC_ROWS = 65535 * 128                   # the most rows 128-row tiles on gridDim.y cover
ARCH = -5                               # MAC_ERR_ARCH: no tensor-map entry point without a driver
KB_B = (2 ** 31 - 1) // 511 + 1         # d = 2044 (d % 8 == 4): kb_attend slices of 4 columns, 511 CTAs per sample

# fp32 at d = 4: 128-row sgemm tiles (at least 512 rows, and more tiles than SMs); small enough to allocate on the GPU
FP32_CASES = [case(c, FP32, 4, UNSUPPORTED, BN=(1, TC_ROWS + 1)) for c in ("fwd", "fwd_inv", "invariant")]
CASES = FP32_CASES + [
    # tensor-core forms and mac_read_invariant's tensor-core products: ceil(B*N / 128) > 65535
    case("fwd", BF16, 128, UNSUPPORTED, BN=(1, TC_ROWS + 1)),
    case("fwd", BF16, 128, UNSUPPORTED, BN=(1, TC_ROWS + 1), keep=0.5),
    case("fwd_inv", BF16, 128, UNSUPPORTED, BN=(TC_ROWS + 1, 1)),
    case("fwd", TC32, 128, UNSUPPORTED, BN=(TC_ROWS + 1, 1)),
    case("fwd_inv", TC32, 128, UNSUPPORTED, BN=(1, TC_ROWS + 1)),
    case("invariant", TC32, 128, UNSUPPORTED, BN=(TC_ROWS + 1, 1)),
    # the fused steps' shapes (B < 2^22, N <= 256): their P and Q are tc_gemm products
    case("invariant", BF16, 512, UNSUPPORTED, BN=(32768, 256)),
    case("invariant", FP8, 512, UNSUPPORTED, BN=(32768, 256)),
    # fp32 at d = 512
    case("fwd", FP32, 512, UNSUPPORTED, BN=(TC_ROWS + 1, 1)),
    # kb_attend: B * 511 CTAs > 2^31 - 1, every product within its row limit
    case("fwd", FP32, 2044, UNSUPPORTED, BN=(KB_B, 1)),
    case("fwd_inv", FP32, 2044, UNSUPPORTED, BN=(KB_B, 1)),
]
# one tile (or one sample) under each limit: the checks pass
AT_LIMIT = [
    case("fwd_inv", FP32, 4, 0, BN=(1, TC_ROWS)),
    case("invariant", FP32, 4, 0, BN=(1, TC_ROWS)),
    case("fwd_inv", BF16, 128, 0, BN=(1, TC_ROWS)),
    case("invariant", BF16, 512, 0, BN=(32767, 256)),
    case("fwd_inv", FP32, 2044, 0, BN=(KB_B - 1, 1)),
]


def _no_gpu():
    if torch.cuda.is_available():
        pytest.skip("host pointers stand in for device buffers: the GPU twin below covers this device")


@pytest.mark.parametrize("c,expect", CASES)
def test_read_limits_refused_before_any_cuda_call(c, expect):
    _no_gpu()
    check_host_refusal(c, expect)


@pytest.mark.parametrize("c,expect", AT_LIMIT)
def test_read_limits_admit_the_largest_shape(c, expect):
    _no_gpu()
    lib = L_.load()
    buf = (ctypes.c_char * 4096)()
    p = (ctypes.addressof(buf) + 15) & ~15
    st = call(lib, c, p, p, p, p, p, p)
    assert st > 0 or st == ARCH, st      # past every check: its first launch or tensor-map encode fails without a driver


def test_kb_attend_refuses_more_ctas_than_a_grid_holds():
    """mac_kb_attend_fwd on its own: d = 4092 runs 4-column slices, 1023 CTAs per sample"""
    _no_gpu()
    lib = L_.load()
    buf = (ctypes.c_char * 4096)()
    p = (ctypes.addressof(buf) + 15) & ~15
    B = (2 ** 31 - 1) // 1023 + 1
    before = lib.mac_b200_launch_count()
    assert lib.mac_kb_attend_fwd(p, 1, 0.0, p, 0, p, p, B, 1, 4092, None) == UNSUPPORTED
    assert lib.mac_b200_launch_count() == before
    assert lib.mac_kb_attend_fwd(p, 1, 0.0, p, 0, p, p, B - 1, 1, 4092, None) == ARCH     # the tensor-map encode


@pytest.mark.gpu
@pytest.mark.parametrize("c,expect", FP32_CASES)
def test_read_limits_refused_before_any_launch_or_write(c, expect):
    check_device_refusal(c, expect)
    torch.cuda.empty_cache()
