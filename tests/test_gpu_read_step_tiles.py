"""The fused read step (csrc/read_step.cuh) at tile counts away from the headline's 196: many tiles per SM, fewer tiles than
SMs, and a tile count one above a multiple of the SM count.  Each shape is checked against the four-launch chain it
replaces (P*y rounded to bf16, H = ELU(P*y @ Wm[0:d] + Q) rounded to bf16, logits, softmax, weighted sum), recomputed in
fp64 from the same operands, with the bounds of tests/test_gpu_fullshape.py::test_fused_read_step_equals_unfused_chain."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

D = 512


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _check_fused_against_chain(B, N):
    from mac_network_b200 import _lib as L_
    lib = L_.load()
    d = D
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + N)

    def rn(*s, scale=1.0):
        return (torch.randn(*s, device="cuda", generator=g) * scale).contiguous()
    W = {"Wx": rn(d, d, scale=d ** -0.5), "bx": rn(d, scale=0.1), "Wy": rn(d, d, scale=d ** -0.5), "by": rn(d, scale=0.1),
         "Wm": rn(2 * d, d, scale=(2 * d) ** -0.5), "bm": rn(d, scale=0.1), "Wm2": rn(d, d, scale=d ** -0.5),
         "bm2": rn(d, scale=0.1), "wr": rn(d, scale=4 * d ** -0.5)}

    def pack(w):
        o = torch.empty((w.shape[1], w.shape[0]), dtype=torch.bfloat16, device="cuda")
        L_.check(lib.mac_pack_weight_bf16(L_.ptr(w), L_.ptr(o), w.shape[0], w.shape[1], L_.stream_ptr()))
        return o
    W16 = [pack(W["Wx"]), pack(W["Wm"]), pack(W["Wm2"])]
    rw = L_.ReadWeights(W["Wx"].data_ptr(), W["bx"].data_ptr(), W["Wy"].data_ptr(), W["by"].data_ptr(),
                        W["Wm"].data_ptr(), W["bm"].data_ptr(), W["Wm2"].data_ptr(), W["bm2"].data_ptr(),
                        W["wr"].data_ptr(), 0.25, W16[0].data_ptr(), W16[1].data_ptr(), W16[2].data_ptr())
    kb = torch.nn.functional.elu(rn(B, N, d)).to(torch.bfloat16).contiguous()
    y, c = rn(B, d), rn(B, d)
    nb = lib.mac_read_invariant_bytes(B, N, d, 1)
    inv = torch.empty(nb, dtype=torch.uint8, device="cuda")
    L_.check(lib.mac_read_invariant(None, L_.ptr(kb), ctypes.byref(rw), 1, L_.ptr(inv), nb, B, N, d, L_.stream_ptr()))
    assert lib.mac_read_step_fused_supported(B, N, d) == 1
    info1, att1 = torch.full((B, d), float("nan"), device="cuda"), torch.full((B, N), float("nan"), device="cuda")
    L_.check(lib.mac_read_step_fused(L_.ptr(inv), L_.ptr(kb), L_.ptr(y), L_.ptr(c), ctypes.byref(rw), L_.ptr(info1),
                                     L_.ptr(att1), B, N, d, L_.stream_ptr()), "mac_read_step_fused")
    M = B * N
    slab = (M * d * 2 + 1023) & ~1023
    off = ((inv.data_ptr() + 1023) & ~1023) - inv.data_ptr()
    P = inv[off:off + M * d * 2].view(torch.bfloat16).view(M, d).float()
    Q = inv[off + slab:off + slab + M * d * 2].view(torch.bfloat16).view(M, d).float()
    PY = (P.view(B, N, d) * y[:, None, :]).to(torch.bfloat16).float().view(M, d)
    H = torch.nn.functional.elu(PY.double() @ W16[1][:, :d].double().T + Q.double()).float().to(torch.bfloat16).float()
    I1 = H.double() @ W16[2].double().T + W["bm2"].double()
    I2 = torch.nn.functional.elu(I1.view(B, N, d) * c.double()[:, None, :])
    logits = (I2 * W["wr"].double()).sum(-1) + 0.25
    att0 = torch.softmax(logits, dim=-1)
    info0 = (att0[:, :, None] * kb.double()).sum(1)
    torch.cuda.synchronize()
    assert float((att1.double() - att0).abs().max()) < 2e-3 * float(att0.max()) + 1e-6, (B, N)
    assert float((info1.double() - info0).abs().max()) < 2e-3 * float(info0.abs().max()), (B, N)
    assert float((att1.sum(1) - 1).abs().max()) < 1e-5


@pytest.mark.parametrize("B,N", [
    (384, 196),    # 1176 tiles: the two-stream batched-request shape, ~9 tiles per SM
    (1000, 17),    # 266 tiles, each spanning four or five samples, so control rows past the second sample come from global
])
def test_fused_read_step_many_tiles(B, N):
    _check_fused_against_chain(B, N)


@pytest.mark.parametrize("B,N", [
    (4, 196),      # 13 tiles
    (3, 49),       # 3 tiles, the last one partial
])
def test_fused_read_step_fewer_tiles_than_sms(B, N):
    assert (B * N + 63) // 64 < _sms()
    _check_fused_against_chain(B, N)


@pytest.mark.parametrize("waves", [1, 2])
def test_fused_read_step_tile_count_one_above_a_multiple_of_the_sms(waves):
    tiles = waves * _sms() + 1                       # one 64-row sample per tile
    _check_fused_against_chain(tiles, 64)
