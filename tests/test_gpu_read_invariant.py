"""The read unit's step-invariant products at d = 512 (csrc/read_inv.cuh): P = KB @ Wx + bx and Q = P @ Wm[d:2d] + bm in
bf16, from a bf16 knowledge base (mac_read_invariant) or from an fp32 one that the same launch casts into kb_bf16
(mac_read_invariant_cast).

Each result must be bit for bit the one of the chain it replaces, run through the generic entry points: mac_cast_bf16,
then mac_linear_tc_fwd (tc_gemm) with Wx and with the packed Wm[d:2d] slice.  Both are also held to an fp64 restatement
of their own operation, within the bf16 rounding of the stored outputs.  Shapes: the headline (B = 64, N = 196), GQA
(N = 49), B*N in {1, 127, 128, 129, 255, 12545} (one row, tiles one short of, equal to and one past 128 rows, a tail that
is not a multiple of 128) and N > 256 (the kernel does not depend on sample boundaries).  The fp8 form's P8 and sP come
from the same P.  The CPU test checks mac_read_invariant_cast's refusals, which come before any launch."""
import ctypes

import pytest
import torch

D = 512
BF16, FP8 = 1, 3
INVALID, ALIGN, UNSUPPORTED, WORKSPACE = -1, -2, -3, -4
SHAPES = [(64, 196), (64, 49), (1, 1), (1, 127), (1, 128), (3, 43), (5, 51), (5, 2509), (2, 300)]


def _lib():
    from mac_network_b200 import _lib as L_
    return L_, L_.load()


def _al(b):
    return (b + 1023) & ~1023


def _slab(inv, off, M, dtype=torch.bfloat16, cols=D):
    """rows [0, M) of a [M, cols] slab at byte `off` behind the 1 KB aligned base of `inv`"""
    o = ((inv.data_ptr() + 1023) & ~1023) - inv.data_ptr() + off
    esz = torch.empty((), dtype=dtype).element_size()
    return inv[o:o + M * cols * esz].view(dtype).view(M, cols)


def _case(B, N, seed):
    L_, lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *s, scale=1.0: (torch.randn(*s, device="cuda", generator=g) * scale).contiguous()
    W = {"Wx": rn(D, D, scale=D ** -0.5), "bx": rn(D, scale=0.1), "Wm": rn(2 * D, D, scale=(2 * D) ** -0.5),
         "bm": rn(D, scale=0.1), "Wm2": rn(D, D, scale=D ** -0.5), "bm2": rn(D, scale=0.1), "wr": rn(D, scale=0.2)}

    def pack(w):
        o = torch.empty((w.shape[1], w.shape[0]), dtype=torch.bfloat16, device="cuda")
        L_.check(lib.mac_pack_weight_bf16(L_.ptr(w), L_.ptr(o), w.shape[0], w.shape[1], L_.stream_ptr()), "pack")
        return o
    keep = {"Wx": pack(W["Wx"]), "Wm": pack(W["Wm"]), "Wm2": pack(W["Wm2"]), "Wmb": pack(W["Wm"][D:])}
    rw = L_.ReadWeights(W["Wx"].data_ptr(), W["bx"].data_ptr(), None, None, W["Wm"].data_ptr(), W["bm"].data_ptr(),
                        W["Wm2"].data_ptr(), W["bm2"].data_ptr(), W["wr"].data_ptr(), 0.0, keep["Wx"].data_ptr(),
                        keep["Wm"].data_ptr(), keep["Wm2"].data_ptr())
    # ELU-like values with a wide exponent range, so the bf16 cast rounds in every binade it meets
    kb = (torch.nn.functional.elu(rn(B * N, D)) * torch.exp2(rn(B * N, D, scale=3.0).round())).contiguous()
    return W, keep, rw, kb


def _chain(L_, lib, W, keep, kb):
    """mac_cast_bf16, then P and Q through mac_linear_tc_fwd (tc_gemm's TC_EPI_ACT epilogue)"""
    M = kb.shape[0]
    kb16 = torch.empty(M, D, dtype=torch.bfloat16, device="cuda")
    L_.check(lib.mac_cast_bf16(L_.ptr(kb), L_.ptr(kb16), kb.numel(), L_.stream_ptr()), "mac_cast_bf16")
    P = torch.empty(M, D, dtype=torch.bfloat16, device="cuda")
    Q = torch.empty(M, D, dtype=torch.bfloat16, device="cuda")
    L_.check(lib.mac_linear_tc_fwd(L_.ptr(kb16), L_.ptr(keep["Wx"]), L_.ptr(W["bx"]), 0, L_.ptr(P), 1, M, D, D,
                                   L_.stream_ptr()), "P")
    L_.check(lib.mac_linear_tc_fwd(L_.ptr(P), L_.ptr(keep["Wmb"]), L_.ptr(W["bm"]), 0, L_.ptr(Q), 1, M, D, D,
                                   L_.stream_ptr()), "Q")
    return kb16, P, Q


def _bits_equal(a, b):
    return torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


def _fp64_bound(out, a16, wt16, bias):
    """|out - (a @ W + b)| in fp64 against the bf16 rounding of out (half an ulp, <= 2^-8 |ref|) plus the fp32
    accumulation over K = 512 (<= 2^-16 of the absolute-value product)"""
    a, w = a16.double(), wt16.double()
    ref = a @ w.T + bias.double()
    absprod = a.abs() @ w.abs().T + bias.double().abs()
    err = (out.double() - ref).abs()
    bar = 2.0 ** -8 * ref.abs() + 2.0 ** -16 * absprod
    return float((err - bar).max()), float((err / absprod.clamp_min(1e-30)).max())


@pytest.mark.gpu
@pytest.mark.parametrize("B,N", SHAPES)
def test_read_invariant_bit_identical_to_cast_and_tc_gemm_chain(B, N):
    L_, lib = _lib()
    M = B * N
    W, keep, rw, kb = _case(B, N, 1000 * B + N)
    kb16_ref, P_ref, Q_ref = _chain(L_, lib, W, keep, kb)
    nb = lib.mac_read_invariant_bytes(B, N, D, BF16)
    q_off = _al(M * D * 2)

    # bf16 knowledge base in (the serving paths, the gather)
    inv = torch.full((nb,), 0xA5, dtype=torch.uint8, device="cuda")
    L_.check(lib.mac_read_invariant(None, L_.ptr(kb16_ref), ctypes.byref(rw), BF16, L_.ptr(inv), nb, B, N, D,
                                    L_.stream_ptr()), "mac_read_invariant")
    # fp32 knowledge base in: kb_bf16 is written by the same launch
    inv2 = torch.full((nb,), 0x5A, dtype=torch.uint8, device="cuda")
    kb16 = torch.full((M, D), float("nan"), dtype=torch.bfloat16, device="cuda")
    L_.check(lib.mac_read_invariant_cast(L_.ptr(kb), L_.ptr(kb16), ctypes.byref(rw), BF16, L_.ptr(inv2), nb, B, N, D,
                                         L_.stream_ptr()), "mac_read_invariant_cast")
    torch.cuda.synchronize()
    assert _bits_equal(kb16, kb16_ref), (B, N)
    for buf, form in ((inv, "bf16 in"), (inv2, "fp32 in")):
        assert _bits_equal(_slab(buf, 0, M), P_ref), (B, N, form, "P")
        assert _bits_equal(_slab(buf, q_off, M), Q_ref), (B, N, form, "Q")

    P, Q = _slab(inv2, 0, M), _slab(inv2, q_off, M)
    excess, _ = _fp64_bound(P, kb16_ref, keep["Wx"], W["bx"])
    assert excess <= 0.0, (B, N, "P", excess)
    excess, _ = _fp64_bound(Q, P, keep["Wmb"], W["bm"])
    assert excess <= 0.0, (B, N, "Q", excess)


@pytest.mark.gpu
@pytest.mark.parametrize("B,N", [(64, 196), (3, 43)])
def test_read_invariant_cast_fp8_form(B, N):
    """MAC_PREC_FP8: P and Q of the chain bit for bit, and P8 / sP as mac_read_invariant makes them from kb_bf16"""
    L_, lib = _lib()
    M = B * N
    W, keep, rw, kb = _case(B, N, 7 * B + N)
    kb16_ref, P_ref, Q_ref = _chain(L_, lib, W, keep, kb)
    nb = lib.mac_read_invariant_bytes(B, N, D, FP8)
    o_sP = _al(M * D)
    o_Q = o_sP + _al(M * 4)
    o_P = o_Q + _al(M * D * 2) + _al(M * 4)
    inv = torch.full((nb,), 0xA5, dtype=torch.uint8, device="cuda")
    L_.check(lib.mac_read_invariant(None, L_.ptr(kb16_ref), ctypes.byref(rw), FP8, L_.ptr(inv), nb, B, N, D,
                                    L_.stream_ptr()), "mac_read_invariant")
    inv2 = torch.full((nb,), 0x5A, dtype=torch.uint8, device="cuda")
    kb16 = torch.full((M, D), float("nan"), dtype=torch.bfloat16, device="cuda")
    L_.check(lib.mac_read_invariant_cast(L_.ptr(kb), L_.ptr(kb16), ctypes.byref(rw), FP8, L_.ptr(inv2), nb, B, N, D,
                                         L_.stream_ptr()), "mac_read_invariant_cast")
    torch.cuda.synchronize()
    assert _bits_equal(kb16, kb16_ref)
    for buf in (inv, inv2):
        assert _bits_equal(_slab(buf, o_P, M), P_ref) and _bits_equal(_slab(buf, o_Q, M), Q_ref)
    assert torch.equal(_slab(inv, 0, M, torch.uint8), _slab(inv2, 0, M, torch.uint8))                     # P8
    assert torch.equal(_slab(inv, o_sP, M, torch.float32, 1), _slab(inv2, o_sP, M, torch.float32, 1))    # sP


def test_read_invariant_cast_refusals():
    """mac_read_invariant_cast refuses before any launch (no GPU needed): the fp32 / tc32 precisions, a missing fp32 or bf16
    knowledge base, pack or weights, misalignment, a short `inv`, d != 512, an fp8 shape outside the read step, B <= 0"""
    from mac_network_b200 import _lib as L_
    lib = L_.load()
    buf = (ctypes.c_float * 4096)()
    p = (ctypes.addressof(buf) + 15) & ~15                 # 16-byte aligned fake "device" pointer (never dereferenced)
    rw = L_.ReadWeights(p, p, p, p, p, p, p, p, p, 0.0, p, p, p)
    rw_nopack = L_.ReadWeights(p, p, p, p, p, p, p, p, p, 0.0, None, p, p)
    B, N = 2, 49
    nb = lib.mac_read_invariant_bytes(B, N, D, BF16)

    def call(kb=p, kb16=p, w=rw, prec=BF16, inv=p, inv_bytes=nb, B=B, N=N, d=D):
        return lib.mac_read_invariant_cast(kb, kb16, ctypes.byref(w) if w is not None else None, prec, inv, inv_bytes,
                                           B, N, d, None)
    assert call(prec=0) == UNSUPPORTED and call(prec=2) == UNSUPPORTED
    assert call(kb=None) == INVALID and call(kb16=None) == INVALID and call(inv=None) == INVALID
    assert call(w=None) == INVALID and call(w=rw_nopack) == INVALID
    assert call(B=0) == INVALID and call(N=0) == INVALID
    assert call(kb=p + 4) == ALIGN and call(kb16=p + 4) == ALIGN and call(inv=p + 4) == ALIGN
    assert call(inv_bytes=nb - 1) == WORKSPACE
    assert call(d=256, inv_bytes=1 << 30) == UNSUPPORTED
    assert call(prec=FP8, N=300, inv_bytes=1 << 30) == UNSUPPORTED
