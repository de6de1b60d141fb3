"""Kernel-level GPU tests through the C ABI: K1 (control attention), K3 (KB attention), dropout RNG, the tensor-core
linear.  mac_linear_fwd is checked in tests/test_gpu_forward_kernels.py."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import mac_oracle as O
from tests._util import max_rel

pytestmark = pytest.mark.gpu


def _lib():
    from mac_network_b200 import _lib as L
    return L, L.load()


# (B, N, d, nparts): N = 1 and N < 64 load one box; N >= 64 four resident boxes; N = 1500 and 5000 a ring of recycled boxes
# whose stage count is not a multiple of the buffer count and whose last box is partial.  B = 3 with N = 257: the last
# batch row's last box runs past B*N (zero fill).  fp32 d covers every slice width (128 .. 4 columns); bf16 runs where
# d % 64 == 0.
KB_CASES_MAXNORM = [(64, 196, 512, 4), (3, 49, 512, 1), (2, 1, 64, 2), (5, 700, 128, 3), (2, 1500, 512, 1),
                    (7, 33, 16, 1)]
KB_CASES = (KB_CASES_MAXNORM
            + [(3, N, d, (1, 8, 32)[(i + j) % 3]) for i, d in enumerate((4, 8, 16, 32, 64, 128, 512))
               for j, N in enumerate((1, 63, 64, 257, 1500, 5000))])


@pytest.mark.parametrize("B,N,d,nparts", KB_CASES)
def test_kb_attend(B, N, d, nparts):
    """mac_kb_attend_fwd against fp64, element-wise (tests/test_gpu_forward_kernels.py, softmax_bound), with the logits
    at their drawn values and offset by +80 and -80 (only the max subtraction keeps expf finite there)"""
    from tests.test_gpu_forward_kernels import TOL_ATT, kb_attend_reference
    from tests.test_gpu_backward_kernels import Report, run_twice
    L, lib = _lib()
    rng = np.random.RandomState(B * 10000 + N * 10 + d)
    kb = rng.standard_normal((B, N, d)).astype(np.float32)
    br = 0.3
    tk = torch.from_numpy(kb).cuda()
    kbs = [(0, tk)] + ([(1, tk.to(torch.bfloat16))] if d % 64 == 0 else [])
    for off in (0.0, 80.0, -80.0):
        parts = (rng.standard_normal((B, N, nparts)) + off / nparts).astype(np.float32)
        tp = torch.from_numpy(parts).cuda()
        for is16, kbt in kbs:
            att = torch.full((B, N), float("nan"), device="cuda")
            info = torch.full((B, d), float("nan"), device="cuda")
            got, same = run_twice(lambda: L.check(lib.mac_kb_attend_fwd(L.ptr(tp), nparts, br, L.ptr(kbt), is16, L.ptr(att),
                                                                        L.ptr(info), B, N, d, L.stream_ptr())),
                                  {"att": att, "info": info})
            a, aa, r, ar = kb_attend_reference(tp, br, kbt.float())
            rep = Report("mac_kb_attend_fwd B=%d N=%d d=%d nparts=%d offset %g%s" % (B, N, d, nparts, off,
                                                                                     " bf16" if is16 else ""))
            rep.add("att", got["att"], a, aa, TOL_ATT)
            rep.add("info", got["info"], r, ar, TOL_ATT)
            rep.check(same, "bit-identical rerun")
            rep.done()
            if off == 0.0 and (B, N, d, nparts) in KB_CASES_MAXNORM:    # the max-norm bars of these cases
                a_np, r_np = a.cpu().numpy(), r.cpu().numpy()
                assert np.max(np.abs(got["att"].cpu().numpy() - a_np)) < 1e-6
                assert max_rel(got["info"].cpu().numpy(), r_np) < 1e-5


# (T, B, S, d): nsteps 1, 12, 13 at B = 3 (steps split over gridDim.y) and B = 300 (one step group: B > 2 x SMs); S*d at
# the shared-memory limit with separate words (S = 54, d = 512: 221 KB); d = 20
CTRL_FWD_CASES = [(12, 64, 40, 512), (1, 3, 1, 64), (4, 5, 45, 512), (3, 2, 7, 16),
                  (1, 3, 40, 512), (12, 3, 40, 64), (13, 3, 40, 64), (1, 300, 30, 128), (12, 300, 30, 128),
                  (13, 300, 30, 128), (3, 3, 54, 512), (13, 5, 7, 20)]


@pytest.mark.parametrize("T,B,S,d", CTRL_FWD_CASES)
def test_control_attend(T, B, S, d):
    """mac_control_attend_fwd against fp64, element-wise: shared and separate words, batch-major words (one bulk copy per
    batch row) and the step-major history layout (rstride = B*d, bstride = d: one bulk copy per word row), lengths of 0
    (uniform attention), > S and negative (clamped)"""
    from tests.test_gpu_forward_kernels import TOL_ATT, softmax_bound
    from tests.test_gpu_backward_kernels import Report, run_twice
    L, lib = _lib()
    rng = np.random.RandomState(1)
    cc = rng.standard_normal((T, B, d)).astype(np.float32)
    words = rng.standard_normal((B, S, d)).astype(np.float32)
    outw = rng.standard_normal((B, S, d)).astype(np.float32)
    w = rng.standard_normal((d,)).astype(np.float32) * 0.1
    lengths = rng.randint(1, S + 1, size=(B,)).astype(np.int32)
    lengths[0] = S
    if B > 1:
        lengths[1] = 1
    for i, n in zip(range(2, B), (0, S + 5, -3)):
        lengths[i] = n
    lens = np.clip(lengths, 0, S)
    b = -0.2
    for layout in ("batch", "history"):
        for separate in (False, True):
            ov = outw if separate else words
            if layout == "batch":
                wbuf, obuf, bstride, rstride = words, ov, S * d, d
            else:
                wbuf, obuf = (np.ascontiguousarray(x.transpose(1, 0, 2)) for x in (words, ov))
                bstride, rstride = d, B * d
            t = {k: torch.from_numpy(v).cuda() for k, v in dict(cc=cc, words=wbuf, ov=obuf, w=w, lengths=lengths).items()}
            att = torch.full((T, B, S), float("nan"), device="cuda")
            out = torch.full((T, B, d), float("nan"), device="cuda")

            def call():
                L.check(lib.mac_control_attend_fwd(L.ptr(t["cc"]), B * d, d, L.ptr(t["words"]), bstride, rstride,
                                                   L.ptr(t["ov"] if separate else t["words"]), bstride, rstride,
                                                   L.ptr(t["lengths"]), L.ptr(t["w"]), b, L.ptr(att), L.ptr(out), T, B, S, d,
                                                   L.stream_ptr()))

            got, same = run_twice(call, {"att": att, "out": out})
            c64 = cc.astype(np.float64)
            logits = np.einsum("tbk,bsk,k->tbs", c64, words.astype(np.float64), w.astype(np.float64)) + b
            alog = np.einsum("tbk,bsk,k->tbs", np.abs(c64), np.abs(words.astype(np.float64)), np.abs(w.astype(np.float64))) + abs(b)
            valid = np.arange(S)[None, :] < lens[:, None]
            valid |= (lens == 0)[:, None]           # length 0: every logit is -1e30 in both, the softmax is uniform
            tl = torch.from_numpy(np.where((lens == 0)[None, :, None], 0.0, logits))
            ta = torch.from_numpy(np.where((lens == 0)[None, :, None], 0.0, alog))
            a, aa = softmax_bound(tl, ta, torch.from_numpy(np.broadcast_to(valid, logits.shape).copy()))
            ovd = torch.from_numpy(ov.astype(np.float64))
            rep = Report("mac_control_attend_fwd T=%d B=%d S=%d d=%d %s%s" % (T, B, S, d, layout,
                                                                               " separate" if separate else ""))
            rep.add("att", got["att"].cpu(), a, aa, TOL_ATT)
            rep.add("out", got["out"].cpu(), torch.einsum("tbs,bsk->tbk", a, ovd), torch.einsum("tbs,bsk->tbk", aa, ovd.abs()),
                    TOL_ATT)
            rep.check(same, "bit-identical rerun")
            rep.done()
            # the bars this test has always had
            a_np = a.numpy()
            g_att = got["att"].cpu().numpy()
            assert np.max(np.abs(g_att - a_np)) < 2e-6
            for bi, n in enumerate(lens):
                if n > 0:
                    assert np.all(g_att[:, bi, n:] == 0.0)
            assert max_rel(got["out"].cpu().numpy(), torch.einsum("tbs,bsk->tbk", a, ovd).numpy()) < 1e-5


def test_dropout_rng_matches_independent_philox():
    """The in-kernel Philox4x32-10 against a numpy restatement; keep-mask == floor(keep + u) (ops.py:1054-1059)."""
    L, lib = _lib()
    from oracle.philox import philox_uniform
    n = 4099
    for site, step, seed in [(1, 0, 7), (3, 11, 2 ** 40 + 5)]:
        u = torch.empty(n, device="cuda")
        L.check(lib.mac_dropout_uniform(seed, site, step, L.ptr(u), n, L.stream_ptr()))
        ref = philox_uniform(seed, site, step, n)
        assert np.array_equal(u.cpu().numpy().astype(np.float64), ref)
        x = torch.ones(n, device="cuda")
        o = torch.empty(n, device="cuda")
        keep = 0.85
        L.check(lib.mac_dropout_fwd(L.ptr(x), keep, seed, site, step, L.ptr(o), n, L.stream_ptr()))
        mask = np.floor(keep + ref)
        assert np.allclose(o.cpu().numpy(), mask / np.float32(keep), rtol=1e-6)
    assert 0.8 < mask.mean() < 0.9


@pytest.mark.parametrize("M,K,N,act", [(12544, 512, 512, "NON"), (300, 1024, 256, "ELU"), (128, 64, 256, "NON"),
                                       (3136, 512, 512, "TANH")])
def test_linear_tensor_core(M, K, N, act):
    """wgmma GEMM (bf16 operands, fp32 accumulate) against an fp64 product of the same bf16-rounded operands."""
    L, lib = _lib()
    rng = np.random.RandomState(3)
    x = torch.from_numpy(rng.standard_normal((M, K)).astype(np.float32)).cuda().to(torch.bfloat16)
    W = torch.from_numpy((rng.standard_normal((K, N)) / np.sqrt(K)).astype(np.float32)).cuda()
    b = torch.from_numpy(rng.standard_normal((N,)).astype(np.float32)).cuda()
    Wt = torch.empty(N, K, dtype=torch.bfloat16, device="cuda")
    L.check(lib.mac_pack_weight_bf16(L.ptr(W), L.ptr(Wt), K, N, L.stream_ptr()))
    torch.cuda.synchronize()
    assert torch.equal(Wt, W.t().contiguous().to(torch.bfloat16))
    y = torch.zeros(M, N, device="cuda")
    L.check(lib.mac_linear_tc_fwd(L.ptr(x), L.ptr(Wt), L.ptr(b), L.ACT[act], L.ptr(y), 0, M, K, N, L.stream_ptr()))
    torch.cuda.synchronize()
    z = x.float().cpu().numpy().astype(np.float64) @ Wt.float().cpu().numpy().astype(np.float64).T + b.cpu().numpy()
    ref = {"NON": z, "ELU": O.elu(z), "TANH": np.tanh(z)}[act]
    assert max_rel(y.cpu().numpy(), ref) < 1e-4
    if act in ("NON", "ELU"):        # bf16 output form used inside the read-unit chain
        yb = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
        L.check(lib.mac_linear_tc_fwd(L.ptr(x), L.ptr(Wt), L.ptr(b), L.ACT[act], L.ptr(yb), 1, M, K, N, L.stream_ptr()))
        torch.cuda.synchronize()
        assert max_rel(yb.float().cpu().numpy(), ref) < 6e-3
