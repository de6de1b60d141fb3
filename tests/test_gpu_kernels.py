"""Kernel-level GPU tests through the C ABI: K1 (control attention), K3 (KB attention), linear, dropout RNG."""
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


@pytest.mark.parametrize("B,N,d,nparts", [(64, 196, 512, 4), (3, 49, 512, 1), (2, 1, 64, 2), (5, 700, 128, 3),
                                          (2, 1500, 512, 1), (7, 33, 16, 1)])
def test_kb_attend(B, N, d, nparts):
    L, lib = _lib()
    rng = np.random.RandomState(0)
    parts = rng.standard_normal((B, N, nparts)).astype(np.float32)
    kb = rng.standard_normal((B, N, d)).astype(np.float32)
    br = 0.3
    tp, tk = torch.from_numpy(parts).cuda(), torch.from_numpy(kb).cuda()
    att = torch.empty(B, N, device="cuda")
    info = torch.empty(B, d, device="cuda")
    L.check(lib.mac_kb_attend_fwd(L.ptr(tp), nparts, br, L.ptr(tk), 0, L.ptr(att), L.ptr(info), B, N, d,
                                  L.stream_ptr()))
    torch.cuda.synchronize()
    logits = parts.astype(np.float64).sum(-1) + br
    a = O.softmax(logits)
    r = O.att2smry(a, kb.astype(np.float64))
    assert np.max(np.abs(att.cpu().numpy() - a)) < 1e-6
    assert max_rel(info.cpu().numpy(), r) < 1e-5
    # bf16 knowledge base (headline configuration): same attention, summary within bf16 rounding of KB
    if d % 64 == 0:
        tkb = tk.to(torch.bfloat16)
        L.check(lib.mac_kb_attend_fwd(L.ptr(tp), nparts, br, L.ptr(tkb), 1, L.ptr(att), L.ptr(info), B, N, d,
                                      L.stream_ptr()))
        torch.cuda.synchronize()
        r16 = O.att2smry(a, tkb.float().cpu().numpy().astype(np.float64))
        assert max_rel(info.cpu().numpy(), r16) < 1e-5


@pytest.mark.parametrize("T,B,S,d", [(12, 64, 40, 512), (1, 3, 1, 64), (4, 5, 45, 512), (3, 2, 7, 16)])
def test_control_attend(T, B, S, d):
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
    b = -0.2
    for separate in (False, True):
        ov = outw if separate else words
        t = {k: torch.from_numpy(v).cuda() for k, v in dict(cc=cc, words=words, ov=ov, w=w, lengths=lengths).items()}
        att = torch.empty(T, B, S, device="cuda")
        out = torch.empty(T, B, d, device="cuda")
        L.check(lib.mac_control_attend_fwd(L.ptr(t["cc"]), B * d, d, L.ptr(t["words"]), S * d, d,
                                           L.ptr(t["ov"] if separate else t["words"]), S * d, d, L.ptr(t["lengths"]),
                                           L.ptr(t["w"]), b, L.ptr(att), L.ptr(out), T, B, S, d, L.stream_ptr()))
        torch.cuda.synchronize()
        c64 = cc.astype(np.float64)
        logits = np.einsum("tbk,bsk,k->tbs", c64, words.astype(np.float64), w.astype(np.float64)) + b
        a = O.softmax(np.stack([O.exp_mask(l, lengths) for l in logits]))
        r = np.einsum("tbs,bsk->tbk", a, ov.astype(np.float64))
        got = att.cpu().numpy()
        assert np.max(np.abs(got - a)) < 2e-6
        for bi, n in enumerate(lengths):
            assert np.all(got[:, bi, n:] == 0.0)
        assert max_rel(out.cpu().numpy(), r) < 1e-5


@pytest.mark.parametrize("M,ks,n_out,act", [(64, [512], 512, "TANH"), (64, [512, 512], 512, "NON"),
                                            (64, [512, 512, 512], 512, "ELU"), (12544, [512], 512, "NON"),
                                            (37, [64, 16], 20, "SIGMOID"), (64, [512], 6144, "NON"),
                                            (700, [128], 128, "RELU_STD")])
def test_linear(M, ks, n_out, act):
    L, lib = _lib()
    rng = np.random.RandomState(2)
    xs = [rng.standard_normal((M, k)).astype(np.float32) for k in ks]
    K = sum(ks)
    W = (rng.standard_normal((K, n_out)) / np.sqrt(K)).astype(np.float32)
    b = rng.standard_normal((n_out,)).astype(np.float32)
    txs = [torch.from_numpy(x).cuda() for x in xs]
    tW, tb = torch.from_numpy(W).cuda(), torch.from_numpy(b).cuda()
    y = torch.empty(M, n_out, device="cuda")
    wsb = int(lib.mac_linear_workspace_bytes(M, K, n_out))
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    n = len(xs)
    for rep in range(2):      # twice: the split-K counters must be left at zero
        arr_p = (ctypes.c_void_p * n)(*[t.data_ptr() for t in txs])
        arr_k = (ctypes.c_int * n)(*ks)
        L.check(lib.mac_linear_fwd(arr_p, arr_k, arr_k, n, L.ptr(tW), L.ptr(tb), 0.25, L.ACT[act], L.ptr(y), n_out,
                                   M, n_out, L.ptr(ws), wsb, L.stream_ptr()))
        torch.cuda.synchronize()
        z = np.concatenate(xs, -1).astype(np.float64) @ W.astype(np.float64) + b + 0.25
        ref = {"NON": z, "TANH": np.tanh(z), "ELU": O.elu(z), "SIGMOID": 1 / (1 + np.exp(-z)),
               "RELU_STD": np.maximum(z, 0)}[act]
        assert max_rel(y.cpu().numpy(), ref) < 2e-5
    assert int(ws[:4096].to(torch.int32).abs().sum().item()) == 0


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
