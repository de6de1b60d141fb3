"""CPU side of the e4m3 read step (MAC_PREC_FP8): the fp64 restatement of the scheme (oracle/fp8_read_oracle.py), the host
plumbing of MACCell(prec="fp8") against the prototype table (tests/_mocklib.py), and the C ABI's rejections, which return
before any CUDA call."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import fp8_read_oracle as F8
from tests import _mocklib

D = 512


def test_e4m3_rounding_is_round_to_nearest_even_and_saturating():
    x = torch.tensor([1.0, 1.0625, 1.1875, 17.0, 448.0, 464.0, 1e6, -1e6, 2.0 ** -9, 2.0 ** -11, 0.0], dtype=torch.float64)
    # 1.0625 is the midpoint of 1 and 1.125 (ties to the even 1), 1.1875 of 1.125 and 1.25 (to 1.25); 17 of 16 and 18 (to 16)
    want = [1.0, 1.0, 1.25, 16.0, 448.0, 448.0, 448.0, -448.0, 2.0 ** -9, 0.0, 0.0]
    assert F8.e4m3(x).tolist() == want


def test_quantisation_scales_and_zero_rows():
    X = torch.randn(5, 64, dtype=torch.float64)
    X[2] = 0
    X8, s = F8.quant_rows(X)
    assert s.shape == (5, 1) and float(s[2]) == 0.0 and bool((X8[2] == 0).all())
    assert float(X8.abs().max()) == 448.0                      # each nonzero row's largest element maps to 448
    assert float(((X8 * s - X).abs() / X.abs().amax(1, keepdim=True).clamp_min(1e-300))[[0, 1, 3, 4]].max()) < 2 ** -4
    W8, sw = F8.pack_weight(X.T)                              # per output column of an [in, out] weight
    assert torch.equal(W8, X8.T) and torch.equal(sw, s.T)


def test_restatement_error_matches_the_emulated_scheme():
    """At a small slice of the headline configuration (args weights from init_params) the scheme's distance from fp64 is of
    the order the design estimate gives (att_kb ~2e-2, info ~7e-3 at B=64), about ten times the bf16 roundings'."""
    from mac_network_b200.config import MACConfig
    from mac_network_b200.params import init_params, perturb_biases
    from mac_network_b200.synthetic import make_inputs
    B, S, N, d, L = 8, 10, 196, D, 2
    cfg = MACConfig.args("args", netLength=L)
    pv = perturb_biases(init_params(cfg, L, seed=100, dtype=np.float64), seed=101)
    inp = make_inputs(B, S, N, d, seed=1234, dtype=np.float64)
    sc = "MACnetwork/MACCell/read/"
    T = lambda k: torch.tensor(pv[k])
    lin = lambda s: (T(s + "weights/weight"), T(s + "biases/bias"))
    Wx, bx = lin(sc + "mulmemInter/linearLayerprojX/")
    Wy, by = lin(sc + "mulmemInter/linearLayerprojY/")
    Wm, bm = lin(sc + "linearLayermemKbProj/")
    Wm2, bm2 = lin(sc + "linearLayermemKbProj/linearLayermemKbProj_2/")
    wr, br = lin(sc + "inter2att/inter2logits/linearLayerlogits/")
    KB = torch.tensor(inp["knowledgeBase"]).reshape(B * N, d)
    ctrl = torch.tensor(inp["vecQuestions"])
    mem = torch.randn(B, d, dtype=torch.float64, generator=torch.Generator().manual_seed(7))
    y = mem @ Wy + by
    att8, info8 = F8.read_step_from_weights(KB, y, ctrl, Wx, bx, Wm, bm, Wm2, bm2, wr, float(br), N)
    rows = lambda v: v.repeat_interleave(N, 0)
    elu = torch.nn.functional.elu
    P = KB @ Wx + bx
    H = elu((P * rows(y)) @ Wm[:d] + P @ Wm[d:] + bm)
    att0 = torch.softmax((elu((H @ Wm2 + bm2) * rows(ctrl)) @ wr + float(br)).reshape(B, N), 1)
    info0 = torch.einsum("bn,bnd->bd", att0, KB.reshape(B, N, d))
    mr = lambda a, b: float((a - b).abs().max() / b.abs().max())
    e_att, e_info = mr(att8, att0), mr(info8, info0)
    assert 2e-3 < e_att < 6e-2, e_att
    assert 5e-4 < e_info < 2e-2, e_info


def _fp8_cell(monkeypatch, B=2, S=5, N=49, d=D, L=2, flags="args", keeps=(1.0, 1.0, 1.0), cfg_kw=None, **kw):
    mock = _mocklib.install(monkeypatch)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True), raising=False)
    from mac_network_b200.config import MACConfig
    from mac_network_b200.mac_cell import MACCell, MACParams
    from mac_network_b200.synthetic import make_inputs
    cfg = MACConfig.args(flags, netLength=L, memDim=d, ctrlDim=d, attDim=d, **(cfg_kw or {}))
    params = MACParams(cfg, L, seed=1, device="cpu")
    x = {k: torch.from_numpy(v) for k, v in make_inputs(B, S, N, d, seed=2).items()}
    make = lambda: MACCell(x["vecQuestions"], x["questionWords"], x["questionCntxWords"], x["questionLengths"],
                           x["knowledgeBase"], keeps[0], keeps[1], keeps[2], B, False, config=cfg, params=params,
                           prec="fp8", **kw)
    return mock, make


@pytest.mark.parametrize("small_tc", [False, True])
def test_fp8_cell_host_calls(monkeypatch, small_tc):
    """MACCell(prec="fp8"): the bf16 packs (P and Q) and the e4m3 packs of Wm[0:d] and Wm2 once per parameter version, the
    bf16 knowledge base, one mac_read_invariant and one mac_read_fwd_inv per step, both with MAC_PREC_FP8 and the e4m3
    weights in mac_read_weights; the batch-sized projections as in bf16 (small_tc included)."""
    from mac_network_b200.mac_cell import mac_network
    L = 3
    mock, make = _fp8_cell(monkeypatch, L=L, small_tc=small_tc)
    seen = {}
    for name in ("mac_read_invariant", "mac_read_fwd_inv", "mac_pack_weight_fp8"):
        fn = getattr(mock, name)

        def spy(*a, _fn=fn, _name=name):
            seen.setdefault(_name, []).append(a)
            return _fn(*a)
        setattr(mock, name, spy)
    cell = make()
    control, memory = mac_network(cell, L)
    assert control.shape == (2, D) and memory.shape == (2, D) and len(cell.attentions["kb"]) == L
    assert mock.calls.count("mac_read_invariant") == 1 and mock.calls.count("mac_read_fwd_inv") == L
    assert mock.calls.count("mac_pack_weight_fp8") == 2 and mock.calls.count("mac_pack_weight_bf16") == 3
    assert mock.calls.count("mac_cast_bf16") == 1 and "mac_read_fwd" not in mock.calls
    assert all(a[3] == 3 for a in seen["mac_read_invariant"]) and all(a[7] == 3 for a in seen["mac_read_fwd_inv"])
    assert [(a[3], a[4]) for a in seen["mac_pack_weight_fp8"]] == [(D, D), (D, D)]     # Wm[0:d] and Wm2, K x n_out
    rw = seen["mac_read_fwd_inv"][0][6]._obj
    assert rw.Wm_fp8 and rw.Wm_fp8_scale and rw.Wm2_fp8 and rw.Wm2_fp8_scale and rw.Wx_bf16 and rw.Wm_bf16
    assert ("mac_linear_tc_small_fwd" in mock.calls) == small_tc
    # a second pass reuses the packs; a parameter update repacks
    mac_network(make(), L)
    assert mock.calls.count("mac_pack_weight_fp8") == 2
    cell.params.touch()
    mac_network(make(), L)
    assert mock.calls.count("mac_pack_weight_fp8") == 4


@pytest.mark.parametrize("what", ["train", "read_dropout", "unshared", "N", "d"])
def test_fp8_cell_rejections(monkeypatch, what):
    """prec="fp8" is the inference read step only: training, read dropout, unshared cells and shapes the kernel does not
    take raise NotImplementedError before the library is asked to compute anything."""
    kw = {"train": dict(save_for_backward=True), "read_dropout": dict(keeps=(1.0, 0.85, 1.0)),
          "unshared": dict(cfg_kw={"unsharedCells": True}), "N": dict(N=257), "d": dict(d=256)}[what]
    mock, make = _fp8_cell(monkeypatch, **kw)
    with pytest.raises(NotImplementedError):
        make()
    assert all(c.endswith("_bytes") or c == "mac_b200_abi_version" for c in mock.calls), mock.calls


def test_fp8_c_abi_rejections_need_no_gpu():
    """MAC_PREC_FP8 outside the inference read step comes back as MAC_ERR_UNSUPPORTED before any CUDA call."""
    from mac_network_b200 import _lib
    lib = _lib.load()
    UNSUPPORTED, INVALID = -3, -1
    buf = (ctypes.c_float * 4096)()
    p = (ctypes.addressof(buf) + 15) & ~15                 # 16-byte aligned fake "device" pointer (never dereferenced)
    rw = _lib.ReadWeights()
    assert lib.mac_read_fwd(p, p, p, p, ctypes.byref(rw), 1.0, 0, 0, 3, p, p, None, p, 1 << 30, 2, 49, D, None) == UNSUPPORTED
    assert lib.mac_read_fwd_inv(None, p, p, None, p, p, ctypes.byref(rw), 3, p, p, p, 1 << 30, 2, 300, D, None) == UNSUPPORTED
    assert lib.mac_read_fwd_inv(None, p, p, None, p, p, ctypes.byref(rw), 3, p, p, p, 1 << 30, 2, 49, 256, None) == UNSUPPORTED
    assert lib.mac_read_fwd_inv(p, None, p, None, p, p, ctypes.byref(rw), 3, p, p, p, 1 << 30, 2, 49, D, None) == UNSUPPORTED
    assert lib.mac_read_invariant(None, p, ctypes.byref(rw), 3, p, 1 << 30, 2, 300, D, None) == UNSUPPORTED
    assert lib.mac_read_invariant(p, None, ctypes.byref(rw), 3, p, 1 << 30, 2, 49, D, None) == UNSUPPORTED
    assert lib.mac_pack_weight_fp8(None, p, p, 4, 4, None) == INVALID
    M = 64 * 196
    assert lib.mac_read_invariant_bytes(64, 196, D, 3) >= M * D * 5 + M * 8
