"""Host plumbing of tensor-core training and inference for the flag sets outside the shipped flag files ("P2", SURVEY section
8(a)), against the dry-run library (tests/_mocklib.py): which products go to `mac_linear_tc_seg_fwd` / `mac_linear_bwd_tc` /
`mac_read_bwd_tc`, the bf16 weight packs and their cache, and every rejection (raised before any compute call).  Numerics are
in tests/test_gpu_linear_tc.py and tests/test_gpu_tape_tc.py."""
import numpy as np
import pytest
import torch

from mac_network_b200 import _lib as L_
from mac_network_b200.config import MACConfig
from tests import _mocklib
from tests._util import load_golden

P2_CASES = ["p2_control", "p2_control_feed", "p2_ablations", "p2_wholeq", "p2_unshared", "p2_read_bl", "p2_read_add",
            "p2_read_plain", "p2_read_noproj", "p2_write_info", "p2_write_sum", "p2_write_mem", "p2_write_mul",
            "p2_read_add_train", "p2_read_plain_train", "p2_memory_bn", "p2_memory_bn_train"]
SHIPPED = ["args", "args1", "args2", "args3", "args4", "gqa"]
NEW_ENTRY_POINTS = ("mac_linear_tc_seg_fwd", "mac_linear_bwd_tc")


class _Recorder(object):
    """Wraps the dry-run library and keeps each call's arguments."""

    def __init__(self, mock):
        self.mock, self.log = mock, []

    def __getattr__(self, name):
        fn = getattr(self.mock, name)

        def rec(*args):
            self.log.append((name, args))
            return fn(*args)
        return rec

    def args_of(self, name):
        return [a for n, a in self.log if n == name]

    def compute_calls(self):
        return [n for n, _ in self.log if not n.endswith("_workspace_bytes") and not n.endswith("_invariant_bytes")]


@pytest.fixture
def rec(monkeypatch):
    mock = _mocklib.install(monkeypatch)
    r = _Recorder(mock)
    monkeypatch.setattr(L_, "load", lambda: r)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True), raising=False)
    # the mock's size queries return 64 KB; give the read workspace its real extent so the bf16 slab views exist
    monkeypatch.setattr(mock, "mac_read_workspace_bytes",
                        lambda b, n, dd, pr: 4096 + (2 + pr * 3) * b * n * dd * 4 + 8192, raising=False)
    return r


def _cfg(case, d=128):
    meta, _ = load_golden(case)
    flags = dict(meta["cell_flags"], memDim=d, ctrlDim=d, attDim=d)
    return MACConfig(**flags).validate(), meta


def _cell(case, B=2, N=32, S=5, d=128, prec="bf16", train=True, save=True):
    from mac_network_b200.mac_cell import MACCell, MACParams
    from mac_network_b200.synthetic import make_inputs
    cfg, meta = _cfg(case, d)
    L = meta["shape"]["L"]
    params = MACParams(cfg, L, seed=1, device="cpu")
    x = {k: torch.from_numpy(v) for k, v in make_inputs(B, S, N, d, seed=2).items()}
    dm = meta["dropouts"]
    cell = MACCell(x["vecQuestions"], x["questionWords"], x["questionCntxWords"], x["questionLengths"], x["knowledgeBase"],
                   dm["memory"], dm["read"], dm["write"], B, train, config=cfg, params=params, prec=prec,
                   save_for_backward=save)
    return cell, cfg, L


def _bn_linears_per_step(cfg):
    """The composed read unit's [B*N, .] ops.linear calls per step (mac_cell.py:209-277, ops.py:668-725)."""
    n = 0
    if cfg.readProjInputs:
        n += 1                                                   # projX / proj on the knowledge base
    if cfg.readMemAttType == "BL":
        n += 1
    if cfg.readMemProj:
        n += 1 + (cfg.readMemAct != "NON")                       # memKbProj and its nested "_2" layer
    if cfg.readCtrl and cfg.readCtrlAttType == "BL":
        n += 1
    return n


def _M(name, args):
    return args[10] if name == "mac_linear_tc_seg_fwd" else args[12]


@pytest.mark.parametrize("case", P2_CASES)
def test_p2_bf16_training_routes_the_bn_rows_to_tensor_cores(rec, case):
    from mac_network_b200.autograd import mac_backward
    from mac_network_b200.mac_cell import mac_network
    B, N, d = 2, 32, 128
    cell, cfg, L = _cell(case, B=B, N=N, d=d)
    assert cell._use_tape, "every P2 flag set is differentiated on the tape"
    mac_network(cell, L)
    fused = cell._fused_read
    seg = rec.args_of("mac_linear_tc_seg_fwd")
    assert all(_M("mac_linear_tc_seg_fwd", a) == B * N for a in seg)
    assert all(_M("mac_linear_fwd", a) != B * N for a in rec.args_of("mac_linear_fwd"))
    assert len(seg) == (0 if fused else L * _bn_linears_per_step(cfg))
    assert rec.args_of("mac_read_fwd") == [] if not fused else len(rec.args_of("mac_read_fwd")) == L
    rec.log.clear()
    g = mac_backward(cell, torch.zeros(B, d), torch.zeros(B, d), tc=True)
    assert g["knowledgeBase"].shape == (B, N, d)
    assert len(rec.args_of("mac_linear_bwd_tc")) == len(seg)
    assert all(_M("mac_linear_bwd_tc", a) == B * N for a in rec.args_of("mac_linear_bwd_tc"))
    assert all(_M("mac_linear_bwd", a) != B * N for a in rec.args_of("mac_linear_bwd"))
    assert rec.args_of("mac_read_bwd") == []
    assert len(rec.args_of("mac_read_bwd_tc")) == (L if fused else 0)
    # the fp32 backward of the same bf16 forward never reaches the new entry points
    mac_network(cell, L)
    rec.log.clear()
    mac_backward(cell, torch.zeros(B, d), torch.zeros(B, d), tc=False)
    assert not any(n in NEW_ENTRY_POINTS + ("mac_read_bwd_tc",) for n, _ in rec.log)
    assert len(rec.args_of("mac_read_bwd")) == (L if fused else 0)


@pytest.mark.parametrize("case", P2_CASES)
def test_p2_bf16_cell_constructs_at_d128(rec, case):
    cell, cfg, L = _cell(case, save=False, train=False)
    assert cell._tc_general == (not cfg.is_fast_path)


def test_packs_are_cached_per_parameter_version(rec):
    from mac_network_b200.mac_cell import mac_network
    cell, cfg, L = _cell("p2_read_bl", save=False, train=False)
    mac_network(cell, L)
    first = len(rec.args_of("mac_pack_weight_bf16"))
    assert first == 5                   # shared proj, memInter BL, memKbProj, memKbProj_2 (readMemAct=TANH), ctrlInter BL
    rec.log.clear()
    mac_network(cell, L)
    assert rec.args_of("mac_pack_weight_bf16") == [] and len(rec.args_of("mac_linear_tc_seg_fwd")) > 0
    cell.params.touch()
    rec.log.clear()
    mac_network(cell, L)
    assert len(rec.args_of("mac_pack_weight_bf16")) == first


@pytest.mark.parametrize("variant", SHIPPED)
def test_shipped_flag_files_never_reach_the_new_entry_points(rec, variant):
    from mac_network_b200.autograd import mac_backward
    from mac_network_b200.mac_cell import MACCell, MACParams, mac_network
    from mac_network_b200.synthetic import make_inputs
    B, S, N, d, L = 2, 5, 32, 128, 2
    cfg = MACConfig.args(variant, netLength=L, memDim=d, ctrlDim=d, attDim=d)
    params = MACParams(cfg, L, seed=1, device="cpu")
    x = {k: torch.from_numpy(v) for k, v in make_inputs(B, S, N, d, seed=2).items()}
    for train in (False, True):
        cell = MACCell(x["vecQuestions"], x["questionWords"], x["questionCntxWords"], x["questionLengths"],
                       x["knowledgeBase"], 0.85 if train else 1.0, 0.85 if train else 1.0, 1.0, B, train, config=cfg,
                       params=params, prec="bf16", save_for_backward=train)
        mac_network(cell, L)
        if train:
            mac_backward(cell, torch.zeros(B, d), torch.zeros(B, d), tc=True)
    assert not any(n in NEW_ENTRY_POINTS for n, _ in rec.log)


def test_composed_bf16_rejects_d_not_a_multiple_of_128(rec):
    with pytest.raises(NotImplementedError, match="composed read unit"):
        _cell("p2_read_add", d=192, save=False, train=False)
    assert rec.compute_calls() == []


@pytest.mark.parametrize("prec", ["tc32", "fp8"])
@pytest.mark.parametrize("case", ["p2_read_bl", "p2_read_add", "p2_read_noproj", "p2_unshared", "p2_memory_bn_train"])
def test_tc32_and_fp8_keep_their_rejections(rec, prec, case):
    meta, _ = load_golden(case)
    for save in (False, True):
        if not save and MACConfig(**meta["cell_flags"]).is_fast_path and not meta["cell_flags"]["unsharedCells"]:
            continue                     # the shared-cell fused read unit in inference is what tc32 / fp8 cover
        rec.log.clear()
        with pytest.raises(NotImplementedError):
            _cell(case, d=512 if prec == "fp8" else 128, N=196 if prec == "fp8" else 32, prec=prec, save=save, train=save)
        assert rec.compute_calls() == []


def test_tape_tc_rejects_a_fused_read_with_bn_not_a_multiple_of_64(rec):
    from mac_network_b200.autograd import mac_backward
    from mac_network_b200.mac_cell import mac_network
    B, N, d = 3, 7, 128                                          # B*N = 21
    cell, cfg, L = _cell("p2_unshared", B=B, N=N, d=d)
    mac_network(cell, L)
    rec.log.clear()
    with pytest.raises(NotImplementedError, match="B\\*N"):
        mac_backward(cell, torch.zeros(B, d), torch.zeros(B, d), tc=True)
    assert rec.compute_calls() == []
    # the composed read unit has no such rule (B*N = 147 here)
    cell, cfg, L = _cell("p2_read_add_train", B=3, N=49, d=d)
    mac_network(cell, L)
    rec.log.clear()
    mac_backward(cell, torch.zeros(3, d), torch.zeros(3, d), tc=True)
    assert {a[12] for a in rec.args_of("mac_linear_bwd_tc")} == {147}


def test_tape_tc_needs_a_bf16_cell(rec):
    from mac_network_b200.autograd import mac_backward
    from mac_network_b200.mac_cell import mac_network
    cell, cfg, L = _cell("p2_read_bl", prec="fp32")
    mac_network(cell, L)
    rec.log.clear()
    with pytest.raises(NotImplementedError, match="fp32 kernels"):
        mac_backward(cell, torch.zeros(2, 128), torch.zeros(2, 128), tc=True)
    assert rec.compute_calls() == []


def test_entry_point_status_codes():
    """Shape and argument errors come back before any CUDA call (the real library, no GPU needed)."""
    import ctypes
    lib = L_.load()
    INVALID, ALIGN, UNSUPPORTED, WORKSPACE = -1, -2, -3, -4
    buf = (ctypes.c_float * 4096)()
    p = (ctypes.addressof(buf) + 15) & ~15
    ints = lambda *v: (ctypes.c_int * len(v))(*v)
    ptrs = lambda *v: (ctypes.c_void_p * len(v))(*v)
    big = 1 << 40

    def fwd(k=(128, 256), ld=None, n_out=128, ws=big, x=p, y=p, act=0):
        ld = ld or k
        return lib.mac_linear_tc_seg_fwd(ptrs(*[x] * len(k)), ints(*k), ints(*ld), len(k), p, None, 0.0, act, y, n_out, 70,
                                         n_out, p, ws, None)
    assert fwd(k=(128, 192)) == UNSUPPORTED
    assert fwd(n_out=192) == UNSUPPORTED
    assert fwd(x=None) == INVALID
    assert fwd(act=5) == INVALID
    assert fwd(k=(128, 128, 128, 128, 128)) == INVALID
    assert fwd(x=p + 4) == ALIGN
    assert fwd(ld=(132, 258)) == ALIGN
    assert fwd(ws=lib.mac_linear_tc_seg_workspace_bytes(70, 384) - 1) == WORKSPACE
    assert lib.mac_linear_tc_seg_workspace_bytes(70, 384) >= 70 * 384 * 2

    def bwd(k=(128,), n_out=128, ws=big, ldy=None, db=p, dW=p, dx=p, W=p):
        ldy = ldy or n_out
        return lib.mac_linear_bwd_tc(ptrs(*[p] * len(k)), ints(*k), ints(*k), len(k), W, p, ldy, ptrs(*[dx] * len(k)),
                                     ints(*k), ints(*[1] * len(k)), dW, db, 70, n_out, p, ws, None)
    assert bwd(k=(64,)) == UNSUPPORTED
    assert bwd(n_out=64) == UNSUPPORTED
    assert bwd(ldy=256) == UNSUPPORTED                          # the bias gradient reads dy as [M, n_out]
    assert bwd(W=None) == INVALID                               # data gradients need the weight
    assert bwd(dx=p + 4) == ALIGN
    need = lib.mac_linear_bwd_tc_workspace_bytes(70, ints(128), 1, 128)
    # bf16 dy, dy^T over Mp = 128 columns, x^T, the bf16 weight, the bias partials
    assert need >= 70 * 128 * 2 + 128 * 128 * 2 + 128 * 128 * 2 + 128 * 128 * 2 + 2 * 128 * 4
    assert bwd(ws=need - 1) == WORKSPACE
