"""Host plumbing of split-bf16 ("tc32") training against the dry-run library (tests/_mocklib.py): which entry points the
training forward and both backward forms reach, the Wm_s3 pack and its cache, and every rejection (raised before any
compute call).  Numerics are in tests/test_gpu_tc32_training.py."""
import ctypes

import pytest
import torch

from mac_network_b200 import _lib as L_
from mac_network_b200.config import MACConfig
from tests.test_linear_tc_host import SHIPPED, _cell, rec  # noqa: F401  (rec is a fixture)


def _shipped_cell(variant, B=2, N=32, d=128, L=2, prec="tc32", tape_bwd=False, kb_dtype=None):
    from mac_network_b200.mac_cell import MACCell, MACParams
    from mac_network_b200.synthetic import make_inputs
    cfg = MACConfig.args(variant, netLength=L, memDim=d, ctrlDim=d, attDim=d)
    params = MACParams(cfg, L, seed=1, device="cpu")
    x = {k: torch.from_numpy(v) for k, v in make_inputs(B, 5, N, d, seed=2).items()}
    kb = x["knowledgeBase"] if kb_dtype is None else x["knowledgeBase"].to(kb_dtype)
    return MACCell(x["vecQuestions"], x["questionWords"], x["questionCntxWords"], x["questionLengths"], kb, 0.85, 0.85, 1.0,
                   B, True, config=cfg, params=params, prec=prec, save_for_backward=True, tape_bwd=tape_bwd), L


def _rw(args):
    return ctypes.cast(args[4], ctypes.POINTER(L_.ReadWeights)).contents if isinstance(args[4], int) else args[4]._obj


@pytest.mark.parametrize("variant", SHIPPED)
@pytest.mark.parametrize("shared_qinput", [True, False])
def test_tc32_training_reaches_the_split_entry_points(rec, variant, shared_qinput):
    from mac_network_b200.autograd import mac_backward
    from mac_network_b200.mac_cell import MACCell, MACParams, mac_network
    from mac_network_b200.synthetic import make_inputs
    B, N, d, L = (5, 49, 128, 2) if variant == "gqa" else (2, 32, 128, 2)        # gqa: B*N = 245
    cfg = MACConfig.args(variant, netLength=L, memDim=d, ctrlDim=d, attDim=d, controlInputUnshared=not shared_qinput)
    params = MACParams(cfg, L, seed=1, device="cpu")
    x = {k: torch.from_numpy(v) for k, v in make_inputs(B, 5, N, d, seed=2).items()}
    cell = MACCell(x["vecQuestions"], x["questionWords"], x["questionCntxWords"], x["questionLengths"], x["knowledgeBase"],
                   0.85, 0.85, 1.0, B, True, config=cfg, params=params, prec="tc32", save_for_backward=True)
    mac_network(cell, L)
    fwd = rec.args_of("mac_read_fwd")
    assert len(fwd) == L and all(a[8] == 2 and a[11] is not None for a in fwd)
    rw = _rw(fwd[0])
    assert rw.Wx_s3 and rw.Wm_s3 and rw.Wm2_s3
    assert rec.args_of("mac_read_fwd_inv") == [] and rec.args_of("mac_read_invariant") == []
    rec.log.clear()
    mac_backward(cell, torch.zeros(B, d), torch.zeros(B, d), tc=True)
    assert len(rec.args_of("mac_read_bwd_tc32")) == L
    assert rec.args_of("mac_read_bwd_tc") == [] and rec.args_of("mac_read_bwd") == []
    assert {a[-4:-1] for a in rec.args_of("mac_read_bwd_tc32")} == {(B, N, d)}
    # tc=False: the fp32 backward of the same tc32 forward
    mac_network(cell, L)
    rec.log.clear()
    mac_backward(cell, torch.zeros(B, d), torch.zeros(B, d), tc=False)
    assert len(rec.args_of("mac_read_bwd")) == L
    assert rec.args_of("mac_read_bwd_tc32") == [] and rec.args_of("mac_read_bwd_tc") == []


def test_wm_s3_is_cached_and_repacked_after_touch(rec):
    from mac_network_b200.mac_cell import mac_network
    d = 128
    cell, L = _shipped_cell("args", d=d)
    whole = lambda: [a for a in rec.args_of("mac_pack_weight_split3") if a[2] == 2 * d]     # K = 2d: the whole Wm
    mac_network(cell, L)
    assert len(whole()) == 1
    rec.log.clear()
    mac_network(cell, L)
    assert whole() == []
    cell.params.touch()
    rec.log.clear()
    mac_network(cell, L)
    assert len(whole()) == 1


def test_tc32_inference_does_not_pack_wm_s3(rec):
    from mac_network_b200.mac_cell import MACCell, MACParams, mac_network
    from mac_network_b200.synthetic import make_inputs
    B, N, d, L = 2, 32, 128, 2
    cfg = MACConfig.args("args", netLength=L, memDim=d, ctrlDim=d, attDim=d)
    x = {k: torch.from_numpy(v) for k, v in make_inputs(B, 5, N, d, seed=2).items()}
    cell = MACCell(x["vecQuestions"], x["questionWords"], x["questionCntxWords"], x["questionLengths"], x["knowledgeBase"],
                   1.0, 1.0, 1.0, B, False, config=cfg, params=MACParams(cfg, L, seed=1, device="cpu"), prec="tc32")
    mac_network(cell, L)
    assert all(a[2] == d for a in rec.args_of("mac_pack_weight_split3"))
    assert rec.args_of("mac_read_fwd") == [] and len(rec.args_of("mac_read_fwd_inv")) == L


@pytest.mark.parametrize("what", ["tape_bwd", "p2_unshared", "p2_memory_bn_train", "bf16_kb", "d192"])
def test_tc32_training_rejections_launch_nothing(rec, what):
    with pytest.raises(NotImplementedError):
        if what == "tape_bwd":
            _shipped_cell("args", tape_bwd=True)
        elif what == "bf16_kb":
            _shipped_cell("args", kb_dtype=torch.bfloat16)
        elif what == "d192":
            _shipped_cell("args", d=192)
        else:
            _cell(what, prec="tc32", save=True, train=True)
    assert rec.compute_calls() == []
