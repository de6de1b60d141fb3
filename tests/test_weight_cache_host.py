"""The weight-derived tensors (mac_network_b200/packs.py) follow the parameter values, against the dry-run library
(tests/_mocklib.py): a cell kept across `params.touch()` hands the read unit pointers into the new packs, a view and its
base get packs of their own, and the stem / output unit drop their packs when their `version` moves."""
import numpy as np
import torch

from mac_network_b200 import packs
from mac_network_b200.config import MACConfig
from tests.test_linear_tc_host import rec  # noqa: F401  (a fixture)

B, N, d, L = 2, 32, 128, 2


def _cell(prec, train):
    from mac_network_b200.mac_cell import MACCell, MACParams
    from mac_network_b200.synthetic import make_inputs
    cfg = MACConfig.args("args", netLength=L, memDim=d, ctrlDim=d, attDim=d)
    x = {k: torch.from_numpy(v) for k, v in make_inputs(B, 5, N, d, seed=2).items()}
    keep = 0.85 if train else 1.0
    return MACCell(x["vecQuestions"], x["questionWords"], x["questionCntxWords"], x["questionLengths"], x["knowledgeBase"],
                   keep, keep, 1.0, B, train, config=cfg, params=MACParams(cfg, L, seed=1, device="cpu"), prec=prec,
                   save_for_backward=train)


def _read_weights(rec, name, i):
    """The ReadWeights struct each call of `name` was handed (argument i, passed by reference)."""
    return [a[i]._obj for a in rec.args_of(name)]


def _outputs(rec, name):
    """The output addresses of every call of the pack entry point `name`."""
    return {a[1].value for a in rec.args_of(name)}


def test_a_cell_kept_across_touch_reads_the_new_packs(rec):
    from mac_network_b200.autograd import mac_backward
    from mac_network_b200.mac_cell import mac_network
    # bf16 inference: Wx, Wm, Wm2 in bf16
    cell = _cell("bf16", train=False)
    mac_network(cell, L)
    cell.params.touch()
    rec.log.clear()
    mac_network(cell, L)
    new = _outputs(rec, "mac_pack_weight_bf16")
    assert len(new) == 3
    rws = _read_weights(rec, "mac_read_invariant", 2) + _read_weights(rec, "mac_read_fwd_inv", 6)
    assert len(rws) == 1 + L
    assert all({rw.Wx_bf16, rw.Wm_bf16, rw.Wm2_bf16} == new for rw in rws)
    # tc32 training: Wx, Wm[:d], Wm[d:], Wm2 and the whole Wm in split bf16, forward and backward
    cell = _cell("tc32", train=True)
    mac_network(cell, L)
    mac_backward(cell, torch.zeros(B, d), torch.zeros(B, d), tc=True)
    cell.params.touch()
    rec.log.clear()
    mac_network(cell, L)
    mac_backward(cell, torch.zeros(B, d), torch.zeros(B, d), tc=True)
    new = _outputs(rec, "mac_pack_weight_split3")
    assert len(new) == 5
    rws = _read_weights(rec, "mac_read_fwd", 4) + _read_weights(rec, "mac_read_bwd_tc32", 3)
    assert len(rws) == 2 * L
    assert all({rw.Wx_s3, rw.Wma_s3, rw.Wmb_s3, rw.Wm2_s3, rw.Wm_s3} == new for rw in rws)


def test_a_view_and_its_base_get_distinct_split3_packs(rec):
    from mac_network_b200.mac_cell import mac_network
    cell = _cell("tc32", train=True)
    mac_network(cell, L)
    npack = len(rec.args_of("mac_pack_weight_split3"))
    p = cell.params
    Wm, _ = p.lin("MACCell/read/", "memKbProj")
    assert Wm.shape == (2 * d, d) and Wm[:d].data_ptr() == Wm.data_ptr()
    head, whole = p.cache.pack(packs.split3, Wm[:d]), p.cache.pack(packs.split3, Wm)
    assert head.shape == (d, 3 * d) and whole.shape == (d, 3 * 2 * d)
    assert len(rec.args_of("mac_pack_weight_split3")) == npack                  # both were built by the forward
    rw = _read_weights(rec, "mac_read_fwd", 4)[-1]
    assert (rw.Wma_s3, rw.Wm_s3) == (head.data_ptr(), whole.data_ptr())


def test_stem_and_output_unit_drop_their_packs_when_the_version_moves(rec):
    from mac_network_b200.output_unit import OutputUnit, init_output_params, output_specs
    from mac_network_b200.stem import Stem, init_stem_params, stem_specs
    cpu = lambda values: {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in values.items()}
    version = [0]
    st = Stem(cpu(init_stem_params(stem_specs(128, 128), seed=1)), relu="ELU", prec="bf16", version=lambda: version[0])
    st.forward(torch.zeros(2, 3, 3, 128))
    packed = [st._weights(i)[1] for i in range(2)]
    assert [st._weights(i)[1] for i in range(2)] == packed and len(rec.args_of("mac_pack_weight_bf16")) == 2
    version[0] += 1
    st.forward(torch.zeros(2, 3, 3, 128))
    assert len(rec.args_of("mac_pack_weight_bf16")) == 4
    assert all(st._weights(i)[1] is not packed[i] for i in range(2))

    p = cpu(init_output_params(output_specs(8, 8, [16], 8), seed=1))
    ou = OutputUnit(p, relu="ELU", version=lambda: version[0])
    grads = {k: torch.zeros_like(v) for k, v in p.items()}
    wn = "classifier/linearLayerfc_1/weights/weight"

    def backward():
        ou.forward(torch.zeros(2, 8), torch.zeros(2, 8), torch.zeros(2, dtype=torch.int32))
        rec.log.clear()
        ou.backward(grads, torch.zeros(2, 8), torch.zeros(2, 8))
        Wt = ou._cache.pack(packs.transposed, p[wn])
        assert rec.args_of("mac_linear_bwd")[0][4].value == Wt.data_ptr()     # fc_1 first: the sweep runs backwards
        return Wt
    Wt = backward()
    assert backward() is Wt
    version[0] += 1
    assert backward() is not Wt
