"""GPU tests of the tensor-core question encoder (QuestionEncoder(prec="bf16"), csrc/encoder_tc.cuh): the entry points against
the fp64 restatement of their own bf16 operands (oracle/encoder_tc_oracle.py), the encoder against the fp64 model, bit-exact
repeats, and whole-model training with DPTrainer(enc_prec="bf16")."""
import json
import os

import numpy as np
import pytest
import torch

from mac_network_b200.encoder import encoder_specs, init_encoder_params
from oracle import encoder_torch_autograd
from oracle.encoder_oracle import encoder_forward
from oracle.encoder_tc_oracle import EncoderTC
from tests._util import GOLDEN_DIR

# ---- bounds; measured worst value on the H100 beside each
# against the restatement of the kernels' own bf16 operands (max-abs error / max-abs reference, per tensor); the gap is
# fp32 against fp64 arithmetic moving a bf16 rounding of h or of a gate gradient now and then          measured
TOL_OWN = {"out": 8e-4,              # questionCntxWords, vecQuestions                                2.6e-4
           "saved": 1e-3,            # gates, c, h_prev                                               3.3e-4
           "grad": 1.8e-3}           # kernels, biases, embeddings                                    5.8e-4
# QuestionEncoder(prec="bf16") against the fp64 encoder at B=64, S=40, E=300, 2 x 256 (max-rel per tensor)
TOL_FP64 = {"out": 1.2e-2,                                                                          # 3.9e-3
            "grad": 9e-3}                                                                           # 2.9e-3
# encoder slice of the whole-model gradient bucket, enc_prec="bf16" against "fp32" (max-rel per tensor)
TOL_TRAINER_ENC = 1e-2                                                                              # 3.2e-3


def _rel(got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    return float(np.max(np.abs(got - ref)) / max(np.max(np.abs(ref)), 1e-30))


def _batch(B, S, V, seed):
    rng = np.random.RandomState(seed)
    lengths = rng.randint(1, S + 1, size=(B,)).astype(np.int32)
    lengths[0] = S                                 # lengths include S and 1
    if B > 1:
        lengths[1] = 1
    q = rng.randint(1, V + 1, size=(B, S)).astype(np.int32)
    q[np.arange(S)[None, :] >= lengths[:, None]] = 0
    return q, lengths


def _dev(pv):
    return {k: torch.from_numpy(np.ascontiguousarray(v, dtype=np.float32)).cuda() for k, v in pv.items()}


def _run(pv, q, lengths, keeps, d_cntx, d_vecq, seed=5, step=1):
    from mac_network_b200.encoder import QuestionEncoder
    dev = _dev(pv)
    enc = QuestionEncoder(dev, keep_input=keeps[0], keep_question=keeps[1], seed=seed, prec="bf16")
    words, cntx, vecq = enc.forward(torch.from_numpy(q).cuda(), torch.from_numpy(lengths).cuda(), step=step,
                                    save_for_backward=True)
    grads = {k: torch.zeros_like(v) for k, v in dev.items()}
    enc.backward(torch.from_numpy(d_cntx.astype(np.float32)).cuda(), torch.from_numpy(d_vecq.astype(np.float32)).cuda(),
                 grads)
    torch.cuda.synchronize()
    sv = enc._saved
    out = dict(words=words.cpu().numpy(), cntx=cntx.cpu().numpy(), vecq=vecq.cpu().numpy(),
               sg=sv["sg"].cpu().numpy(), sc=sv["sc"].cpu().numpy(), shp=sv["shp"].cpu().numpy(),
               grads={k: v.cpu().numpy() for k, v in grads.items()})
    return enc, out


def _inputs(B, S, V, E, D, seed):
    pv = init_encoder_params(encoder_specs(V, E, D), seed=seed, dtype=np.float32)      # the values the device holds
    pv = {k: v.astype(np.float64) for k, v in pv.items()}
    q, lengths = _batch(B, S, V, seed + 1)
    rng = np.random.RandomState(seed + 2)
    return pv, q, lengths, rng.standard_normal((B, S, D)) / np.sqrt(S), rng.standard_normal((B, D))


@pytest.mark.gpu
@pytest.mark.parametrize("keeps", [(1.0, 1.0), (0.85, 0.92)])
@pytest.mark.parametrize("B,S,E", [(64, 40, 300), (13, 11, 256), (65, 7, 300), (1, 1, 256), (64, 40, 256), (13, 11, 300)])
def test_entry_points_against_own_operand_restatement(B, S, E, keeps):
    """Outputs, saved tensors and every gradient against fp64 products of the same bf16 operands (h rounded before each
    step's product, the gate gradients before each of theirs).  B = 65 runs two clusters per direction with a one-row
    second; padded rows of B*S and E are zeros in every operand."""
    V, D = 50, 512
    pv, q, lengths, d_cntx, d_vecq = _inputs(B, S, V, E, D, seed=B + S + E)
    enc, got = _run(pv, q, lengths, keeps, d_cntx, d_vecq)
    us = enc.dropout_uniforms(B, S, step=1)
    ref = EncoderTC(pv, keeps[0], keeps[1], uniforms=us)
    fo = ref.forward(q, lengths)
    gr = ref.backward(d_cntx, d_vecq)
    nd, M = 2, B * S
    errs = {"cntx": _rel(got["cntx"], fo["questionCntxWords"]), "vecq": _rel(got["vecq"], fo["vecQuestions"])}
    assert _rel(got["words"], fo["questionWords"]) == 0.0
    for name, key in (("sg", "gates"), ("sc", "c"), ("shp", "hprev")):
        errs[name] = _rel(got[name], np.stack([a.reshape(M, -1) for a in fo[key]]).reshape(nd, M, -1))
    for k, g in gr.items():
        errs[k] = _rel(got["grads"][k], g)
    print("own-operand (B=%d S=%d E=%d keeps=%s):" % (B, S, E, keeps), {k: "%.1e" % v for k, v in errs.items()})
    pad = np.arange(S)[None, :] >= lengths[:, None]
    assert np.all(got["cntx"][pad] == 0)
    bad = {k: v for k, v in errs.items()
           if not v < TOL_OWN["out" if k in ("cntx", "vecq") else "saved" if k in ("sg", "sc", "shp") else "grad"]}
    assert not bad, bad


@pytest.mark.gpu
@pytest.mark.parametrize("keeps", [(1.0, 1.0), (0.85, 0.92)])
def test_encoder_bf16_against_fp64(keeps):
    """The bf16 encoder at the headline question shape against the fp64 encoder (oracle/encoder_oracle.py) and its
    torch.autograd gradients."""
    B, S, V, E, D = 64, 40, 90, 300, 512
    pv, q, lengths, d_cntx, d_vecq = _inputs(B, S, V, E, D, seed=41)
    enc, got = _run(pv, q, lengths, keeps, d_cntx, d_vecq)
    us = enc.dropout_uniforms(B, S, step=1)
    ref = encoder_forward(pv, q, lengths, keeps[0], keeps[1], uniforms=us)
    errs = {"cntx": _rel(got["cntx"], ref["questionCntxWords"]), "vecq": _rel(got["vecq"], ref["vecQuestions"])}
    _, _, gref = encoder_torch_autograd.run(pv, q, lengths, keeps[0], keeps[1], us, d_cntx=d_cntx, d_vecq=d_vecq)
    for k, g in gref.items():
        errs[k] = _rel(got["grads"][k], g)
    print("bf16 vs fp64 (keeps=%s):" % (keeps,), {k: "%.1e" % v for k, v in errs.items()})
    bad = {k: v for k, v in errs.items() if not v < TOL_FP64["out" if k in ("cntx", "vecq") else "grad"]}
    assert not bad, bad


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["encoder_eval", "encoder_train", "encoder_proj", "encoder_uni"])
def test_golden_fixture_shapes_raise(case):
    """Every encoder fixture has h = 8, which the bf16 path does not support: it raises before any launch."""
    from mac_network_b200.encoder import QuestionEncoder
    z = np.load(os.path.join(GOLDEN_DIR, case + ".npz"))
    meta = json.loads(bytes(z["meta_json"]).decode())
    sh = meta["shape"]
    specs = encoder_specs(sh["V"], sh["E"], sh["encDim"], ctrl_dim=sh["ctrlDim"], bi=meta.get("bi", True), proj=meta["proj"])
    pv = init_encoder_params(specs, seed=meta["param_seed"])
    with pytest.raises(NotImplementedError):
        QuestionEncoder(_dev(pv), prec="bf16")


@pytest.mark.gpu
def test_encoder_bf16_is_deterministic():
    B, S, V, E, D = 65, 23, 40, 300, 512
    pv, q, lengths, d_cntx, d_vecq = _inputs(B, S, V, E, D, seed=9)
    _, a = _run(pv, q, lengths, (0.85, 0.92), d_cntx, d_vecq)
    _, b = _run(pv, q, lengths, (0.85, 0.92), d_cntx, d_vecq)
    for k in ("words", "cntx", "vecq", "sg", "sc", "shp"):
        assert np.array_equal(a[k], b[k]), k
    for k in a["grads"]:
        assert np.array_equal(a["grads"][k], b["grads"][k]), k


def _full_setup(seed):
    from tests.test_full_model import _make
    B, S, V, E, d, H, W, C, A, L = 16, 7, 13, 300, 512, 4, 4, 128, 8, 2      # ctrlDim 512: h = 256 per direction
    cfg, data = _make(B, S, V, E, d, H, W, C, A, L, seed=seed)
    return cfg, data, dict(classifier=(A, [32]), encoder=(V, E), stem=(C, 2)), B, L


@pytest.mark.gpu
def test_full_model_bf16_encoder_train_steps_reduce_loss():
    """12 whole-model steps with the encoder, the cell and the stem on tensor cores: the loss goes down, the encoder moves."""
    from mac_network_b200.dp import DPTrainer
    cfg, data, kw, B, L = _full_setup(21)
    tr = DPTrainer(cfg, L, seed=6, lr=3e-4, prec="bf16", bwd_tc=True, stem_prec="bf16", enc_prec="bf16", **kw)
    dev = {k: torch.from_numpy(v).cuda() for k, v in data.items()}
    before = {k: v.clone() for k, v in tr.params.t.items()}
    hist = []
    for _ in range(12):
        _, losses = tr.train_step_full("t", dev, global_batch=B)
        hist.append(float(losses.mean().item()))
    print("losses", [round(h, 4) for h in hist])
    assert np.all(np.isfinite(hist)) and min(hist[-3:]) < hist[0], hist
    for prefix in ("encoder/", "qEmbeddings/"):
        moved = [float((tr.params.t[k] - before[k]).abs().max().item()) for k in before if k.startswith(prefix)]
        assert moved and max(moved) > 0, prefix


@pytest.mark.gpu
def test_full_model_bf16_encoder_gradient_matches_fp32_encoder():
    """Dropouts off, same parameters and data: the encoder's slice of the gradient bucket with enc_prec="bf16" against the
    enc_prec="fp32" twin (cell and stem on tensor cores in both)."""
    from mac_network_b200.dp import DPTrainer
    cfg, data, kw, B, L = _full_setup(31)
    off = dict(dropouts=(1.0, 1.0, 1.0), output_dropout=1.0, enc_dropouts=(1.0, 1.0), stem_dropout=1.0)
    dev = {k: torch.from_numpy(v).cuda() for k, v in data.items()}
    buckets, ref_flat = {}, None
    for ep in ("fp32", "bf16"):
        tr = DPTrainer(cfg, L, seed=7, prec="bf16", bwd_tc=True, stem_prec="bf16", enc_prec=ep, **kw, **off)
        if ref_flat is None:
            ref_flat = tr.params.flat.clone()
        tr.params.flat.copy_(ref_flat)
        tr.params.touch()
        tr.full_forward_backward("t", dev, global_batch=B)
        torch.cuda.synchronize()
        buckets[ep] = tr.bucket.double().cpu()
    errs = {}
    for n in (n for n in tr.params.specs if n.startswith(("encoder/", "qEmbeddings/"))):
        o, k = tr.params.offsets[n], int(np.prod(tr.params.specs[n][0]))
        ref = buckets["fp32"][o:o + k]
        errs[n] = float((buckets["bf16"][o:o + k] - ref).abs().max() / ref.abs().max())
    print("encoder gradient bf16 vs fp32 encoder:", {k: "%.2e" % v for k, v in errs.items()})
    bad = {k: v for k, v in errs.items() if not v < TOL_TRAINER_ENC}
    assert not bad, bad
