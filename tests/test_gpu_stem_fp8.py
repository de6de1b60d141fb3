"""The e4m3 inference stem (Stem(prec="fp8"), csrc/tc_gemm_fp8.cuh) on the GPU.

- mac_im2col3x3_fp8 against the restatement (oracle/fp8_stem_oracle.py), which uses the kernel's own fp32 operations: the
  e4m3 bytes and the row scales are equal bit for bit.
- mac_linear_fp8_fwd against fp64 products of its own e4m3 operands and scales, at the stem's K and n_out and at M that are
  not multiples of 128; two runs give identical bits.
- The stem at the headline shape against the fp64 restatement of the fp32 stem, and the whole MACnet evaluation with the
  e4m3 stem and read step against the fp32 model.
Each bound is about three times the value measured on an H100 80GB HBM3 (700 W power limit, 1980 MHz max SM clock),
written beside it."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import fp8_stem_oracle as F8S

pytestmark = pytest.mark.gpu

# mac_linear_fp8_fwd against fp64 of its own operands, max|y - ref| / max|ref|: the e4m3 wgmma's own accumulation inside
# each 128-element k-block (a single-level accumulator over all of K measured 1.5e-3 to 4.3e-3)       measured
TOL_LINEAR = 5e-4                                                                               # 0.9e-4 .. 1.7e-4
# the stem at B=64, 14x14, 1024 -> 512 -> 512 (max-norm relative)
TOL_STEM = 1.5e-1            # against the fp64 fp32 stem (the bf16 stem: 3.3e-3)                  4.9e-2
TOL_STEM_REST = 1.2e-2       # against the e4m3 restatement: layer 1's roundings flip where layer 0 differs   4.0e-3
# MACnet evaluation, prec="fp8" with eval_stem_prec="fp8", against prec="fp32" (max-norm relative; with the bf16 stem:
# 2.2e-3, 2.4e-3 and 6.1e-3)
TOL_MODEL = {"logits": 8e-2,                                                                    # 2.8e-2
             "memory": 1.2e-1,                                                                  # 3.8e-2
             "att_kb": 3e-2}                                                                    # 9.0e-3


def _lib():
    from mac_network_b200 import _lib as L_
    return L_, L_.load()


def _im2col8(x):
    L_, lib = _lib()
    B, H, W, C = x.shape
    M = B * H * W
    cols = torch.empty((M, 9 * C), dtype=torch.uint8, device="cuda")
    sa = torch.empty(M, dtype=torch.float32, device="cuda")
    nb = lib.mac_im2col3x3_fp8_workspace_bytes(B, H, W, C)
    ws = torch.empty(nb, dtype=torch.uint8, device="cuda")
    L_.check(lib.mac_im2col3x3_fp8(L_.ptr(x), L_.ptr(cols), L_.ptr(sa), L_.ptr(ws), nb, B, H, W, C, L_.stream_ptr()),
             "mac_im2col3x3_fp8")
    return cols, sa


def _pack8(W):
    L_, lib = _lib()
    o = torch.empty((W.shape[1], W.shape[0]), dtype=torch.uint8, device="cuda")
    s = torch.empty(W.shape[1], dtype=torch.float32, device="cuda")
    L_.check(lib.mac_pack_weight_fp8(L_.ptr(W), L_.ptr(o), L_.ptr(s), W.shape[0], W.shape[1], L_.stream_ptr()), "pack8")
    return o, s


def _linear8(cols, sa, W8, sw, b, act):
    L_, lib = _lib()
    M, K = cols.shape
    y = torch.full((M, W8.shape[0]), float("nan"), device="cuda")
    L_.check(lib.mac_linear_fp8_fwd(L_.ptr(cols), L_.ptr(sa), L_.ptr(W8), L_.ptr(sw), L_.ptr(b), L_.ACT[act], L_.ptr(y), M,
                                    K, W8.shape[0], L_.stream_ptr()), "mac_linear_fp8_fwd")
    return y


def _e4m3(u8):
    return u8.view(torch.float8_e4m3fn).double()


def _mr(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


@pytest.mark.parametrize("B,H,W,C,zeros", [(1, 7, 7, 128, False), (3, 14, 14, 512, False), (64, 14, 14, 1024, False),
                                           (2, 14, 14, 256, True)])
def test_im2col3x3_fp8_equals_restatement_bit_for_bit(B, H, W, C, zeros):
    g = torch.Generator(device="cuda").manual_seed(B * 100 + C)
    x = torch.nn.functional.elu(torch.randn(B, H, W, C, device="cuda", generator=g))
    if zeros:
        x[0, :6, :6] = 0                        # windows inside this block have no nonzero pixel: sA = 0
        x[1] = 0
        x[1, 7, 7, :5] = 1.0                    # one pixel: only its 3x3 neighbourhood has nonzero windows
    cols, sa = _im2col8(x)
    torch.cuda.synchronize()
    ref8, sa_ref = F8S.quant_patches(x)
    assert torch.equal(sa, sa_ref), float((sa - sa_ref).abs().max())
    want = ref8.to(torch.float8_e4m3fn).view(torch.uint8)
    bad = int((cols != want).sum())
    assert bad == 0, (bad, int((_e4m3(cols) != ref8).sum()))
    if zeros:
        nz = sa > 0
        assert int((~nz).sum()) > 0 and int(cols[~nz].count_nonzero()) == 0
        assert int(nz[H * W:].sum()) == 9


# (M, K, n_out, act): M = 49 (one partial tile), 588 (partial last tile), 12544 (the stem's B=64, 14x14); K = 9C for
# C = 128, 512, 1024; n_out = 128 and 512
LINEAR_CASES = [(49, 1152, 128, "NON"), (49, 9216, 512, "ELU"), (588, 4608, 512, "NON"), (588, 1152, 128, "ELU"),
                (12544, 9216, 512, "ELU"), (12544, 4608, 128, "NON"), (12544, 1152, 512, "NON")]


@pytest.mark.parametrize("M,K,N,act", LINEAR_CASES)
def test_linear_fp8_fwd_against_fp64_of_its_operands(M, K, N, act):
    g = torch.Generator(device="cuda").manual_seed(M + K + N)
    X = torch.relu(torch.randn(M, K, device="cuda", generator=g))
    X[M // 3] = 0                                            # an all-zero row: sA = 0, y = act(b)
    am = X.abs().amax(1)
    sa = am / torch.tensor(448.0)
    inv = torch.where(am > 0, torch.tensor(448.0) / torch.where(am > 0, am, torch.ones_like(am)), torch.zeros_like(am))
    cols = (X * inv[:, None]).to(torch.float8_e4m3fn).view(torch.uint8).contiguous()
    Wf = torch.randn(K, N, device="cuda", generator=g) * K ** -0.5
    b = torch.randn(N, device="cuda", generator=g) * 0.1
    W8, sw = _pack8(Wf)
    y = _linear8(cols, sa, W8, sw, b, act)
    y2 = _linear8(cols, sa, W8, sw, b, act)
    torch.cuda.synchronize()
    ref = F8S.linear(_e4m3(cols), sa, _e4m3(W8).T, sw, b, relu=None)
    if act == "ELU":
        ref = torch.nn.functional.elu(ref)
    assert torch.equal(y, y2)                                # deterministic
    assert bool(torch.isfinite(y).all())
    row0 = y[M // 3]
    assert torch.allclose(row0, ref[M // 3].float(), rtol=0, atol=1e-6)
    e = _mr(y, ref)
    print("mac_linear_fp8_fwd M=%d K=%d N=%d %s: max-rel vs fp64 of its operands %.3e" % (M, K, N, act, e))
    assert e < TOL_LINEAR, e


def _stem_fp64(params, images):
    """oracle/stem_oracle.py's fp32 stem (SAME 3x3 convolution + bias, ELU after each layer) in fp64, on the GPU."""
    x = images.double()
    B, H, W, _ = x.shape
    i = 0
    while "stem/cnnLayercnn_%d/kernels/kernel" % i in params:
        K = params["stem/cnnLayercnn_%d/kernels/kernel" % i].double()
        b = params["stem/cnnLayercnn_%d/biases/bias" % i].double()
        y = F8S.im2col3x3(x) @ K.reshape(-1, K.shape[3]) + b
        x = torch.nn.functional.elu(y).reshape(B, H, W, -1)
        i += 1
    return x.reshape(B, H * W, -1)


def test_stem_fp8_headline_shape():
    """Stem(prec="fp8") at B=64, 14x14, 1024 -> 512 -> 512 against the fp64 fp32 stem, and against the e4m3 restatement."""
    from mac_network_b200.stem import Stem, init_stem_params, stem_specs
    p = {k: torch.from_numpy(v).cuda() for k, v in init_stem_params(stem_specs(1024, 512), seed=5).items()}
    g = torch.Generator(device="cuda").manual_seed(6)
    images = torch.relu(torch.randn(64, 14, 14, 1024, device="cuda", generator=g))
    kb = Stem(p, relu="ELU", prec="fp8").forward(images)
    kb16 = Stem(p, relu="ELU", prec="bf16").forward(images)
    torch.cuda.synchronize()
    ref = _stem_fp64(p, images)
    rest = F8S.stem_forward("ELU", p, images)
    e, e16, e_rest = _mr(kb, ref), _mr(kb16, ref), _mr(kb, rest)
    print("fp8 stem at the headline shape: vs fp64 %.3e (bf16 stem %.3e), vs the e4m3 restatement %.3e" % (e, e16, e_rest))
    assert bool(torch.isfinite(kb).all())
    assert e < TOL_STEM, e
    assert e_rest < TOL_STEM_REST, (e_rest, e)


def _eval_parts(net, data, images):
    """runBatch(train=False)'s evaluation chain, keeping the logits, the last memory and the knowledge-base attentions."""
    from mac_network_b200.mac_cell import MACCell, mac_network
    dev = net._to_device(net.trimData(dict(data)), images)
    words, cntx, vecq = net._enc.forward(dev["questions"], dev["questionLengths"])
    kb = net._stem.forward(dev["images"])
    B = dev["questions"].shape[0]
    cell = MACCell(vecq, words, cntx, dev["questionLengths"], kb, 1.0, 1.0, 1.0, B, False, config=net.cfg,
                   params=net.trainer.params, prec=net.prec)
    _, memory = mac_network(cell, net.L)
    logits, _, _ = net._out.forward(memory, vecq, dev["answers"])
    torch.cuda.synchronize()
    return {"logits": logits.double(), "memory": memory.double(),
            "att_kb": torch.stack([torch.as_tensor(a) for a in cell.attentions["kb"]]).double().cuda()}


def test_macnet_eval_with_fp8_stem_against_fp32_model():
    """MACnet(prec="fp8", eval_stem_prec="fp8") against MACnet(prec="fp32") with the same parameters, B=16 at the headline
    cell shape (14x14 grid, 1024 image channels, d=512, 12 steps): logits, memory and att_kb; runBatch runs end to end."""
    from mac_network_b200.config import MACConfig
    from mac_network_b200.model import MACnet
    B, S, V, E, C, A, L = 16, 12, 90, 300, 1024, 28, 12
    cfg = MACConfig.args("args", netLength=L)
    rng = np.random.RandomState(9)
    lengths = rng.randint(4, S + 1, size=(B,)).astype(np.int32)
    q = rng.randint(1, V + 1, size=(B, S)).astype(np.int32)
    q[np.arange(S)[None, :] >= lengths[:, None]] = 0
    data = {"questions": q, "questionLengths": lengths, "answers": rng.randint(0, A, size=(B,)).astype(np.int32)}
    images = {"images": np.maximum(rng.standard_normal((B, C, 14, 14)), 0).astype(np.float32)}
    kw = dict(wrd_emb_dim=E, image_in_dim=C, classifier_dims=(512,), seed=3)
    ref = _eval_parts(MACnet(cfg, L, V, A, prec="fp32", **kw), data, images)
    net8 = MACnet(cfg, L, V, A, prec="fp8", eval_stem_prec="fp8", **kw)
    got = _eval_parts(net8, data, images)
    net16 = MACnet(cfg, L, V, A, prec="fp8", **kw)
    got16 = _eval_parts(net16, data, images)
    errs = {k: _mr(got[k], ref[k]) for k in ref}
    errs16 = {k: _mr(got16[k], ref[k]) for k in ref}
    print("MACnet eval vs the fp32 model: fp8 stem %s; bf16 stem (prec='fp8' alone) %s" % (errs, errs16))
    for k in TOL_MODEL:
        assert errs[k] < TOL_MODEL[k], (k, errs)
    res = net8.runBatch(None, data, images, train=False)
    assert np.isfinite(res["loss"]) and len(res["preds"]) == B


def test_fp8_stem_rejections_launch_nothing():
    """Training, dropout and unsupported channel counts raise before any launch; the C entry points reject arguments
    before any launch."""
    from mac_network_b200.stem import Stem, init_stem_params, stem_specs
    L_, lib = _lib()
    p = {k: torch.from_numpy(v).cuda() for k, v in init_stem_params(stem_specs(128, 128), seed=1).items()}
    st = Stem(p, relu="ELU", prec="fp8")
    x = torch.zeros(1, 3, 3, 128, device="cuda")
    n0 = lib.mac_b200_launch_count()
    for kw in (dict(save_for_backward=True), dict(keep=0.82)):
        with pytest.raises(NotImplementedError):
            st.forward(x, **kw)
    with pytest.raises(NotImplementedError):
        Stem(p, relu="ELU", prec="fp8").forward(torch.zeros(1, 3, 3, 96, device="cuda"))
    cols = torch.zeros(9, 9 * 128, dtype=torch.uint8, device="cuda")
    sa = torch.zeros(9, device="cuda")
    ws = torch.zeros(64, dtype=torch.uint8, device="cuda")
    assert lib.mac_im2col3x3_fp8(L_.ptr(x), L_.ptr(cols), L_.ptr(sa), L_.ptr(ws), 16, 1, 3, 3, 128, None) == -4
    assert lib.mac_im2col3x3_fp8(L_.ptr(x), L_.ptr(cols), L_.ptr(sa), L_.ptr(ws), 64, 1, 3, 3, 96, None) == -3
    assert lib.mac_linear_fp8_fwd(L_.ptr(cols), L_.ptr(sa), L_.ptr(cols), L_.ptr(sa), None, 3, L_.ptr(x), 0, 1152, 128,
                                  None) == -1
    assert lib.mac_linear_fp8_fwd(L_.ptr(cols), L_.ptr(sa), L_.ptr(cols), L_.ptr(sa), None, 3, L_.ptr(x), 9, 1152, 96,
                                  None) == -3
    torch.cuda.synchronize()
    assert lib.mac_b200_launch_count() == n0
