"""The split-bf16 image stem (`Stem(prec="bf16x3")`, DESIGN.md section 9 item 6) on the GPU.

- mac_im2col3x3_split bit for bit against the host split of mac_im2col3x3's fp32 patch matrix.
- mac_linear_tc32_fwd and mac_conv3x3_bwd_tc32 against fp64 references on their fp32 operands, error as a fraction of the
  same reference on absolute values (`excess` of tests/test_gpu_wgmma.py), up to the stem's K = 9216 and Mp = 12 544.
- The stem against torch.autograd on the fp64 restatement, the whole-model trainer against its fp32-stem twin, and the MACnet
  evaluation against the fp32 stem: the fp32 path's bars (1e-4 forward, 2e-4 of each gradient tensor's maximum).
tests/test_stem_bf16x3_bounds.py shows on the CPU that these bounds reject plain bf16 products, a dropped term, unwritten
padding columns and a shifted Philox index.  Each bound is about three times the value measured on an H100 80GB HBM3
(700 W power limit, 1980 MHz max SM clock), written beside it."""
import numpy as np
import pytest
import torch

from mac_network_b200 import _lib as L_
from oracle.model_torch_autograd import mask_uniforms, stem_grads
from tests.test_gpu_wgmma import excess, pack3, split_hi_lo
from tests.test_stem_tc_training import _col2im, _patches, _uniform_mask

pytestmark = pytest.mark.gpu

ACT_ELU = L_.ACT["ELU"]
# fraction of the absolute-value reference                                                        measured
# mac_linear_tc32_fwd, worst over M = 49, 245, 12 544.  One fp32 wgmma accumulator over the whole K measured 2.6e-6, 3.9e-6
# and 4.9e-6 at K = 1152, 4608 and 9216: from K = 4608 on these bars reject it.                     measured
TOL_LINEAR = {1152: 4.5e-6,                                                                  # 1.5e-6
              4608: 2.1e-6,                                                                  # 7.0e-7
              9216: 1.6e-6,                                                                  # 5.3e-7
              18432: 1.1e-6}                                                                 # 3.6e-7
TOL_CONV = {"dkernel": 3.6e-5,      # 8.8e-6 over Mp = 12 544; over M = 49 single terms show: the dropped lo*lo product is
                                    # up to 2^-16 of a term and does not average out                1.2e-5
            "dbias": 2.5e-7,                                                                 # 8.1e-8
            "dx": 3.5e-6}           # contraction over Cout, then nine fp32 adds                    1.2e-6
# Stem(prec="bf16x3") against the fp64 restatement: the fp32 stem's own bars (tests/test_stem.py), not looser.  Measured at
# B=64, 14x14, 1024 -> 512 -> 512, keep 0.82: kb 7.1e-6, layer 0's kernel gradient 7.6e-5, layer 1's 7.4e-5, d_images 6.8e-6
BAR_FWD, BAR_GRAD = 1e-4, 2e-4
# whole-model trainer, stem_prec="bf16x3" against "fp32" under the tc32 cell, two steps (the tc32 cell against the fp32
# cell: 1.8e-5, DESIGN.md section 9 item 5)
TOL_TRAINER_LOSS = 1e-5             # relative                                                      3.9e-7
TOL_TRAINER = 1e-4                  # every gradient tensor, of its max: 3.2e-5 (a cell tensor); stem tensors 6.4e-6
# MACnet(prec="bf16") evaluation, the bf16x3 stem against the fp32 stem (max-norm relative)
TOL_EVAL = {"kb": 1e-4,             # the forward bar                                               6.2e-6
            "logits": 2e-4}                                                                  # 1.3e-5


def _mr(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


# ------------------------------------------------------------------------------------------------ mac_im2col3x3_split
@pytest.mark.parametrize("keep", [1.0, 0.82])
@pytest.mark.parametrize("shape", [(1, 7, 7, 128), (3, 14, 14, 320)])
def test_im2col3x3_split_equals_the_host_split_bit_for_bit(shape, keep):
    lib = L_.load()
    B, H, W, C = shape
    M, K = B * H * W, 9 * C
    x = torch.randn(B, H, W, C, device="cuda", generator=torch.Generator(device="cuda").manual_seed(C + B))
    cols = torch.empty(M, K, device="cuda")
    L_.check(lib.mac_im2col3x3(L_.ptr(x), L_.ptr(cols), 0, keep, 77, 33, 6, B, H, W, C, L_.stream_ptr()), "mac_im2col3x3")
    cols2 = torch.full((M, 2 * K), float("nan"), dtype=torch.bfloat16, device="cuda")
    L_.check(lib.mac_im2col3x3_split(L_.ptr(x), L_.ptr(cols2), keep, 77, 33, 6, B, H, W, C, L_.stream_ptr()),
             "mac_im2col3x3_split")
    torch.cuda.synchronize()
    hi = cols.to(torch.bfloat16)
    lo = (cols - hi.float()).to(torch.bfloat16)
    assert keep == 1.0 or 0.1 < float((cols == 0).float().mean()) < 0.5          # the mask is in the fp32 patches
    assert torch.equal(cols2.view(torch.int16), torch.cat([hi, lo], 1).view(torch.int16))


# ------------------------------------------------------------------------------------------------ mac_linear_tc32_fwd
@pytest.mark.parametrize("K", [1152, 4608, 9216, 18432])
@pytest.mark.parametrize("M", [49, 245, 12544])
def test_linear_tc32_fwd_against_fp64(M, K):
    """y = ELU(A W + b) from [A_hi | A_lo] and [W_hi | W_hi | W_lo], two-level accumulation (tc_gemm_kernel's PROMOTE
    form), up to the stem's K = 9 C at C = 1024 and 2048."""
    lib = L_.load()
    N = 256
    g = torch.Generator(device="cuda").manual_seed(M + K)
    A = torch.relu(torch.randn(M, K, device="cuda", generator=g))
    Wt = torch.randn(K, N, device="cuda", generator=g) * K ** -0.5
    b = torch.randn(N, device="cuda", generator=g) * 0.1
    hi, lo = split_hi_lo(A)
    a2 = torch.cat([hi, lo], 1).to(torch.bfloat16).contiguous()
    w3 = pack3(Wt)
    ys = []
    for _ in range(2):
        y = torch.full((M, N), float("nan"), device="cuda")
        L_.check(lib.mac_linear_tc32_fwd(L_.ptr(a2), L_.ptr(w3), L_.ptr(b), ACT_ELU, L_.ptr(y), M, K, N, L_.stream_ptr()),
                 "mac_linear_tc32_fwd")
        ys.append(y)
    torch.cuda.synchronize()
    assert torch.equal(ys[0].view(torch.int32), ys[1].view(torch.int32))
    pre = A.double() @ Wt.double() + b.double()
    absref = A.double().abs() @ Wt.double().abs() + b.double().abs()
    # ELU is 1-Lipschitz: the pre-activation's bound carries over; 2e-7 for the epilogue's fp32 exponential
    e = excess(ys[0], torch.where(pre > 0, pre, torch.expm1(pre)), absref, tiny=2e-7)
    print("mac_linear_tc32_fwd M=%d K=%d: %.2e of the absolute-value product" % (M, K, e))
    assert e <= TOL_LINEAR[K], e


# ------------------------------------------------------------------------------------------------ mac_conv3x3_bwd_tc32
def _run_conv(lib, x, y, dy, kernel, keep, seed, site, step, dkernel, dbias, dx, shape):
    B, H, W, C, Cout = shape
    nbytes = int(lib.mac_conv3x3_bwd_tc32_workspace_bytes(B, H, W, C, Cout, int(dx is not None)))
    ws = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device="cuda")    # NaN everywhere: the workspace is not assumed zero
    L_.check(lib.mac_conv3x3_bwd_tc32(L_.ptr(x), L_.ptr(y), L_.ptr(dy), L_.ptr(kernel), ACT_ELU, keep, seed, site, step,
                                      L_.ptr(dkernel), L_.ptr(dbias), L_.ptr(dx), L_.ptr(ws), nbytes, B, H, W, C, Cout,
                                      L_.stream_ptr()), "mac_conv3x3_bwd_tc32")


@pytest.mark.parametrize("shape,keep,with_dx", [((1, 7, 7, 128, 128), 0.82, True),      # M = 49: one partly filled k-block
                                                ((5, 7, 7, 128, 256), 0.82, True),      # M = 245, Mp = 256
                                                ((5, 7, 7, 256, 128), 0.82, False),
                                                ((3, 14, 14, 256, 128), 1.0, True),
                                                ((64, 14, 14, 1024, 512), 0.82, False),  # headline layer 0
                                                ((64, 14, 14, 512, 512), 0.82, True)])   # headline layer 1
def test_conv3x3_bwd_tc32_against_fp64(shape, keep, with_dx):
    """against the fp64 backward of the layer on its fp32 operands; `+=` onto non-zero gradients; two runs bit-identical"""
    lib = L_.load()
    B, H, W, C, Cout = shape
    M = B * H * W
    g = torch.Generator(device="cuda").manual_seed(sum(shape))
    x = torch.relu(torch.randn(B, H, W, C, device="cuda", generator=g))
    kernel = torch.randn(3, 3, C, Cout, device="cuda", generator=g) * (2.0 / (9 * (C + Cout))) ** 0.5
    y = torch.nn.functional.elu(torch.randn(M, Cout, device="cuda", generator=g))
    dy = torch.randn(M, Cout, device="cuda", generator=g)
    seed, site, step = 4321, 33, 5
    pre_k = torch.randn(3, 3, C, Cout, device="cuda", generator=g) * 0.1
    pre_b = torch.randn(Cout, device="cuda", generator=g)
    runs = []
    for _ in range(2):
        dkernel, dbias = pre_k.clone(), pre_b.clone()
        dx = torch.full((B, H, W, C), float("nan"), device="cuda") if with_dx else None
        _run_conv(lib, x, y, dy, kernel, keep, seed, site, step, dkernel, dbias, dx, shape)
        runs.append((dkernel, dbias, dx))
    torch.cuda.synchronize()
    same = lambda a, b: torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert same(runs[0][0], runs[1][0]) and same(runs[0][1], runs[1][1])
    if with_dx:
        assert same(runs[0][2], runs[1][2])
    dkernel, dbias, dx = runs[0]
    dz = (dy * torch.where(y > 0, torch.ones_like(y), y + 1)).double()           # fp32, as the kernel forms it
    scale = float(np.float32(1.0) / np.float32(keep))
    mask = _uniform_mask(lib, seed, site, step, (B, H, W, C), keep) if keep < 1.0 else torch.ones(B, H, W, C, device="cuda",
                                                                                                     dtype=torch.bool)
    cols = _patches((x * np.float32(scale)).double() * mask)                     # fp32 dropout(x)
    ref_k, abs_k = cols.t() @ dz, cols.abs().t() @ dz.abs()
    del cols
    rows = {"dkernel": excess(dkernel.view(-1, Cout), pre_k.double().view(-1, Cout) + ref_k,
                              abs_k + pre_k.double().view(-1, Cout).abs()),
            "dbias": excess(dbias, pre_b.double() + dz.sum(0), dz.abs().sum(0) + pre_b.double().abs())}
    if with_dx:
        k64 = kernel.double().view(-1, Cout)
        f = mask.double() * scale
        assert bool(torch.isfinite(dx).all())                                     # every element written
        rows["dx"] = excess(dx, _col2im(dz @ k64.t(), B, H, W, C) * f, _col2im(dz.abs() @ k64.abs().t(), B, H, W, C) * f)
    print("conv3x3_bwd_tc32 %s keep=%s: %s" % (shape, keep, ", ".join("%s %.2e" % kv for kv in rows.items())))
    bad = {k: v for k, v in rows.items() if not v <= TOL_CONV[k]}
    assert not bad, bad


# ------------------------------------------------------------------------------------------------ the stem
@pytest.mark.parametrize("keep,shape", [(0.82, (2, 5, 7, 128, 128)), (1.0, (4, 14, 14, 256, 256)),
                                        (0.82, (64, 14, 14, 1024, 512))])
def test_stem_bf16x3_training_against_fp64_autograd(keep, shape):
    from mac_network_b200.stem import Stem, SITE_STEM, stem_specs, init_stem_params
    lib = L_.load()
    B, H, W, cin, cout = shape
    params = {k: torch.from_numpy(v).cuda() for k, v in init_stem_params(stem_specs(cin, cout), seed=8).items()}
    g = torch.Generator(device="cuda").manual_seed(9)
    images = torch.relu(torch.randn(B, H, W, cin, device="cuda", generator=g))
    st = Stem(params, relu="ELU", prec="bf16x3", seed=13)
    kb = st.forward(images, keep=keep, step=4, save_for_backward=True)
    d_kb = torch.randn(kb.shape, device="cuda", generator=g)
    grads = {k: torch.zeros_like(v) for k, v in params.items()}
    d_img = st.backward(d_kb, grads, need_d_images=True)
    kb_inf = st.forward(images, keep=keep, step=4)                               # the inference form: the same products
    torch.cuda.synchronize()
    assert torch.equal(kb_inf, kb)
    us = [mask_uniforms(_uniform_mask(lib, 13, SITE_STEM + i, 4, (B, H, W, c), keep)) for i, c in ((0, cin), (1, cout))] \
        if keep < 1.0 else None
    kb_ref, gref, dimg_ref = stem_grads("ELU", params, images, keep, us, d_kb)
    errs = {"kb": _mr(kb, kb_ref), "d_images": _mr(d_img, dimg_ref)}
    errs.update({k: _mr(grads[k], gref[k]) for k in gref})
    print("bf16x3 stem keep=%s %s: %s" % (keep, shape, ", ".join("%s %.2e" % (k.split("/")[1] + "/" + k.split("/")[-1]
                                                                            if "/" in k else k, v) for k, v in errs.items())))
    assert errs.pop("kb") < BAR_FWD
    bad = {k: v for k, v in errs.items() if not v < BAR_GRAD}
    assert not bad, bad


def test_full_model_bf16x3_stem_matches_its_fp32_stem_twin_over_two_steps():
    """DPTrainer(prec="tc32", bwd_tc=True).train_step_full with the training dropouts (the same masks in both arms), two
    steps: the loss and every tensor of the gradient bucket, stem_prec="bf16x3" against "fp32"."""
    from mac_network_b200.dp import DPTrainer
    from tests.test_gpu_tc32_training import NULL_GRADIENTS
    from tests.test_stem_tc_training import _full_setup
    cfg, data, kw, B, L = _full_setup(31)
    dev = {k: torch.from_numpy(v).cuda() for k, v in data.items()}
    out = {}
    for sp in ("fp32", "bf16x3"):
        tr = DPTrainer(cfg, L, seed=7, prec="tc32", bwd_tc=True, stem_prec=sp, **kw)
        out[sp] = []
        for _ in range(2):
            _, losses = tr.train_step_full("t", dev, global_batch=B)
            torch.cuda.synchronize()
            out[sp].append((float(losses.mean()), tr.bucket.double().clone()))
    worst = {}
    for s in range(2):
        (l32, g32), (l3, g3) = out["fp32"][s], out["bf16x3"][s]
        assert abs(l3 - l32) <= TOL_TRAINER_LOSS * abs(l32), (s, l3, l32)
        for name in tr.params.specs:
            o, n = tr.params.offsets[name], int(np.prod(tr.params.specs[name][0]) or 1)
            scale = float(g32[o:o + n].abs().max())
            if scale > 1e-12 and not name.endswith(NULL_GRADIENTS):      # a softmax logit bias: true gradient exactly 0
                worst[(s, name)] = float((g3[o:o + n] - g32[o:o + n]).abs().max()) / scale
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:4]
    print("bf16x3 vs fp32 stem under the tc32 cell: losses %s vs %s; worst gradient tensors %s" % (
        [l for l, _ in out["bf16x3"]], [l for l, _ in out["fp32"]], [(s, n.split("/", 1)[0], "%.2e" % v) for (s, n), v in top]))
    stem = max(v for (s, n), v in worst.items() if n.startswith("stem/"))
    print("stem tensors: %.2e" % stem)
    bad = {k: v for k, v in worst.items() if v > TOL_TRAINER}
    assert not bad, bad


def test_macnet_eval_with_bf16x3_stem_against_the_fp32_stem():
    """MACnet(prec="bf16", eval_stem_prec="bf16x3") against the same net with an fp32 evaluation stem: the knowledge base
    and the logits; runBatch(train=False) runs end to end."""
    from mac_network_b200.config import MACConfig
    from mac_network_b200.model import MACnet
    from mac_network_b200.stem import Stem
    from tests.test_gpu_stem_fp8 import _eval_parts
    B, S, V, E, C, A, L = 8, 12, 90, 300, 1024, 28, 4
    cfg = MACConfig.args("args", netLength=L)
    rng = np.random.RandomState(9)
    lengths = rng.randint(4, S + 1, size=(B,)).astype(np.int32)
    q = rng.randint(1, V + 1, size=(B, S)).astype(np.int32)
    q[np.arange(S)[None, :] >= lengths[:, None]] = 0
    data = {"questions": q, "questionLengths": lengths, "answers": rng.randint(0, A, size=(B,)).astype(np.int32)}
    images = {"images": np.maximum(rng.standard_normal((B, C, 14, 14)), 0).astype(np.float32)}
    net = MACnet(cfg, L, V, A, prec="bf16", eval_stem_prec="bf16x3", wrd_emb_dim=E, image_in_dim=C, classifier_dims=(512,),
                 seed=3)
    assert net._stem.prec == "bf16x3" and net.trainer.stem.prec == "fp32"
    res = net.runBatch(None, data, images, train=False)
    assert np.isfinite(res["loss"]) and len(res["preds"]) == B
    got = _eval_parts(net, data, images)
    x = net._to_device(net.trimData(dict(data)), images)["images"]
    kb3 = net._stem.forward(x)
    net._stem = Stem(net._stem.p, relu=cfg.relu, prec="fp32")
    ref = _eval_parts(net, data, images)
    errs = {"kb": _mr(kb3, net._stem.forward(x)), "logits": _mr(got["logits"], ref["logits"])}
    print("MACnet eval, bf16x3 stem vs fp32 stem: %s" % errs)
    bad = {k: v for k, v in errs.items() if not v < TOL_EVAL[k]}
    assert not bad, bad
