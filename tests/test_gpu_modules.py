"""The `torch.nn` modules on the H100 (mac_network_b200/modules.py): a training step of `MACModel` bit for bit
`DPTrainer.full_forward_backward`; `MACNetwork`'s input and parameter gradients against fp64 autograd; the version refresh
after `torch.optim`; two forwards before their backwards; torch layers and extra loss terms around the modules."""
import numpy as np
import pytest
import torch

from mac_network_b200.config import MACConfig
from mac_network_b200.params import init_params, perturb_biases
from mac_network_b200.synthetic import make_inputs
from tests._util import load_golden, max_rel

pytestmark = pytest.mark.gpu

B, S, V, A, L, C, H, W = 4, 6, 20, 8, 2, 128, 4, 4          # B * H * W = 64 rows for the bf16 tensor-core backward
E = 300


def _cfg(variant, d):
    if variant.startswith("p2_"):
        meta, _ = load_golden(variant)
        return MACConfig(**dict(meta["cell_flags"], memDim=d, ctrlDim=d, attDim=d, netLength=L)).validate()
    return MACConfig.args(variant, netLength=L, memDim=d, ctrlDim=d, attDim=d)


def _data(seed, k=B, index=None, nchw=True):
    rng = np.random.RandomState(seed)
    lens = np.array([S, 2, 5, 3], dtype=np.int32)
    q = rng.randint(1, V + 1, size=(B, S)).astype(np.int32)
    q[np.arange(S)[None, :] >= lens[:, None]] = 0
    img = np.maximum(rng.standard_normal((k, C, H, W)), 0).astype(np.float32)
    d = {"questions": torch.from_numpy(q).cuda(), "questionLengths": torch.from_numpy(lens).cuda(),
         "answers": torch.from_numpy(rng.randint(0, A, size=B).astype(np.int32)).cuda()}
    if nchw:
        d["images_nchw"] = torch.from_numpy(img).cuda()
    else:
        d["images"] = torch.from_numpy(img).cuda().permute(0, 2, 3, 1).contiguous()
    if index is not None:
        d["imageIndex"] = torch.tensor(index, dtype=torch.int32, device="cuda")
    return d


def _images(d):
    return {k: d[k] for k in ("images", "images_nchw") if k in d}


def _trainer(variant, d, kw):
    from mac_network_b200.dp import DPTrainer
    return DPTrainer(_cfg(variant, d), L, seed=7, classifier=(A, [64]), encoder=(V, E), stem=(C, 2), **kw)


# ------------------------------------------------------------------------------------------------ against the trainer
CASES = [
    ("args", 128, dict(), None),
    ("args", 128, dict(), [1, 0, 1, 1]),
    ("args", 512, dict(prec="bf16", bwd_tc=True, stem_prec="bf16", enc_prec="bf16"), None),
    ("args", 512, dict(prec="bf16", bwd_tc=True, stem_prec="bf16", enc_prec="bf16"), [2, 0, 2, 1]),
    ("args", 128, dict(prec="tc32", bwd_tc=True, stem_prec="bf16x3"), None),
    ("args", 128, dict(prec="tc32", bwd_tc=True, stem_prec="bf16x3"), [0, 1, 2, 0]),
    ("args1", 128, dict(), None),
    ("args3", 128, dict(), [0, 0, 1, 0]),
    ("args4", 128, dict(prec="tc32", bwd_tc=True), None),
    ("p2_read_add", 128, dict(), None),
]


@pytest.mark.parametrize("variant,d,kw,index", CASES)
def test_model_step_equals_the_trainer_bit_for_bit(variant, d, kw, index):
    """After one trainer step (so the model starts from trained values, step 1): the model's logits, and every parameter's
    .grad after answer_loss(...).backward(), equal the trainer's logits and gradient bucket; the loss is the mean of the
    trainer's per-sample losses."""
    from mac_network_b200.modules import MACModel, answer_loss
    t = _trainer(variant, d, kw)
    k = B if index is None else max(index) + 1
    t.train_step_full((B, S), _data(1, k, index), global_batch=B)
    m = MACModel.from_trainer(t)
    data = _data(2, k, index, nchw=variant != "args3")           # args3: the NHWC images
    logits, _ = m(data["questions"], data["questionLengths"], imageIndex=data.get("imageIndex"), **_images(data))
    loss = answer_loss(logits, data["answers"])
    loss.backward()
    t_logits, t_losses = t.full_forward_backward((B, S), data, global_batch=B)
    torch.cuda.synchronize()
    assert torch.equal(logits.detach(), t_logits)
    want = float(t_losses.double().sum()) / B
    assert abs(float(loss.detach()) - want) <= 1e-6 * abs(want), (float(loss.detach()), want)
    bad = []
    for name, p in m.named_parameters():
        o = t.params.offsets[name]
        if not torch.equal(p.grad.reshape(-1), t.bucket[o:o + p.numel()]):
            bad.append(name)
    assert not bad, bad


# ------------------------------------------------------------------------------------------------ against fp64
@pytest.mark.parametrize("prec,bwd_tc,tol", [("fp32", False, 2e-4), ("tc32", True, 2e-4), ("bf16", True, 5e-2)])
def test_network_gradients_match_fp64_autograd(prec, bwd_tc, tol):
    """MACNetwork in training (the cell's dropouts from cfg): control / memory and the gradients of
    sum(control * gc) + sum(memory * gm) w.r.t. every parameter and input, against oracle/mac_torch_autograd.py at the
    bars of the cell's own tests (2e-4 of each tensor's max for fp32 and tc32, 5e-2 for the bf16 tensor-core backward)."""
    from mac_network_b200.modules import MACNetwork
    from oracle import mac_torch_autograd as TA
    Bn, Sn, N, d, Ln = 4, 6, 16, 128, 3
    cfg = MACConfig.args("args", netLength=Ln, memDim=d, ctrlDim=d, attDim=d)
    inputs = make_inputs(Bn, Sn, N, d, seed=51, dtype=np.float64)
    pv = perturb_biases(init_params(cfg, Ln, seed=52, dtype=np.float64), seed=53)
    rng = np.random.RandomState(54)
    gc, gm = rng.standard_normal((Bn, d)), rng.standard_normal((Bn, d))
    net = MACNetwork(cfg, Ln, prec=prec, bwd_tc=bwd_tc, values={k: v.astype(np.float32) for k, v in pv.items()}, seed=9)
    x = {k: torch.from_numpy(np.ascontiguousarray(v if v.dtype == np.int32 else v.astype(np.float32))).cuda()
         for k, v in inputs.items()}
    for k in ("vecQuestions", "questionCntxWords", "knowledgeBase"):
        x[k].requires_grad_(True)
    control, memory = net(x["vecQuestions"], x["questionWords"], x["questionCntxWords"], x["questionLengths"],
                          x["knowledgeBase"])
    tc_, tm_ = (torch.from_numpy(a.astype(np.float32)).cuda() for a in (gc, gm))
    ((control * tc_).sum() + (memory * tm_).sum()).backward()
    torch.cuda.synchronize()
    cell = next(reversed(net.cells._idle.values()))          # the forward's cell, back in the pool after its backward
    rc, rm, rg = TA.run(cfg, pv, inputs, Ln, (cfg.memoryDropout, cfg.readDropout, cfg.writeDropout),
                        cell.dropout_uniforms(), gc, gm)
    fwd = max(max_rel(memory.detach().cpu().numpy(), rm), max_rel(control.detach().cpu().numpy(), rc))
    got = {n: p.grad for n, p in net.named_parameters()}
    got.update({k: x[k].grad for k in ("vecQuestions", "questionCntxWords", "knowledgeBase")})
    worst = {}
    for k, ref in rg.items():
        g = got[k].cpu().numpy().reshape(ref.shape)
        scale = np.max(np.abs(ref))
        if scale < 1e-12:
            assert np.max(np.abs(g)) < 1e-4, k
            continue
        worst[k] = float(np.max(np.abs(g - ref)) / scale)
    print("MACNetwork %s: forward %.2e, worst gradients %s" % (prec, fwd, sorted(worst.items(), key=lambda kv: -kv[1])[:3]))
    assert fwd < (1e-4 if prec != "bf16" else 2.5e-2), fwd
    assert not {k: v for k, v in worst.items() if v > tol}


def test_an_extra_loss_on_memory_is_mac_backwards_d_memory():
    """Gradients of sum(control * gc) + sum(memory * gm) through MACNetwork equal mac_backward(cell, gc, gm) on a cell fed
    the same seed, bit for bit."""
    from mac_network_b200.autograd import mac_backward
    from mac_network_b200.mac_cell import MACCell, mac_network
    from mac_network_b200.modules import MACNetwork, _seed
    Bn, Sn, N, d = 4, 6, 16, 128
    cfg = MACConfig.args("args", netLength=L, memDim=d, ctrlDim=d, attDim=d)
    x = {k: torch.from_numpy(v).cuda() for k, v in make_inputs(Bn, Sn, N, d, seed=3).items()}
    rng = np.random.RandomState(4)
    gc, gm = (torch.from_numpy(rng.standard_normal((Bn, d)).astype(np.float32)).cuda() for _ in range(2))
    net = MACNetwork(cfg, L, prec="tc32", bwd_tc=True, seed=11)
    kb = x["knowledgeBase"].clone().requires_grad_(True)
    control, memory = net(x["vecQuestions"], x["questionWords"], x["questionCntxWords"], x["questionLengths"], kb)
    ((control * gc).sum() + (memory * gm).sum()).backward()
    cell = MACCell(x["vecQuestions"], x["questionWords"], x["questionCntxWords"], x["questionLengths"], x["knowledgeBase"],
                   cfg.memoryDropout, cfg.readDropout, cfg.writeDropout, Bn, True, config=cfg, params=net.params,
                   prec="tc32", seed=_seed(11, 0), save_for_backward=True)
    c2, m2 = mac_network(cell, L)
    g = mac_backward(cell, gc, gm, tc=True)
    torch.cuda.synchronize()
    assert torch.equal(memory.detach(), m2) and torch.equal(control.detach(), c2)
    assert torch.equal(kb.grad, g["knowledgeBase"])
    assert all(torch.equal(p.grad.reshape(-1), g[n].reshape(-1)) for n, p in net.named_parameters())


# ------------------------------------------------------------------------------------------------ versions
@pytest.mark.parametrize("kw", [dict(prec="bf16", bwd_tc=True, stem_prec="bf16", enc_prec="bf16"),
                                dict(prec="tc32", bwd_tc=True, stem_prec="bf16x3")])
def test_forward_after_an_optimizer_step_is_a_fresh_models(kw):
    """torch.optim.Adam updates the parameters in place; the next forward (training and eval) is bit for bit a model built
    from the updated values, and differs from the pre-step output (the packs were rebuilt)."""
    from mac_network_b200.modules import MACModel, answer_loss
    d = 512 if kw["prec"] == "bf16" else 128
    args = (_cfg("args", d), L, V, A)
    opts = dict(wrd_emb_dim=E, image_in_dim=C, classifier_dims=(64,), seed=3, **kw)
    m = MACModel(*args, **opts)
    opt = torch.optim.Adam(m.parameters(), lr=1e-2)
    data = _data(5)
    q, ql, img = data["questions"], data["questionLengths"], _images(data)
    m.eval()
    before = m(q, ql, **img)[0].clone()
    m.train()
    answer_loss(m(q, ql, **img)[0], data["answers"]).backward()
    opt.step()
    step = m.step
    train_after = m(q, ql, **img)[0].detach()
    m.eval()
    eval_after = m(q, ql, **img)[0]
    fresh = MACModel(*args, values={k: v.detach().cpu().numpy() for k, v in m.state_dict().items()}, **opts)
    fresh.step = step
    train_fresh = fresh(q, ql, **img)[0].detach()
    fresh.eval()
    eval_fresh = fresh(q, ql, **img)[0]
    torch.cuda.synchronize()
    assert torch.equal(train_after, train_fresh) and torch.equal(eval_after, eval_fresh)
    assert not torch.equal(eval_after, before)


# ------------------------------------------------------------------------------------------------ ownership of saved state
def test_two_forwards_then_one_backward():
    """f(a); f(b); (la + lb).backward() equals the sum of the separate backwards of a twin at the same seed and step; a
    second backward through the freed graph raises."""
    from mac_network_b200.modules import MACModel, answer_loss
    kw = dict(prec="bf16", bwd_tc=True, stem_prec="bf16", enc_prec="bf16")
    t = _trainer("args", 512, kw)
    m, twin = MACModel.from_trainer(t), MACModel.from_trainer(t)
    a, b = _data(6), _data(7)
    run = lambda mod, x: answer_loss(mod(x["questions"], x["questionLengths"], **_images(x))[0], x["answers"])
    la, lb = run(m, a), run(m, b)
    (la + lb).backward()
    run(twin, a).backward()
    ga = {n: p.grad.clone() for n, p in twin.named_parameters()}
    twin.zero_grad()
    run(twin, b).backward()
    torch.cuda.synchronize()
    bad = [n for n, p in m.named_parameters() if not torch.equal(p.grad, ga[n] + dict(twin.named_parameters())[n].grad)]
    assert not bad, bad
    with pytest.raises(RuntimeError, match="already run"):
        la.backward()


# ------------------------------------------------------------------------------------------------ composition
def test_a_torch_layer_in_front_of_the_stem_gets_the_finite_difference_gradient():
    """nn.Linear (fp32) -> ImageStem(NHWC, fp32, no dropout) -> sum(kb * r): the Linear's weight and bias gradients against
    central differences of the fp64 stem (oracle/stem_oracle.py)."""
    from mac_network_b200.modules import ImageStem
    from oracle.stem_oracle import stem_forward
    rng = np.random.RandomState(8)
    cin, cmid, cout = 8, 16, 32
    lin = torch.nn.Linear(cin, cmid).cuda()
    stem = ImageStem(cmid, cout, num_layers=2, seed=2)
    stem.stem_keep = 1.0
    x = torch.from_numpy(rng.standard_normal((2, 3, 5, cin)).astype(np.float32)).cuda()
    r = torch.from_numpy(rng.standard_normal((2, 15, cout)).astype(np.float32)).cuda()
    (stem(images=lin(x)) * r).sum().backward()
    torch.cuda.synchronize()
    sp = {k: v.detach().cpu().numpy().astype(np.float64) for k, v in stem.named_parameters()}
    x64, r64 = x.cpu().numpy().astype(np.float64), r.cpu().numpy().astype(np.float64)
    W0, b0 = lin.weight.detach().cpu().numpy().astype(np.float64), lin.bias.detach().cpu().numpy().astype(np.float64)

    def f(Wl, bl):
        return float(np.sum(stem_forward("ELU", sp, x64 @ Wl.T + bl).reshape(2, 15, cout) * r64))
    eps = 1e-5
    got_w, got_b = lin.weight.grad.cpu().numpy(), lin.bias.grad.cpu().numpy()
    worst = 0.0
    scale = max(np.abs(got_w).max(), np.abs(got_b).max())
    for i, j in [(i, j) for i in range(cmid) for j in range(cin)][::5]:
        dW = np.zeros_like(W0)
        dW[i, j] = eps
        fd = (f(W0 + dW, b0) - f(W0 - dW, b0)) / (2 * eps)
        worst = max(worst, abs(fd - got_w[i, j]) / scale)
    for i in range(cmid):
        db = np.zeros_like(b0)
        db[i] = eps
        fd = (f(W0, b0 + db) - f(W0, b0 - db)) / (2 * eps)
        worst = max(worst, abs(fd - got_b[i]) / scale)
    assert worst < 1e-4, worst
