"""Whole-model serving from host buffers (serving.ModelPipeline) and the pieces it adds, on the GPU.

- mac_ingest_nchw, both modes, fp32 and bf16 input: bit for bit the permuted tensor / the bf16 patch matrix mac_im2col3x3
  makes of it; refusals return their status and leave the output untouched.
- mac_answer_topk against numpy (ties to the lower id, A not a multiple of 32, one very large logit).
- OutputUnit.logits and Stem.forward_nchw bit for bit their labelled / NHWC forms.
- The pipeline against MACnet.runBatch(train=False, getAtt=True) on the same weights and batches: bit for bit when the longest
  question fills S, exactly zero attention beyond each length and 1e-6 agreement when every question is shorter; re-capture
  after the weights move, also when they were moved on the caller's stream with no device synchronise before the submit;
  old tickets stay readable until their slot is reused."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

INVALID, ALIGN, UNSUPPORTED = -1, -2, -3


def _lib():
    from mac_network_b200 import _lib as L_
    return L_, L_.load()


def _features(B, C, H, W, seed):
    """Post-ReLU-like features whose fp32 values include exact bf16 ties (round-to-nearest-even both ways) and values one
    ulp either side of a tie."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, C, H, W, device="cuda", generator=g).clamp_(min=0)
    bits = x.view(torch.int32)
    flat = bits.view(-1)
    n = flat.numel()
    for k, low in enumerate((0x8000, 0x18000, 0x7fff, 0x8001)):            # tie to even down / up, just below, just above
        idx = torch.arange(k, n, 7, device="cuda")
        flat[idx] = (flat[idx] & ~0x1ffff) | low
    return bits.view(torch.float32)


def _ingest(x, mode, out=None):
    L_, lib = _lib()
    B, C, H, W = x.shape
    if out is None:
        out = (torch.empty((B * H * W, 9 * C), dtype=torch.bfloat16, device="cuda") if mode == 1 else
               torch.empty((B, H, W, C), dtype=torch.float32, device="cuda"))
    st = lib.mac_ingest_nchw(L_.ptr(x), int(x.dtype == torch.bfloat16), L_.ptr(out), mode, B, C, H, W, L_.stream_ptr())
    return st, out


def _im2col_bf16(x_nhwc):
    L_, lib = _lib()
    B, H, W, C = x_nhwc.shape
    cols = torch.empty((B * H * W, 9 * C), dtype=torch.bfloat16, device="cuda")
    L_.check(lib.mac_im2col3x3(L_.ptr(x_nhwc), L_.ptr(cols), 1, 1.0, 0, 32, 0, B, H, W, C, L_.stream_ptr()), "mac_im2col3x3")
    return cols


@pytest.mark.parametrize("C", [64, 128, 1024, 2048])
@pytest.mark.parametrize("B,H,W", [(1, 14, 14), (64, 7, 7), (3, 14, 14), (2, 5, 9)])
def test_ingest_nchw_equals_permute_and_im2col_bit_for_bit(B, H, W, C):
    if B == 64 and C == 2048:
        B = 16
    x = _features(B, C, H, W, seed=C + B)
    nhwc = x.permute(0, 2, 3, 1).contiguous()
    want_cols = _im2col_bf16(nhwc)
    st, y = _ingest(x, 0)
    assert st == 0 and torch.equal(y, nhwc)
    st, cols = _ingest(x, 1)
    assert st == 0 and torch.equal(cols.view(torch.int16), want_cols.view(torch.int16))
    # bf16 input (the host cast's output): a move into the patch matrix, a widening into NHWC
    x16 = x.to(torch.bfloat16)
    st, cols16 = _ingest(x16, 1)
    assert st == 0 and torch.equal(cols16.view(torch.int16), want_cols.view(torch.int16))
    st, y16 = _ingest(x16, 0)
    assert st == 0 and torch.equal(y16, x16.float().permute(0, 2, 3, 1).contiguous())


def test_ingest_nchw_refusals_leave_the_output_untouched():
    L_, lib = _lib()
    x = torch.ones(2, 64, 3, 3, device="cuda")
    out = torch.full((2 * 9, 9 * 64), 7.0, dtype=torch.bfloat16, device="cuda")
    p, o = x.data_ptr(), out.data_ptr()
    call = lambda xp, op, mode, B, C, H, W: lib.mac_ingest_nchw(xp, 0, op, mode, B, C, H, W, None)
    assert call(None, o, 1, 2, 64, 3, 3) == INVALID and call(p, None, 1, 2, 64, 3, 3) == INVALID
    assert call(p, o, 1, 0, 64, 3, 3) == INVALID and call(p, o, 1, 2, 64, 3, -1) == INVALID
    assert call(p + 4, o, 1, 2, 64, 3, 3) == ALIGN and call(p, o + 2, 1, 2, 64, 3, 3) == ALIGN
    assert call(p, o, 1, 2, 96, 3, 3) == UNSUPPORTED and call(p, o, 2, 2, 64, 3, 3) == UNSUPPORTED
    assert call(p, o, 0, 2, 64, 40, 40) == UNSUPPORTED                    # a slab beyond one SM's shared memory
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())


def _topk_numpy(logits, k):
    z = logits.astype(np.float32)
    order = np.lexsort((np.arange(z.shape[1])[None, :].repeat(z.shape[0], 0), -z), axis=1)[:, :k]
    e = np.exp(z - z.max(axis=1, keepdims=True), dtype=np.float32)
    p = e / e.sum(axis=1, keepdims=True, dtype=np.float32)
    return order.astype(np.int32), np.take_along_axis(p, order, axis=1)


@pytest.mark.parametrize("k", [1, 8])
@pytest.mark.parametrize("B,A", [(64, 28), (5, 1845), (9, 8), (1, 33)])
def test_answer_topk_against_numpy(B, A, k):
    from mac_network_b200.output_unit import answer_topk
    rng = np.random.RandomState(A + k)
    z = (3 * rng.standard_normal((B, A))).astype(np.float32)
    z[0, :] = np.round(z[0, :])                                             # many exact ties
    z[-1, A // 2] = 3.0e4                                                   # one very large logit: no overflow
    if B > 2:
        z[1, :] = 0.25                                                      # a constant row: ids 0..k-1
    ids, probs = answer_topk(torch.from_numpy(z).cuda(), k)
    want_ids, want_p = _topk_numpy(z, k)
    assert np.array_equal(ids.cpu().numpy(), want_ids)
    got_p = probs.cpu().numpy()
    assert np.isfinite(got_p).all() and np.allclose(got_p, want_p, rtol=2e-6, atol=1e-9)
    assert np.array_equal(ids[:, 0].cpu().numpy(), torch.argmax(torch.from_numpy(z), dim=-1).numpy())
    if k == A:
        assert np.abs(got_p.sum(axis=1) - 1).max() < 1e-6
    assert got_p[-1, 0] == 1.0


def test_answer_topk_refuses_k_out_of_range():
    L_, lib = _lib()
    from mac_network_b200.output_unit import answer_topk
    z = torch.zeros(4, 6, device="cuda")
    ids = torch.full((4, 8), -7, dtype=torch.int32, device="cuda")
    probs = torch.zeros(4, 8, device="cuda")
    for k in (0, 7, 9):
        assert lib.mac_answer_topk(L_.ptr(z), 4, 6, k, L_.ptr(ids), L_.ptr(probs), None) == INVALID
        with pytest.raises(ValueError):
            answer_topk(z, k)
    torch.cuda.synchronize()
    assert bool((ids == -7).all())


def test_output_unit_logits_equals_forward_bit_for_bit():
    from mac_network_b200.output_unit import OutputUnit, init_output_params, output_specs
    B, d, A = 64, 512, 28
    p = {k: torch.from_numpy(v).cuda() for k, v in init_output_params(output_specs(d, d, (512,), A), seed=3).items()}
    unit = OutputUnit(p, relu="ELU", keep=1.0)
    g = torch.Generator(device="cuda").manual_seed(5)
    mem, vq = torch.randn(B, d, device="cuda", generator=g), torch.randn(B, d, device="cuda", generator=g)
    answers = torch.zeros(B, dtype=torch.int32, device="cuda")
    want = unit.forward(mem, vq, answers)[0].clone()
    assert torch.equal(unit.logits(mem, vq), want)
    assert torch.equal(OutputUnit(p, relu="ELU", keep=0.85).logits(mem, vq), want)      # the label-free form never drops


@pytest.mark.parametrize("prec", ["fp32", "bf16", "bf16x3", "fp8"])
@pytest.mark.parametrize("B,H,W", [(4, 14, 14), (3, 7, 7)])
def test_stem_forward_nchw_equals_forward_of_the_permuted_image(prec, B, H, W):
    from mac_network_b200.stem import Stem, init_stem_params, stem_specs
    C = 256
    p = {k: torch.from_numpy(v).cuda() for k, v in init_stem_params(stem_specs(C, 128), seed=6).items()}
    stem = Stem(p, relu="ELU", prec=prec)
    x = _features(B, C, H, W, seed=11)
    want = stem.forward(x.permute(0, 2, 3, 1).contiguous())
    assert torch.equal(stem.forward_nchw(x), want)
    if prec == "bf16":
        assert torch.equal(stem.forward_nchw(x.to(torch.bfloat16)), want)
    else:
        with pytest.raises(ValueError):
            stem.forward_nchw(x.to(torch.bfloat16))
    with pytest.raises(ValueError):
        stem.forward_nchw(x.permute(0, 2, 3, 1))


# ------------------------------------------------------------------------------------------------ the pipeline
MODELS = {"fp32": dict(prec="fp32"), "bf16": dict(prec="bf16"),
          "fp8": dict(prec="fp8", eval_stem_prec="fp8", eval_enc_prec="bf16")}
V, E, C, A = 90, 300, 128, 28


def _net(variant, model, L=3, seed=3):
    from mac_network_b200.config import MACConfig
    from mac_network_b200.model import MACnet
    cfg = MACConfig.args(variant, netLength=L)
    return MACnet(cfg, L, V, A, wrd_emb_dim=E, image_in_dim=C, classifier_dims=(512,), seed=seed, **MODELS[model])


def _batches(n, B, S, H, W, seed, longest):
    """n host batches; every batch's longest question has length `longest` (<= S), questions 0-padded to S."""
    rng = np.random.RandomState(seed)
    out = []
    for _ in range(n):
        lengths = rng.randint(1, longest + 1, size=(B,)).astype(np.int32)
        lengths[rng.randint(B)] = longest
        q = rng.randint(1, V + 1, size=(B, S)).astype(np.int32)
        q[np.arange(S)[None, :] >= lengths[:, None]] = 0
        out.append({"questions": q, "questionLengths": lengths,
                    "images": np.maximum(rng.standard_normal((B, C, H, W)), 0).astype(np.float32)})
    return out


def _reference(net, batch):
    """runBatch(train=False, getAtt=True) on one batch: predictions and attention maps from its result, logits and memory
    from the units it leaves behind."""
    data = dict(batch, answers=np.zeros(len(batch["questionLengths"]), dtype=np.int32))
    res = net.runBatch(None, data, {"images": batch["images"]}, train=False, getAtt=True)
    torch.cuda.synchronize()
    cell = net.macCell
    ref = {"answers": np.array([p["prediction"] for p in res["preds"]], dtype=np.int32),
           "logits": net._out.last_logits.cpu().numpy(), "memory": cell._hm[net.L].cpu().numpy(),
           "att_kb": torch.stack(cell.attentions["kb"]).cpu().numpy(),
           "att_question": torch.stack(cell.attentions["question"]).cpu().numpy()}
    if cell.attentions["gate"]:
        ref["gate"] = torch.stack(cell.attentions["gate"]).cpu().numpy()
    if cell.attentions["self"]:
        ref["self"] = [a.cpu().numpy() for a in cell.attentions["self"]]
    # the attention maps runBatch hands its caller are these tensors
    assert np.array_equal(np.array(res["preds"][0]["attentions"]["kb"], dtype=np.float32).reshape(net.L, -1),
                          ref["att_kb"][:, 0])
    return ref


def _assert_same(out, ref, L):
    got = {k: v.numpy() for k, v in out.items()}
    assert np.array_equal(got["answers"][:, 0], ref["answers"])
    for k in ("logits", "memory", "att_kb", "att_question"):
        assert np.array_equal(got[k], ref[k]), k
    assert ("gate" in got) == ("gate" in ref) and ("self" in got) == ("self" in ref)
    if "gate" in ref:
        assert np.array_equal(got["gate"], ref["gate"])
    if "self" in ref:
        for i in range(L):
            assert np.array_equal(got["self"][i, :, :i + 1], ref["self"][i]) and not got["self"][i, :, i + 1:].any()


@pytest.mark.parametrize("variant,H,W", [("args", 14, 14), ("gqa", 7, 7)])
@pytest.mark.parametrize("model", ["fp32", "bf16", "fp8"])
def test_pipeline_equals_run_batch_bit_for_bit(variant, H, W, model):
    """The longest question of every batch fills S.  With and without the host cast, with and without the graph, 1 and 4
    slots; nine submits, so every slot and every staging buffer is used again."""
    from mac_network_b200.serving import ModelPipeline
    B, S, L = 8, 10, 3
    net = _net(variant, model, L)
    batches = _batches(9, B, S, H, W, seed=21, longest=S)
    refs = [_reference(net, b) for b in batches]
    for slots, use_graph, host_cast in ((4, True, True), (1, True, False), (4, False, True), (2, False, False)):
        pipe = ModelPipeline(net, (B, S, H, W), slots=slots, use_graph=use_graph, host_cast=host_cast, topk=3,
                             cast_threads=3)
        assert pipe.host_cast == (host_cast and model == "bf16")
        assert pipe.h2d_bytes == B * C * H * W * (2 if pipe.host_cast else 4) + B * S * 4 + B * 4
        tickets = []
        for i, b in enumerate(batches):
            tickets.append(pipe.submit(b, next_batch=batches[i + 1] if i + 1 < len(batches) else None))
            if len(tickets) >= slots:                       # read each result before its slot is taken again
                j = len(tickets) - slots
                _assert_same(pipe.result(tickets[j]), refs[j], L)
        for j in range(max(0, len(batches) - slots + 1), len(batches)):
            out = pipe.result(tickets[j])
            _assert_same(out, refs[j], L)
            p = out["probs"].numpy()
            assert (p[:, :-1] >= p[:, 1:]).all() and (p > 0).all() and p.sum(axis=1).max() <= 1 + 1e-6
        assert pipe.predictions(out) == [int(a) for a in refs[-1]["answers"]]
        pipe.drain()


@pytest.mark.parametrize("variant,H,W", [("args", 14, 14), ("gqa", 7, 7)])
@pytest.mark.parametrize("model", ["fp32", "bf16", "fp8"])
def test_pipeline_padding_beyond_the_longest_question(variant, H, W, model):
    """Every question shorter than S: runBatch trims the batch to its longest question, the pipeline cannot.  Attention at
    positions >= length is exactly 0 and nothing else moves by more than the changed reduction length allows."""
    from mac_network_b200.serving import ModelPipeline
    B, S, L, longest = 8, 12, 3, 7
    net = _net(variant, model, L)
    batch = _batches(1, B, S, H, W, seed=31, longest=longest)[0]
    ref = _reference(net, batch)
    pipe = ModelPipeline(net, (B, S, H, W), slots=1)
    out = {k: v.numpy() for k, v in pipe.result(pipe.submit(batch)).items()}
    beyond = np.arange(S)[None, :] >= batch["questionLengths"][:, None]
    assert not out["att_question"][:, beyond].any()
    assert np.array_equal(out["answers"][:, 0], ref["answers"])
    rel = lambda a, b: float(np.abs(a.astype(np.float64) - b).max() / np.abs(b).max())
    errs = {"att_question": rel(out["att_question"][:, :, :longest], ref["att_question"]),
            "att_kb": rel(out["att_kb"], ref["att_kb"]), "memory": rel(out["memory"], ref["memory"]),
            "logits": rel(out["logits"], ref["logits"])}
    print("padded to S = %d against trimmed to %d: %s" % (S, longest, errs))
    assert max(errs.values()) <= 1e-6, errs


def test_pipeline_follows_the_weights_and_keeps_old_tickets():
    """After the parameter values move (`params.touch()`), the next result is runBatch's on the new weights; results of
    earlier tickets stay readable until `slots` further submits; a ticket older than that is refused."""
    from mac_network_b200.serving import ModelPipeline
    B, S, H, W, L = 8, 10, 14, 14, 3
    net = _net("args", "bf16", L)
    batches = _batches(4, B, S, H, W, seed=41, longest=S)
    pipe = ModelPipeline(net, (B, S, H, W), slots=2)
    ref0 = _reference(net, batches[0])
    t0 = pipe.submit(batches[0])
    t1 = pipe.submit(batches[1])
    _assert_same(pipe.result(t0), ref0, L)                  # still there after one further submit
    p = net.trainer.params
    with torch.no_grad():
        p.flat.mul_(1.03)
    p.touch()
    ref2 = _reference(net, batches[2])
    t2 = pipe.submit(batches[2])                            # drains and captures again before it takes the batch
    _assert_same(pipe.result(t2), ref2, L)
    with pytest.raises(ValueError):
        pipe.result(t0)                                     # its slot now holds t2
    pipe.result(t1)
    # the same batch before and after the move differs: the pipeline did not serve stale packs
    t3 = pipe.submit(batches[0])
    assert not np.array_equal(pipe.result(t3)["logits"].numpy(), ref0["logits"])
    with pytest.raises(ValueError):
        pipe.submit(dict(batches[0], questions=batches[0]["questions"][:, :S - 1]))
    pipe.drain()


@pytest.mark.parametrize("use_graph", [True, False])
def test_pipeline_waits_for_the_stream_that_moved_the_weights(use_graph):
    """The weights are moved on the caller's stream behind a long queue of other work -- an in-place update + `touch()`,
    then a `DPTrainer` optimizer step, which does not synchronise -- and `submit` follows with no device synchronise in
    between: the slots' streams must wait for that stream before they rebuild their packs, or they serve the old weights."""
    from mac_network_b200.serving import ModelPipeline
    B, S, H, W, L = 8, 10, 14, 14, 3
    net = _net("args", "bf16", L)
    batches = _batches(3, B, S, H, W, seed=51, longest=S)
    pipe = ModelPipeline(net, (B, S, H, W), slots=2, use_graph=use_graph)
    pipe.result(pipe.submit(batches[0]))
    p = net.trainer.params
    busy = torch.randn(8192, 8192, device="cuda")

    def queue_work():                                       # tens of milliseconds ahead of whatever is enqueued next
        a = busy
        for _ in range(12):
            a = (a @ busy).clamp_(-1, 1)

    queue_work()
    with torch.no_grad():
        p.flat.mul_(1.03)
    p.touch()
    out = {k: v.clone() for k, v in pipe.result(pipe.submit(batches[1])).items()}
    _assert_same(out, _reference(net, batches[1]), L)
    # an optimizer step of the trainer on the same stream
    data = dict(batches[0], answers=np.arange(B, dtype=np.int32) % A)
    dev = net._to_device(net.trimData(dict(data)), {"images": batches[0]["images"]})
    version = p.version
    queue_work()
    net.trainer.train_step_full((B, S), dev, global_batch=B)
    assert p.version != version
    out = {k: v.clone() for k, v in pipe.result(pipe.submit(batches[2])).items()}
    _assert_same(out, _reference(net, batches[2]), L)
    pipe.drain()
