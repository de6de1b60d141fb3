"""ORACLE (test infrastructure only): the reference's whole training loss (`MACnet.build`, model.py:774-821) as one
differentiable fp64 PyTorch graph, used to check the trainer's hand-written backward element by element against
`torch.autograd` (the reference uses TF autodiff, model.py:626-636):

    embeddings + bi-LSTM (`encoder_torch_autograd.graph`) -> image stem (`stem_graph`) -> optional gather of each question's
    knowledge base by `imageIndex` -> netLength MAC steps (`mac_torch_autograd.graph`) -> output unit and classifier
    (`output_graph`) -> sum of the per-sample softmax cross-entropies / global_batch.

Each unit consumes its own list of uniforms in the reference's call order, with tf.nn.dropout's x / keep * floor(keep + U).
The forward is pinned to the chain of numpy oracles (each pinned to the reference's own code on the TF1 shim) and the
gradient to central differences of this graph in tests/test_model_autograd_oracle.py."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import encoder_torch_autograd, mac_torch_autograd

UNITS = ("encoder", "stem", "cell", "output")


def _dropout(x, keep, us):
    if float(keep) == 1.0:
        return x
    return x / float(keep) * torch.floor(float(keep) + torch.as_tensor(next(us), dtype=torch.float64).to(x.device))


def _act(relu, x):
    """ops.py:161-187: the "RELU" activation of the stem and the classifier under `config.relu`."""
    return F.elu(x) if relu == "ELU" else torch.relu(x)


def mask_uniforms(mask):
    """Uniforms whose tf.nn.dropout mask floor(keep + U) is exactly `mask` (0 / 1) for any keep in (2^-30, 1)."""
    return torch.as_tensor(mask, dtype=torch.float64) * (1.0 - 2.0 ** -30)


def stem_graph(relu, p, images, keep=1.0, uniforms=None):
    """ops.CNNLayer (ops.py:380-438): per layer, dropout on the input, 3x3 stride-1 SAME conv2d with the HWIO kernel, bias,
    activation.  `images` fp64 NHWC [B, H, W, C]; returns the knowledge base [B, H*W, d]."""
    us = iter(uniforms or [])
    cur = images
    n = len([k for k in p if k.startswith("stem/") and k.endswith("kernels/kernel")])
    for i in range(n):
        cur = _dropout(cur, keep, us)
        K = p["stem/cnnLayercnn_%d/kernels/kernel" % i]                       # HWIO -> OIHW
        y = F.conv2d(cur.permute(0, 3, 1, 2), K.permute(3, 2, 0, 1), padding=K.shape[0] // 2).permute(0, 2, 3, 1)
        cur = _act(relu, y + p["stem/cnnLayercnn_%d/biases/bias" % i])
    return cur.reshape(cur.shape[0], -1, cur.shape[-1])


def output_graph(relu, p, memory, vecQuestions, answers, keep=1.0, uniforms=None):
    """outputOp + classifier + the per-sample sparse softmax cross-entropy (model.py:512-596): returns (logits, losses)."""
    us = iter(uniforms or [])
    eq = vecQuestions @ p["outputUnit/linearLayeroutQuestion/weights/weight"] + p["outputUnit/linearLayeroutQuestion/biases/bias"]
    x = torch.cat([memory, eq], -1)
    nfc = len([k for k in p if k.startswith("classifier/linearLayerfc_") and k.endswith("weights/weight")])
    for i in range(nfc):
        sc = "classifier/linearLayerfc_%d/" % i
        x = _dropout(x, keep, us) @ p[sc + "weights/weight"] + p[sc + "biases/bias"]
        if i < nfc - 1:
            x = _act(relu, x)
    losses = torch.logsumexp(x, -1) - x.gather(1, answers.view(-1, 1)).squeeze(1)
    return x, losses


def stem_grads(relu, params, images, keep, uniforms, d_kb):
    """The stem's fp64 forward and its gradients for the upstream gradient `d_kb`: (kb, {name: grad}, d_images), on the
    device and in the array kind (numpy or torch) of `images`."""
    as_np = isinstance(images, np.ndarray)
    dev = torch.device("cpu") if as_np else images.device
    t64 = lambda a: torch.as_tensor(np.asarray(a) if isinstance(a, np.ndarray) else a, dtype=torch.float64).to(dev)
    p = {k: t64(v).requires_grad_(True) for k, v in params.items()}
    x = t64(images).requires_grad_(True)
    kb = stem_graph(relu, p, x, keep, uniforms)
    (kb * t64(d_kb)).sum().backward()
    out = lambda t: t.detach().cpu().numpy() if as_np else t.detach()
    return out(kb), {k: out(v.grad) for k, v in p.items()}, out(x.grad)


def stem_graph_for(geometry):
    """The stem `run` calls for a model with the stem options `geometry`, with the signature of `stem_graph`: a dict as
    `DPTrainer(stem=(C, layers, geometry))` takes it, of which "strides", "linear" and "location" (with "location_bias"
    and "location_dim", defaulting as the library's do) select the graph; the kernel sizes are the kernels' own.  The
    stem's uniforms are the reference's: with location features the first draw covers layer 0's whole input
    [k, H, W, C + l] (`oracle/stem_geometry.py`, `oracle/stem_location.py`)."""
    # imported here: oracle/output_options.py imports this module, and these two are only needed with the options
    from oracle.stem_geometry import stem_torch
    from oracle.stem_location import stem_loc_torch
    strides, linear = geometry.get("strides"), bool(geometry.get("linear", False))
    location = geometry.get("location")
    if location is not None:
        location = (location, geometry.get("location_bias", 1.0), geometry.get("location_dim", 32))

    def graph(relu, p, images, keep=1.0, uniforms=None):
        ps = {k: v for k, v in p.items() if k.startswith("stem/")}
        if location is not None:
            return stem_loc_torch(relu, ps, images, location, keep, uniforms, strides)
        return stem_torch(relu, ps, images, keep, uniforms, strides, linear)
    return graph


def run(cfg, L, values, data, keeps, uniforms=None, global_batch=None, device="cpu", grad=True, trace=None, stem=None,
        output=None, train=True, moving=None):
    """The training loss of one shard.

    `values`: every variable by its TF name (numpy or torch); `data`: "questions" [B, S] (0 = padding),
    "questionLengths" [B], "answers" [B], the images as exactly one of "images" (NHWC [k, H, W, C]) and "images_nchw"
    ([k, C, H, W], permuted here), and optionally "imageIndex" [B] (question b asks about image imageIndex[b]; without it
    k = B).  `keeps`: {"encoder": (input, question), "stem": keep, "cell": (memory, read, write), "output": keep}.
    `uniforms`: {unit: list of draws in the reference's call order} for the units in UNITS; each list must be consumed
    exactly.  `global_batch`: the loss is sum(losses) / global_batch (default B).

    Returns {"logits", "losses", "loss"} and, with `grad`, "grads" (every variable's gradient, zeros for the stored
    batch-norm statistics) and "d_images" (in the layout of the images given), all fp64 tensors on `device`.

    `trace`: a list that receives the cell's per-step control, memory, info, "att_question" and "att_kb" (numpy, see
    `mac_torch_autograd.graph`); with it the result also holds the units' outputs the cell reads: "knowledgeBase" (the
    stem's, one per image [k, H*W, d], before the imageIndex gather), "vecQuestions", "questionWords" and
    "questionCntxWords".  It changes nothing else.

    `stem`: the stem options (see `stem_graph_for`; None: `stem_graph`, the shipped 3x3 stride-1 stem).  `output`: the
    output unit's options {"question", "mul", "bn"} (`oracle/output_options.output_graph`; None: `output_graph`, the
    shipped layout).  `train`: the batch norms' form, of the cell's memoryBN and the output unit's: batch statistics (True)
    or the stored ones (False, the reference's evaluation).  `moving`: a dict that receives the output unit's stored
    statistics after a training forward."""
    dev = torch.device(device)
    t64 = lambda a: torch.as_tensor(np.asarray(a) if isinstance(a, np.ndarray) else a).to(dev, torch.float64)
    p = {k: t64(v).requires_grad_(grad and "/BatchNorm/moving_" not in k) for k, v in values.items()}
    lng = lambda a: torch.as_tensor(np.asarray(a) if isinstance(a, np.ndarray) else a).to(dev, torch.long)
    uniforms = uniforms or {}
    assert set(uniforms) <= set(UNITS), sorted(uniforms)
    its = {u: iter(uniforms.get(u, [])) for u in UNITS}
    if ("images" in data) == ("images_nchw" in data):
        raise ValueError("data needs exactly one of images and images_nchw")
    nchw = "images_nchw" in data
    x_img = t64(data["images_nchw" if nchw else "images"]).requires_grad_(grad)
    questions, lengths, answers = lng(data["questions"]), lng(data["questionLengths"]), lng(data["answers"])
    B = questions.shape[0]
    words, cntx, vecq = encoder_torch_autograd.graph(p, questions, lengths, keeps["encoder"][0], keeps["encoder"][1],
                                                     its["encoder"])
    stem_fn = stem_graph if stem is None else stem_graph_for(stem)
    kb = stem_kb = stem_fn(cfg.relu, p, x_img.permute(0, 2, 3, 1) if nchw else x_img, keeps["stem"], its["stem"])
    if data.get("imageIndex") is not None:
        kb = kb[lng(data["imageIndex"])]
    assert kb.shape[0] == B, (kb.shape, B)
    x = {"vecQuestions": vecq, "questionWords": words, "questionCntxWords": cntx, "knowledgeBase": kb}
    _, memory = mac_torch_autograd.graph(cfg, p, x, lengths, L, keeps["cell"], its["cell"], train=train, trace=trace)
    # the cell's vecQuestions is the encoder's output: the output unit reads the same tensor (model.py:512-528)
    if output is None:
        logits, losses = output_graph(cfg.relu, p, memory, vecq, answers, keeps["output"], its["output"])
    else:
        from oracle.output_options import output_graph as options_graph
        logits, losses = options_graph(cfg.relu, p, memory, vecq, answers, keeps["output"], its["output"], train=train,
                                       decay=cfg.bnDecay, moving=moving, **output)
    for u in UNITS:
        assert next(its[u], None) is None, "%s: uniform draws left over: the dropout calls differ from the reference's" % u
    loss = losses.sum() / float(B if global_batch is None else global_batch)
    out = {"logits": logits.detach(), "losses": losses.detach(), "loss": loss.detach()}
    if trace is not None:
        out.update({"knowledgeBase": stem_kb.detach(), "vecQuestions": vecq.detach(), "questionWords": words.detach(),
                    "questionCntxWords": cntx.detach()})
    if grad:
        names = [k for k, v in p.items() if v.requires_grad]
        got = torch.autograd.grad(loss, [p[k] for k in names] + [x_img], allow_unused=True)
        g = dict(zip(names, got[:-1]))
        out["grads"] = {k: (g[k] if g.get(k) is not None else torch.zeros_like(v)).detach() for k, v in p.items()}
        out["d_images"] = (got[-1] if got[-1] is not None else torch.zeros_like(x_img)).detach()
    return out
