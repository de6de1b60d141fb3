"""ORACLE (test infrastructure only): the reference's output unit, classifier and answer loss with the output-unit flags
`--outQuestion` (on or off), `--outQuestionMul` and `--outputBN`, as a numpy restatement (`output_forward`) and as a
differentiable fp64 PyTorch graph (`output_graph`, a drop-in for `model_torch_autograd.output_graph` with the same
defaults).  `oracle/output_oracle.py` and `oracle/model_torch_autograd.py` keep the shipped layout (question on, no
product, no batch norm), which these reproduce with the default keywords.

  * `model.py:512-528`  outputOp:    features = memory, [memory, q'] or [memory, q', memory * q'] (ops.concat, ops.py:65-78)
                                     with q' = linear_outQuestion(vecQuestions); outQuestionMul has no effect without
                                     outQuestion
  * `model.py:547-576`  classifier:  ops.FCLayer(features, [F] + outClassifierDims + [answerWordsNum], batchNorm, dropout)
  * `ops.py:298-359`    ops.linear:  batch_norm (outputBN), then the input dropout, then the matmul; `act` (RELU ->
                                     config.relu) between layers
  * `ops.py:307-309`    batch_norm:  tf.contrib.layers.batch_norm(decay=bnDecay, center, scale, updates_collections=None),
                                     epsilon 1e-3: batch mean / biased variance in training with the stored statistics
                                     moved towards the batch mean / Bessel-corrected variance; the stored ones at eval
Pinned by `tests/golden/output_<layout>_<widths>_<mode>.npz` (`oracle/gen_output_options.py`)."""
import numpy as np
import torch

from oracle.mac_oracle import elu
from oracle.model_torch_autograd import _act, _dropout

EPS = 1e-3


def batch_norm_np(x, p, scope, train, decay, dtype=np.float64):
    """(y, stored mean, stored variance after the call) of the batch norm under `scope` + "BatchNorm/"."""
    sc = scope + "BatchNorm/"
    beta, gamma, mm, mv = (p[sc + n] for n in ("beta", "gamma", "moving_mean", "moving_variance"))
    if not train:
        return (x - mm) / np.sqrt(mv + dtype(EPS)) * gamma + beta, mm, mv
    n = x.shape[0]
    mean = x.mean(0)
    var = ((x - mean) ** 2).mean(0)
    unbiased = var * (dtype(n) / max(n - 1, 1))
    y = (x - mean) / np.sqrt(var + dtype(EPS)) * gamma + beta
    return y, mm - (mm - mean) * (1.0 - dtype(decay)), mv - (mv - unbiased) * (1.0 - dtype(decay))


def output_forward(relu, params, memory, vecQuestions, answers, keep=1.0, uniforms=None, question=True, mul=False,
                   bn=False, train=None, decay=0.999, dtype=np.float64):
    """numpy forward: {"logits", "losses", "loss", "preds"} and, with `bn`, "moving" (the stored statistics after the call,
    by variable name).  `train` (the batch norm's is_training) defaults to keep < 1."""
    p = {k: np.asarray(v, dtype) for k, v in params.items()}
    us = iter(uniforms or [])
    train = float(keep) < 1.0 if train is None else bool(train)
    moving = {}

    def dropout(x):
        if float(keep) == 1.0:
            return x
        return x / dtype(keep) * np.floor(dtype(keep) + np.asarray(next(us), dtype))

    x = np.asarray(memory, dtype)
    if question:
        sc = "outputUnit/linearLayeroutQuestion/"
        eq = np.asarray(vecQuestions, dtype) @ p[sc + "weights/weight"] + p[sc + "biases/bias"]
        x = np.concatenate([x, eq] + ([x * eq] if mul else []), axis=-1)
    nfc = len([k for k in p if k.startswith("classifier/linearLayerfc_") and k.endswith("weights/weight")])
    for i in range(nfc):
        sc = "classifier/linearLayerfc_%d/" % i
        if bn:
            x, moving[sc + "BatchNorm/moving_mean"], moving[sc + "BatchNorm/moving_variance"] = \
                batch_norm_np(x, p, sc, train, decay, dtype)
        x = dropout(x) @ p[sc + "weights/weight"] + p[sc + "biases/bias"]
        if i < nfc - 1:
            x = elu(x) if relu == "ELU" else np.maximum(x, 0)
    m = x.max(-1, keepdims=True)
    lse = m[:, 0] + np.log(np.exp(x - m).sum(-1))
    losses = lse - x[np.arange(x.shape[0]), np.asarray(answers)]
    out = {"logits": x, "losses": losses, "loss": losses.mean(), "preds": x.argmax(-1)}
    if bn:
        out["moving"] = moving
    return out


def batch_norm(x, p, sc, train, decay, moving, eps=EPS):
    """torch form of `batch_norm_np` under the scope `sc` (ending in "BatchNorm/"); the stored statistics are constants,
    and their update goes into the dict `moving` (when given)."""
    mm, mv = p[sc + "moving_mean"].detach(), p[sc + "moving_variance"].detach()
    if not train:
        mean, var = mm, mv
    else:
        n = x.shape[0]
        mean = x.mean(0)
        var = ((x - mean) ** 2).mean(0)
        if moving is not None:
            unbiased = var.detach() * (float(n) / max(n - 1, 1))
            moving[sc + "moving_mean"] = mm - (mm - mean.detach()) * (1.0 - decay)
            moving[sc + "moving_variance"] = mv - (mv - unbiased) * (1.0 - decay)
    return (x - mean) / torch.sqrt(var + eps) * p[sc + "gamma"] + p[sc + "beta"]


def output_graph(relu, p, memory, vecQuestions, answers, keep=1.0, uniforms=None, question=True, mul=False, bn=False,
                 train=True, decay=0.999, moving=None):
    """outputOp + classifier + the per-sample sparse softmax cross-entropy as an fp64 torch graph: (logits, losses).
    Without the question no gradient reaches `vecQuestions`.  With `bn`, `train` picks the batch statistics (True) or the
    stored ones, and `moving` (a dict) receives the stored statistics after the call."""
    us = iter(uniforms or [])
    x = memory
    if question:
        sc = "outputUnit/linearLayeroutQuestion/"
        eq = vecQuestions @ p[sc + "weights/weight"] + p[sc + "biases/bias"]
        x = torch.cat([memory, eq] + ([memory * eq] if mul else []), -1)
    nfc = len([k for k in p if k.startswith("classifier/linearLayerfc_") and k.endswith("weights/weight")])
    for i in range(nfc):
        sc = "classifier/linearLayerfc_%d/" % i
        if bn:
            x = batch_norm(x, p, sc + "BatchNorm/", train, decay, moving)
        x = _dropout(x, keep, us) @ p[sc + "weights/weight"] + p[sc + "biases/bias"]
        if i < nfc - 1:
            x = _act(relu, x)
    losses = torch.logsumexp(x, -1) - x.gather(1, answers.view(-1, 1)).squeeze(1)
    return x, losses


def output_graph_for(options, decay, moving):
    """`output_graph` with `options` ({"question", "mul", "bn"}) and the batch norm's training form bound, with the
    signature of `model_torch_autograd.output_graph`: what `model_torch_autograd.run` calls in its place for a model with
    those options.  `moving` receives the stored statistics after the training forward."""
    def graph(relu, p, memory, vecQuestions, answers, keep=1.0, uniforms=None):
        return output_graph(relu, p, memory, vecQuestions, answers, keep, uniforms, train=True, decay=decay, moving=moving,
                            **options)
    return graph
