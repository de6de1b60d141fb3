"""Output unit, classifier and answer loss of the reference model on the same CUDA primitives as the cell
(SURVEY.md section 8(f), "next" row 2): `MACnet.outputOp` (`model.py:512-528`, `outQuestion` on), `MACnet.classifier`
(`model.py:547-576` -> `ops.FCLayer`, `ops.py:349-359`), `addAnswerLossOp` (`model.py:593-596`).

    features = [memory, vecQuestions @ W_oq + b_oq]                       (2 * memDim)
    h        = act(dropout(features) @ W_fc0 + b_fc0) ...                 (outClassifierDims, act = RELU -> config.relu)
    logits   = dropout(h) @ W_fcK + b_fcK                                 (answerWordsNum)
    loss     = mean_b( logsumexp(logits_b) - logits_b[answer_b] )

It supplies dL/dmemory and dL/dvecQuestions to the cell's backward, so data-parallel training runs on the reference's
real loss.  Variable names follow the reference's scopes (siblings of "MACnetwork/" under "macModel/")."""
import collections

import numpy as np
import torch

from . import _lib, packs
from ._lib import act_code, check, ptr, segments, stream_ptr

SITE_OUTPUT = 16          # Philox site base for the output unit's dropouts (site + layer index)


def output_specs(ctrl_dim, mem_dim, hidden, n_answers):
    s = collections.OrderedDict()
    s["outputUnit/linearLayeroutQuestion/weights/weight"] = ((ctrl_dim, mem_dim), "xavier")
    s["outputUnit/linearLayeroutQuestion/biases/bias"] = ((mem_dim,), "zeros")
    dims = [2 * mem_dim] + list(hidden) + [n_answers]
    for i in range(len(dims) - 1):
        s["classifier/linearLayerfc_%d/weights/weight" % i] = ((dims[i], dims[i + 1]), "xavier")
        s["classifier/linearLayerfc_%d/biases/bias" % i] = ((dims[i + 1],), "zeros")
    return s


def init_output_params(specs, seed=0, dtype=np.float32, bias_scale=0.1):
    rng = np.random.RandomState(seed)
    out = collections.OrderedDict()
    for name, (shape, kind) in specs.items():
        if kind == "zeros":
            v = bias_scale * rng.standard_normal(shape)       # non-trivial biases so bias handling is exercised
        else:
            lim = np.sqrt(6.0 / (shape[0] + shape[1]))
            v = rng.uniform(-lim, lim, size=shape)
        out[name] = np.asarray(v, dtype=dtype)
    return out


def answer_topk(logits, k=1, ids=None, probs=None):
    """(ids int32 [B, k], probs fp32 [B, k]): the k most probable answers of each row of `logits` [B, A] and their softmax
    probabilities, equal logits in ascending id order (`mac_answer_topk`); ids[:, 0] is the prediction of `addPredOp`
    (`model.py:603-612`).  1 <= k <= min(8, A).  `ids` / `probs`: optional output tensors to write into."""
    B, A = logits.shape
    if not 1 <= int(k) <= min(8, A):
        raise ValueError("k must be in 1..min(8, A = %d), got %r" % (A, k))
    ids = torch.empty((B, k), dtype=torch.int32, device=logits.device) if ids is None else ids
    probs = torch.empty((B, k), dtype=torch.float32, device=logits.device) if probs is None else probs
    check(_lib.load().mac_answer_topk(ptr(logits), B, A, int(k), ptr(ids), ptr(probs), stream_ptr()), "mac_answer_topk")
    return ids, probs


class OutputUnit(object):
    """Forward / loss / backward of the output unit on device tensors.  `params` / `grads`: dict name -> tensor
    (e.g. views into the trainer's flat buckets)."""

    def __init__(self, params, relu="ELU", keep=1.0, seed=0, version=None):
        """`version`: optional callable returning a counter that changes whenever the parameter values do
        (`MACParams.version`): the transposed weight copies of the backward are rebuilt when it moves."""
        self.lib = _lib.load()
        self.p = params
        self._cache = packs.Cache(version)
        self.relu, self.keep, self.seed = relu, float(keep), int(seed)
        self.nfc = len([k for k in params if k.startswith("classifier/linearLayerfc_") and k.endswith("weights/weight")])
        for k, v in params.items():
            if k.endswith("weights/weight") and (v.shape[0] % 4 or v.shape[1] % 4):
                raise ValueError("%s is %s: the fp32 GEMM needs every dimension to be a multiple of 4 (pad the answer "
                                 "vocabulary / classifier width)" % (k, tuple(v.shape)))
        dev = next(iter(params.values())).device
        self.lws_bytes = 4096 + 32 * 64 * 2048 * 4
        self.lws = torch.zeros(self.lws_bytes, dtype=torch.uint8, device=dev)

    def _new(self, *shape):
        return torch.empty(shape, dtype=torch.float32, device=self.lws.device)

    def _linear(self, xs, W, b, act=0):
        n, M = len(xs), xs[0].shape[0]
        y = self._new(M, W.shape[1])
        arr_p, arr_k, arr_ld = segments(xs)
        check(self.lib.mac_linear_fwd(arr_p, arr_k, arr_ld, n, ptr(W), ptr(b), 0.0, act, ptr(y), y.stride(0), M, W.shape[1],
                                      ptr(self.lws), self.lws_bytes, stream_ptr()), "mac_linear_fwd")
        return y

    def _dropout(self, x, layer, step):
        if self.keep >= 1.0:
            return x
        out = self._new(*x.shape)
        check(self.lib.mac_dropout_fwd(ptr(x), self.keep, self.seed, SITE_OUTPUT + layer, step, ptr(out), x.numel(),
                                       stream_ptr()), "mac_dropout_fwd")
        return out

    def forward(self, memory, vecQuestions, answers, step=0, loss_scale=None):
        """Returns (logits, losses [B], dlogits [B, A]) -- dlogits = (softmax - onehot) * loss_scale (default 1/B).  The three
        stay reachable as `last_logits`, `losses` and `dlogits` (`logits` is the label-free method)."""
        B = memory.shape[0]
        self.forward_logits(memory, vecQuestions, step)
        A = self.last_logits.shape[1]
        self.losses = self._new(B)
        self.dlogits = self._new(B, A)
        scale = (1.0 / B) if loss_scale is None else float(loss_scale)
        check(self.lib.mac_softmax_xent(ptr(self.last_logits), ptr(answers), ptr(self.losses), ptr(self.dlogits), scale, B, A,
                                        stream_ptr()), "mac_softmax_xent")
        return self.last_logits, self.losses, self.dlogits

    def forward_logits(self, memory, vecQuestions, step=0):
        """The training forward up to the logits (this unit's dropouts, its inputs kept for `backward`), without the loss:
        `backward(dlogits=)` then takes the gradient of the logits from the caller.  Returns the logits [B, A]."""
        act = act_code("RELU", self.relu)
        self.eq = self._linear([vecQuestions], self.p["outputUnit/linearLayeroutQuestion/weights/weight"],
                               self.p["outputUnit/linearLayeroutQuestion/biases/bias"])
        self.memory, self.vecq, self.step = memory, vecQuestions, step
        self.inputs = []            # per layer: list of input segments after dropout
        xs = [memory, self.eq]
        x = None
        for i in range(self.nfc):
            W = self.p["classifier/linearLayerfc_%d/weights/weight" % i]
            b = self.p["classifier/linearLayerfc_%d/biases/bias" % i]
            if i == 0:
                # dropout over the concatenated features: one Philox stream over [B, 2*memDim], applied per segment
                if self.keep < 1.0:
                    cat = torch.cat(xs, dim=1)                                # plumbing: layout for the flat mask index
                    xs = [self._dropout(cat, 0, step)]
            else:
                xs = [self._dropout(x, i, step)]
            self.inputs.append(xs)
            x = self._linear(xs, W, b, act if i < self.nfc - 1 else 0)
            if i < self.nfc - 1:
                setattr(self, "_h%d" % i, x)
        self.last_logits = x
        return x

    def logits(self, memory, vecQuestions):
        """The answer logits [B, A] without labels: the linears of `forward` with every dropout at 1, no loss, no `dlogits`,
        nothing kept for a backward.  Bit for bit `forward(...)[0]` of a unit with keep = 1."""
        act = act_code("RELU", self.relu)
        eq = self._linear([vecQuestions], self.p["outputUnit/linearLayeroutQuestion/weights/weight"],
                          self.p["outputUnit/linearLayeroutQuestion/biases/bias"])
        xs = [memory, eq]
        for i in range(self.nfc):
            xs = [self._linear(xs, self.p["classifier/linearLayerfc_%d/weights/weight" % i],
                               self.p["classifier/linearLayerfc_%d/biases/bias" % i], act if i < self.nfc - 1 else 0)]
        return xs[0]

    def backward(self, grads, d_memory, d_vecq, dlogits=None):
        """Accumulates parameter gradients into `grads` (dict name -> tensor) and ADDS dL/dmemory, dL/dvecQuestions.
        `dlogits`: the gradient of the logits [B, A]; by default the loss's, `self.dlogits`, from `forward`."""
        B = self.memory.shape[0]
        dy = self.dlogits if dlogits is None else dlogits
        act = act_code("RELU", self.relu)

        def lin_bwd(xs, wname, bname, dy, dxs, accum):
            _lib.linear_bwd(xs, self._cache.pack(packs.transposed, self.p[wname]), dy, dxs, accum, grads[wname],
                            grads[bname], self.lws, self.lws_bytes, stream_ptr())
        for i in reversed(range(self.nfc)):
            xs = self.inputs[i]
            wn, bn = "classifier/linearLayerfc_%d/weights/weight" % i, "classifier/linearLayerfc_%d/biases/bias" % i
            if i == 0 and len(xs) == 2:
                dmem, deq = self._new(B, xs[0].shape[1]), self._new(B, xs[1].shape[1])
                lin_bwd(xs, wn, bn, dy, [dmem, deq], [0, 0])
            else:
                dx = self._new(B, xs[0].shape[1])
                lin_bwd(xs, wn, bn, dy, [dx], [0])
                if self.keep < 1.0:       # through the input dropout of this layer
                    check(self.lib.mac_dropout_fwd(ptr(dx), self.keep, self.seed, SITE_OUTPUT + i, self.step, ptr(dx),
                                                   dx.numel(), stream_ptr()), "dropout bwd")
                if i == 0:
                    md = self.memory.shape[1]
                    dmem, deq = dx[:, :md].contiguous(), dx[:, md:].contiguous()
                else:
                    h = getattr(self, "_h%d" % (i - 1))
                    dpre = self._new(*h.shape)
                    check(self.lib.mac_activation_bwd(ptr(h), ptr(dx), act, ptr(dpre), h.numel(), stream_ptr()), "act bwd")
                    dy = dpre
        check(self.lib.mac_axpy(ptr(d_memory), ptr(dmem), 1.0, dmem.numel(), stream_ptr()), "axpy")
        lin_bwd([self.vecq], "outputUnit/linearLayeroutQuestion/weights/weight",
                "outputUnit/linearLayeroutQuestion/biases/bias", deq, [d_vecq], [1])
