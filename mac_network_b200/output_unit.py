"""Output unit, classifier and answer loss of the reference model on the same CUDA primitives as the cell
(SURVEY.md section 8(f), "next" row 2): `MACnet.outputOp` (`model.py:512-528`), `MACnet.classifier` (`model.py:547-576` ->
`ops.FCLayer`, `ops.py:298-359`), `addAnswerLossOp` (`model.py:593-596`).

    q'       = vecQuestions @ W_oq + b_oq                                  (--outQuestion)
    features = [memory, q']  or  [memory, q', memory * q']  or  memory     (2, 3 or 1 x memDim; --outQuestionMul)
    h        = act(dropout(bn(features)) @ W_fc0 + b_fc0) ...              (outClassifierDims, act = RELU -> config.relu)
    logits   = dropout(bn(h)) @ W_fcK + b_fcK                              (answerWordsNum)
    loss     = mean_b( logsumexp(logits_b) - logits_b[answer_b] )

`bn` is tf.contrib.layers.batch_norm (center, scale, epsilon 1e-3, decay --bnDecay) on the input of every FC layer, present
with --outputBN only: batch statistics and the update of the stored ones in training, the stored statistics at evaluation.
`--outQuestionMul` without `--outQuestion` does nothing, as in the reference (the product is taken with q' only).  The
default options (question on, no product, no batch normalisation) are the shipped flag files' output unit.

It supplies dL/dmemory and dL/dvecQuestions to the cell's backward, so data-parallel training runs on the reference's
real loss.  Variable names follow the reference's scopes (siblings of "MACnetwork/" under "macModel/")."""
import collections

import numpy as np
import torch

from . import _lib, packs
from ._lib import act_code, check, ptr, segments, stream_ptr

SITE_OUTPUT = 16          # Philox site base for the output unit's dropouts (site + layer index)


BN_EPS = 1e-3             # tf.contrib.layers.batch_norm's default epsilon (ops.py:307-309)
OUTPUT_OPTIONS = ("question", "mul", "bn")


def output_options(options=None):
    """The output unit's layout as a dict {"question", "mul", "bn"} (--outQuestion, --outQuestionMul, --outputBN), from a
    dict of some of those keys; missing keys take the shipped flag files' values (True, False, False).  Unknown keys and
    values that are not booleans raise ValueError.  `mul` is recorded as given: it has no effect without `question`."""
    out = {"question": True, "mul": False, "bn": False}
    extra = dict(options or {})
    unknown = sorted(set(extra) - set(out))
    if unknown:
        raise ValueError("unknown output unit options %s (known: %s)" % (unknown, list(OUTPUT_OPTIONS)))
    for k, v in extra.items():
        if not isinstance(v, (bool, np.bool_)):
            raise ValueError("output unit option %r must be a bool, got %r" % (k, v))
        out[k] = bool(v)
    return out


def feature_width(mem_dim, question=True, mul=False):
    """Width of the classifier's input: memDim, 2 memDim with the question, 3 memDim with its product (ops.concat)."""
    return mem_dim * ((3 if mul else 2) if question else 1)


def is_moving_stat(name):
    """The output unit's stored batch-norm statistics: not trainable (no gradient, Adam update or EMA shadow)."""
    return name.startswith("classifier/") and "/BatchNorm/moving_" in name


def output_specs(ctrl_dim, mem_dim, hidden, n_answers, question=True, mul=False, bn=False):
    s = collections.OrderedDict()
    if question:
        s["outputUnit/linearLayeroutQuestion/weights/weight"] = ((ctrl_dim, mem_dim), "xavier")
        s["outputUnit/linearLayeroutQuestion/biases/bias"] = ((mem_dim,), "zeros")
    dims = [feature_width(mem_dim, question, mul)] + list(hidden) + [n_answers]
    for i in range(len(dims) - 1):
        s["classifier/linearLayerfc_%d/weights/weight" % i] = ((dims[i], dims[i + 1]), "xavier")
        s["classifier/linearLayerfc_%d/biases/bias" % i] = ((dims[i + 1],), "zeros")
        if bn:            # ops.linear (ops.py:306-309): batch_norm on the layer's input, under the layer's scope
            sc = "classifier/linearLayerfc_%d/BatchNorm/" % i
            s[sc + "beta"] = ((dims[i],), "zeros")
            s[sc + "gamma"] = ((dims[i],), "ones")
            s[sc + "moving_mean"] = ((dims[i],), "zeros")
            s[sc + "moving_variance"] = ((dims[i],), "ones")
    return s


def init_output_params(specs, seed=0, dtype=np.float32, bias_scale=0.1):
    rng = np.random.RandomState(seed)
    out = collections.OrderedDict()
    for name, (shape, kind) in specs.items():
        if kind == "zeros":
            v = bias_scale * rng.standard_normal(shape)       # non-trivial biases so bias handling is exercised
        elif kind == "ones":                                  # gamma, moving_variance: 1 (+ a perturbation that stays > 0)
            v = 1.0 + bias_scale * np.tanh(rng.standard_normal(shape))
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

    def __init__(self, params, relu="ELU", keep=1.0, seed=0, version=None, question=True, mul=False, bn=False,
                 bn_decay=0.999):
        """`version`: optional callable returning a counter that changes whenever the parameter values do
        (`MACParams.version`): the transposed weight copies of the backward are rebuilt when it moves.
        `question`, `mul`, `bn`: the layout (--outQuestion, --outQuestionMul, --outputBN; `output_specs`), which `params`
        must hold; `bn_decay` (--bnDecay) moves the stored batch-norm statistics in a training forward."""
        opts = output_options({"question": question, "mul": mul, "bn": bn})
        self.lib = _lib.load()
        self.p = params
        self._cache = packs.Cache(version)
        self.relu, self.keep, self.seed = relu, float(keep), int(seed)
        self.question, self.mul, self.bn = opts["question"], opts["mul"] and opts["question"], opts["bn"]
        self.options = opts
        self.bn_decay = float(bn_decay)
        self.nfc = len([k for k in params if k.startswith("classifier/linearLayerfc_") and k.endswith("weights/weight")])
        for k, v in params.items():
            if k.endswith("weights/weight") and (v.shape[0] % 4 or v.shape[1] % 4):
                raise ValueError("%s is %s: the fp32 GEMM needs every dimension to be a multiple of 4 (pad the answer "
                                 "vocabulary / classifier width)" % (k, tuple(v.shape)))
        self._check_layout()
        dev = next(iter(params.values())).device
        self.lws_bytes = 4096 + 32 * 64 * 2048 * 4
        self.lws = torch.zeros(self.lws_bytes, dtype=torch.uint8, device=dev)

    def _check_layout(self):
        """`params` against the options: raises ValueError before anything is allocated or launched."""
        p = self.p
        if not 0 < self.nfc or any("classifier/linearLayerfc_%d/weights/weight" % i not in p for i in range(self.nfc)):
            raise ValueError("the classifier's layers must be fc_0 .. fc_%d" % (self.nfc - 1))
        has_q = "outputUnit/linearLayeroutQuestion/weights/weight" in p
        if has_q != self.question:
            raise ValueError("question=%s but the parameters %s the outQuestion linear" % (self.question,
                                                                                          "hold" if has_q else "lack"))
        rows = p["classifier/linearLayerfc_0/weights/weight"].shape[0]
        if self.question:
            mem = p["outputUnit/linearLayeroutQuestion/weights/weight"].shape[1]
            if rows != feature_width(mem, True, self.mul):
                raise ValueError("fc_0 takes %d features, but memDim %d with mul=%s gives %d"
                                 % (rows, mem, self.mul, feature_width(mem, True, self.mul)))
        for i in range(self.nfc):
            sc = "classifier/linearLayerfc_%d/BatchNorm/" % i
            width = p["classifier/linearLayerfc_%d/weights/weight" % i].shape[0]
            have = [n for n in ("beta", "gamma", "moving_mean", "moving_variance") if sc + n in p]
            if len(have) != (4 if self.bn else 0):
                raise ValueError("bn=%s but fc_%d has the batch-norm variables %s" % (self.bn, i, have))
            if self.bn and any(tuple(p[sc + n].shape) != (width,) for n in have):
                raise ValueError("fc_%d's batch-norm variables must be [%d]" % (i, width))

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

    def _check_memory(self, memory):
        rows = self.p["classifier/linearLayerfc_0/weights/weight"].shape[0]
        if memory.dim() != 2 or feature_width(memory.shape[1], self.question, self.mul) != rows:
            raise ValueError("memory %s does not give fc_0's %d features" % (tuple(memory.shape), rows))

    def _features(self, memory, vecQuestions):
        """outputOp (model.py:512-528): the classifier's input as segments [memory(, q'(, memory * q'))], never concatenated."""
        if not self.question:
            return [memory]
        eq = self._linear([vecQuestions], self.p["outputUnit/linearLayeroutQuestion/weights/weight"],
                          self.p["outputUnit/linearLayeroutQuestion/biases/bias"])
        if not self.mul:
            return [memory, eq]
        B, d = memory.shape
        mq = self._new(B, d)
        check(self.lib.mac_bcast_mul(ptr(memory), ptr(eq), 0.0, ptr(mq), B, 1, d, stream_ptr()), "mac_bcast_mul")
        return [memory, eq, mq]

    def _batch_norm(self, xs, layer, train, saved=None):
        """batch_norm on the input of fc_<layer> (ops.py:306-309), segment by segment: the statistics are per column, so
        each segment uses its columns of beta, gamma and the stored statistics.  `saved`: a list that receives
        (x, mean, invstd, column offset) per segment for the backward."""
        sc = "classifier/linearLayerfc_%d/BatchNorm/" % layer
        p, out, off = self.p, [], 0
        for x in xs:
            x = x.contiguous()
            B, w = x.shape
            cols = lambda n: p[sc + n][off:off + w]
            y = self._new(B, w)
            mean, invstd = (self._new(w), self._new(w)) if saved is not None else (None, None)
            check(self.lib.mac_batchnorm_fwd(ptr(x), ptr(cols("gamma")), ptr(cols("beta")), ptr(cols("moving_mean")),
                                             ptr(cols("moving_variance")), self.bn_decay, BN_EPS, int(train), ptr(y),
                                             ptr(mean), ptr(invstd), B, w, stream_ptr()), "mac_batchnorm_fwd")
            if saved is not None:
                saved.append((x, mean, invstd, off))
            out.append(y)
            off += w
        return out

    def forward(self, memory, vecQuestions, answers, step=0, loss_scale=None, train=True):
        """Returns (logits, losses [B], dlogits [B, A]) -- dlogits = (softmax - onehot) * loss_scale (default 1/B).  The three
        stay reachable as `last_logits`, `losses` and `dlogits` (`logits` is the label-free method).  `train`: the batch
        norm's mode (see `forward_logits`)."""
        B = memory.shape[0]
        self.forward_logits(memory, vecQuestions, step, train=train)
        A = self.last_logits.shape[1]
        self.losses = self._new(B)
        self.dlogits = self._new(B, A)
        scale = (1.0 / B) if loss_scale is None else float(loss_scale)
        check(self.lib.mac_softmax_xent(ptr(self.last_logits), ptr(answers), ptr(self.losses), ptr(self.dlogits), scale, B, A,
                                        stream_ptr()), "mac_softmax_xent")
        return self.last_logits, self.losses, self.dlogits

    def forward_logits(self, memory, vecQuestions, step=0, train=True):
        """The training forward up to the logits (this unit's dropouts, its inputs kept for `backward`), without the loss:
        `backward(dlogits=)` then takes the gradient of the logits from the caller.  Returns the logits [B, A].
        With bn, `train=True` normalises with the batch statistics and moves the stored ones in place (is_training), and
        `train=False` normalises with the stored statistics; the backward follows the same mode."""
        self._check_memory(memory)
        act = act_code("RELU", self.relu)
        self.memory, self.vecq, self.step, self.train = memory, vecQuestions, step, bool(train)
        feats = self._features(memory, vecQuestions)
        self.eq = feats[1] if self.question else None
        self.widths = [f.shape[1] for f in feats]
        self.inputs = []            # per layer: list of input segments after batch norm and dropout
        self.bn_saved = []          # per layer (bn): list of (input, mean, invstd, offset) per segment
        xs, x = feats, None
        for i in range(self.nfc):
            W = self.p["classifier/linearLayerfc_%d/weights/weight" % i]
            b = self.p["classifier/linearLayerfc_%d/biases/bias" % i]
            if i > 0:
                xs = [x]
            if self.bn:
                saved = []
                xs = self._batch_norm(xs, i, self.train, saved)
                self.bn_saved.append(saved)
            if self.keep < 1.0:
                # dropout over the concatenated features: one Philox stream over [B, F], the flat mask index of [B, F]
                xs = [self._dropout(torch.cat(xs, dim=1) if len(xs) > 1 else xs[0], i, step)]   # plumbing: layout
            self.inputs.append(xs)
            x = self._linear(xs, W, b, act if i < self.nfc - 1 else 0)
            if i < self.nfc - 1:
                setattr(self, "_h%d" % i, x)
        self.last_logits = x
        return x

    def logits(self, memory, vecQuestions, train=False):
        """The answer logits [B, A] without labels: the linears of `forward` with every dropout at 1, no loss, no `dlogits`,
        nothing kept for a backward (capturable in a CUDA graph).  The batch norm normalises with its stored statistics, or
        with `train=True` with the batch's, moving the stored ones.  Bit for bit `forward(..., train=train)[0]` of a unit
        with keep = 1."""
        self._check_memory(memory)
        act = act_code("RELU", self.relu)
        xs = self._features(memory, vecQuestions)
        for i in range(self.nfc):
            if self.bn:
                xs = self._batch_norm(xs, i, train)
            xs = [self._linear(xs, self.p["classifier/linearLayerfc_%d/weights/weight" % i],
                               self.p["classifier/linearLayerfc_%d/biases/bias" % i], act if i < self.nfc - 1 else 0)]
        return xs[0]

    def backward(self, grads, d_memory, d_vecq, dlogits=None):
        """Accumulates parameter gradients into `grads` (dict name -> tensor) and ADDS dL/dmemory, dL/dvecQuestions
        (`d_vecq` is untouched without the question).  `dlogits`: the gradient of the logits [B, A]; by default the loss's,
        `self.dlogits`, from `forward`.  The stored batch-norm statistics get no gradient."""
        B = self.memory.shape[0]
        dy = self.dlogits if dlogits is None else dlogits
        act = act_code("RELU", self.relu)

        def lin_bwd(xs, wname, bname, dy, dxs, accum):
            _lib.linear_bwd(xs, self._cache.pack(packs.transposed, self.p[wname]), dy, dxs, accum, grads[wname],
                            grads[bname], self.lws, self.lws_bytes, stream_ptr())
        for i in reversed(range(self.nfc)):
            xs = self.inputs[i]
            wn, bn = "classifier/linearLayerfc_%d/weights/weight" % i, "classifier/linearLayerfc_%d/biases/bias" % i
            dxs = [self._new(B, x.shape[1]) for x in xs]
            lin_bwd(xs, wn, bn, dy, dxs, [0] * len(xs))
            if self.keep < 1.0:           # through the input dropout of this layer (one segment)
                check(self.lib.mac_dropout_fwd(ptr(dxs[0]), self.keep, self.seed, SITE_OUTPUT + i, self.step, ptr(dxs[0]),
                                               dxs[0].numel(), stream_ptr()), "dropout bwd")
            widths = self.widths if i == 0 else [dxs[0].shape[1]]
            if len(dxs) != len(widths):   # the dropout's concatenation, split back into the features' segments
                offs = np.cumsum([0] + widths)
                dxs = [dxs[0][:, offs[k]:offs[k + 1]].contiguous() for k in range(len(widths))]
            if self.bn:
                dxs = self._batch_norm_bwd(grads, i, dxs)
            if i > 0:
                h = getattr(self, "_h%d" % (i - 1))
                dpre = self._new(*h.shape)
                check(self.lib.mac_activation_bwd(ptr(h), ptr(dxs[0]), act, ptr(dpre), h.numel(), stream_ptr()), "act bwd")
                dy = dpre
        dfeats = dxs
        if self.mul:                      # memory * q': d_memory += g * q', dq' += g * memory
            check(self.lib.mac_bcast_op_bwd(ptr(self.memory), ptr(self.eq), None, ptr(dfeats[2]), 0, 0.0, ptr(d_memory),
                                            ptr(dfeats[1]), None, B, 1, self.memory.shape[1], stream_ptr()),
                  "mac_bcast_op_bwd")
        check(self.lib.mac_axpy(ptr(d_memory), ptr(dfeats[0]), 1.0, dfeats[0].numel(), stream_ptr()), "axpy")
        if self.question:
            lin_bwd([self.vecq], "outputUnit/linearLayeroutQuestion/weights/weight",
                    "outputUnit/linearLayeroutQuestion/biases/bias", dfeats[1], [d_vecq], [1])

    def _batch_norm_bwd(self, grads, layer, dys):
        """Gradients of the segments' batch-norm inputs from those of their outputs; dgamma, dbeta into `grads`."""
        sc = "classifier/linearLayerfc_%d/BatchNorm/" % layer
        out = []
        for (x, mean, invstd, off), dy in zip(self.bn_saved[layer], dys):
            B, w = x.shape
            dx = torch.zeros_like(x)
            check(self.lib.mac_batchnorm_bwd(ptr(x), ptr(self.p[sc + "gamma"][off:off + w]), ptr(mean), ptr(invstd), ptr(dy),
                                             int(self.train), ptr(dx), ptr(grads[sc + "gamma"][off:off + w]),
                                             ptr(grads[sc + "beta"][off:off + w]), B, w, stream_ptr()), "mac_batchnorm_bwd")
            out.append(dx)
        return out
