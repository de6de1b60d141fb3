"""`torch.nn` modules over the sm_90a kernels: the MAC network, its question encoder, image stem and output unit, and the
whole model, trained through `torch.autograd` -- `loss.backward()`, extra loss terms, torch layers around them, `torch.optim`.

Each unit's forward and backward are the library's kernels, as `DPTrainer` runs them; torch only allocates, views and routes
gradients.  The boundary with autograd is one `torch.autograd.Function` per unit (`_CellFunction`, `_EncoderFunction`,
`_StemFunction`, `_OutputFunction`, `_LossFunction`):

  * forward runs the unit's training forward and keeps what its backward reads -- a shallow copy of the unit object (the
    encoder, stem and output unit keep one forward's activations on themselves), or the cell itself -- in the Function's
    `ctx`, so two forwards before their backwards each differentiate their own activations.  The backward consumes that
    state: a second backward through the same graph raises, and so does `create_graph=True`.
  * every parameter is an `nn.Parameter` view into one flat fp32 buffer laid out like `MACParams.flat`, named by the
    reference's TF variable name.  The views share the buffer's version counter, so an in-place update by anyone
    (`optimizer.step()`, `load_state_dict`, `copy_`) moves `flat._version`; the next forward then calls `touch()`, which
    drops every weight-derived tensor (bf16 / split / e4m3 packs, transposes, the cached scalar logit biases).
  * parameter gradients come back as views of a flat buffer allocated, zeroed, for each training forward and shared by
    the Functions of that forward (so `.grad` never aliases a buffer that a later step writes again).
  * `train()` with something requiring grad runs the training forms with the reference's training dropouts, drawing one
    Philox seed per forward from `seed` and the module's `step`, the stream `DPTrainer` draws; `eval()`, `torch.no_grad()`
    or nothing requiring grad runs the inference forms (hoisted read, fused read step, folded write, `eval_prec="fp8"`)
    and saves nothing.
"""
import collections
import copy

import numpy as np
import torch
from torch import nn

from . import _lib
from ._lib import check, ptr, stream_ptr
from .autograd import check_backward, mac_backward
from .encoder import QuestionEncoder as _Encoder, encoder_specs, init_encoder_params
from .mac_cell import MACCell, MACParams, flat_layout, mac_network, views_of
from .output_unit import OutputUnit as _Output, init_output_params, is_moving_stat, output_specs
from .params import param_specs
from .stem import Stem, init_stem_params, stem_specs

ENCODER_KEEP = (0.85, 0.92)      # the reference's training dropouts (config.py:202-206), as DPTrainer's defaults
STEM_KEEP = 0.82
OUTPUT_KEEP = 0.85


def _seed(base, step):
    """The Philox seed of one training forward: DPTrainer's per-step stream (of rank 0)."""
    return (int(base) * 1000003 + int(step) * 7919 + 1) & 0x7FFFFFFFFFFFFFFF


class _Params(object):
    """The variables of `specs` as views into one flat fp32 buffer in `MACParams`' layout, with its version counter."""

    def __init__(self, specs, values, device):
        self.specs, self.offsets = specs, flat_layout(specs)
        self.flat = torch.zeros(self.offsets["__total__"], dtype=torch.float32, device=device)
        self.t = views_of(self.flat, specs, self.offsets)
        for name, view in self.t.items():
            view.copy_(torch.from_numpy(np.ascontiguousarray(values[name], dtype=np.float32)).reshape(view.shape))
        self.version = 0

    def touch(self):
        self.version += 1


# ------------------------------------------------------------------------------------------------ the autograd boundary
class _KernelFunction(torch.autograd.Function):
    """apply(op, *tensors): `op.forward(*tensors)` runs the unit's forward and returns (outputs, state, non-differentiable
    outputs); `op.backward(state, *output grads)` runs its backward and returns one gradient (or None) per tensor.  The
    state lives in ctx until the one backward that consumes it."""

    @staticmethod
    def forward(ctx, op, *tensors):
        ctx.set_materialize_grads(False)
        outs, state, nondiff = op.forward(*tensors)
        ctx.op, ctx.state, ctx.version = op, state, op.flat._version
        if nondiff:
            ctx.mark_non_differentiable(*nondiff)
        return outs

    @staticmethod
    def backward(ctx, *grads):
        name = type(ctx.op).__name__[1:-2]          # _CellOp -> Cell
        if torch.is_grad_enabled():
            raise RuntimeError("%s has no double backward (create_graph=True): its backward is the library's kernels"
                               % name)
        if ctx.state is None:
            raise RuntimeError("%s: backward through this graph has already run and freed the saved activations; run the "
                               "forward again (retain_graph cannot keep them)" % name)
        if ctx.op.flat._version != ctx.version:
            raise RuntimeError("%s: the parameters were modified in place between this forward and its backward" % name)
        state, ctx.state = ctx.state, None
        return (None,) + tuple(ctx.op.backward(state, *grads))


class _CellFunction(_KernelFunction):
    pass


class _EncoderFunction(_KernelFunction):
    pass


class _StemFunction(_KernelFunction):
    pass


class _OutputFunction(_KernelFunction):
    pass


class _LossFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, answers, global_batch):
        lib = _lib.load()
        B, A = logits.shape
        losses = torch.empty(B, dtype=torch.float32, device=logits.device)
        dlogits = torch.empty((B, A), dtype=torch.float32, device=logits.device)
        check(lib.mac_softmax_xent(ptr(logits), ptr(answers), ptr(losses), ptr(dlogits), 1.0 / global_batch, B, A,
                                   stream_ptr()), "mac_softmax_xent")
        total = torch.empty(1, dtype=torch.float32, device=logits.device)
        check(lib.mac_colsum(ptr(losses), ptr(total), 1, B, 1, 0, stream_ptr()), "mac_colsum")
        loss = torch.zeros((), dtype=torch.float32, device=logits.device)
        check(lib.mac_axpy(ptr(loss), ptr(total), 1.0 / global_batch, 1, stream_ptr()), "mac_axpy")
        ctx.dlogits = dlogits
        return loss

    @staticmethod
    def backward(ctx, g):
        if torch.is_grad_enabled():
            raise RuntimeError("answer_loss has no double backward (create_graph=True)")
        if ctx.dlogits is None:
            raise RuntimeError("answer_loss: backward through this graph has already run; run the forward again")
        dlogits, ctx.dlogits = ctx.dlogits, None
        B, A = dlogits.shape
        out = torch.empty_like(dlogits)
        # dlogits * g, g the incoming scalar on the device: mac_bcast_op's MUL with one row of one column
        check(_lib.load().mac_bcast_op(ptr(dlogits), ptr(g.contiguous()), 0, 0.0, None, ptr(out), 1, B * A, 1,
                                       stream_ptr()), "mac_bcast_op")
        return out, None, None


def answer_loss(logits, answers, global_batch=None):
    """The reference's answer loss (model.py:593-596): sum_b softmax-CE(logits[b], answers[b]) / global_batch (default B),
    a 0-d tensor, on `mac_softmax_xent`; its backward is the kernel's dlogits times the incoming gradient.  `answers`:
    contiguous int32 [B] on the logits' device."""
    if not (answers.dtype == torch.int32 and answers.is_contiguous() and answers.shape == logits.shape[:1]):
        raise ValueError("answers must be a contiguous int32 tensor of shape [%d]" % logits.shape[0])
    if not (logits.dtype == torch.float32 and logits.dim() == 2):
        raise ValueError("logits must be an fp32 [B, A] tensor")
    G = logits.shape[0] if global_batch is None else int(global_batch)
    return _LossFunction.apply(logits.contiguous(), answers, float(G))


# ------------------------------------------------------------------------------------------------ one unit's forward/backward
class _Op(object):
    """One call of a unit: its engine, the parameter names it differentiates, the gradient views of this forward."""

    def __init__(self, unit, flat, names, grads, seed, step):
        self.unit, self.flat, self.names, self.grads, self.seed, self.step = unit, flat, names, grads, seed, step

    def param_grads(self):
        """Fresh views of this forward's gradient buffer, referenced nowhere else, so that AccumulateGrad keeps them as
        `.grad` instead of copying them."""
        bucket, g = self.grads["__bucket__"], self.grads
        return tuple(bucket[g[n].storage_offset():g[n].storage_offset() + g[n].numel()].view(g[n].shape) for n in self.names)


class _EncoderOp(_Op):
    def forward(self, questions, lengths, *params):
        self.unit.seed = self.seed
        words, cntx, vecq = self.unit.forward(questions, lengths, step=self.step, save_for_backward=True)
        return (words, cntx, vecq), copy.copy(self.unit), (words,)

    def backward(self, unit, _, d_cntx, d_vecq):
        sv = unit._saved
        if d_cntx is None:
            d_cntx = torch.zeros_like(sv["cntx"])
        if d_vecq is None:
            d_vecq = torch.zeros_like(sv["vecq"])
        unit.backward(d_cntx, d_vecq, self.grads)
        return (None, None) + self.param_grads()


class _StemOp(_Op):
    def __init__(self, unit, flat, names, grads, seed, step, keep, nchw):
        _Op.__init__(self, unit, flat, names, grads, seed, step)
        self.keep, self.nchw = keep, nchw

    def forward(self, images, *params):
        self.unit.seed = self.seed
        fwd = self.unit.forward_nchw if self.nchw else self.unit.forward
        kb = fwd(images, keep=self.keep, step=self.step, save_for_backward=True)
        return kb, (copy.copy(self.unit), images.requires_grad), ()

    def backward(self, state, d_kb):
        unit, need_d_images = state
        if d_kb is None:
            return (None,) + self.param_grads()
        dx = unit.backward(d_kb, self.grads, need_d_images=need_d_images)
        if dx is not None and self.nchw:
            dx = dx.permute(0, 3, 1, 2)
        return (dx,) + self.param_grads()


class _OutputOp(_Op):
    def forward(self, memory, vecq, *params):
        self.unit.seed = self.seed
        logits = self.unit.forward_logits(memory, vecq, step=self.step)
        return logits, copy.copy(self.unit), ()

    def backward(self, unit, d_logits):
        d_mem = torch.zeros_like(unit.memory)
        d_vecq = torch.zeros_like(unit.vecq)
        if d_logits is not None:
            unit.backward(self.grads, d_mem, d_vecq, dlogits=d_logits.contiguous())
        return (d_mem, d_vecq) + self.param_grads()


class _CellOp(_Op):
    """The cell's training call.  Outputs (control, memory, vecQuestions): the third is the input itself, handed on so that a
    consumer of the question vector after the cell (the output unit) sends its gradient into the cell's backward as
    `d_vecq`, as DPTrainer does, instead of autograd adding the two gradients."""

    def __init__(self, cells, flat, names, grads, seed, key, cell, kbIndex):
        _Op.__init__(self, cells, flat, names, grads, seed, 0)
        self.key, self.cell, self.kbIndex = key, cell, kbIndex

    def forward(self, vecq, words, cntx, lengths, kb, *params):
        cells, cell = self.unit, self.cell
        if self.kbIndex is not None:   # DPTrainer._gather_kb: each question's knowledge base into the cell's fp32 input
            self.U = kb.shape[0]
            kb_q = cell.knowledgeBase
            check(cells.lib.mac_kb_gather(ptr(kb), ptr(self.kbIndex), ptr(kb_q), 0, cell.B, self.U, cell.N, cell.d,
                                          stream_ptr()), "mac_kb_gather")
            kb = kb_q
        cells.bind(cell, vecq, words, cntx, lengths, kb)
        cell.seed = self.seed
        control, memory = mac_network(cell, cell.L)
        cells.attentions = {k: list(v) for k, v in cell.attentions.items()}
        return (control, memory, vecq), cell, ()

    def backward(self, cell, d_control, d_memory, d_vecq):
        cells = self.unit
        g = mac_backward(cell, d_control, d_memory, bucket=self.grads["__bucket__"], zero_bucket=False, d_vecq=d_vecq,
                         tc=cells.bwd_tc)
        d_kb = g["knowledgeBase"]
        if self.kbIndex is not None:   # DPTrainer._sum_kb_grad: each image's gradient summed over its questions
            d_u = torch.empty((self.U, cell.N, cell.d), dtype=torch.float32, device=cell.device)
            check(cells.lib.mac_kb_gather_bwd(ptr(d_kb.contiguous()), ptr(self.kbIndex), ptr(d_u), cell.B, self.U, cell.N,
                                              cell.d, stream_ptr()), "mac_kb_gather_bwd")
            d_kb = d_u
        cells.release(self.key, cell)
        return (g["vecQuestions"], g.get("questionWords"), g.get("questionCntxWords"), None, d_kb) + self.param_grads()


class _Cells(object):
    """The MAC cells of one parameter set: built over placeholder inputs (so a cell refuses its configuration before anything
    runs), bound to each call's tensors, and reused -- one idle cell per input shape and form, at most MAX_KEYS shapes
    (each idle training cell keeps its last forward's activations, as DPTrainer's cached cells do)."""
    MAX_KEYS = 4

    def __init__(self, cfg, L, params, prec, bwd_tc, eval_prec, dropouts):
        self.cfg, self.L, self.params = cfg, L, params
        self.prec, self.bwd_tc, self.eval_prec = prec, bool(bwd_tc), eval_prec or prec
        self.dropouts = tuple(float(k) for k in dropouts)
        self.lib = _lib.load()
        self._idle = collections.OrderedDict()
        self.attentions = None

    def acquire(self, train, B, S, E, N, U=None):
        """(key, cell) for `B` questions of `S` words (E-wide word vectors) over knowledge bases of N rows; U: the distinct
        images an inference cell gathers from (MACCell(kbIndex=)).  Raises every refusal of the configuration here."""
        key = (bool(train), B, S, E, N, U)
        idle = self._idle.pop(key, None)
        if idle is not None:
            return key, idle
        d, dev = self.cfg.memDim, self.params.device
        e = lambda *shape: torch.empty(shape, dtype=torch.float32, device=dev)
        lengths = torch.ones(B, dtype=torch.int32, device=dev)
        kbIndex = torch.zeros(B, dtype=torch.int32, device=dev) if U is not None and not train else None
        keep = self.dropouts if train else (1.0, 1.0, 1.0)
        cell = MACCell(e(B, d), e(B, S, E), e(B, S, d), lengths, e(U if kbIndex is not None else B, N, d), keep[0], keep[1],
                       keep[2], B, bool(train), config=self.cfg, params=self.params,
                       prec=self.prec if train else self.eval_prec, save_for_backward=bool(train), kbIndex=kbIndex)
        if train:
            check_backward(cell, self.bwd_tc)
            if U is not None:
                if d % 8:
                    raise NotImplementedError("imageIndex needs memDim %% 8 == 0 (mac_kb_gather's 16-byte vectors), got %d"
                                              % d)
        return key, cell

    def release(self, key, cell):
        self._idle.pop(key, None)
        self._idle[key] = cell
        while len(self._idle) > self.MAX_KEYS:
            self._idle.popitem(last=False)

    @staticmethod
    def bind(cell, vecq, words, cntx, lengths, kb, kbIndex=None):
        cell.rebind(vecq, words, cntx, kb, kbIndex=kbIndex)
        cell.questionLengths = lengths

    def infer(self, vecq, words, cntx, lengths, kb, kbIndex):
        B, S, E = words.shape
        key, cell = self.acquire(False, B, S, E, kb.shape[1], None if kbIndex is None else kb.shape[0])
        self.bind(cell, vecq, words, cntx, lengths, kb, kbIndex)
        control, memory = mac_network(cell, self.L)
        self.attentions = {k: list(v) for k, v in cell.attentions.items()}
        self.release(key, cell)
        return control, memory


def _int32(t):
    return t.to(torch.int32).contiguous()


# ------------------------------------------------------------------------------------------------ modules
class _KernelModule(nn.Module):
    """Parameters as named views of one flat buffer (`params.flat`), the version refresh and the per-forward seed."""

    def _register(self, params, seed):
        self.params = params
        for name, view in params.t.items():     # scalars as the reference's 0-d variables (the kernels' views are [1])
            if is_moving_stat(name):            # the classifier's stored batch-norm statistics: state, not parameters
                self.register_buffer(name, view.view(params.specs[name][0]))
            else:
                self.register_parameter(name, nn.Parameter(view.view(params.specs[name][0])))
        self._seen = params.flat._version
        self.seed, self.step = int(seed), 0

    def _refresh(self):
        """After an in-place update of the values (anyone's), drop every tensor derived from the old ones."""
        v = self.params.flat._version
        if v != self._seen:
            self.params.touch()
            self._seen = v

    def _trains(self, *inputs):
        """The training form: train mode, grad mode on, and a parameter or an input that requires grad."""
        if not (self.training and torch.is_grad_enabled()):
            return False
        return (any(t is not None and t.requires_grad for t in inputs)
                or any(p.requires_grad for p in self._parameters.values()))

    def _next(self):
        """(seed, step) of this training forward; advances the step."""
        step = self.step
        self.step += 1
        return _seed(self.seed, step), step

    def _grads(self):
        bucket = torch.zeros_like(self.params.flat)
        specs = self.params.specs
        g = {n: v.view(specs[n][0]) for n, v in views_of(bucket, specs, self.params.offsets).items()}
        g["__bucket__"] = bucket
        return g

    def _plist(self, names):
        return [self._parameters[n] for n in names]


class MACNetwork(_KernelModule):
    """The MAC cell unrolled `netLength` steps (`MACnet.MACnetwork`, model.py:447-458).  `prec`: the training cell's
    arithmetic ("fp32", "bf16", "tc32"), `bwd_tc`: the read unit's backward products on tensor cores (`mac_backward(tc=)`),
    `eval_prec`: the inference cell's (default `prec`; "fp8" is inference only), `values`: name -> array (default
    `init_params(cfg, netLength, seed)`).  Training draws the cell's dropouts from `cfg`."""

    def __init__(self, cfg, netLength, prec="fp32", bwd_tc=False, eval_prec=None, values=None, seed=0, device="cuda"):
        super(MACNetwork, self).__init__()
        self.cfg, self.L = cfg, netLength
        self._register(MACParams(cfg, netLength, values=values, seed=seed, device=device), seed)
        self.cells = _Cells(cfg, netLength, self.params, prec, bwd_tc, eval_prec,
                            (cfg.memoryDropout, cfg.readDropout, cfg.writeDropout))
        self._names = list(self.params.specs)

    @property
    def attentions(self):
        """The last forward's attention maps, {"kb" | "question" | "self" | "gate": [per step]}, not differentiable."""
        return self.cells.attentions

    def forward(self, vecQuestions, questionWords, questionCntxWords, questionLengths, knowledgeBase, kbIndex=None):
        """fp32 CUDA inputs as `MACCell` takes them; `kbIndex` (int32 [B]): knowledgeBase holds U distinct images' [U, N, d]
        and question b reads image kbIndex[b].  Returns (control, memory) [B, d] after the last step."""
        self._refresh()
        vecq, words, cntx = (t.contiguous() for t in (vecQuestions, questionWords, questionCntxWords))
        kb, lengths = knowledgeBase.contiguous(), _int32(questionLengths)
        if not self._trains(vecq, words, cntx, kb):
            return self.cells.infer(vecq, words, cntx, lengths, kb, kbIndex)
        B, S, E = words.shape
        key, cell = self.cells.acquire(True, B, S, E, kb.shape[1], None if kbIndex is None else kb.shape[0])
        if kbIndex is not None:
            cell._check_kb_index(kbIndex, B, cell.device)
        seed, _ = self._next()
        op = _CellOp(self.cells, self.params.flat, self._names, self._grads(), seed, key, cell, kbIndex)
        control, memory, _ = _CellFunction.apply(op, vecq, words, cntx, lengths, kb, *self._plist(self._names))
        return control, memory


class QuestionEncoder(_KernelModule):
    """The question input unit (embeddings + bi-LSTM, model.py:208-220, 279-307): `forward(questions, questionLengths)` ->
    (questionWords, questionCntxWords, vecQuestions); questionWords is not differentiable (the embeddings get their
    gradient through the LSTM).  `prec="bf16"`: the LSTM on tensor cores (encDim 512)."""

    def __init__(self, vocab, wrd_emb_dim, enc_dim, prec="fp32", values=None, seed=0, device="cuda"):
        super(QuestionEncoder, self).__init__()
        specs = encoder_specs(vocab, wrd_emb_dim, enc_dim, ctrl_dim=enc_dim, bi=True)
        values = values if values is not None else init_encoder_params(specs, seed=seed + 19, bias_scale=0.0)
        self._register(_Params(specs, values, device), seed)
        self._enc = _encoder_units(self.params, prec)
        self._enc_names = list(specs)

    def forward(self, questions, questionLengths):
        self._refresh()
        lengths = _int32(questionLengths)
        if not self._trains():
            return self._enc[1].forward(questions, lengths)
        return _encoder_fn(self, self._grads(), self._next(), questions, lengths)


def _encoder_units(params, prec, keep=ENCODER_KEEP):
    """(training unit, inference unit) over the encoder's views of `params`."""
    t = {k: params.t[k] for k in params.t if k.startswith(("qEmbeddings/", "encoder/"))}
    version = lambda: params.version
    return (_Encoder(t, keep_input=keep[0], keep_question=keep[1], prec=prec, version=version),
            _Encoder(t, prec=prec, version=version))


def _encoder_fn(mod, grads, seed_step, questions, lengths):
    op = _EncoderOp(mod._enc[0], mod.params.flat, mod._enc_names, grads, *seed_step)
    return _EncoderFunction.apply(op, questions, lengths, *mod._plist(mod._enc_names))


class ImageStem(_KernelModule):
    """The image stem (model.py:165-204): `forward(images=NHWC fp32)` or `forward(images_nchw=NCHW fp32 or fp16)` -> the
    knowledge base [B, Ho*Wo, out_dim] on the stem's output grid (`grid`).  The gradient w.r.t. the images is computed
    exactly when they require grad, and comes back in their dtype.  `prec`: "fp32", "bf16" or "bf16x3" (training and
    inference) or "fp8" (inference).  `ksizes`, `strides`, `linear`, `stem_dim`: the reference's --stemKernelSizes,
    --stemStrideSizes, --stemLinear and --stemDim; `location`: --locationAware as `Stem(location=)` takes it."""

    def __init__(self, in_dim, out_dim, num_layers=2, relu="ELU", prec="fp32", values=None, seed=0, device="cuda",
                 ksizes=None, strides=None, linear=False, stem_dim=None, location=None):
        super(ImageStem, self).__init__()
        specs = stem_specs(in_dim, out_dim, num_layers=num_layers, ksizes=ksizes, linear=linear, stem_dim=stem_dim,
                           location=location)
        values = values if values is not None else init_stem_params(specs, seed=seed + 23, bias_scale=0.0)
        self._register(_Params(specs, values, device), seed)
        self._stem = _stem_unit(self.params, relu, prec, {"strides": strides, "linear": linear, "location": location})
        self._stem_names, self.stem_keep = list(specs), STEM_KEEP

    def forward(self, images=None, images_nchw=None):
        self._refresh()
        x, nchw = _pick_images(images, images_nchw)
        if not self._trains(x):
            return self._stem.forward_nchw(x) if nchw else self._stem.forward(x)
        return _stem_fn(self, self._grads(), self._next(), x, nchw)


def _stem_unit(params, relu, prec, geometry):
    return Stem({k: params.t[k] for k in params.t if k.startswith("stem/")}, relu=relu, prec=prec,
                version=lambda: params.version, strides=geometry["strides"], linear=geometry["linear"],
                location=geometry["location"])


def _pick_images(images, images_nchw):
    if (images is None) == (images_nchw is None):
        raise ValueError("give exactly one of images (NHWC) and images_nchw")
    return (images, False) if images_nchw is None else (images_nchw, True)


def _stem_fn(mod, grads, seed_step, x, nchw):
    op = _StemOp(mod._stem, mod.params.flat, mod._stem_names, grads, seed_step[0], seed_step[1], mod.stem_keep, nchw)
    return _StemFunction.apply(op, x, *mod._plist(mod._stem_names))


class OutputUnit(_KernelModule):
    """The output unit and classifier (model.py:512-528, 547-576): `forward(memory, vecQuestions)` -> logits [B, A]; the
    loss is `answer_loss`.  `question`, `mul`, `bn`: --outQuestion, --outQuestionMul, --outputBN (`output_specs`); with
    `bn` the stored statistics are buffers (`moving_mean`, `moving_variance` under the reference's names), the batch
    normalisation follows `training` -- batch statistics and an in-place update of the stored ones in train mode, the
    stored statistics in eval mode -- and `bn_decay` is --bnDecay."""

    def __init__(self, ctrl_dim, mem_dim, hidden, n_answers, relu="ELU", values=None, seed=0, device="cuda",
                 question=True, mul=False, bn=False, bn_decay=0.999):
        super(OutputUnit, self).__init__()
        opts = {"question": question, "mul": mul, "bn": bn}
        specs = output_specs(ctrl_dim, mem_dim, list(hidden), n_answers, **opts)
        values = values if values is not None else init_output_params(specs, seed=seed + 17, bias_scale=0.0)
        self._register(_Params(specs, values, device), seed)
        self._out = _output_unit(self.params, relu, opts=opts, bn_decay=bn_decay)
        self._out_names = [k for k in specs if not is_moving_stat(k)]

    def forward(self, memory, vecQuestions):
        self._refresh()
        memory, vecq = memory.contiguous(), vecQuestions.contiguous()
        if not self._trains(memory, vecq):
            return self._out.logits(memory, vecq, train=self.training)
        return _output_fn(self, self._grads(), self._next(), memory, vecq)


def _output_unit(params, relu, keep=OUTPUT_KEEP, opts=None, bn_decay=0.999):
    return _Output({k: params.t[k] for k in params.t if k.startswith(("outputUnit/", "classifier/"))}, relu=relu,
                   keep=keep, version=lambda: params.version, bn_decay=bn_decay, **(opts or {}))


def _output_fn(mod, grads, seed_step, memory, vecq):
    op = _OutputOp(mod._out, mod.params.flat, mod._out_names, grads, *seed_step)
    return _OutputFunction.apply(op, memory, vecq, *mod._plist(mod._out_names))


class MACModel(_KernelModule):
    """The whole model as `MACnet` builds it (model.py:762-829): embeddings + bi-LSTM encoder -> stem -> netLength MAC steps ->
    output unit -> classifier.  Constructor arguments as `MACnet` / `DPTrainer`: `prec`, `bwd_tc` (the cell), `stem_prec`
    ("fp32", "bf16", "bf16x3"), `enc_prec` ("fp32", "bf16"), `eval_prec` (the inference cell, default `prec`; may be
    "fp8").  `values`: name -> array for every variable (default: `DPTrainer(seed=seed)`'s initial values).  A training
    forward runs exactly the launches of `DPTrainer.full_forward_backward`, and its backward gives the same gradients."""

    def __init__(self, cfg, netLength, vocab, n_answers, wrd_emb_dim=300, image_in_dim=1024, classifier_dims=(512,),
                 stem_layers=2, prec="fp32", bwd_tc=False, stem_prec="fp32", enc_prec="fp32", eval_prec=None, values=None,
                 seed=0, device="cuda", stem_geometry=None, out_question=True, out_question_mul=False, output_bn=False):
        super(MACModel, self).__init__()
        from .dp import check_model_precisions, model_parameters, stem_geometry as stem_geometry_of, stem_location
        if not cfg.controlContextual:
            raise NotImplementedError("the raw-word control inputs (controlContextual off) need wrdEmbDim == ctrlDim")
        encoder, stem = (vocab, wrd_emb_dim), (image_in_dim, stem_layers, stem_geometry)
        opts = {"question": out_question, "mul": out_question_mul, "bn": output_bn}
        check_model_precisions(cfg, encoder, stem, stem_prec, enc_prec)
        cell_values, extra_specs, extra_values, enc_specs, stem_specs_ = model_parameters(
            cfg, netLength, seed, (n_answers, list(classifier_dims), opts), encoder, stem, values)
        if values is not None:
            extra_values = {k: values[k] for k in extra_specs}
        self.cfg, self.L = cfg, netLength
        self._register(MACParams(cfg, netLength, values=cell_values, seed=seed, device=device, extra_specs=extra_specs,
                                 extra_values=extra_values), seed)
        self._cell_names = list(param_specs(cfg, netLength))
        self._enc_names, self._stem_names = list(enc_specs), list(stem_specs_)
        self._out_names = [k for k in extra_specs if k.startswith(("outputUnit/", "classifier/")) and not is_moving_stat(k)]
        self._enc = _encoder_units(self.params, enc_prec)
        geom = stem_geometry_of(stem)
        self._stem = _stem_unit(self.params, cfg.relu, stem_prec, dict(geom, location=stem_location(geom)))
        self._out = _output_unit(self.params, cfg.relu, opts=opts, bn_decay=cfg.bnDecay)
        self.stem_keep = STEM_KEEP
        self.cells = _Cells(cfg, netLength, self.params, prec, bwd_tc, eval_prec,
                            (cfg.memoryDropout, cfg.readDropout, cfg.writeDropout))

    @classmethod
    def from_trainer(cls, trainer, eval_prec=None):
        """A model over a copy of a full-model `DPTrainer`'s current values, with its precisions, dropouts, seed and step:
        its next training forward and backward are the trainer's next `full_forward_backward` (of rank 0)."""
        t = trainer
        if t.enc is None:
            raise ValueError("from_trainer needs a trainer built with classifier=, encoder= and stem=")
        specs = t.params.specs
        vocab, E = specs["qEmbeddings/emb"][0]
        fcs = [specs[k][0] for k in specs if k.startswith("classifier/") and k.endswith("weights/weight")]
        values = {k: v.reshape(specs[k][0]) for k, v in t.params.numpy().items()}
        m = cls(t.cfg, t.L, vocab, fcs[-1][1], wrd_emb_dim=E, image_in_dim=t.stem.in_dim,
                classifier_dims=[s[1] for s in fcs[:-1]], stem_layers=t.stem.nlayers, prec=t.prec, bwd_tc=t.bwd_tc,
                stem_prec=t.stem_prec, enc_prec=t.enc_prec, eval_prec=eval_prec, values=values, seed=t.base_seed,
                device=t.params.device, stem_geometry=t.stem_geometry, out_question=t.out.options["question"],
                out_question_mul=t.out.options["mul"], output_bn=t.out.options["bn"])
        m.step = t.step_id
        m.cells.dropouts = tuple(float(k) for k in t.dropouts)
        m._enc[0].keep_input, m._enc[0].keep_question = t.enc.keep_input, t.enc.keep_question
        m.stem_keep, m._out.keep = t.stem_dropout, t.out.keep
        return m

    @property
    def attentions(self):
        """The cell's attention maps of the last forward (see `MACNetwork.attentions`)."""
        return self.cells.attentions

    def forward(self, questions, questionLengths, images=None, images_nchw=None, imageIndex=None):
        """questions int32 [B, S] (0 = padding), questionLengths [B], and the images as exactly one of `images` fp32 NHWC
        [k, H, W, C] or `images_nchw` fp32 or fp16 NCHW [k, C, H, W]; k = B, or with `imageIndex` (int32 [B]) k distinct
        images of which question b asks about imageIndex[b] (the stem runs once per image).  fp16 features are widened on the
        device (`Stem.forward_nchw`): everything equals the forward and backward of `images_nchw.float()` bit for bit, except
        that when the images require grad their gradient comes back in their dtype, fp16, as autograd returns the gradient of
        any input.  Returns (logits [B, A], memory [B, d])."""
        self._refresh()
        x, nchw = _pick_images(images, images_nchw)
        lengths = _int32(questionLengths)
        B, S = questions.shape
        Ho, Wo = self._stem.grid(*(x.shape[2:4] if nchw else x.shape[1:3]))
        N = Ho * Wo
        U = None if imageIndex is None else x.shape[0]
        if not self._trains(x):
            words, cntx, vecq = self._enc[1].forward(questions, lengths)
            kb = self._stem.forward_nchw(x) if nchw else self._stem.forward(x)
            _, memory = self.cells.infer(vecq, words, cntx, lengths, kb, imageIndex)
            return self._out.logits(memory, vecq, train=self.training), memory
        # the training cell first: every refusal of the configuration comes before the first launch
        key, cell = self.cells.acquire(True, B, S, self._enc[0].E, N, U)
        if imageIndex is not None:
            cell._check_kb_index(imageIndex, B, cell.device)
        seed_step = self._next()
        grads = self._grads()          # one flat gradient buffer for every Function of this forward
        words, cntx, vecq = _encoder_fn(self, grads, seed_step, questions, lengths)
        kb = _stem_fn(self, grads, seed_step, x, nchw)
        op = _CellOp(self.cells, self.params.flat, self._cell_names, grads, seed_step[0], key, cell, imageIndex)
        _, memory, vecq = _CellFunction.apply(op, vecq, words, cntx, lengths, kb, *self._plist(self._cell_names))
        return _output_fn(self, grads, seed_step, memory, vecq), memory
