"""Host-side mirror of the reference's MAC cell over the sm_90a kernels in libmac_b200.so.

Same call surface as `/root/reference/mac_cell.py`:

    cell = MACCell(vecQuestions, questionWords, questionCntxWords, questionLengths, knowledgeBase,
                   memoryDropout, readDropout, writeDropout, batchSize, train, reuse=None)   # mac_cell.py:59-61
    state = cell.zero_state(batchSize)                                                      # mac_cell.py:539-592
    for i in range(config.netLength):                                                       # model.py:453-458
        cell.iteration = i
        _, state = cell(none, state)                                                        # mac_cell.py:420-480
    cell.attentions["kb" | "question" | "self" | "gate"][step]                              # model.py:740

plus the three units with the reference signatures (`control` 133-187, `read` 209-277, `write`
305-375).  Differences that the PyTorch/CUDA setting forces (SURVEY.md section 8(b)):
  * the reference reads a module-global `config` and pulls weights out of TF variable scopes; here
    they are the keyword-only arguments `config=` (a `MACConfig`) and `params=` (a `MACParams`, keyed by
    the reference's variable names), defaulting to the module globals set with `set_defaults`.
  * tensors are CUDA float32 `torch.Tensor`s; every arithmetic op is a kernel of libmac_b200.so --
    there is no PyTorch/CPU fallback, and a missing library raises at construction.
"""
import collections
import ctypes

import numpy as np
import torch

from . import _lib, packs
from ._lib import PREC, ReadWeights, act_code, check, ptr, segments, stream_ptr
from .config import MACConfig
from .params import PREFIX, init_params, param_specs

MACCellTuple = collections.namedtuple("MACCellTuple", ("control", "memory"))   # mac_cell.py:8

_defaults = {"config": None, "params": None}


def set_defaults(config=None, params=None):
    """The analogue of the reference's global `config` (config.py:92) and of the enclosing variable scope."""
    if config is not None:
        _defaults["config"] = config
    if params is not None:
        _defaults["params"] = params


def flat_layout(specs):
    """name -> element offset of each variable in the flat parameter / gradient bucket (+ "__total__")."""
    off, out = 0, {}
    for name, (shape, _) in specs.items():
        out[name] = off
        n = int(np.prod(shape)) if shape else 1
        off += (n + 63) // 64 * 64
    out["__total__"] = off
    return out


def views_of(flat, specs, offsets):
    """Per-variable views into a flat buffer laid out by `flat_layout`."""
    out = collections.OrderedDict()
    for name, (shape, _) in specs.items():
        n = int(np.prod(shape)) if shape else 1
        out[name] = flat[offsets[name]:offsets[name] + n].view(shape if shape else (1,))
    return out


class MACParams(object):
    """Cell parameters on the device, keyed by the reference's TF variable names (SURVEY Appendix B)."""

    def __init__(self, cfg, netLength=None, values=None, seed=0, device="cuda", extra_specs=None, extra_values=None):
        self.cfg = cfg
        self.L = cfg.netLength if netLength is None else netLength
        self.specs = param_specs(cfg, self.L)
        if values is None:
            values = init_params(cfg, self.L, seed=seed)
        if extra_specs:            # e.g. the output unit's variables: same flat bucket, same optimizer step
            self.specs = collections.OrderedDict(list(self.specs.items()) + list(extra_specs.items()))
            values = dict(values)
            values.update(extra_values)
        missing = set(self.specs) - set(values)
        if missing:
            raise KeyError("missing parameters: %s" % sorted(missing)[:4])
        self.device = torch.device(device)
        # ONE flat fp32 buffer (the layout of the data-parallel gradient bucket and of the fused optimizer step);
        # every variable is a view into it, offsets padded to 64 elements so rows stay 256-byte aligned
        self.offsets = flat_layout(self.specs)
        self.numel = self.offsets["__total__"]
        self.flat = torch.zeros(self.numel, dtype=torch.float32, device=self.device)
        self.t = collections.OrderedDict()
        for name, (shape, _) in self.specs.items():
            v = np.asarray(values[name], dtype=np.float32)
            assert tuple(v.shape) == tuple(shape), (name, v.shape, shape)
            view = self.flat[self.offsets[name]:self.offsets[name] + max(1, v.size)].view(shape if shape else (1,))
            view.copy_(torch.from_numpy(np.ascontiguousarray(v).reshape(view.shape)))
            self.t[name] = view
        self.version = 0
        self.cache = packs.Cache()          # weight-derived tensors of this version: packs, transposes, folded weights

    def __getitem__(self, name):
        return self.t[PREFIX + name]

    def has(self, name):
        return (PREFIX + name) in self.t

    def lin(self, scope, name):
        sc = scope + "linearLayer" + name + "/"
        return self[sc + "weights/weight"], self[sc + "biases/bias"]

    def numpy(self):
        return collections.OrderedDict((k, v.detach().cpu().numpy()) for k, v in self.t.items())

    def touch(self):
        """Call after updating parameter values in place (optimizer step, checkpoint restore): moves `version` and drops
        every weight-derived tensor."""
        self.version += 1
        self.cache.clear()

    def scalar(self, name):
        """0-d bias of an outDim == 1 linear (ops.py:304-305) as a python float (read once, cached)."""
        return self.cache.get(("scalar", name), lambda: float(self[name].item()))

    def q_input_cat(self):
        """([d, L*d], [L*d]): the per-step qInput{i} weights and biases side by side (controlInputUnshared), so that the
        control inputs of all steps are one product."""
        def build():
            Ws = [self.lin("MACCell/", "qInput%d" % i) for i in range(self.L)]
            return torch.cat([w for w, _ in Ws], dim=1).contiguous(), torch.cat([b for _, b in Ws]).contiguous()
        return self.cache.get("qInputCat", build)


class _Workspaces(object):
    """Device scratch, allocated once per (B, N, d, precision); the first 4 KB of each stays zero (split-K counters)."""

    def __init__(self, lib, B, N, d, prec, device):
        self.read_bytes = int(lib.mac_read_workspace_bytes(B, N, d, prec))
        self.write_bytes = int(lib.mac_write_workspace_bytes(B, d))
        self.lin_bytes = int(lib.mac_linear_workspace_bytes(max(B, 64), 3 * d, max(d, 64) * 16))
        self.read = torch.zeros(self.read_bytes, dtype=torch.uint8, device=device)
        self.write = torch.zeros(self.write_bytes, dtype=torch.uint8, device=device)
        self.lin = torch.zeros(self.lin_bytes, dtype=torch.uint8, device=device)


class MACCell(object):
    """The MAC recurrent cell (stateful, like the reference: mac_cell.py:32-34)."""

    def __init__(self, vecQuestions, questionWords, questionCntxWords, questionLengths, knowledgeBase,
                 memoryDropout, readDropout, writeDropout, batchSize, train, reuse=None, *,
                 config=None, params=None, prec="fp32", seed=0, save_for_backward=False, fold_y=None, small_tc=None,
                 tape_bwd=False, kbIndex=None):
        """`kbIndex` (inference only): CUDA int32 [batchSize], contiguous.  `knowledgeBase` is then the fp32 [U, N, d] of U
        distinct images and question b reads image kbIndex[b]; `zero_state` gathers each question's rows (mac_kb_gather)
        into the operand its read unit reads -- directly into the bf16 copy for the bf16 and fp8 inference forms, which
        read nothing else, into an fp32 [batchSize, N, d] buffer of the cell for every other form."""
        self.lib = _lib.load()
        self.cfg = config if config is not None else _defaults["config"]
        self.params = params if params is not None else _defaults["params"]
        if self.cfg is None or self.params is None:
            raise ValueError("MACCell needs config= and params= (or set_defaults(...))")
        if not isinstance(self.cfg, MACConfig):
            raise TypeError("config must be a MACConfig")
        self.cfg.validate()
        c = self.cfg
        # which units run on the fused sm_90a kernels; everything else goes through the general (composed) path
        self._fused_read = c.is_fast_path
        self._fused_write = (c.writeInputs == "BOTH" and c.writeMemProj and not c.writeConcatMul and not c.writeInfoProj
                             and c.writeInfoAct == "NON" and not c.writeMergeCtrl and c.writeMemAct == "NON")
        self._fused_control = not (c.controlConcatWords or c.controlProj)
        # the knowledge base may arrive already in bf16 (host-cast front end, serving.py): bf16 eval path only
        self._kb_given_bf16 = knowledgeBase.dtype == torch.bfloat16
        for t in (vecQuestions, questionCntxWords) + (() if self._kb_given_bf16 else (knowledgeBase,)):
            if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
                raise ValueError("inputs must be contiguous CUDA float32 tensors")
        if self._kb_given_bf16 and not (knowledgeBase.is_cuda and knowledgeBase.is_contiguous()):
            raise ValueError("a bf16 knowledge base must be a contiguous CUDA tensor")
        self.kbIndex = kbIndex
        if kbIndex is not None:
            # training draws the read dropout per question and needs dKB per image, a sum over each image's questions: the
            # trainer gathers outside the cell instead (DPTrainer.full_forward_backward with data["imageIndex"],
            # mac_kb_gather_bwd), so the cell's shared knowledge bases are an inference form
            if save_for_backward or min(float(memoryDropout), float(readDropout), float(writeDropout)) < 1.0:
                raise NotImplementedError("kbIndex (knowledge bases shared between questions) is inference only: "
                                          "save_for_backward=False and every dropout 1.0")
            if self._kb_given_bf16:
                raise NotImplementedError("kbIndex gathers from the stem's fp32 output: a bf16 knowledge base is not accepted")
            self._check_kb_index(kbIndex, int(batchSize), knowledgeBase.device)
        self.vecQuestions = vecQuestions
        self.questionWords = questionWords
        self.questionCntxWords = questionCntxWords
        self.questionLengths = questionLengths.to(torch.int32).contiguous()
        self.knowledgeBase = knowledgeBase
        self.dropouts = {"memory": float(memoryDropout), "read": float(readDropout), "write": float(writeDropout)}
        self.batchSize = int(batchSize)
        self.train = bool(train)
        self.reuse = reuse
        self.prec = PREC[prec]
        self.seed = int(seed)
        self.device = knowledgeBase.device
        B, N, d = knowledgeBase.shape
        if kbIndex is not None:
            self.U, B = B, self.batchSize
            if d % 8:
                raise NotImplementedError("kbIndex needs memDim %% 8 == 0 (mac_kb_gather's 16-byte vectors), got %d" % d)
        self.B, self.N, self.d = B, N, d
        assert B == self.batchSize and d == c.memDim == c.ctrlDim
        self.none = torch.zeros((B, 1), dtype=torch.float32, device=self.device)     # mac_cell.py:75
        self.iteration = 0
        self.L = self.params.L
        self.ws = _Workspaces(self.lib, B, N, d, self.prec, self.device)
        self._hoist = (not (c.controlFeedPrev or c.controlWholeQ or c.controlContinuous or c.unsharedCells)
                       and self._fused_control)
        self._read_inv = {}
        # eval-mode hoist of the step-invariant read projections (shared cells only)
        self._read_hoist = self._fused_read and not c.unsharedCells and not save_for_backward
        self._y_for = -1
        self.kb_bf16 = None
        self.save_for_backward = bool(save_for_backward)
        # bf16 inference: the batch-sized projections of the step (projY, write unit, gate, ctrlProj) on tensor cores as
        # three-pass split-bf16 products (mac_linear_tc_small_fwd, fp32-class accuracy): 16-32 independent CTAs that can run
        # beside another pass's read kernels, which the 8-CTA-cluster fp32 kernel cannot; its own latency is higher than the
        # cluster kernel's, so it is the THROUGHPUT form: small_tc=True (callers with several passes in flight: bench.py,
        # serving.HostPipeline); default off.  The e4m3 read step (prec="fp8") runs these projections exactly as bf16 does.
        self._small_tc = bool(small_tc and self.prec in (PREC["bf16"], PREC["fp8"]) and not save_for_backward and B <= 128
                              and d % 64 == 0 and self._fused_write)
        # plain write unit: its GEMM also produces the next step's memory projection.  It shortens the dependency chain of
        # ONE pass; with several independent passes in flight the two smaller GEMMs can pack better, so throughput callers
        # may pass fold_y=False.  fold_y=None: on.  The throughput form (small_tc) always folds: one launch for the write
        # unit + the next projY.  With memoryBN the normalised memory is what the next projY sees: no folded form.
        self._fold_y = (self._read_hoist and self._fused_write and not (c.writeSelfAtt or c.writeGate)
                        and not (c.writeDropout < 1.0 and float(writeDropout) < 1.0) and not c.memoryBN
                        and (fold_y is None or bool(fold_y) or self._small_tc))
        recurrent_ctrl_ok = (c.controlFeedPrev and self._fused_control and not (c.controlWholeQ or c.controlContinuous
                                                                                or c.unsharedCells))
        # Backward: the hand-scheduled sweep of autograd._Bwd covers the shipped flag files (fused read + write, control
        # either memory-independent or the plain recurrent chain); every other working flag combination records its
        # primitives on a tape (tape.py) and is differentiated node by node.  tape_bwd=True records the tape even where the
        # scheduled sweep applies (a check of the tape machinery on the shipped flag files).
        scheduled_bwd_ok = (self._fused_read and self._fused_write and (self._hoist or recurrent_ctrl_ok)
                            and not c.memoryBN
                            and not (c.controlInWordsProj or c.controlOutWordsProj)      # wordsProj is outside _Bwd (ADVICE r1)
                            and not (c.controlFeedPrev and not c.controlFeedPrevAtt)
                            and not (c.controlFeedPrev and c.writeSelfAtt and c.writeSelfAttMod == "CONT"))
        self._use_tape = self.save_for_backward and (not scheduled_bwd_ok or tape_bwd)
        self._tape = None
        if self._use_tape:
            if self.prec not in (PREC["fp32"], PREC["bf16"]):
                raise NotImplementedError("the tape backward (flags outside the shipped files) runs the fp32 kernels")
            self._hoist = False              # per-step control(): every launch is a tape node
        if self.save_for_backward and self.prec != PREC["fp32"] and (d % 128 or self._kb_given_bf16):
            raise NotImplementedError("training forward on tensor cores needs d % 128 == 0 and an fp32 knowledge base")
        if self.prec not in (PREC["fp32"], PREC["bf16"]) and not self._fused_read:
            raise NotImplementedError("the tensor-core projections cover the fused read unit only")
        # bf16 with the composed read unit (read flags outside the fused kernel): its [B*N, .] products run on tensor cores
        # (mac_linear_tc_seg_fwd), whose widths (memDim, attDim) must fill whole 128-wide wgmma tiles
        self._tc_general = self.prec == PREC["bf16"] and not self._fused_read
        if self._tc_general and (d % 128 or c.attDim % 128):
            raise NotImplementedError('prec="bf16" with the composed read unit needs d %% 128 == 0 and attDim %% 128 == 0 '
                                      "(got d = %d, attDim = %d)" % (d, c.attDim))
        self._lin_tc_ws = None
        # tc32 training (save_for_backward) runs mac_read_fwd's split-bf16 training form and mac_read_bwd_tc32 under the
        # scheduled backward: the fused read unit, d % 128 == 0 and an fp32 knowledge base (checked above; the tape rejects it)
        if self.prec == PREC["tc32"] and not save_for_backward and (not self._read_hoist or float(readDropout) < 1.0
                                                                    or d % 128):
            raise NotImplementedError('prec="tc32" (split-bf16 tensor-core projections inside the 1e-4 bar) in inference is '
                                      "the hoisted form of the fused read unit: shared cells, readDropout = 1, d % 128 == 0")
        if self.prec == PREC["fp8"] and (save_for_backward or not self._read_hoist or float(readDropout) < 1.0
                                         or not (d == 512 and 1 <= N <= 256 and B < 2 ** 22)):
            raise NotImplementedError('prec="fp8" (e4m3 read step, csrc/read_step_fp8.cuh) is the inference form of the fused '
                                      "read unit: shared cells, readDropout = 1, d = 512, N <= 256")
        if self._kb_given_bf16 and not (self.prec in (PREC["bf16"], PREC["fp8"]) and self._read_hoist
                                        and float(readDropout) >= 1.0):
            raise NotImplementedError("a bf16 knowledge base is accepted by the bf16 and fp8 inference paths only")
        # kbIndex: the bf16 and fp8 hoisted inference forms (fused step or unfused chain) read only kb_bf16, which the gather
        # writes directly; every other form reads an fp32 per-question knowledge base, gathered into this cell's buffer
        self._kb_gather_bf16 = kbIndex is not None and self.prec in (PREC["bf16"], PREC["fp8"]) and self._read_hoist
        self._kb_rows = (torch.empty((B, N, d), dtype=torch.float32, device=self.device)
                         if kbIndex is not None and not self._kb_gather_bf16 else None)

    def _check_kb_index(self, kbIndex, B, device):
        if not (torch.is_tensor(kbIndex) and kbIndex.dtype == torch.int32 and kbIndex.is_cuda and kbIndex.device == device
                and kbIndex.dim() == 1 and kbIndex.is_contiguous() and kbIndex.shape[0] == B):
            raise ValueError("kbIndex must be a contiguous CUDA int32 tensor of shape [batchSize = %d] on the knowledge "
                             "base's device" % B)

    def rebind(self, vecQuestions, questionWords, questionCntxWords, knowledgeBase, kbIndex=None):
        """Point the cell at another batch's input tensors of the same shapes and types (the next `mac_network` reads
        them): what a caller whose encoder and stem produce fresh tensors on every pass needs to keep one cell -- its scratch
        workspaces and cached weight structures; `zero_state` still allocates the histories and attention buffers of each
        pass -- across passes (serving.ModelPipeline).  A cell built with `kbIndex` takes the new index here, one without
        takes none."""
        for new, old in ((vecQuestions, self.vecQuestions), (questionWords, self.questionWords),
                         (questionCntxWords, self.questionCntxWords), (knowledgeBase, self.knowledgeBase)):
            if not (new.shape == old.shape and new.dtype == old.dtype and new.device == old.device and new.is_contiguous()):
                raise ValueError("rebind needs contiguous tensors of the shapes and types the cell was built over")
        if (kbIndex is None) != (self.kbIndex is None):
            raise ValueError("rebind takes a kbIndex exactly when the cell was built with one")
        if kbIndex is not None:
            self._check_kb_index(kbIndex, self.B, self.device)
            self.kbIndex = kbIndex
        self.vecQuestions, self.questionWords = vecQuestions, questionWords
        self.questionCntxWords, self.knowledgeBase = questionCntxWords, knowledgeBase

    # ------------------------------------------------------------------ reference properties
    @property
    def state_size(self):
        return MACCellTuple(self.cfg.ctrlDim, self.cfg.memDim)      # mac_cell.py:84-86

    @property
    def output_size(self):
        return 1                                                     # mac_cell.py:91-93

    # ------------------------------------------------------------------ thin wrappers over the C ABI
    def _linear(self, xs, W, b, out, act="NON", bias_const=0.0, bn_rows=False):
        """ops.linear (ops.py:298-333) on [M, sum k] segments; `xs` is a list of 2-D row-major views.  `bn_rows`: a product
        of the composed read unit over the B*N knowledge-base rows -- on tensor cores with prec="bf16"."""
        n = len(xs)
        M = xs[0].shape[0]
        arr_p, arr_k, arr_ld = segments(xs)
        code = act_code(act, self.cfg.relu)
        if bn_rows and self._tc_general:
            K = sum(x.shape[1] for x in xs)
            need = int(self.lib.mac_linear_tc_seg_workspace_bytes(M, K))
            if self._lin_tc_ws is None or self._lin_tc_ws.numel() < need:
                self._lin_tc_ws = torch.empty(need, dtype=torch.uint8, device=self.device)
            s = stream_ptr()
            W16 = self.params.cache.pack(packs.bf16, W, stream=s)
            check(self.lib.mac_linear_tc_seg_fwd(arr_p, arr_k, arr_ld, n, ptr(W16), ptr(b), float(bias_const), code,
                                                 ptr(out), out.stride(0), M, W.shape[1], ptr(self._lin_tc_ws),
                                                 self._lin_tc_ws.numel(), s),
                  "mac_linear_tc_seg_fwd")
        else:
            check(self.lib.mac_linear_fwd(arr_p, arr_k, arr_ld, n, ptr(W), ptr(b), float(bias_const), code, ptr(out),
                                          out.stride(0), M, W.shape[1], ptr(self.ws.lin), self.ws.lin_bytes, stream_ptr()),
                  "mac_linear_fwd")
        if self._tape is not None:
            self._tape.linear(xs, W, b, out, code, bn_rows=bn_rows)
        return out

    def _linear_tc(self, xs, W, b, out, act="NON", bias_const=0.0, y2=None, n_split=0, gate=None):
        """ops.linear on [M <= 128, sum k] segments as a three-pass split-bf16 wgmma product (mac_linear_tc_small_fwd).
        `gate` = (new, old, z_out): the write gate epilogue (mac_cell.py:358-367)."""
        n = len(xs)
        s = stream_ptr()
        hi, lo = self.params.cache.pack(packs.bf16_split, W, stream=s)
        arr_p, arr_k, arr_ld = segments(xs)
        gn, go, gz = gate if gate is not None else (None, None, None)
        check(self.lib.mac_linear_tc_small_fwd(arr_p, arr_k, arr_ld, n, ptr(hi), ptr(lo), ptr(b), float(bias_const),
                                               act_code(act, self.cfg.relu), ptr(out), out.stride(0), ptr(y2), int(n_split),
                                               ptr(gn), ptr(go), ptr(gz), xs[0].shape[0], W.shape[1], s),
              "mac_linear_tc_small_fwd")
        return out

    def _attend(self, cc, cc_t, cc_b, inw, in_b, in_r, outw, out_b, out_r, lengths, w, b, att, out, nsteps, S):
        check(self.lib.mac_control_attend_fwd(ptr(cc), cc_t, cc_b, ptr(inw), in_b, in_r, ptr(outw), out_b, out_r,
                                              ptr(lengths), ptr(w), float(b), ptr(att), ptr(out), nsteps, self.B, S,
                                              self.d, stream_ptr()), "mac_control_attend_fwd")

    def _dropout(self, x, keep, site, step, out):
        check(self.lib.mac_dropout_fwd(ptr(x), float(keep), self.seed, site, step, ptr(out), x.numel(), stream_ptr()),
              "mac_dropout_fwd")
        if self._tape is not None:
            self._tape.dropout(x, out, keep, site, step)
        return out

    def _new(self, *shape):
        return torch.empty(shape, dtype=torch.float32, device=self.device)

    # ------------------------------------------------------------------ state init (mac_cell.py:496-505, 539-592)
    def initState(self, name, dim, initType, batchSize, out):
        if initType == "PRM":
            out.copy_(self.params[name].unsqueeze(0).expand(batchSize, dim))
        elif initType == "ZERO":
            out.zero_()
        else:  # "Q"
            out.copy_(self.vecQuestions)
        return out

    def zero_state(self, batchSize=None, dtype=None):
        c, B, d, L = self.cfg, self.B, self.d, self.L
        self.attentions = {"kb": [], "question": [], "self": [], "gate": []}        # mac_cell.py:541
        self._read_inv = {}
        # step-major histories [L+1, B, d]; the reference's [B, i+1, d] tensors are permuted views of these
        self._hc = self._new(L + 1, B, d)
        self._hm = self._new(L + 1, B, d)
        self._hi = self._new(L + 1, B, d)
        if self._use_tape:
            from .tape import Tape
            self._tape = Tape(self)
            self._gC, self._gM = self._tape.register_history(self._hc), self._tape.register_history(self._hm)
            self._tape.register_history(self._hi)
            self._tape.init_state(self._hc[0], c.initCtrl, "initCtrl")
            self._tape.init_state(self._hm[0], c.initMem, "initMem")
        c0 = self.initState("initCtrl", c.ctrlDim, c.initCtrl, B, self._hc[0])
        m0 = self.initState("initMem", c.memDim, c.initMem, B, self._hm[0])
        self._hi[0].copy_(m0)                                                          # mac_cell.py:551
        self._set_histories(0)
        self.contControl = c0                                                          # mac_cell.py:553
        words = self.questionCntxWords if c.controlContextual else self.questionWords  # mac_cell.py:570
        self.inWords = self.outWords = words
        if c.controlInWordsProj or c.controlOutWordsProj:                                # mac_cell.py:578-581
            Wp, bp = self.params.lin("", "wordsProj")
            S_ = words.shape[1]
            pWords = self._linear([words.view(B * S_, d)], Wp, bp, self._new(B * S_, d)).view(B, S_, d)
            self.inWords = pWords if c.controlInWordsProj else words
            self.outWords = pWords if c.controlOutWordsProj else words
        self._att_q = self._new(L, B, words.shape[1])
        self._att_kb = self._new(L, B, self.N)
        self._gate = self._new(L, B, d) if c.writeGate else None
        # the per-question knowledge base the read unit takes (`_kb_q`): the caller's, or gathered from the U images
        self._kb_q = self.knowledgeBase
        if self._kb_gather_bf16:
            self.kb_bf16 = self._kb_q = torch.empty((B, self.N, d), dtype=torch.bfloat16, device=self.device)
            self._kb_gather(self.kb_bf16, 1)
        elif self.kbIndex is not None:
            self._kb_q = self._kb_gather(self._kb_rows, 0)
        if self._kb_given_bf16:
            self.kb_bf16 = self.knowledgeBase
        elif self.prec in (PREC["bf16"], PREC["fp8"]) and self._fused_read and not self._kb_gather_bf16:
            self.kb_bf16 = torch.empty(self._kb_q.shape, dtype=torch.bfloat16, device=self.device)
            check(self.lib.mac_cast_bf16(ptr(self._kb_q), ptr(self.kb_bf16), self._kb_q.numel(), stream_ptr()),
                  "mac_cast_bf16")
        self._mem_in = self._new(B, d)
        self._y_next = self._new(B, d)
        self._y_for = -1
        if self.save_for_backward:
            self._ctrl_saved = {}
            M = B * self.N
            self._save = [self._new(3 * M * d + B * d) for _ in range(L)]      # [P | H | I1 | y] per step
            self._mem_in_hist = self._new(L, B, d)
            self._mnew = self._new(L, B, d) if c.writeGate else None
            self._ss = self._new(L, B, d) if c.writeSelfAtt else None
            self._sc = self._new(L, B, d) if c.writeSelfAtt else None
        if self._hoist:
            self._control_all_steps()
        return MACCellTuple(c0, m0)

    def _kb_gather(self, out, bf16):
        """out[b] = knowledgeBase[kbIndex[b]] (mac_kb_gather), fp32 or bf16."""
        check(self.lib.mac_kb_gather(ptr(self.knowledgeBase), ptr(self.kbIndex), ptr(out), int(bf16), self.B, self.U, self.N,
                                     self.d, stream_ptr()), "mac_kb_gather")
        return out

    def _set_histories(self, i):
        self.controls = self._hc[:i + 1].permute(1, 0, 2)      # [B, i+1, d] like mac_cell.py:549, 472
        self.memories = self._hm[:i + 1].permute(1, 0, 2)
        self.infos = self._hi[:i + 1].permute(1, 0, 2)

    # ------------------------------------------------------------------ control unit
    def _question_input(self):
        """u = act(linear_qInput(vecQuestions)) (mac_cell.py:442-445): weights shared over steps => once per forward."""
        W, b = self.params.lin("MACCell/", "qInput")
        u = self._linear([self.vecQuestions], W, b, self._new(self.B, self.d), act=self.cfg.controlInputAct)
        self._u_saved = u
        return u

    def _control_all_steps(self):
        """With controlFeedPrev off the control chain does not depend on memory (mac_cell.py:141-151): compute
        ci_i = linear_qInput{i}(u) for every step with ONE GEMM against the packed [d, L*d] weight, then ONE
        attention launch that streams each batch row's words once for all L steps."""
        c, B, d, L = self.cfg, self.B, self.d, self.L
        u = self._question_input()
        if c.controlInputUnshared:
            Wc, bc = self.params.q_input_cat()
            self._ci = self._linear([u], Wc, bc, self._new(B, L * d))              # [B, L*d]: ci_i = [:, i*d:(i+1)*d]
            cc_t, cc_b = d, L * d
        else:
            W, b = self.params.lin("MACCell/", "qInputU")
            self._ci = self._linear([u], W, b, self._new(B, d))
            cc_t, cc_b = 0, d                                                       # same query for every step
        sc = "MACCell/control/inter2logits/linearLayerlogits/"
        w = self.params[sc + "weights/weight"]
        bl = self.params.scalar(sc + "biases/bias")
        S = self.inWords.shape[1]
        self._attend(self._ci, cc_t, cc_b, self.inWords, S * d, d, self.outWords, S * d, d, self.questionLengths,
                     w, bl, self._att_q, self._hc[1:], L, S)

    def control(self, controlInput, inWords, outWords, questionLengths, control, contControl=None, name="",
                reuse=None, _att_out=None, _out=None):
        """mac_cell.py:133-187 (returns newControl, newContControl)."""
        c, B, d = self.cfg, self.B, self.d
        sc = "MACCell/control" + name + "/"
        newContControl = controlInput
        if c.controlFeedPrev:
            prev = control if c.controlFeedPrevAtt else contControl
            xs = [prev, controlInput] if c.controlFeedInputs else [prev]
            W, b = self.params.lin(sc, "contControl")
            newContControl = self._linear(xs, W, b, self._new(B, d), act=c.controlContAct)
            hidden = newContControl
            if c.controlContAct != "NON":                                            # nested "_2" layer, ops.py:325-328
                W2, b2 = self.params.lin(sc + "linearLayercontControl/", "contControl_2")
                newContControl = self._linear([newContControl], W2, b2, self._new(B, d))
            if self.save_for_backward:      # what the recurrent control chain's backward needs, per step
                self._ctrl_saved[self.iteration] = (prev, controlInput, hidden, newContControl)
        S = inWords.shape[1]
        att = _att_out if _att_out is not None else self._new(B, S)
        out = _out if _out is not None else self._new(B, d)
        lsc = sc + "inter2logits/linearLayerlogits/"
        if not self._fused_control:
            # general path (mac_cell.py:155-181 with controlConcatWords / controlProj)
            inter = self._bcast(inWords.reshape(B * S, d), newContControl, 0, S, mul_bias=0.0)   # plain product, mac_cell.py:155
            segs = [inter] + ([inWords.reshape(B * S, d)] if c.controlConcatWords else [])
            if c.controlProj:
                segs = [self._ops_linear(segs, sc, "", act=c.controlProjAct)]
            logits = self._rowdot(segs, lsc)
            check(self.lib.mac_attend_fwd(ptr(logits), ptr(questionLengths), ptr(outWords), S * d, d, ptr(att), ptr(out),
                                          B, S, d, stream_ptr()), "mac_attend_fwd")
            if self._tape is not None:
                self._tape.attend(logits, outWords, att, out, B, S, d)
            self.attentions["question"].append(att)
            return (newContControl if c.controlContinuous else out), newContControl
        self._attend(newContControl, 0, d, inWords, S * d, d, outWords, S * d, d, questionLengths,
                     self.params[lsc + "weights/weight"], self.params.scalar(lsc + "biases/bias"), att, out, 1, S)
        if self._tape is not None:
            self._tape.control_attend(newContControl, inWords, outWords, lsc, att, out, S)
        self.attentions["question"].append(att)
        newControl = out
        if c.controlContinuous:
            newControl = newContControl
        return newControl, newContControl

    # ------------------------------------------------------------------ read unit
    def _read_weights(self, name):
        """The read unit's weights as the library reads them, with the packs of this cell's precision.  An entry of the
        parameters' cache, so it is rebuilt together with the packs it points into whenever the values move."""
        return self.params.cache.get(("ReadWeights", name, self.prec, self.save_for_backward),
                                     lambda: self._build_read_weights(name))

    def _build_read_weights(self, name):
        p, sc, d, s = self.params, "MACCell/read" + name + "/", self.d, stream_ptr()
        pack = lambda builder, W: p.cache.pack(builder, W, stream=s)
        Wx, bx = p.lin(sc + "mulmemInter/", "projX")
        Wy, by = p.lin(sc + "mulmemInter/", "projY")
        Wm, bm = p.lin(sc, "memKbProj")
        Wm2, bm2 = p.lin(sc + "linearLayermemKbProj/", "memKbProj_2")
        lsc = sc + "inter2att/inter2logits/linearLayerlogits/"
        rw = ReadWeights(Wx.data_ptr(), bx.data_ptr(), Wy.data_ptr(), by.data_ptr(), Wm.data_ptr(), bm.data_ptr(),
                         Wm2.data_ptr(), bm2.data_ptr(), p[lsc + "weights/weight"].data_ptr(),
                         p.scalar(lsc + "biases/bias"), None, None, None)
        if self.prec in (PREC["bf16"], PREC["fp8"]):     # fp8: P and Q are the bf16 path's (mac_read_invariant)
            rw.Wx_bf16, rw.Wm_bf16, rw.Wm2_bf16 = (pack(packs.bf16, t).data_ptr() for t in (Wx, Wm, Wm2))
        if self.prec == PREC["tc32"]:
            rw.Wx_s3, rw.Wma_s3, rw.Wmb_s3, rw.Wm2_s3 = (pack(packs.split3, t).data_ptr()
                                                         for t in (Wx, Wm[:d], Wm[d:], Wm2))
            if self.save_for_backward:   # training form: H = ELU([P*y | P] @ Wm + bm) as one product over K = 2d
                rw.Wm_s3 = pack(packs.split3, Wm).data_ptr()
        if self.prec == PREC["fp8"]:
            (w8, s8), (w8_2, s8_2) = pack(packs.fp8, Wm[:d]), pack(packs.fp8, Wm2)
            rw.Wm_fp8, rw.Wm_fp8_scale, rw.Wm2_fp8, rw.Wm2_fp8_scale = (t.data_ptr() for t in (w8, s8, w8_2, s8_2))
        return rw

    def read(self, knowledgeBase, memory, control, name="", reuse=None, _att_out=None, _out=None, _save=None,
             _y_pre=None):
        """mac_cell.py:209-277 (returns the retrieved information [B, memDim])."""
        c, B, N, d = self.cfg, self.B, self.N, self.d
        i = self.iteration
        keep_m = self.dropouts["memory"]
        if keep_m < 1.0:
            mem_in = self._mem_in if self._tape is None else self._new(B, d)     # the tape keeps every step's tensor
            if c.memoryVariationalDropout:     # one mask per forward (mac_cell.py:589-590): site MEM_VAR, step 0
                memory = self._dropout(memory, keep_m, _lib.SITE_MEM_VAR, 0, mem_in)
            else:
                memory = self._dropout(memory, keep_m, _lib.SITE_MEM_PLAIN, i, mem_in)
        att = _att_out if _att_out is not None else self._new(B, N)
        info = _out if _out is not None else self._new(B, d)
        if not self._fused_read:
            return self._read_general(knowledgeBase, memory, control, name, att, info)
        if self.save_for_backward and _save is None:
            _save = self._save[i]
            self._mem_in_hist[i].copy_(memory)
        rw = self._read_weights(name)
        if self._read_hoist and self.dropouts["read"] >= 1.0 and _save is None:
            # eval mode: P and Q = P @ Wm[d:2d] + bm do not depend on the step -> once per forward (mac_b200.h)
            kb32 = None if knowledgeBase.dtype == torch.bfloat16 else ptr(knowledgeBase)
            if name not in self._read_inv:
                nbytes = self.lib.mac_read_invariant_bytes(B, N, d, self.prec)
                inv = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
                check(self.lib.mac_read_invariant(kb32, ptr(self.kb_bf16), ctypes.byref(rw), self.prec,
                                                  ptr(inv), nbytes, B, N, d, stream_ptr()), "mac_read_invariant")
                self._read_inv[name] = inv
            if _y_pre is None and self._small_tc:
                Wy, by = self.params.lin("MACCell/read" + name + "/mulmemInter/", "projY")
                _y_pre = self._linear_tc([memory], Wy, by, self._y_next)
            check(self.lib.mac_read_fwd_inv(kb32, ptr(self.kb_bf16), ptr(self._read_inv[name]), ptr(_y_pre),
                                            ptr(memory), ptr(control), ctypes.byref(rw), self.prec, ptr(info), ptr(att),
                                            ptr(self.ws.read), self.ws.read_bytes, B, N, d, stream_ptr()),
                  "mac_read_fwd_inv")
            self.attentions["kb"].append(att)
            return info
        check(self.lib.mac_read_fwd(ptr(knowledgeBase), ptr(self.kb_bf16), ptr(memory), ptr(control),
                                    ctypes.byref(rw), float(self.dropouts["read"]), self.seed, i, self.prec,
                                    ptr(info), ptr(att), ptr(_save), ptr(self.ws.read), self.ws.read_bytes, B, N, d,
                                    stream_ptr()), "mac_read_fwd")
        if self._tape is not None:
            self._tape.fused_read(i, name, knowledgeBase, memory, control, info)
        self.attentions["kb"].append(att)
        return info

    # ------------------------------------------------------------------ write unit
    def _folded_write_weights(self, name):
        """[Ww | Ww @ Wy], [bw | bw @ Wy + by]: the plain write unit and the next step's memory projection as one
        linear map of [memory, info] (mac_b200.h, mac_write_fwd_next_y); rebuilt when the parameters change."""
        def build():
            d = self.d
            Ww, bw = self.params.lin("MACCell/write" + name + "/", "newMemory")
            Wy, by = self.params.lin("MACCell/read" + name + "/mulmemInter/", "projY")
            Wf = self._new(2 * d, 2 * d)
            bf = self._new(2 * d)
            Wf[:, :d].copy_(Ww)
            bf[:d].copy_(bw)
            self._linear([Ww], Wy, None, Wf[:, d:])                       # Ww @ Wy        (ldy = 2d)
            self._linear([bw.view(1, d)], Wy, by, bf[d:].view(1, d))      # bw @ Wy + by
            return Wf, bf
        return self.params.cache.get(("foldY", name), build)

    def write(self, memory, info, control, contControl=None, name="", reuse=None, _out=None, _gate_out=None,
              _y_next=None):
        """mac_cell.py:305-375 (returns the new memory [B, memDim])."""
        if not self.cfg.memoryBN:
            return self._write_unit(memory, info, control, contControl, name, _out, _gate_out, _y_next)
        pre = self._write_unit(memory, info, control, contControl, name, self._new(self.B, self.d), _gate_out, None)
        return self._batch_norm(pre, name, _out if _out is not None else self._new(self.B, self.d))

    def _batch_norm(self, x, name, out, eps=1e-3):
        """mac_cell.py:369-373: tf.contrib.layers.batch_norm(newMemory, decay=bnDecay, center=bnCenter, scale=bnScale,
        is_training=self.train, updates_collections=None) -- batch statistics (and the in-place update of the stored ones, once
        per reasoning step) in training, the stored statistics at eval; epsilon is the layer's default 0.001."""
        c, B, d = self.cfg, self.B, self.d
        sc = "MACCell/write" + name + "/BatchNorm/"
        gamma = self.params[sc + "gamma"] if c.bnScale else None
        beta = self.params[sc + "beta"] if c.bnCenter else None
        mean, invstd = self._new(d), self._new(d)
        check(self.lib.mac_batchnorm_fwd(ptr(x), ptr(gamma), ptr(beta), ptr(self.params[sc + "moving_mean"]),
                                         ptr(self.params[sc + "moving_variance"]), float(c.bnDecay), float(eps),
                                         int(self.train), ptr(out), ptr(mean), ptr(invstd), B, d, stream_ptr()),
              "mac_batchnorm_fwd")
        if self._tape is not None:
            self._tape.batch_norm(x, out, gamma, beta, mean, invstd, int(self.train))
        return out

    def _write_unit(self, memory, info, control, contControl, name, _out, _gate_out, _y_next):
        c, B, d = self.cfg, self.B, self.d
        sc = "MACCell/write" + name + "/"
        i = self.iteration
        if not self._fused_write:
            return self._write_general(memory, info, control, contControl, name, _out, _gate_out)
        if _y_next is not None and self._small_tc:
            Wf, bf = self._folded_write_weights(name)
            out = _out if _out is not None else self._new(B, d)
            return self._linear_tc([memory, info], Wf, bf, out, y2=_y_next, n_split=d)
        if _y_next is not None:
            Wf, bf = self._folded_write_weights(name)
            out = _out if _out is not None else self._new(B, d)
            check(self.lib.mac_write_fwd_next_y(ptr(memory), ptr(info), ptr(Wf), ptr(bf), ptr(out), ptr(_y_next),
                                                ptr(self.ws.write), self.ws.write_bytes, B, d, stream_ptr()),
                  "mac_write_fwd_next_y")
            return out
        selfSmry = None
        if c.writeSelfAtt:
            selfControl = contControl if c.writeSelfAttMod == "CONT" else control
            W, b = self.params.lin(sc, "ctrlProj")
            keep = self.save_for_backward
            if self._small_tc:
                selfControl = self._linear_tc([selfControl], W, b, self._new(B, d))
            else:
                selfControl = self._linear([selfControl], W, b, self._sc[i] if keep else self._new(B, d))
            lsc = sc + "inter2attselfAttention/inter2logits/linearLayerlogits/"
            att = self._new(B, i + 1)
            selfSmry = self._ss[i] if keep else self._new(B, d)
            # interactions = controls * selfControl; attention over the i+1 history rows; summary of memories
            self._attend(selfControl, 0, selfControl.stride(0), self._hc, d, B * d, self._hm, d, B * d, None,
                         self.params[lsc + "weights/weight"], self.params.scalar(lsc + "biases/bias"), att, selfSmry,
                         1, i + 1)
            if self._tape is not None:
                self._tape.self_attend(selfControl, lsc, att, selfSmry, i + 1, self._gC, self._gM)
            self.attentions["self"].append(att)
        Ww, bw = self.params.lin(sc, "newMemory")
        Wg = bg = None
        gate = None
        if c.writeGate:
            Wg, bg = self.params.lin(sc, "gate")
            gate = _gate_out if _gate_out is not None else self._new(B, d)
        out = _out if _out is not None else self._new(B, d)
        if self._small_tc:
            segs = [memory, info] + ([selfSmry] if selfSmry is not None else [])
            if c.writeGate:
                mnew = self._linear_tc(segs, Ww, bw, self._new(B, d))
                self._linear_tc([control], Wg, bg, out, bias_const=float(c.writeGateBias),
                                gate=(mnew, memory, gate))
                self.attentions["gate"].append(gate)
            else:
                self._linear_tc(segs, Ww, bw, out)
            return out
        check(self.lib.mac_write_fwd(ptr(memory), ptr(info), ptr(selfSmry), ptr(control), ptr(Ww), ptr(bw), ptr(Wg),
                                     ptr(bg), float(c.writeGateBias), ptr(out), ptr(gate), ptr(self.ws.write),
                                     self.ws.write_bytes, B, d, stream_ptr()), "mac_write_fwd")
        if self.save_for_backward and c.writeGate:
            # the pre-gate memory m' is the first [B,d] block of the write workspace after its 4 KB header
            self._mnew[i].copy_(self.ws.write[4096:4096 + B * d * 4].view(torch.float32).view(B, d))
        if self._tape is not None:
            self._tape.fused_write(i, name, memory, info, selfSmry, control, out)
        if c.writeGate:
            self.attentions["gate"].append(gate)
        return out

    # ------------------------------------------------------------------ general (composed) path
    def _ops_linear(self, xs, scope, name, act="NON", bias_const=0.0, bn_rows=False):
        """ops.linear incl. the nested "<name>_2" layer when act != NON (ops.py:298-333); xs: list of 2-D segments."""
        W, b = self.params.lin(scope, name)
        y = self._linear(xs, W, b, self._new(xs[0].shape[0], W.shape[1]), act=act, bias_const=bias_const, bn_rows=bn_rows)
        if act != "NON":
            W2, b2 = self.params.lin(scope + "linearLayer" + name + "/", name + "_2")
            y = self._linear([y], W2, b2, self._new(y.shape[0], W2.shape[1]), bn_rows=bn_rows)
        return y

    def _rowdot(self, xs, lscope):
        """outDim == 1 linear (vector weight, scalar bias) over concatenated segments -> [R]."""
        n, R = len(xs), xs[0].shape[0]
        out = self._new(R)
        arr_p, arr_k, arr_ld = segments(xs)
        check(self.lib.mac_rowdot_fwd(arr_p, arr_k, arr_ld, n, ptr(self.params[lscope + "weights/weight"]),
                                      self.params.scalar(lscope + "biases/bias"), ptr(out), R, stream_ptr()), "mac_rowdot_fwd")
        if self._tape is not None:
            self._tape.rowdot(xs, lscope, out)
        return out

    def _bcast(self, x2d, v, mode, N, bias=None, mul_bias=None):
        """ops.mul interaction of x [B*N, d] with the per-sample vector v [B, d] (MUL / BL tail / ADD)."""
        out = self._new(*x2d.shape)
        mb = self.cfg.mulBias if mul_bias is None else mul_bias
        check(self.lib.mac_bcast_op(ptr(x2d), ptr(v), mode, float(mb), ptr(bias), ptr(out), self.B, N,
                                    x2d.shape[1], stream_ptr()), "mac_bcast_op")
        if self._tape is not None:
            self._tape.bcast(x2d, v, mode, mb, bias, out, self.B, N)
        return out

    def _add_scaled(self, a, b, alpha):
        """a + alpha * b as a new tensor (the copy is memory plumbing, the arithmetic is mac_axpy)."""
        out = a.clone()
        check(self.lib.mac_axpy(ptr(out), ptr(b), float(alpha), out.numel(), stream_ptr()), "mac_axpy")
        if self._tape is not None:
            self._tape.add_scaled(a, b, float(alpha), out)
        return out

    def _act(self, x, act):
        if act == "NON":
            return x
        out = self._new(*x.shape)
        code = act_code(act, self.cfg.relu)
        check(self.lib.mac_activation(ptr(x), code, ptr(out), x.numel(), stream_ptr()), "mac_activation")
        if self._tape is not None:
            self._tape.act(x, out, code)
        return out

    def _mul_general(self, x2d, y, dim, N, scope, name, proj, inter_mod, concat_x, concat_proj):
        """ops.mul (ops.py:668-725) -> (list of segments [B*N, .], projected x or None)."""
        sc = scope + "mul" + name + "/"
        orig_x, proj_x = x2d, None
        if proj is not None:
            if proj.get("dropout", 1.0) < 1.0:          # ops.py:678-679: both operands, before their projections
                i = self.iteration
                x2d = self._dropout(x2d, proj["dropout"], _lib.SITE_READ_KB, i, self._new(*x2d.shape))
                y = self._dropout(y, proj["dropout"], _lib.SITE_READ_MEM, i, self._new(*y.shape))
            xn, yn = ("proj", "proj") if proj["shared"] else ("projX", "projY")
            x2d = self._ops_linear([x2d], sc, xn, bn_rows=True)
            y = self._ops_linear([y], sc, yn)
            proj_x = x2d
        if inter_mod == "MUL":
            inter = self._bcast(x2d, y, 0, N)
        elif inter_mod == "BL":
            W, b = self.params[sc + "weights/weight"], self.params[sc + "biases/bias"]
            xw = self._linear([x2d], W, None, self._new(x2d.shape[0], W.shape[1]), bn_rows=True)
            inter = self._bcast(xw, y, 1, N, bias=b)
        else:  # ADD
            inter = self._bcast(x2d, y, 2, N)
        segs = [inter]
        if concat_x:
            segs.append(proj_x if concat_proj else orig_x)
        return segs, proj_x

    def _read_general(self, knowledgeBase, memory, control, name, att, info):
        """mac_cell.py:209-277 composed from primitives (flag sets outside the fused read kernel)."""
        c, B, N, d = self.cfg, self.B, self.N, self.d
        keep_r = self.dropouts["read"]
        sc = "MACCell/read" + name + "/"
        kb2 = knowledgeBase.view(B * N, d)
        proj = {"shared": c.readProjShared, "dropout": keep_r} if c.readProjInputs else None
        segs, projectedKB = self._mul_general(kb2, memory, c.memDim, N, sc, "memInter", proj, c.readMemAttType,
                                              c.readMemConcatKB, c.readMemConcatProj)
        if c.readMemProj:
            segs = [self._ops_linear(segs, sc, "memKbProj", act=c.readMemAct, bn_rows=True)]
        if c.readCtrl:
            segs, _ = self._mul_general(segs[0], control, 0, N, sc, "ctrlInter", None, c.readCtrlAttType, False, False)
            if c.readCtrlConcatKB:
                segs.append(projectedKB if c.readCtrlConcatProj else kb2)
            segs = [self._act(x, c.readCtrlAct) for x in segs]          # act(concat) == concat(act)
        if keep_r < 1.0:
            # inter2att's linear drops its (concatenated) input (mac_cell.py:266, ops.py:312): ONE mask over [B, N, total
            # width], so the concat is materialised for the flat mask index (memory plumbing) and dropped as one tensor
            cat = segs[0] if len(segs) == 1 else torch.cat(segs, dim=1)
            if self._tape is not None and len(segs) > 1:
                self._tape.cat(list(segs), cat)
            segs = [self._dropout(cat, keep_r, _lib.SITE_READ_INTER, self.iteration, self._new(*cat.shape))]
        logits = self._rowdot(segs, sc + "inter2att/inter2logits/linearLayerlogits/")
        feats = projectedKB if c.readSmryKBProj else kb2
        dd = feats.shape[1]
        check(self.lib.mac_attend_fwd(ptr(logits), None, ptr(feats), N * dd, dd, ptr(att), ptr(info), B, N, dd,
                                      stream_ptr()), "mac_attend_fwd")
        if self._tape is not None:
            self._tape.attend(logits, feats, att, info, B, N, dd)
        self.attentions["kb"].append(att)
        return info

    def _write_general(self, memory, info, control, contControl, name, _out, _gate_out):
        """mac_cell.py:305-375 composed from primitives."""
        c, B, d = self.cfg, self.B, self.d
        sc = "MACCell/write" + name + "/"
        i = self.iteration
        if c.writeInfoProj:
            info = self._ops_linear([info], sc, "info")
        info = self._act(info, c.writeInfoAct)
        selfSmry = None
        if c.writeSelfAtt:
            selfControl = contControl if c.writeSelfAttMod == "CONT" else control
            selfControl = self._ops_linear([selfControl], sc, "ctrlProj")
            lsc = sc + "inter2attselfAttention/inter2logits/linearLayerlogits/"
            satt, selfSmry = self._new(B, i + 1), self._new(B, d)
            self._attend(selfControl, 0, selfControl.stride(0), self._hc, d, B * d, self._hm, d, B * d, None,
                         self.params[lsc + "weights/weight"], self.params.scalar(lsc + "biases/bias"), satt, selfSmry,
                         1, i + 1)
            if self._tape is not None:
                self._tape.self_attend(selfControl, lsc, satt, selfSmry, i + 1, self._gC, self._gM)
            self.attentions["self"].append(satt)
        if c.writeInputs == "INFO":
            segs = [info]
        elif c.writeInputs == "SUM":
            segs = [self._add_scaled(memory, info, 1.0)]
        elif c.writeInputs == "BOTH":
            segs = [memory, info]
            if c.writeConcatMul:                                                          # ops.py:65-78
                segs.append(self._bcast(memory, info, 0, 1, mul_bias=0.0))
        else:  # MEM
            segs = [memory]
        if selfSmry is not None:
            segs.append(selfSmry)
        if c.writeMergeCtrl:
            segs.append(control)
        dim = sum(x.shape[1] for x in segs)
        out = _out if _out is not None else self._new(B, d)
        if c.writeMemProj or dim != c.memDim:
            if len(segs) > 4:
                raise NotImplementedError("more than four concatenated write inputs")
            W, b = self.params.lin(sc, "newMemory")
            newMemory = self._linear(segs, W, b, self._new(B, d))
        else:
            newMemory = segs[0]
        newMemory = self._act(newMemory, c.writeMemAct)
        if c.writeGate:
            Wg, bg = self.params.lin(sc, "gate")
            z = self._linear([control], Wg, bg, _gate_out if _gate_out is not None else self._new(B, d), act="SIGMOID",
                             bias_const=c.writeGateBias)
            self.attentions["gate"].append(z)
            # m' * z + m * (1 - z) = m + z * (m' - m)
            diff = self._add_scaled(newMemory, memory, -1.0)
            zd = self._bcast(diff, z, 0, 1, mul_bias=0.0)
            newMemory = self._add_scaled(memory, zd, 1.0)
        out.copy_(newMemory)
        if self._tape is not None:
            self._tape.copy(out, newMemory)
        return out

    # ------------------------------------------------------------------ one reasoning step (mac_cell.py:420-480)
    def __call__(self, inputs, state, scope=None):
        c, B, d = self.cfg, self.B, self.d
        i = self.iteration
        if i >= self.L:
            raise IndexError("iteration %d >= netLength %d the parameters were built for" % (i, self.L))
        control, memory = state.control, state.memory
        cellName = str(i) if c.unsharedCells else ""                                    # mac_cell.py:434-438
        if self._hoist:
            newControl = self._hc[i + 1]
            self.contControl = self._ci[:, i * d:(i + 1) * d] if c.controlInputUnshared else self._ci
            self.attentions["question"].append(self._att_q[i])
        else:
            u = self._question_input() if i == 0 else self._u
            self._u = u
            nameU = ("qInput%d" % i) if c.controlInputUnshared else "qInputU"
            W, b = self.params.lin("MACCell/", nameU)
            ci = self._linear([u], W, b, self._new(B, d))
            newControl, self.contControl = self.control(ci, self.inWords, self.outWords, self.questionLengths,
                                                        control, self.contControl, name=cellName,
                                                        _att_out=self._att_q[i], _out=self._hc[i + 1])
            if c.controlContinuous:
                self._hc[i + 1].copy_(newControl)
                if self._tape is not None:
                    self._tape.copy(self._hc[i + 1], newControl)
                newControl = self._hc[i + 1]
        if c.controlWholeQ:                                                            # mac_cell.py:455-456
            self._hc[i + 1].copy_(self.vecQuestions)
            if self._tape is not None:
                self._tape.copy(self._hc[i + 1], self.vecQuestions)
            newControl = self._hc[i + 1]
        info = self.read(self._kb_q, memory, newControl, name=cellName, _att_out=self._att_kb[i],
                         _out=self._hi[i + 1], _y_pre=self._y_next if self._y_for == i else None)
        if c.writeDropout < 1.0 and self.dropouts["write"] < 1.0:                      # mac_cell.py:461-463
            info = self._dropout(info, self.dropouts["write"], _lib.SITE_WRITE_INFO, i, self._hi[i + 1])
        fold = self._fold_y and i + 1 < self.L and self.dropouts["read"] >= 1.0 and self.dropouts["memory"] >= 1.0
        newMemory = self.write(memory, info, newControl, self.contControl, name=cellName, _out=self._hm[i + 1],
                               _gate_out=None if self._gate is None else self._gate[i],
                               _y_next=self._y_next if fold else None)
        self._y_for = i + 1 if fold else -1
        self._set_histories(i + 1)                                                     # mac_cell.py:472-474
        return self.none, MACCellTuple(newControl, newMemory)

    def _read_inter_width(self):
        """Width of the tensor inter2att drops (mac_cell.py:209-266): the fused family ends in memDim columns."""
        c = self.cfg
        if self._fused_read:
            return self.d
        dim = c.attDim if c.readProjInputs else c.memDim
        inter = dim + ((c.attDim if c.readMemConcatProj else c.memDim) if c.readMemConcatKB else 0)
        if c.readMemProj:
            inter = dim
        if c.readCtrl and c.readCtrlConcatKB:
            inter += c.attDim if c.readCtrlConcatProj else c.memDim
        return inter

    # ------------------------------------------------------------------ test support
    def dropout_uniforms(self):
        """The uniforms the kernels draw for this forward, in the reference's call order (zero_state mask, then per
        step KB / memory / interactions / write) -- tests hand them to the oracle."""
        c, B, N, d, L = self.cfg, self.B, self.N, self.d, self.L
        out = []

        def draw(site, step, shape):
            u = torch.empty(shape, dtype=torch.float32, device=self.device)
            check(self.lib.mac_dropout_uniform(self.seed, site, step, ptr(u), u.numel(), stream_ptr()), "uniform")
            return u.cpu().numpy().astype(np.float64)
        km, kr, kw = self.dropouts["memory"], self.dropouts["read"], self.dropouts["write"]
        if c.memoryVariationalDropout and km < 1.0:
            out.append(draw(_lib.SITE_MEM_VAR, 0, (B, d)))
        for i in range(L):
            if not c.memoryVariationalDropout and km < 1.0:
                out.append(draw(_lib.SITE_MEM_PLAIN, i, (B, d)))
            if kr < 1.0:
                if self._fused_read or c.readProjInputs:
                    out.append(draw(_lib.SITE_READ_KB, i, (B, N, d)))
                    out.append(draw(_lib.SITE_READ_MEM, i, (B, d)))
                out.append(draw(_lib.SITE_READ_INTER, i, (B, N, self._read_inter_width())))
            if c.writeDropout < 1.0 and kw < 1.0:
                out.append(draw(_lib.SITE_WRITE_INFO, i, (B, d)))
        return out


def mac_network(cell, netLength):
    """The caller of the cell, `MACnet.MACnetwork` (model.py:447-458, 486-487): zero_state + static unroll."""
    state = cell.zero_state(cell.batchSize)
    none = cell.none
    for i in range(netLength):
        cell.iteration = i
        _, state = cell(none, state)
    return state.control, state.memory
