"""Data-parallel training of the MAC cell: one process per GPU, the batch sharded over ranks, ONE collective per step.

The reference's multi-GPU path is a stub (towers >= 1 are ignored, `model.py:671-679`), so there is nothing to match
except single-process semantics: the all-reduced gradient of the global-mean loss must equal the 1-process gradient on
the concatenated batch.  Per step (SURVEY.md section 8(e)):
    forward (train-mode dropouts, per-rank Philox streams) -> hand-written backward into the flat gradient bucket ->
    `all_reduce(SUM)` of the bucket over NCCL/NVLink -> global-norm clip, Adam, EMA fused in one kernel (replicated).
The loss of this cell-level harness is a linear probe of the final state, sum(memory_L * t_m + control_L * t_c) / B_global,
standing in for the out-of-scope output unit / classifier (it supplies dL/dmemory and dL/dcontrol exactly as they would).
"""

import numpy as np
import torch

from . import _lib
from ._lib import check, ptr, stream_ptr


def shard_rows(global_batch, rank, world):
    """Rank r takes samples [r*B/world, (r+1)*B/world) of the global batch (mirrors initTowerBatch, model.py:139-149)."""
    if global_batch % world:
        raise ValueError("global batch %d is not divisible by world size %d" % (global_batch, world))
    per = global_batch // world
    return slice(rank * per, (rank + 1) * per)


def allreduce_sum_(bucket, group=None):
    """The path's only exchange step.  Returns the bucket (summed over ranks in place)."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(bucket, op=dist.ReduceOp.SUM, group=group)
    return bucket


def allreduce_sum_with_stats_(bucket, flat, start, group=None):
    """The step's one exchange when the flat layout ends in stored batch-norm statistics (elements `start:` of `flat`,
    `DPTrainer.n_train`), which each rank has just moved with its own batch: the bucket's tail, which holds no gradient,
    carries each rank's statistics / world, so the SUM leaves the mean over ranks, copied back into `flat`.  Every rank
    then holds the same statistics, moved by the mean over ranks of the per-rank batch statistics (the update is linear in
    them).  The gradient norm, clipping, Adam and the EMA read elements `:start` only.  At world = 1 nothing is touched."""
    import torch.distributed as dist
    world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
    tail = world > 1 and start < flat.numel()
    if tail:
        torch.mul(flat[start:], 1.0 / world, out=bucket[start:])
    allreduce_sum_(bucket, group)
    if tail:
        flat[start:].copy_(bucket[start:])
    return bucket


def classifier_options(classifier):
    """The output unit options of `classifier=(answerWordsNum, outClassifierDims[, options])` (`output_options`)."""
    from .output_unit import output_options
    return output_options(classifier[2] if len(classifier) > 2 else None)


def check_model_precisions(cfg, encoder, stem, stem_prec, enc_prec):
    """The stem's and the encoder's training precisions against the model's shapes (DPTrainer, modules.MACModel): raises
    before anything is allocated or launched."""
    if stem_prec not in ("fp32", "bf16", "bf16x3"):
        raise ValueError("stem_prec must be 'fp32', 'bf16' or 'bf16x3', got %r" % (stem_prec,))
    if stem_prec != "fp32":
        if stem is None:
            raise ValueError("stem_prec=%r needs stem=" % (stem_prec,))
        stem_dim = stem_geometry(stem)["stem_dim"]
        if stem[0] % 128 or cfg.memDim % 128 or (stem_dim is not None and stem_dim % 128):
            raise NotImplementedError("stem_prec=%r needs the image channels (%d), memDim (%d) and stem_dim (%s) to be "
                                      "multiples of 128 (the wgmma tiles of mac_conv3x3_bwd_tc)"
                                      % (stem_prec, stem[0], cfg.memDim, stem_dim))
    if enc_prec not in ("fp32", "bf16"):
        raise ValueError("enc_prec must be 'fp32' or 'bf16', got %r" % (enc_prec,))
    if enc_prec != "fp32":
        if encoder is None:
            raise ValueError("enc_prec=%r needs encoder=" % (enc_prec,))
        if cfg.ctrlDim != 512:
            raise NotImplementedError("enc_prec='bf16' needs ctrlDim = 512 (h = 256 per LSTM direction), got %d"
                                      % cfg.ctrlDim)


STEM_GEOMETRY = {"ksizes": None, "strides": None, "linear": False, "stem_dim": None, "location": None, "location_bias": 1.0,
                 "location_dim": 32}


def stem_geometry(stem):
    """The geometry of `stem=(imageInDim, stemNumLayers[, geometry])`: a dict with the keys of STEM_GEOMETRY --
    `ksizes` (--stemKernelSizes, one kernel size per layer; None: 3x3), `strides` (--stemStrideSizes; None: 1),
    `linear` (--stemLinear), `stem_dim` (--stemDim; None: memDim) and `location`, `location_bias`, `location_dim`
    (--locationAware with --locationType "L" or "PE", --locationBias, --locationDim; None: off) -- defaults filled in.
    Location features with the linear stem, an unknown type, a dim < 1 or a non-finite bias raise ValueError."""
    geom = dict(STEM_GEOMETRY)
    extra = dict(stem[2]) if len(stem) > 2 and stem[2] is not None else {}
    unknown = sorted(set(extra) - set(geom))
    if unknown:
        raise ValueError("unknown stem geometry keys %s (known: %s)" % (unknown, sorted(geom)))
    geom.update(extra)
    if geom["linear"] and (geom["ksizes"] is not None or geom["stem_dim"] is not None
                           or geom["strides"] not in (None, [1], (1,))):
        raise ValueError("the linear stem is one 1x1 stride-1 layer: it takes no ksizes, strides or stem_dim, got %s" % extra)
    if geom["location"] is not None and geom["linear"]:
        raise ValueError("the linear stem takes no location features (the reference adds them in the CNN stem only)")
    stem_location(geom)
    return geom


def stem_location(geom):
    """The `Stem(location=)` of a filled-in geometry: None or the checked (type, bias, dim)."""
    from .stem import location_spec
    if geom["location"] is None:
        return None
    return location_spec((geom["location"], geom["location_bias"], geom["location_dim"]))


def model_parameters(cfg, netLength, seed, classifier=None, encoder=None, stem=None, param_values=None):
    """The variables of the model DPTrainer trains, initialised as the reference does from `seed`: (cell values -- the
    caller's `param_values` when given --, output / encoder / stem specs and values in one OrderedDict each, encoder specs,
    stem specs).  The last four are None where the model has no such part."""
    from .params import init_params
    extra_specs = extra_values = None
    if classifier is not None:
        from .output_unit import output_specs, init_output_params
        extra_specs = output_specs(cfg.ctrlDim, cfg.memDim, list(classifier[1]), classifier[0],
                                   **classifier_options(classifier))
        extra_values = init_output_params(extra_specs, seed=seed + 17, bias_scale=0.0)
    enc_specs = stem_specs_ = None
    if encoder is not None or stem is not None:
        import collections
        if classifier is None or encoder is None or stem is None:
            raise ValueError("the full model needs classifier=, encoder= and stem= together")
        from .encoder import encoder_specs, init_encoder_params
        from .stem import stem_specs, init_stem_params
        enc_specs = encoder_specs(encoder[0], encoder[1], cfg.ctrlDim, ctrl_dim=cfg.ctrlDim, bi=True)
        geom = stem_geometry(stem)
        stem_specs_ = stem_specs(stem[0], cfg.memDim, num_layers=stem[1], ksizes=geom["ksizes"], stem_dim=geom["stem_dim"],
                                 linear=geom["linear"], location=stem_location(geom))
        extra_specs = collections.OrderedDict(list(extra_specs.items()) + list(enc_specs.items())
                                              + list(stem_specs_.items()))
        extra_values = dict(extra_values)
        extra_values.update(init_encoder_params(enc_specs, seed=seed + 19, bias_scale=0.0))   # TF: zero biases
        extra_values.update(init_stem_params(stem_specs_, seed=seed + 23, bias_scale=0.0))
    if extra_specs is not None:
        from .output_unit import is_moving_stat
        # the classifier's stored batch-norm statistics last: the optimizer and the EMA run over the flat buffer before them
        import collections
        extra_specs = collections.OrderedDict([kv for kv in extra_specs.items() if not is_moving_stat(kv[0])]
                                              + [kv for kv in extra_specs.items() if is_moving_stat(kv[0])])
    if extra_specs is not None and param_values is None:
        param_values = init_params(cfg, netLength, seed=seed)
    return param_values, extra_specs, extra_values, enc_specs, stem_specs_


class DPTrainer(object):
    def __init__(self, cfg, netLength, param_values=None, seed=0, rank=0, world=1, lr=1e-4, clip=8.0, ema_decay=0.999,
                 beta1=0.9, beta2=0.999, eps=1e-8, dropouts=None, device="cuda", classifier=None, output_dropout=0.85,
                 encoder=None, stem=None, enc_dropouts=(0.85, 0.92), stem_dropout=0.82, prec="fp32", bwd_tc=False,
                 stem_prec="fp32", enc_prec="fp32"):
        """`classifier=(answerWordsNum, outClassifierDims)` adds the reference's output unit + answer loss
        (model.py:512-528, 547-576, 593-596), and `classifier=(answerWordsNum, outClassifierDims, options)` the one of
        the options {"question", "mul", "bn"} (--outQuestion, --outQuestionMul, --outputBN; `output_unit.output_options`,
        unknown keys raise ValueError).  With "bn" the stored statistics sit at the end of the flat buffer, from `n_train`:
        they get no gradient, clipping, Adam update or EMA shadow, and after each step every rank holds their mean over
        ranks (`allreduce_sum_with_stats_`); `encoder=(vocabulary rows, wrdEmbDim)` the question input unit
        (model.py:208-220, 279-307) and `stem=(imageInDim, stemNumLayers)` the image stem (model.py:165-204) -- or
        `stem=(imageInDim, stemNumLayers, geometry)` with the stem's kernel sizes, strides, linear form and width
        (`stem_geometry`) --, with the
        reference's training dropouts (config.py:202-206).  All variables join the same flat buckets, so the one
        all-reduce and the one fused optimizer pass cover the whole model (`train_step_full`).
        `prec="bf16"` runs the read unit's forward projections on tensor cores in training too (activations saved in bf16,
        widened for the backward); `bwd_tc=True` runs its six backward products on tensor cores (`mac_read_bwd_tc`).
        Both hold for every working flag combination, not only the shipped flag files: with read-unit flags outside the
        fused kernel the composed read unit's [B*N, .] products run on `mac_linear_tc_seg_fwd` / `mac_linear_bwd_tc`
        (memDim and attDim multiples of 128), and a cell differentiated on the tape (`tape.py`) runs its fused read unit
        backward on `mac_read_bwd_tc` (B*N a multiple of 64); the batch-sized products stay fp32 (DESIGN.md section 9).
        `prec="tc32"` trains the fused read unit's [B*N, .] products as split-bf16 tensor-core products inside the fp32
        parity bar (shipped flag files, memDim a multiple of 128, any B*N); with `bwd_tc=True` its backward products are
        split-bf16 too (`mac_read_bwd_tc32`), with `bwd_tc=False` they run on the fp32 `mac_read_bwd`.
        `stem_prec="bf16"` trains the image stem on tensor cores too (forward `mac_linear_tc_fwd`, backward
        `mac_conv3x3_bwd_tc`; every stem channel count must be a multiple of 128).  `enc_prec="bf16"` trains the question
        encoder's LSTM on tensor cores (`QuestionEncoder(prec="bf16")`; needs ctrlDim = 512, i.e. h = 256 per direction).
        `stem_prec="bf16x3"` trains the stem as split-bf16 tensor-core products inside the fp32 parity bar (the stem's
        counterpart of `prec="tc32"`: `mac_linear_tc32_fwd`, `mac_conv3x3_bwd_tc32`; same channel rule, independent of `prec`
        and `bwd_tc`).  The others are mixed precision: bf16 operands, fp32 accumulation, fp32 master weights / gradients /
        optimizer state (DESIGN.md section 9)."""
        from .mac_cell import MACParams, views_of
        check_model_precisions(cfg, encoder, stem, stem_prec, enc_prec)
        self.cfg, self.L, self.rank, self.world = cfg, netLength, rank, world
        self.prec, self.bwd_tc, self.stem_prec, self.enc_prec = prec, bool(bwd_tc), stem_prec, enc_prec
        self.lib = _lib.load()
        param_values, extra_specs, extra_values, self._enc_specs, self._stem_specs = model_parameters(
            cfg, netLength, seed, classifier, encoder, stem, param_values)
        self.params = MACParams(cfg, netLength, values=param_values, seed=seed, device=device, extra_specs=extra_specs,
                                extra_values=extra_values)   # replicated
        self.out = None
        self.n_train = self.params.numel      # the optimizer's and the EMA's elements of the flat buffer
        if classifier is not None:
            from .output_unit import OutputUnit, is_moving_stat
            self.out = OutputUnit({k: self.params.t[k] for k in extra_specs
                                   if k.startswith(("outputUnit/", "classifier/"))}, relu=cfg.relu, keep=output_dropout,
                                  seed=seed, version=lambda: self.params.version, bn_decay=cfg.bnDecay,
                                  **classifier_options(classifier))
            self._views_of = views_of
            tail = [self.params.offsets[k] for k in extra_specs if is_moving_stat(k)]
            self.n_train = min(tail) if tail else self.params.numel
        self.enc = self.stem = None
        if self._enc_specs is not None:
            from .encoder import QuestionEncoder
            from .stem import Stem
            self.enc = QuestionEncoder({k: self.params.t[k] for k in self._enc_specs}, keep_input=enc_dropouts[0],
                                       keep_question=enc_dropouts[1], seed=seed, prec=enc_prec,
                                       version=lambda: self.params.version)
            geom = self.stem_geometry = stem_geometry(stem)
            self.stem = Stem({k: self.params.t[k] for k in self._stem_specs}, relu=cfg.relu, prec=stem_prec, seed=seed,
                             version=lambda: self.params.version, strides=geom["strides"], linear=geom["linear"],
                             location=stem_location(geom))
            self.stem_dropout = float(stem_dropout)
            self._full_bufs = {}
        n = self.params.numel
        z = lambda: torch.zeros(n, dtype=torch.float32, device=self.params.device)
        self.bucket, self.adam_m, self.adam_v = z(), z(), z()
        self.ema = self.params.flat.clone()
        self.norm = torch.zeros(2, dtype=torch.float32, device=self.params.device)
        self.ows_bytes = int(self.lib.mac_optimizer_workspace_bytes())
        self.ows = torch.zeros(self.ows_bytes, dtype=torch.uint8, device=self.params.device)
        self.hp = dict(lr=lr, clip=clip, ema=ema_decay, b1=beta1, b2=beta2, eps=eps)
        self.dropouts = dropouts or (cfg.memoryDropout, cfg.readDropout, cfg.writeDropout)
        self.step_id = 0
        self.base_seed = seed
        self._cells = {}

    MAX_CACHED_CELLS = 4      # a save-for-backward cell holds L x (3 B N d + B d) floats (~1.2 GB at B=64, N=196, d=512, L=16)

    def cell_for(self, key, batch):
        """The training cell of shape-key `key`, fed with `batch`.

        The reference cell captures its input tensors at construction (mac_cell.py:59-79), and so does `MACCell`; the
        trainer therefore owns PERSISTENT input buffers per key and copies the caller's batch into them on every call, so
        a cached cell can never run on the tensors of an earlier batch (ADVICE r1).  A batch that already lives in these
        buffers (`full_forward_backward` writes into them directly) is not copied again.  At most MAX_CACHED_CELLS keys
        are kept (least recently used first out): callers with many distinct shapes -- e.g. one per trimmed question
        length -- should bucket / pad instead (attention masks the padding)."""
        from .mac_cell import MACCell
        names = ("vecQuestions", "questionWords", "questionCntxWords", "questionLengths", "knowledgeBase")
        ent = self._cells.pop(key, None)
        if ent is None:
            bufs = {}
            for n in names:
                src = batch[n]
                bufs[n] = src.to(torch.int32).clone().contiguous() if n == "questionLengths" else src.clone().contiguous()
            dm, dr, dw = self.dropouts
            cell = MACCell(bufs["vecQuestions"], bufs["questionWords"], bufs["questionCntxWords"], bufs["questionLengths"],
                           bufs["knowledgeBase"], dm, dr, dw, bufs["knowledgeBase"].shape[0], True, config=self.cfg,
                           params=self.params, prec=self.prec, save_for_backward=True)
            ent = (cell, bufs)
            while len(self._cells) >= self.MAX_CACHED_CELLS:
                old_key = next(iter(self._cells))
                del self._cells[old_key]
                if hasattr(self, "_full_bufs"):
                    self._full_bufs.pop(old_key, None)
        else:
            cell, bufs = ent
            for n in names:
                src = batch[n]
                if src.data_ptr() != bufs[n].data_ptr():
                    if tuple(src.shape) != tuple(bufs[n].shape):
                        raise ValueError("batch tensor %s has shape %s but key %r was built for %s"
                                         % (n, tuple(src.shape), key, tuple(bufs[n].shape)))
                    bufs[n].copy_(src)
        self._cells[key] = ent                 # (re-)insert as most recently used
        return ent[0]

    def grads(self, key, batch, t_control, t_memory, global_batch):
        """Forward + backward of the local shard into the flat bucket (not yet reduced)."""
        from .autograd import mac_backward
        from .mac_cell import mac_network
        cell = self.cell_for(key, batch)
        # per-(step, rank) dropout stream: masks differ across ranks and steps, reproducibly
        cell.seed = (self.base_seed * 1000003 + self.step_id * 7919 + self.rank * 104729 + 1) & 0x7FFFFFFFFFFFFFFF
        control, memory = mac_network(cell, self.L)
        scale = 1.0 / float(global_batch)
        g = mac_backward(cell, None if t_control is None else t_control * scale,
                         None if t_memory is None else t_memory * scale, bucket=self.bucket, tc=self.bwd_tc)
        return control, memory, g

    def apply(self):
        """all-reduce the bucket, then clip + Adam + EMA (model.py:645-667) in one fused pass; refresh derived weights."""
        allreduce_sum_with_stats_(self.bucket, self.params.flat, self.n_train)
        self.step_id += 1
        h = self.hp
        check(self.lib.mac_clip_adam_ema_step(ptr(self.params.flat), ptr(self.bucket), ptr(self.adam_m), ptr(self.adam_v),
                                              ptr(self.ema), self.n_train, 1.0, h["clip"], h["lr"], h["b1"], h["b2"],
                                              h["eps"], self.step_id, h["ema"], ptr(self.norm), ptr(self.ows),
                                              self.ows_bytes, stream_ptr()), "mac_clip_adam_ema_step")
        self.params.touch()

    def train_step_answers(self, key, batch, answers, global_batch):
        """One DP step on the reference's loss: cell forward -> output unit -> mean softmax-CE over the GLOBAL batch ->
        output-unit backward -> cell backward -> all-reduce -> clip/Adam/EMA.  Returns (logits, per-sample losses)."""
        from .autograd import mac_backward
        from .mac_cell import mac_network
        cell = self.cell_for(key, batch)
        cell.seed = (self.base_seed * 1000003 + self.step_id * 7919 + self.rank * 104729 + 1) & 0x7FFFFFFFFFFFFFFF
        self.out.seed = cell.seed
        control, memory = mac_network(cell, self.L)
        self.bucket.zero_()
        gviews = self._views_of(self.bucket, self.params.specs, self.params.offsets)
        logits, losses, _ = self.out.forward(memory, getattr(cell, "vecQuestions", batch["vecQuestions"]), answers, step=self.step_id,
                                             loss_scale=1.0 / float(global_batch))
        d_mem, d_q = torch.zeros_like(memory), torch.zeros_like(memory)
        self.out.backward(gviews, d_mem, d_q)
        mac_backward(cell, None, d_mem, bucket=self.bucket, zero_bucket=False, d_vecq=d_q, tc=self.bwd_tc)
        self.apply()
        return logits, losses

    def full_forward_backward(self, key, data, global_batch):
        """The reference's whole training graph (`MACnet.build`, model.py:774-821) on the local shard, gradients into the
        flat bucket (not yet reduced):  embeddings + bi-LSTM encoder -> stem -> netLength MAC steps -> output unit ->
        classifier -> mean softmax-CE over the GLOBAL batch, then the hand-written backward of each in reverse order.
        `data`: questions int32 [B,S] (0 = padding), questionLengths int32 [B], answers int32 [B], and the images as exactly
        one of `images` fp32 [B,H,W,C] (NHWC: the reference transposes its NCHW feed first, model.py:68) or `images_nchw`
        fp32 or fp16 [B,C,H,W], contiguous, as the features are stored (`Stem.forward_nchw`: the ingest kernel replaces the
        permute and, for the bf16 and bf16x3 stems, layer 0's patch pass; the same results bit for bit; fp16 features are
        widened on the device and give the step of `images_nchw.float()` bit for bit).  Returns (logits, per-sample losses).

        Several questions per image: with `imageIndex`, a contiguous int32 [B] tensor on the trainer's device, the images
        carry k <= B distinct rows and question b asks about image imageIndex[b], which must lie in [0, k) (the caller's
        contract; `serving.TrainPipeline(images=U)` checks it on the host).  The stem runs over the k images, so its
        dropout is drawn once per image -- image u gets the mask that batch row u gets without an index -- where the
        per-question step draws one per question.  `mac_kb_gather` writes each question's knowledge base into the cell's
        fp32 input, and after the cell's backward `mac_kb_gather_bwd` sums each image's knowledge-base gradient over its
        questions (fp32, ascending question order) for the stem's backward: the exact gradient of that objective.
        Everything after the stem -- the cell and its per-question read dropout, the encoder, the output unit, the loss --
        is the step without an index.  With imageIndex = arange(B) and all B images the step is that step bit for bit."""
        from .autograd import mac_backward
        from .mac_cell import mac_network
        if self.enc is None:
            raise RuntimeError("construct the trainer with classifier=, encoder= and stem=")
        if ("images" in data) == ("images_nchw" in data):
            raise ValueError("data needs exactly one of images (NHWC) and images_nchw, got %s"
                             % sorted(k for k in data if k.startswith("images")))
        nchw = data.get("images_nchw")
        if nchw is not None and (nchw.device != self.params.flat.device or nchw.dtype not in (torch.float32, torch.float16)
                                 or nchw.dim() != 4 or not nchw.is_contiguous()):
            raise ValueError("images_nchw must be a contiguous fp32 or fp16 [B, C, H, W] tensor on %s" % self.params.flat.device)
        idx = data.get("imageIndex")
        if idx is not None:
            self._check_image_index(idx, data["questions"].shape[0], (data["images"] if nchw is None else nchw).shape[0])
        seed = (self.base_seed * 1000003 + self.step_id * 7919 + self.rank * 104729 + 1) & 0x7FFFFFFFFFFFFFFF
        self.enc.seed = self.stem.seed = self.out.seed = seed
        words, cntx, vecq = self.enc.forward(data["questions"], data["questionLengths"], step=self.step_id,
                                             save_for_backward=True)
        if nchw is not None:
            kb = self.stem.forward_nchw(nchw, keep=self.stem_dropout, step=self.step_id, save_for_backward=True)
        else:
            kb = self.stem.forward(data["images"], keep=self.stem_dropout, step=self.step_id, save_for_backward=True)
        if idx is not None:
            kb_u, kb = kb, self._gather_kb(key, kb, idx)
        # the cell captures its inputs at construction (mac_cell.py:59-79): cell_for owns persistent buffers per key and
        # copies this step's encoder / stem outputs into them
        bufs = {"vecQuestions": vecq, "questionWords": words, "questionCntxWords": cntx, "knowledgeBase": kb,
                "questionLengths": data["questionLengths"]}
        cell = self.cell_for(key, bufs)
        cell.seed = seed
        control, memory = mac_network(cell, self.L)
        self.bucket.zero_()
        gviews = self._views_of(self.bucket, self.params.specs, self.params.offsets)
        logits, losses, _ = self.out.forward(memory, getattr(cell, "vecQuestions", vecq), data["answers"], step=self.step_id,
                                             loss_scale=1.0 / float(global_batch))
        d_mem, d_q = torch.zeros_like(memory), torch.zeros_like(memory)
        self.out.backward(gviews, d_mem, d_q)
        g = mac_backward(cell, None, d_mem, bucket=self.bucket, zero_bucket=False, d_vecq=d_q, tc=self.bwd_tc)
        d_kb = g["knowledgeBase"]
        if idx is not None:
            d_kb = self._sum_kb_grad(d_kb.contiguous(), idx, kb_u.shape[0])
        self.stem.backward(d_kb, gviews)
        if not self.cfg.controlContextual:
            raise NotImplementedError("the raw-word control inputs (controlContextual off) need wrdEmbDim == ctrlDim")
        self.enc.backward(g["questionCntxWords"], g["vecQuestions"], gviews)
        return logits, losses

    def _check_image_index(self, idx, B, k):
        """Refuse a malformed `imageIndex` or image count before any launch (no synchronise: the values are not read)."""
        dev = self.params.flat.device
        if not (torch.is_tensor(idx) and idx.dtype == torch.int32 and idx.is_cuda and idx.device == dev and idx.dim() == 1
                and idx.is_contiguous() and idx.shape[0] == B and idx.data_ptr() % 16 == 0):
            raise ValueError("imageIndex must be a contiguous, 16-byte aligned int32 tensor of shape [%d] on %s" % (B, dev))
        if not 1 <= k <= B:
            raise ValueError("with imageIndex the images carry 1..%d distinct rows (one per image), got %d" % (B, k))
        if self.cfg.memDim % 8:
            raise NotImplementedError("imageIndex needs memDim %% 8 == 0 (mac_kb_gather's 16-byte vectors), got %d"
                                      % self.cfg.memDim)

    def _gather_kb(self, key, kb_u, idx):
        """Each question's knowledge base from the k images' [k, N, d]: straight into the persistent buffer of `key`'s cell
        when it exists (so `cell_for` copies nothing), else into a new tensor that the new cell's buffer is made from."""
        B, (_, N, d) = idx.shape[0], kb_u.shape
        ent = self._cells.get(key)
        out = ent[1]["knowledgeBase"] if ent is not None else None
        if out is None or tuple(out.shape) != (B, N, d) or out.dtype != torch.float32:
            out = torch.empty((B, N, d), dtype=torch.float32, device=kb_u.device)
        check(self.lib.mac_kb_gather(ptr(kb_u), ptr(idx), ptr(out), 0, B, kb_u.shape[0], N, d, stream_ptr()),
              "mac_kb_gather")
        return out

    def _sum_kb_grad(self, d_kb, idx, k):
        """The k images' knowledge-base gradient [k, N, d]: each question's [B, N, d] row summed over its image's questions."""
        B, N, d = d_kb.shape
        out = torch.empty((k, N, d), dtype=torch.float32, device=d_kb.device)
        check(self.lib.mac_kb_gather_bwd(ptr(d_kb), ptr(idx), ptr(out), B, k, N, d, stream_ptr()), "mac_kb_gather_bwd")
        return out

    def train_step_full(self, key, data, global_batch):
        """One data-parallel step of the whole model: `full_forward_backward` -> all-reduce -> clip / Adam / EMA."""
        logits, losses = self.full_forward_backward(key, data, global_batch)
        self.apply()
        return logits, losses

    def train_step(self, key, batch, t_control, t_memory, global_batch):
        control, memory, _ = self.grads(key, batch, t_control, t_memory, global_batch)
        self.apply()
        return control, memory


def adam_reference(p, g, m, v, ema, step, lr=1e-4, clip=8.0, b1=0.9, b2=0.999, eps=1e-8, ema_decay=0.999):
    """numpy restatement of the fused step (tests): tf.clip_by_global_norm + tf.train.AdamOptimizer + EMA.apply."""
    p, g, m, v, ema = (np.asarray(a, np.float64) for a in (p, g, m, v, ema))
    norm = np.sqrt(np.sum(g * g))
    g = g * (clip / max(norm, clip))
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    lr_t = lr * np.sqrt(1 - b2 ** step) / (1 - b1 ** step)
    p = p - lr_t * m / (np.sqrt(v) + eps)
    ema = ema_decay * ema + (1 - ema_decay) * p
    return p, m, v, ema, norm
