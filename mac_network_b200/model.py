"""Run surface of the reference's `MACnet` (`/root/reference/model.py`) over the sm_90a kernels: the one call the reference's
training / evaluation loop makes per batch,

    res = model.runBatch(sess, data, images, train, getAtt)          # model.py:732-760

with the same batch dictionaries (`data["questions"]` int ids padded with 0, `data["questionLengths"]`, `data["answers"]`,
optional `data["instances"]`; `images["images"]` float `[B, C, H, W]`) and the same result dictionary (`loss`, `correctNum`,
`acc`, `preds`, `gradNorm`, `readTime`, `trainTime`).  `sess` has no analogue (there is no graph session) and is accepted and
ignored so the reference's call sites read the same.

    build (model.py:762-829)      embeddings + bi-LSTM encoder -> stem -> netLength MAC steps -> output unit -> classifier
    train=True                    `DPTrainer.train_step_full`: train-mode dropouts (model.py:118-125), mean softmax-CE over the
                                  global batch, hand-written backward, ONE all-reduce, fused clip / Adam / EMA (model.py:645-667)
    train=False                   dropouts = 1.0, optionally the EMA shadow weights (main.py:717-719); the cell runs its
                                  inference form (tensor-core projections when prec="bf16")
    trimData (model.py:681-687)   questions trimmed to the longest question of the batch
    addPredOp (model.py:603-612)  predictions = argmax of the logits, correctNum, accuracy
    buildPredsList (693-710)      per-instance prediction + `attentions[key][step]` maps when getAtt

Composition only: every arithmetic step is a kernel of libmac_b200.so through the classes of this package."""
import time

import numpy as np
import torch

from .checkpoint import attention_maps
from .dp import DPTrainer
from .encoder import QuestionEncoder
from .mac_cell import MACCell, mac_network
from .output_unit import OutputUnit
from .stem import Stem


class MACnet(object):
    def __init__(self, cfg, netLength, vocab, n_answers, wrd_emb_dim=300, image_in_dim=1024, classifier_dims=(512,),
                 stem_layers=2, seed=0, rank=0, world=1, lr=1e-4, prec="bf16", use_ema=False, answer_decoder=None,
                 device="cuda", eval_stem_prec=None, eval_enc_prec=None, train_prec="fp32", stem_kernel_sizes=None,
                 stem_strides=None, stem_linear=False, stem_dim=None, stem_location=None, stem_location_bias=1.0,
                 stem_location_dim=32, out_question=True, out_question_mul=False, output_bn=False, **trainer_kw):
        """`vocab`: rows of the question-embedding variable (ids 1..vocab; 0 is padding); `answer_decoder`: optional
        id -> answer string (`answerDict.decodeId`, model.py:699).  `prec`: arithmetic of the evaluation forward; with
        "fp8" the cell's read step runs on e4m3 and the image stem in bf16.  `eval_stem_prec="fp8"` runs the evaluation
        stem in e4m3 (`Stem(prec="fp8")`) and `eval_stem_prec="bf16x3"` in split bf16 inside the fp32 parity bar
        (`Stem(prec="bf16x3")`), whatever `prec` is; None keeps the stem `prec` implies.  `eval_enc_prec="bf16"` runs
        the evaluation question encoder on tensor cores (`QuestionEncoder(prec="bf16")`); None keeps it fp32.  Training is
        unaffected (see `DPTrainer(enc_prec=)`).  `train_prec` is the training cell's arithmetic (`DPTrainer(prec=)`: "fp32",
        "bf16" or "tc32"); the other training precisions pass through as `DPTrainer` keywords (`bwd_tc`, `stem_prec`,
        `enc_prec`).  `stem_kernel_sizes`, `stem_strides`, `stem_linear` and `stem_dim` are the reference's
        --stemKernelSizes, --stemStrideSizes, --stemLinear and --stemDim (`dp.stem_geometry`); the knowledge base then has
        the stem's output grid (`Stem.grid`).  `stem_location` ("L" or "PE"; None: off), `stem_location_bias` and
        `stem_location_dim` are --locationAware with --locationType, --locationBias and --locationDim.
        `out_question`, `out_question_mul` and `output_bn` are the output unit's --outQuestion, --outQuestionMul and
        --outputBN (`DPTrainer(classifier=)`).  The default keeps the shipped flag files' output unit; note that the
        reference's own default for --outQuestion is off (a model trained without the flag files needs
        out_question=False), and that --outQuestionMul does nothing without --outQuestion.  With output_bn, evaluation
        (`runBatch(train=False)`) normalises with the stored statistics, which are not trainable: `use_ema=True` swaps the
        trained weights only, so evaluation reads the live statistics, as the reference's EMA (trainable variables only,
        model.py:658-667) does."""
        if eval_stem_prec not in (None, "fp8", "bf16x3"):
            raise ValueError("eval_stem_prec must be None, 'fp8' or 'bf16x3', got %r" % (eval_stem_prec,))
        if eval_enc_prec not in (None, "bf16"):
            raise ValueError("eval_enc_prec must be None or 'bf16', got %r" % (eval_enc_prec,))
        default_geometry = not stem_linear and all(int(k) == 3 for k in (stem_kernel_sizes or [3])) and \
            all(int(s) == 1 for s in (stem_strides or [1]))
        if eval_stem_prec == "fp8" and stem_location is not None:
            raise NotImplementedError("the fp8 stem does not run location features; use eval_stem_prec=None or 'bf16x3'")
        if eval_stem_prec == "fp8" and not default_geometry:
            raise NotImplementedError("the fp8 stem runs the 3x3 stride-1 geometry only, got kernel sizes %s, strides %s%s"
                                      % (stem_kernel_sizes, stem_strides, ", linear" if stem_linear else ""))
        self.cfg, self.L, self.prec, self.use_ema = cfg, netLength, prec, bool(use_ema)
        self.decode = answer_decoder
        self.trainer = DPTrainer(cfg, netLength, seed=seed, rank=rank, world=world, lr=lr, device=device,
                                 classifier=(n_answers, list(classifier_dims),
                                             {"question": out_question, "mul": out_question_mul, "bn": output_bn}),
                                 encoder=(vocab, wrd_emb_dim),
                                 stem=(image_in_dim, stem_layers, {"ksizes": stem_kernel_sizes, "strides": stem_strides,
                                                                   "linear": stem_linear, "stem_dim": stem_dim,
                                                                   "location": stem_location,
                                                                   "location_bias": stem_location_bias,
                                                                   "location_dim": stem_location_dim}),
                                 prec=train_prec, **trainer_kw)
        p = self.trainer.params
        t = self.trainer
        # evaluation-mode views of the same variables: every dropout at 1.0 (model.py:118-125)
        self._enc = QuestionEncoder({k: p.t[k] for k in t._enc_specs}, keep_input=1.0, keep_question=1.0,
                                    prec=eval_enc_prec or "fp32", version=lambda: p.version)
        stem_prec = eval_stem_prec or ("bf16" if prec == "fp8" else prec)
        self._stem = Stem({k: p.t[k] for k in t._stem_specs}, relu=cfg.relu, prec=stem_prec, version=lambda: p.version,
                          strides=t.stem.strides, linear=t.stem.linear, location=t.stem.location)
        self._out = OutputUnit({k: p.t[k] for k in p.specs if k.startswith(("outputUnit/", "classifier/"))}, relu=cfg.relu,
                               keep=1.0, version=lambda: p.version, bn_decay=cfg.bnDecay, **t.out.options)
        self.device = p.device
        self.macCell = None                      # the cell of the last batch (model.py:740 reads macCell.attentions)

    # ------------------------------------------------------------------ model.py:681-687
    @staticmethod
    def trim2DVectors(vectors, vectorsLengths):
        return vectors[:, :int(np.max(vectorsLengths))]

    def trimData(self, data):
        data["questions"] = self.trim2DVectors(data["questions"], data["questionLengths"])
        return data

    # ------------------------------------------------------------------ model.py:693-710
    def buildPredsList(self, data, predictions, attentionMaps):
        predsList = []
        instances = data.get("instances") or [{"index": i} for i in range(len(predictions))]
        for i, instance in enumerate(instances):
            instance = dict(instance)
            if predictions is not None:
                instance["prediction"] = self.decode(int(predictions[i])) if self.decode else int(predictions[i])
            if attentionMaps is not None:
                instance["attentions"] = {k: [step[i] for step in attentionMaps[k]] for k in attentionMaps}
            predsList.append(instance)
        return predsList

    # ------------------------------------------------------------------ feed (model.py:101-128, 68)
    @staticmethod
    def shared_images(images):
        """(rows, inverse) when `images["imageIds"]` (the reference's key, main.py:325-334) repeats an id, else None:
        `rows` are the batch rows that hold the first occurrence of each distinct id (in ascending id order), `inverse[b]`
        the position in `rows` of question b's image."""
        ids = images.get("imageIds") if isinstance(images, dict) else None
        if ids is None:
            return None
        ids = np.asarray(ids)
        _, rows, inverse = np.unique(ids, return_index=True, return_inverse=True)
        if len(rows) == len(ids):
            return None
        return rows, inverse.reshape(-1).astype(np.int32)

    def _to_device(self, data, images, rows=None):
        """`rows`: copy only these rows of the images (the first occurrence of each distinct image)."""
        q = np.ascontiguousarray(data["questions"], dtype=np.int32)
        dev = {"questions": torch.from_numpy(q).to(self.device),
               "questionLengths": torch.from_numpy(np.ascontiguousarray(data["questionLengths"], dtype=np.int32)).to(self.device),
               "answers": torch.from_numpy(np.ascontiguousarray(data["answers"], dtype=np.int32)).to(self.device)}
        img = images["images"]
        if rows is not None:
            img = img[torch.from_numpy(rows)] if torch.is_tensor(img) else np.asarray(img)[rows]
        img = img if torch.is_tensor(img) else torch.from_numpy(np.ascontiguousarray(img, dtype=np.float32))
        # the reference feeds [B, C, H, W] and transposes to channels-last first (model.py:68)
        dev["images"] = img.to(self.device).permute(0, 2, 3, 1).contiguous()
        return dev

    def _swap_ema(self):
        """Evaluate on the EMA shadows (main.py:717-719): swap them with the live weights (and back).  The EMA covers the
        trainable variables (`DPTrainer.n_train`), so the classifier's stored batch-norm statistics stay the live ones."""
        t = self.trainer
        n = t.n_train
        tmp = t.params.flat[:n].clone()
        t.params.flat[:n].copy_(t.ema[:n])
        t.ema[:n].copy_(tmp)
        t.params.touch()

    # ------------------------------------------------------------------ model.py:732-760
    def runBatch(self, sess, data, images, train, getAtt=False):
        data = self.trimData(dict(data))
        time0 = time.time()
        # evaluation with repeated imageIds: the stem runs once per distinct image and the cell gathers each question's
        # knowledge base (MACCell(kbIndex=)); training draws its dropouts per question, so it keeps one image per question
        shared = None if train else self.shared_images(images)
        dev = self._to_device(data, images, rows=None if shared is None else shared[0])
        B, S = dev["questions"].shape
        time1 = time.time()
        t = self.trainer
        gradNorm = -1
        if train:
            logits, losses = t.train_step_full((B, S), dev, global_batch=B * t.world)
            self.macCell = t._cells[(B, S)][0]
            gradNorm = float(t.norm[0].item())
        else:
            if self.use_ema:
                self._swap_ema()
            try:
                words, cntx, vecq = self._enc.forward(dev["questions"], dev["questionLengths"])
                kb = self._stem.forward(dev["images"])
                kbIndex = None if shared is None else torch.from_numpy(shared[1]).to(self.device)
                cell = MACCell(vecq, words, cntx, dev["questionLengths"], kb, 1.0, 1.0, 1.0, B, False, config=self.cfg,
                               params=t.params, prec=self.prec, kbIndex=kbIndex)
                _, memory = mac_network(cell, self.L)
                logits, losses, _ = self._out.forward(memory, vecq, dev["answers"], train=False)
                self.macCell = cell
            finally:
                if self.use_ema:
                    self._swap_ema()
        preds = torch.argmax(logits, dim=-1).to(torch.int32)                      # model.py:605
        corrects = preds == dev["answers"]
        correctNum = int(corrects.sum().item())
        loss = float(losses.mean().item())
        time2 = time.time()
        attentionMaps = attention_maps(self.macCell, self._stem.grid(*dev["images"].shape[1:3])) if getAtt else None
        predsList = self.buildPredsList(data, preds.cpu().numpy(), attentionMaps)
        return {"loss": loss, "correctNum": correctNum, "acc": correctNum / float(B), "preds": predsList,
                "gradNorm": gradNorm, "readTime": time1 - time0, "trainTime": time2 - time1}
