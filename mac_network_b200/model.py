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
                 device="cuda", **trainer_kw):
        """`vocab`: rows of the question-embedding variable (ids 1..vocab; 0 is padding); `answer_decoder`: optional
        id -> answer string (`answerDict.decodeId`, model.py:699).  `prec`: arithmetic of the evaluation forward."""
        self.cfg, self.L, self.prec, self.use_ema = cfg, netLength, prec, bool(use_ema)
        self.decode = answer_decoder
        self.trainer = DPTrainer(cfg, netLength, seed=seed, rank=rank, world=world, lr=lr, device=device,
                                 classifier=(n_answers, list(classifier_dims)), encoder=(vocab, wrd_emb_dim),
                                 stem=(image_in_dim, stem_layers), **trainer_kw)
        p = self.trainer.params
        t = self.trainer
        # evaluation-mode views of the same variables: every dropout at 1.0 (model.py:118-125)
        self._enc = QuestionEncoder({k: p.t[k] for k in t._enc_specs}, keep_input=1.0, keep_question=1.0)
        self._stem = Stem({k: p.t[k] for k in t._stem_specs}, relu=cfg.relu, prec=prec, version=lambda: p.version)
        self._out = OutputUnit({k: p.t[k] for k in p.specs if k.startswith(("outputUnit/", "classifier/"))}, relu=cfg.relu,
                               keep=1.0, version=lambda: p.version)
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
    def _to_device(self, data, images):
        q = np.ascontiguousarray(data["questions"], dtype=np.int32)
        dev = {"questions": torch.from_numpy(q).to(self.device),
               "questionLengths": torch.from_numpy(np.ascontiguousarray(data["questionLengths"], dtype=np.int32)).to(self.device),
               "answers": torch.from_numpy(np.ascontiguousarray(data["answers"], dtype=np.int32)).to(self.device)}
        img = images["images"]
        img = img if torch.is_tensor(img) else torch.from_numpy(np.ascontiguousarray(img, dtype=np.float32))
        # the reference feeds [B, C, H, W] and transposes to channels-last first (model.py:68)
        dev["images"] = img.to(self.device).permute(0, 2, 3, 1).contiguous()
        return dev

    def _swap_ema(self):
        """Evaluate on the EMA shadows (main.py:717-719): swap them with the live weights (and back)."""
        t = self.trainer
        tmp = t.params.flat.clone()
        t.params.flat.copy_(t.ema)
        t.ema.copy_(tmp)
        t.params.touch()
        self._out.invalidate()
        self._stem._packed.clear()

    # ------------------------------------------------------------------ model.py:732-760
    def runBatch(self, sess, data, images, train, getAtt=False):
        data = self.trimData(dict(data))
        time0 = time.time()
        dev = self._to_device(data, images)
        B, S = dev["questions"].shape
        time1 = time.time()
        t = self.trainer
        gradNorm = -1
        if train:
            logits, losses = t.train_step_full((B, S), dev, global_batch=B * t.world)
            self.macCell = t._cells[(B, S)][0]
            gradNorm = float(t.norm[0].item())
            self._out.invalidate()
            self._stem._packed.clear()
        else:
            if self.use_ema:
                self._swap_ema()
            try:
                words, cntx, vecq = self._enc.forward(dev["questions"], dev["questionLengths"])
                kb = self._stem.forward(dev["images"])
                cell = MACCell(vecq, words, cntx, dev["questionLengths"], kb, 1.0, 1.0, 1.0, B, False, config=self.cfg,
                               params=t.params, prec=self.prec)
                _, memory = mac_network(cell, self.L)
                logits, losses, _ = self._out.forward(memory, vecq, dev["answers"])
                self.macCell = cell
            finally:
                if self.use_ema:
                    self._swap_ema()
        preds = torch.argmax(logits, dim=-1).to(torch.int32)                      # model.py:605
        corrects = preds == dev["answers"]
        correctNum = int(corrects.sum().item())
        loss = float(losses.mean().item())
        time2 = time.time()
        H = W = int(round(np.sqrt(self.macCell.N)))
        attentionMaps = attention_maps(self.macCell, (H, W) if H * W == self.macCell.N else None) if getAtt else None
        predsList = self.buildPredsList(data, preds.cpu().numpy(), attentionMaps)
        return {"loss": loss, "correctNum": correctNum, "acc": correctNum / float(B), "preds": predsList,
                "gradNorm": gradNorm, "readTime": time1 - time0, "trainTime": time2 - time1}
