"""Question input unit -- the producer of the control unit's inputs (SURVEY.md section 8(f), "next" row 3):
`MACnet.qEmbeddingsOp` (`model.py:208-220`) and `MACnet.encoder` (`model.py:279-307`) = `ops.RNNLayer`/`biRNNLayer`
(`ops.py:859-952`): word-embedding lookup (index 0 = padding row of zeros), dropout on the embedded sequence
(`encInputDropout`), a (bi)directional `BasicLSTMCell` of `encDim/2` units per direction under
`tf.nn.bidirectional_dynamic_rnn(sequence_length=questionLengths)`, dropout on the question vector (`qDropout`), and the
optional `projCW` / `projQ` linears (`encProj`, or `encDim != ctrlDim`).

    questionWords      [B,S,E]      = emb[qIndices]
    questionCntxWords  [B,S,encDim] = [h_fw(t), h_bw(t)], zero for t >= length
    vecQuestions       [B,encDim]   = dropout([h_fw(len-1), h_bw(0)])

GPU formulation (csrc/encoder.cu): the input half of both LSTM kernels is one GEMM each over all S steps
(`mac_linear_fwd`), the recurrence is one launch per step for both directions with the gate math, the length masking and
the backward direction's per-row time reversal fused behind the `[B,h] x [h,4h]` product; BPTT mirrors it and turns the
weight / input gradients of all steps into GEMMs over the `[B*S, 4h]` gate-gradient matrix.  Variable names follow the
reference's scopes (`qEmbeddings/emb`, `encoder/birnnLayer/bidirectional_rnn/{fw,bw}/basic_lstm_cell/{kernel,bias}`)."""
import collections
import ctypes

import numpy as np
import torch

from . import _lib
from ._lib import check, ptr, stream_ptr

SITE_ENC_INPUT = 48       # Philox sites of the encoder's two dropouts
SITE_ENC_QUESTION = 49
ENC = "encoder/birnnLayer/bidirectional_rnn/"
ENC_UNI = "encoder/rnnLayer/rnn/"          # ops.fwRNNLayer (encBi off): scope "rnnLayer", dynamic_rnn's default "rnn"


def encoder_specs(vocab, wrd_emb_dim, enc_dim, ctrl_dim=None, bi=True, proj=False):
    """OrderedDict name -> (shape, initialiser kind).  `vocab` = rows of the variable (the padding row is not stored)."""
    s = collections.OrderedDict()
    s["qEmbeddings/emb"] = ((vocab, wrd_emb_dim), "emb_uniform")
    h = enc_dim // 2 if bi else enc_dim
    for d in (("fw", "bw") if bi else ("",)):
        sc = (ENC + d + "/") if bi else ENC_UNI
        s[sc + "basic_lstm_cell/kernel"] = ((wrd_emb_dim + h, 4 * h), "xavier")
        s[sc + "basic_lstm_cell/bias"] = ((4 * h,), "zeros")
    ctrl_dim = enc_dim if ctrl_dim is None else ctrl_dim
    if proj or enc_dim != ctrl_dim:                                        # model.py:786
        for name in ("projCW", "projQ"):
            s["encoder/linearLayer%s/weights/weight" % name] = ((enc_dim, ctrl_dim), "xavier")
            s["encoder/linearLayer%s/biases/bias" % name] = ((ctrl_dim,), "zeros")
    return s


def init_encoder_params(specs, seed=0, dtype=np.float32, bias_scale=0.1, emb_scale=1.0):
    """Embeddings U(-scale, scale) (`wrdEmbRandom` + `wrdEmbUniform`, preprocess.py:583-588); LSTM kernels glorot-uniform
    (TF's default initialiser); biases perturbed away from TF's zeros so that bias handling is exercised."""
    rng = np.random.RandomState(seed)
    out = collections.OrderedDict()
    for name, (shape, kind) in specs.items():
        if kind == "zeros":
            v = bias_scale * rng.standard_normal(shape)
        elif kind == "emb_uniform":
            v = rng.uniform(-emb_scale, emb_scale, size=shape)
        else:
            lim = np.sqrt(6.0 / (shape[0] + shape[1]))
            v = rng.uniform(-lim, lim, size=shape)
        out[name] = np.asarray(v, dtype=dtype)
    return out


class QuestionEncoder(object):
    """Forward / backward of the question input unit on device tensors.  `params` (and `grads` for backward): dict
    TF-name -> CUDA fp32 tensor (e.g. views into the trainer's flat buckets)."""

    def __init__(self, params, keep_input=1.0, keep_question=1.0, seed=0, forget_bias=1.0):
        self.lib = _lib.load()
        self.p = params
        self.keep_input, self.keep_question, self.seed = float(keep_input), float(keep_question), int(seed)
        self.forget_bias = float(forget_bias)
        self.bi = (ENC + "fw/basic_lstm_cell/kernel") in params
        self.scopes = [ENC + "fw/", ENC + "bw/"] if self.bi else [ENC_UNI]
        self.ndir = len(self.scopes)
        k0 = params[self.scopes[0] + "basic_lstm_cell/kernel"]
        self.h = k0.shape[1] // 4
        self.E = k0.shape[0] - self.h
        self.V = params["qEmbeddings/emb"].shape[0]
        if self.E != params["qEmbeddings/emb"].shape[1]:
            raise ValueError("LSTM kernel rows do not match the embedding width")
        self.proj = "encoder/linearLayerprojCW/weights/weight" in params
        self.device = k0.device
        self._lws_bytes = 4096 + 32 * 64 * 4096 * 4
        self._lws = torch.zeros(self._lws_bytes, dtype=torch.uint8, device=self.device)
        self._saved = None

    # ------------------------------------------------------------------ helpers over the C ABI
    def _new(self, *shape):
        return torch.empty(shape, dtype=torch.float32, device=self.device)

    def _linear(self, xs, W, b, out, n_out=None):
        n = len(xs)
        arr_p = (ctypes.c_void_p * n)(*[x.data_ptr() for x in xs])
        arr_k = (ctypes.c_int * n)(*[x.shape[1] for x in xs])
        arr_ld = (ctypes.c_int * n)(*[x.stride(0) for x in xs])
        n_out = W.shape[1] if n_out is None else n_out
        check(self.lib.mac_linear_fwd(arr_p, arr_k, arr_ld, n, ptr(W), ptr(b), 0.0, 0, ptr(out), out.stride(0),
                                      xs[0].shape[0], n_out, ptr(self._lws), self._lws_bytes, stream_ptr()), "mac_linear_fwd")
        return out

    def _linear_bwd(self, xs, Wt, dy, dxs, dx_accum, dW, db):
        n = len(xs)
        arr_p = (ctypes.c_void_p * n)(*[x.data_ptr() for x in xs])
        arr_k = (ctypes.c_int * n)(*[x.shape[1] for x in xs])
        arr_ld = (ctypes.c_int * n)(*[x.stride(0) for x in xs])
        arr_dx = (ctypes.c_void_p * n)(*[None if t is None else t.data_ptr() for t in dxs])
        arr_lddx = (ctypes.c_int * n)(*[0 if t is None else t.stride(0) for t in dxs])
        arr_acc = (ctypes.c_int * n)(*[int(a) for a in dx_accum])
        check(self.lib.mac_linear_bwd(arr_p, arr_k, arr_ld, n, ptr(Wt), ptr(dy), dy.stride(0), arr_dx, arr_lddx, arr_acc,
                                      ptr(dW), ptr(db), xs[0].shape[0], dy.shape[1], ptr(self._lws), self._lws_bytes,
                                      stream_ptr()), "mac_linear_bwd")

    # ------------------------------------------------------------------ forward
    def forward(self, qIndices, questionLengths, step=0, save_for_backward=False):
        """qIndices int32 [B,S] (0 = padding), questionLengths int32 [B] (1 <= len <= S).
        Returns (questionWords [B,S,E], questionCntxWords [B,S,D], vecQuestions [B,D])."""
        if not (qIndices.is_cuda and qIndices.dtype == torch.int32 and qIndices.is_contiguous()):
            raise ValueError("qIndices must be a contiguous CUDA int32 tensor")
        lengths = questionLengths.to(torch.int32).contiguous()
        B, S = qIndices.shape
        E, h, nd = self.E, self.h, self.ndir
        words = self._new(B, S, E)
        x = self._new(B, S, E) if self.keep_input < 1.0 else words
        check(self.lib.mac_embed_fwd(ptr(self.p["qEmbeddings/emb"]), ptr(qIndices), self.keep_input, self.seed,
                                     SITE_ENC_INPUT, step, ptr(words) if x is not words else None, ptr(x), B, S, self.V, E,
                                     stream_ptr()), "mac_embed_fwd")
        x2 = x.view(B * S, E)
        gx, Wh = [], []
        for sc in self.scopes:
            K = self.p[sc + "basic_lstm_cell/kernel"]
            gx.append(self._linear([x2], K, self.p[sc + "basic_lstm_cell/bias"], self._new(B * S, 4 * h)))   # rows 0..E-1 of K
            Wh.append(K[E:])
        cntx = self._new(B, S, nd * h)
        vecq = self._new(B, nd * h)
        sg = sc_ = shp = None
        if save_for_backward:
            sg, sc_, shp = self._new(nd, B * S, 4 * h), self._new(nd, B * S, h), self._new(nd, B * S, h)
        wsb = int(self.lib.mac_lstm_workspace_bytes(B, h, nd))
        ws = torch.empty(wsb, dtype=torch.uint8, device=self.device)
        check(self.lib.mac_lstm_fwd(ptr(gx[0]), ptr(gx[1]) if nd == 2 else None, ptr(Wh[0]), ptr(Wh[1]) if nd == 2 else None,
                                    ptr(lengths), self.forget_bias, ptr(cntx), ptr(vecq), ptr(sg), ptr(sc_), ptr(shp),
                                    ptr(ws), wsb, B, S, h, nd, stream_ptr()), "mac_lstm_fwd")
        if self.keep_question < 1.0:                                                       # model.py:297
            check(self.lib.mac_dropout_fwd(ptr(vecq), self.keep_question, self.seed, SITE_ENC_QUESTION, step, ptr(vecq),
                                           vecq.numel(), stream_ptr()), "mac_dropout_fwd")
        cntx_out, vecq_out = cntx, vecq
        if self.proj:                                                                      # model.py:300-305
            Wc, bc = self.p["encoder/linearLayerprojCW/weights/weight"], self.p["encoder/linearLayerprojCW/biases/bias"]
            Wq, bq = self.p["encoder/linearLayerprojQ/weights/weight"], self.p["encoder/linearLayerprojQ/biases/bias"]
            cntx_out = self._linear([cntx.view(B * S, nd * h)], Wc, bc, self._new(B * S, Wc.shape[1])).view(B, S, -1)
            vecq_out = self._linear([vecq], Wq, bq, self._new(B, Wq.shape[1]))
        if save_for_backward:
            self._saved = dict(qIndices=qIndices, lengths=lengths, x2=x2, sg=sg, sc=sc_, shp=shp, cntx=cntx, vecq=vecq,
                               step=step, B=B, S=S, ws=ws, wsb=wsb)
        return words, cntx_out, vecq_out

    # ------------------------------------------------------------------ backward
    def backward(self, d_cntx, d_vecq, grads):
        """Accumulates (+=) the parameter gradients into `grads` (dict name -> tensor, zeroed once per step by the
        caller).  d_cntx [B,S,D] / d_vecq [B,D]: gradients w.r.t. questionCntxWords / vecQuestions."""
        sv = self._saved
        if sv is None:
            raise RuntimeError("forward(save_for_backward=True) must run first")
        B, S, E, h, nd = sv["B"], sv["S"], self.E, self.h, self.ndir
        d_cntx = d_cntx.contiguous()
        d_vecq = d_vecq.contiguous()
        if self.proj:
            Wc, Wq = self.p["encoder/linearLayerprojCW/weights/weight"], self.p["encoder/linearLayerprojQ/weights/weight"]
            dc, dq = self._new(B * S, nd * h), self._new(B, nd * h)
            self._linear_bwd([sv["cntx"].view(B * S, nd * h)], Wc.t().contiguous(), d_cntx.view(B * S, -1), [dc], [0],
                             grads["encoder/linearLayerprojCW/weights/weight"], grads["encoder/linearLayerprojCW/biases/bias"])
            self._linear_bwd([sv["vecq"]], Wq.t().contiguous(), d_vecq, [dq], [0],
                             grads["encoder/linearLayerprojQ/weights/weight"], grads["encoder/linearLayerprojQ/biases/bias"])
            d_cntx, d_vecq = dc.view(B, S, nd * h), dq
        if self.keep_question < 1.0:                 # gradient through tf.nn.dropout: the same mask and 1/keep
            dq = self._new(B, nd * h)
            check(self.lib.mac_dropout_fwd(ptr(d_vecq), self.keep_question, self.seed, SITE_ENC_QUESTION, sv["step"],
                                           ptr(dq), dq.numel(), stream_ptr()), "mac_dropout_fwd")
            d_vecq = dq
        Ks = [self.p[sc + "basic_lstm_cell/kernel"] for sc in self.scopes]
        dG = [self._new(B * S, 4 * h) for _ in range(nd)]
        check(self.lib.mac_lstm_bwd(ptr(Ks[0][E:]), ptr(Ks[1][E:]) if nd == 2 else None, ptr(sv["lengths"]), ptr(sv["sg"]),
                                    ptr(sv["sc"]), ptr(d_cntx), ptr(d_vecq), ptr(dG[0]), ptr(dG[1]) if nd == 2 else None,
                                    ptr(sv["ws"]), sv["wsb"], B, S, h, nd, stream_ptr()), "mac_lstm_bwd")
        dx = self._new(B * S, E)
        for i, sc in enumerate(self.scopes):
            # dKernel += [dropout(X), h_prev]^T @ dG;  dBias += colsum(dG);  dX (+)= dG @ kernel[0:E]^T
            self._linear_bwd([sv["x2"], sv["shp"][i]], Ks[i].t().contiguous(), dG[i], [dx, None], [1 if i else 0, 0],
                             grads[sc + "basic_lstm_cell/kernel"], grads[sc + "basic_lstm_cell/bias"])
        check(self.lib.mac_embed_bwd(ptr(dx), ptr(sv["qIndices"]), self.keep_input, self.seed, SITE_ENC_INPUT, sv["step"],
                                     ptr(grads["qEmbeddings/emb"]), B, S, self.V, E, stream_ptr()), "mac_embed_bwd")

    def dropout_uniforms(self, B, S, step=0):
        """The uniforms the kernels draw, in the reference's call order (input sequence, question vector): for the oracle."""
        out = []
        for keep, site, shape in ((self.keep_input, SITE_ENC_INPUT, (B, S, self.E)),
                                  (self.keep_question, SITE_ENC_QUESTION, (B, self.ndir * self.h))):
            if keep < 1.0:
                u = torch.empty(shape, dtype=torch.float32, device=self.device)
                check(self.lib.mac_dropout_uniform(self.seed, site, step, ptr(u), u.numel(), stream_ptr()), "uniform")
                out.append(u.cpu().numpy().astype(np.float64))
        return out
