"""Backward pass of the MAC cell over the kernels of csrc/backward.cu (fp32 path).

The reference gets its gradients from TF autodiff over the unrolled graph (`model.py:626-636`); here the reverse
sweep is explicit: for i = L-1 .. 0: write-unit backward -> read-unit backward, then ONE control-attention backward for
all L steps (the control chain is memory-independent with `controlFeedPrev` off), then the question projections.
Math: SURVEY.md Appendix E.  Gradients are returned keyed by the reference's TF variable names, plus the three inputs
the enclosing model trains through (`knowledgeBase` -> stem, `questionCntxWords` / `vecQuestions` -> encoder).

Usage:
    cell = MACCell(..., train=True, save_for_backward=True)
    control, memory = mac_network(cell, L)
    grads = mac_backward(cell, d_control, d_memory)        # dict name -> tensor
"""
import collections
import ctypes

import torch

from . import _lib, packs
from ._lib import act_code, check, ptr, stream_ptr
from .params import PREFIX


# the forms of the read unit's backward (csrc/backward.cu): fp32 FMA pipe, bf16 tensor cores, split-bf16 tensor cores
READ_BWD = {"fp32": "mac_read_bwd", "tc": "mac_read_bwd_tc", "tc32": "mac_read_bwd_tc32"}


def read_bwd_workspace_bytes(lib, form, B, N, d):
    return int(getattr(lib, READ_BWD[form] + "_workspace_bytes")(B, N, d))


def read_bwd(lib, form, cell, i, kb, control, rw, Wt, dinfo, grads, ws, ws_bytes):
    """The read unit's backward of step i in `form`.  Wt(name) gives the transposed fp32 weight "Wx", "Wy", "Wm" or "Wm2" (the
    tensor-core forms read only Wy's); grads are the 13 gradient outputs dkb .. dbr_part in the order of the C ABI."""
    wt = ("Wx", "Wy", "Wm", "Wm2") if form == "fp32" else ("Wy",)
    check(getattr(lib, READ_BWD[form])(ptr(kb), ptr(cell._mem_in_hist[i]), ptr(control), ctypes.byref(rw),
                                       *[ptr(Wt(k)) for k in wt], ptr(cell._att_kb[i]), ptr(cell._save[i]), ptr(dinfo),
                                       float(cell.dropouts["read"]), cell.seed, i, *[ptr(g) for g in grads], ptr(ws), ws_bytes,
                                       cell.B, cell.N, cell.d, stream_ptr()), READ_BWD[form])


class _Bwd(object):
    def __init__(self, cell, bucket=None, zero_bucket=True, tc=False):
        self.cell, self.lib = cell, cell.lib
        # tc: the read unit's six big products on wgmma tensor cores (mac_read_bwd_tc) instead of the fp32 FMA GEMMs
        self.tc = bool(tc)
        # a tc32 cell keeps its forward's accuracy class in backward: split-bf16 products (mac_read_bwd_tc32, any B*N)
        self.tc32 = self.tc and cell.prec == _lib.PREC["tc32"]
        check_backward(cell, tc)
        self.form = "tc32" if self.tc32 else "tc" if self.tc else "fp32"
        self.p = cell.params
        c = cell.cfg
        if c.controlWholeQ or c.controlContinuous:
            raise NotImplementedError("backward covers the shipped flag files (args, args1, args2, args3, args4, GQA)")
        self.recurrent = bool(c.controlFeedPrev)
        if self.recurrent and c.writeSelfAtt and c.writeSelfAttMod == "CONT":
            raise NotImplementedError("backward of controlFeedPrev together with writeSelfAttMod=CONT")
        self.B, self.N, self.d, self.L = cell.B, cell.N, cell.d, cell.L
        dev = cell.device
        self.z = lambda *s: torch.zeros(s, dtype=torch.float32, device=dev)
        self.e = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)
        # parameter gradients are views into ONE flat bucket laid out like MACParams.flat (what NCCL all-reduces)
        from .mac_cell import views_of
        self.bucket = bucket if bucket is not None else torch.zeros_like(self.p.flat)
        if bucket is not None and zero_bucket:
            self.bucket.zero_()
        self.g = views_of(self.bucket, self.p.specs, self.p.offsets)
        cache = getattr(cell, "_bwd_ws", None)            # scratch is allocated once per cell and reused every step
        if cache is not None and cache[4] != self.form:
            cache = None
        if cache is None:
            ws_bytes = read_bwd_workspace_bytes(self.lib, self.form, self.B, self.N, self.d)
            lws_bytes = 4096 + 32 * 1536 * 512 * 4
            cache = (ws_bytes, torch.zeros(ws_bytes, dtype=torch.uint8, device=dev), lws_bytes,
                     torch.zeros(lws_bytes, dtype=torch.uint8, device=dev), self.form)
            cell._bwd_ws = cache
        self.ws_bytes, self.ws, self.lws_bytes, self.lws = cache[:4]

    def G(self, name):
        return self.g[PREFIX + name]

    def lin_names(self, scope, name):
        sc = scope + "linearLayer" + name + "/"
        return sc + "weights/weight", sc + "biases/bias"

    def linear_bwd(self, xs, wname, bname, dy, dxs, accum, wgrad=True):
        """ops.linear backward: xs/dxs lists of 2-D views (dxs entries may be None).  wgrad=False: data gradients only (the
        weight / bias gradients of this call are formed later, batched over the steps)."""
        Wt = self.p.cache.pack(packs.transposed, self.p[wname]) if any(d is not None for d in dxs) else None
        _lib.linear_bwd(xs, Wt, dy, dxs, accum, self.G(wname) if wgrad else None,
                        self.G(bname) if (bname and wgrad) else None, self.lws, self.lws_bytes, stream_ptr())

    def axpy(self, dst, src, alpha=1.0):
        check(self.lib.mac_axpy(ptr(dst), ptr(src), float(alpha), src.numel(), stream_ptr()), "mac_axpy")

    def colsum_B(self, part, out_flat):
        """out[k] += sum_b part[b, k]"""
        Bp, d = part.shape
        check(self.lib.mac_colsum(ptr(part), ptr(out_flat), 1, Bp, d, 1, stream_ptr()), "mac_colsum")

    def run(self, d_control, d_memory, d_vecq=None):
        cell, c, lib = self.cell, self.cell.cfg, self.lib
        B, N, d, L = self.B, self.N, self.d, self.L
        z, e = self.z, self.e
        S = cell.inWords.shape[1]
        gC, gM = z(L + 1, B, d), z(L + 1, B, d)          # gradients w.r.t. the history slots c_0..c_L, m_0..m_L
        if d_control is not None:
            gC[L].copy_(d_control)
        if d_memory is not None:
            gM[L].copy_(d_memory)
        dkb = z(B, N, d)
        dwords = z(B, S, d)
        dq = z(B, d)
        if d_vecq is not None:          # e.g. from the output unit (model.py:519), which also consumes vecQuestions
            dq.copy_(d_vecq)
        unshared = c.controlInputUnshared
        dci = z(B, L * d) if unshared else z(B, d)       # gradient w.r.t. ci_i (cell._ci layout)
        du_rec = z(B, d)                                  # recurrent control: gradient w.r.t. u accumulated over the steps
        part = {k: z(B, d) for k in ("wr", "bx", "bm", "bm2", "wc", "ws")}
        spart = {k: z(B) for k in ("br", "bc", "bs")}
        tmp_dm, tmp_dpre, dinfo, dss, dsc, dmem_in, tmp2 = (e(B, d) for _ in range(7))
        wsc = "MACCell/write/"
        rsc = "MACCell/read/"
        rw = cell._read_weights("")
        nWx, nbx = self.lin_names(rsc + "mulmemInter/", "projX")
        nWy, nby = self.lin_names(rsc + "mulmemInter/", "projY")
        nWm, nbm = self.lin_names(rsc, "memKbProj")
        nWm2, nbm2 = self.lin_names(rsc + "linearLayermemKbProj/", "memKbProj_2")
        wnames = {"Wx": nWx, "Wy": nWy, "Wm": nWm, "Wm2": nWm2}
        Wt = lambda k: self.p.cache.pack(packs.transposed, self.p[wnames[k]])
        keep_m, keep_w = cell.dropouts["memory"], cell.dropouts["write"]
        hc, hm, hi = cell._hc, cell._hm, cell._hi

        for i in reversed(range(L)):
            cell.iteration = i
            g_m = gM[i + 1]
            control = hc[i + 1]
            # ---------------- write unit backward (mac_cell.py:305-375)
            dmp = g_m
            if c.writeGate:
                check(lib.mac_gate_bwd(ptr(g_m), ptr(cell._gate[i]), ptr(cell._mnew[i]), ptr(hm[i]), ptr(tmp_dm), ptr(gM[i]),
                                       ptr(tmp_dpre), B * d, stream_ptr()), "mac_gate_bwd")
                nW, nb = self.lin_names(wsc, "gate")
                self.linear_bwd([control], nW, nb, tmp_dpre, [gC[i + 1]], [1])
                dmp = tmp_dm
            nW, nb = self.lin_names(wsc, "newMemory")
            xs = [hm[i], hi[i + 1]] + ([cell._ss[i]] if c.writeSelfAtt else [])
            dxs = [gM[i], dinfo] + ([dss] if c.writeSelfAtt else [])
            # without a gate the gradient of the write unit's output IS the history slot gM[i+1], which nothing modifies
            # afterwards: its weight / bias gradient over all L steps is ONE [L*B]-row product after the loop
            defer_w = not c.writeGate
            self.linear_bwd(xs, nW, nb, dmp, dxs, [1, 0] + ([0] if c.writeSelfAtt else []), wgrad=not defer_w)
            if c.writeSelfAtt:
                lsc = wsc + "inter2attselfAttention/inter2logits/linearLayerlogits/"
                check(lib.mac_control_attend_bwd(ptr(cell._sc[i]), 0, d, ptr(hc), d, B * d, ptr(hm), d, B * d,
                                                 ptr(self.p[lsc + "weights/weight"]), ptr(cell.attentions["self"][i]),
                                                 ptr(dss), 0, d, ptr(gC), ptr(gM), ptr(dsc), 0, d, 0, ptr(part["ws"]),
                                                 ptr(spart["bs"]), 1, B, i + 1, d, stream_ptr()), "self-att bwd")
                nW, nb = self.lin_names(wsc, "ctrlProj")
                if c.writeSelfAttMod == "CONT":
                    x = cell._ci[:, i * d:(i + 1) * d] if unshared else cell._ci
                    dx = dci[:, i * d:(i + 1) * d] if unshared else dci
                else:
                    x, dx = control, gC[i + 1]
                self.linear_bwd([x], nW, nb, dsc, [dx], [1])
            if c.writeDropout < 1.0 and keep_w < 1.0:                    # mac_cell.py:461-463
                check(lib.mac_dropout_fwd(ptr(dinfo), keep_w, cell.seed, _lib.SITE_WRITE_INFO, i, ptr(dinfo), B * d,
                                          stream_ptr()), "dropout bwd")
            # ---------------- read unit backward (mac_cell.py:209-277)
            read_bwd(lib, self.form, cell, i, cell.knowledgeBase, control, rw, Wt, dinfo,
                     [dkb, dmem_in, gC[i + 1], self.G(nWx), part["bx"], self.G(nWy), self.G(nby), self.G(nWm), part["bm"],
                      self.G(nWm2), part["bm2"], part["wr"], spart["br"]], self.ws, self.ws_bytes)
            # memory_in = (variational) dropout of m_{i-1}  (mac_cell.py:214-217)
            if keep_m < 1.0:
                site, st = (_lib.SITE_MEM_VAR, 0) if c.memoryVariationalDropout else (_lib.SITE_MEM_PLAIN, i)
                check(lib.mac_dropout_fwd(ptr(dmem_in), keep_m, cell.seed, site, st, ptr(tmp2), B * d, stream_ptr()), "dp")
                self.axpy(gM[i], tmp2)
            else:
                self.axpy(gM[i], dmem_in)

            if self.recurrent:
                self._control_step_bwd(i, gC, dwords, du_rec, part, spart, S)

        if not c.writeGate:             # deferred weight / bias gradient of write/newMemory (see the loop): K = L*B rows at once
            nW, nb = self.lin_names(wsc, "newMemory")
            LB = L * B
            xs = [hm[:L].reshape(LB, d), hi[1:L + 1].reshape(LB, d)] + ([cell._ss.reshape(LB, d)] if c.writeSelfAtt else [])
            self.linear_bwd(xs, nW, nb, gM[1:L + 1].reshape(LB, d), [None] * len(xs), [0] * len(xs))
        lsc = "MACCell/control/inter2logits/linearLayerlogits/"
        if self.recurrent:
            return self._finish(gC, gM, dkb, dwords, dq, du_rec, part, spart, rsc, wsc, lsc, nbx, nbm, nbm2)
        # ---------------- control unit, all L steps in one launch (mac_cell.py:155-181)
        cc_t, cc_b = (d, L * d) if unshared else (0, d)
        check(lib.mac_control_attend_bwd(ptr(cell._ci), cc_t, cc_b, ptr(cell.inWords), S * d, d, ptr(cell.outWords), S * d, d,
                                         ptr(self.p[lsc + "weights/weight"]), ptr(cell._att_q), ptr(gC[1:]), B * d, d,
                                         ptr(dwords), ptr(dwords), ptr(dci), cc_t, cc_b, 1, ptr(part["wc"]),
                                         ptr(spart["bc"]), L, B, S, d, stream_ptr()), "control bwd")
        # ---------------- question projections (mac_cell.py:442-448)
        u = cell._u_saved
        du = z(B, d)
        if unshared:
            # one backward against the packed [d, L*d] weight; gradients scattered back to the per-step variables
            Wc, bc = self.p.q_input_cat()
            gW, gb = torch.zeros_like(Wc), torch.zeros_like(bc)
            _lib.linear_bwd([u], self.p.cache.pack(packs.transposed, Wc), dci, [du], [0], gW, gb, self.lws, self.lws_bytes,
                            stream_ptr())
            for i in range(L):
                nW, nb = self.lin_names("MACCell/", "qInput%d" % i)
                self.G(nW).copy_(gW[:, i * d:(i + 1) * d])
                self.G(nb).copy_(gb[i * d:(i + 1) * d])
        else:
            nW, nb = self.lin_names("MACCell/", "qInputU")
            self.linear_bwd([u], nW, nb, dci, [du], [0])
        return self._finish(gC, gM, dkb, dwords, dq, du, part, spart, rsc, wsc, lsc, nbx, nbm, nbm2)

    def _control_step_bwd(self, i, gC, dwords, du_rec, part, spart, S):
        """Recurrent control unit of step i (mac_cell.py:141-181 with controlFeedPrev):
        cc_i = linear_2(act(linear_1([prev, ci_i]))), c_i = attention(cc_i); ci_i = linear_qInputU/qInput{i}(u)."""
        cell, c, lib = self.cell, self.cell.cfg, self.lib
        B, d = self.B, self.d
        prev, ci, hidden, cc = cell._ctrl_saved[i]
        sc = "MACCell/control/"
        lsc = sc + "inter2logits/linearLayerlogits/"
        dcc = self.e(B, d)
        check(lib.mac_control_attend_bwd(ptr(cc), 0, d, ptr(cell.inWords), S * d, d, ptr(cell.outWords), S * d, d,
                                         ptr(self.p[lsc + "weights/weight"]), ptr(cell._att_q[i]), ptr(gC[i + 1]), 0, d,
                                         ptr(dwords), ptr(dwords), ptr(dcc), 0, d, 0, ptr(part["wc"]), ptr(spart["bc"]),
                                         1, B, S, d, stream_ptr()), "control bwd")
        dy = dcc
        if c.controlContAct != "NON":
            nW2, nb2 = self.lin_names(sc + "linearLayercontControl/", "contControl_2")
            dh = self.e(B, d)
            self.linear_bwd([hidden], nW2, nb2, dcc, [dh], [0])
            dpre = self.e(B, d)
            check(lib.mac_activation_bwd(ptr(hidden), ptr(dh), act_code(c.controlContAct, c.relu), ptr(dpre), B * d,
                                         stream_ptr()), "act bwd")
            dy = dpre
        nW, nb = self.lin_names(sc, "contControl")
        dci = self.e(B, d)
        # prev = c_{i-1} (controlFeedPrevAtt) lives in history slot i; the continuous variant feeds cc_{i-1}
        if not c.controlFeedPrevAtt:
            raise NotImplementedError("backward of controlFeedPrev without controlFeedPrevAtt")
        if c.controlFeedInputs:
            self.linear_bwd([prev, ci], nW, nb, dy, [gC[i], dci], [1, 0])
        else:
            self.linear_bwd([prev], nW, nb, dy, [gC[i]], [1])
            dci.zero_()
        nameU = ("qInput%d" % i) if c.controlInputUnshared else "qInputU"
        nWu, nbu = self.lin_names("MACCell/", nameU)
        self.linear_bwd([cell._u_saved], nWu, nbu, dci, [du_rec], [1])

    def _finish(self, gC, gM, dkb, dwords, dq, du, part, spart, rsc, wsc, lsc, nbx, nbm, nbm2):
        cell, c, lib = self.cell, self.cell.cfg, self.lib
        B, d = self.B, self.d
        u = cell._u_saved
        dpre = self.e(B, d)
        check(lib.mac_activation_bwd(ptr(u), ptr(du), act_code(c.controlInputAct, c.relu), ptr(dpre), B * d, stream_ptr()),
              "act bwd")
        nW, nb = self.lin_names("MACCell/", "qInput")
        self.linear_bwd([cell.vecQuestions], nW, nb, dpre, [dq], [1])
        # ---------------- initial state (mac_cell.py:496-505)
        for name, kind, gslot in (("initCtrl", c.initCtrl, gC[0]), ("initMem", c.initMem, gM[0])):
            if kind == "PRM":
                self.colsum_B(gslot, self.G(name))
            elif kind == "Q":
                self.axpy(dq, gslot)
        # ---------------- reduce the per-sample partial sums over the batch
        self.colsum_B(part["wr"], self.G(rsc + "inter2att/inter2logits/linearLayerlogits/weights/weight"))
        self.colsum_B(part["bx"], self.G(nbx))
        self.colsum_B(part["bm"], self.G(nbm))
        self.colsum_B(part["bm2"], self.G(nbm2))
        self.colsum_B(part["wc"], self.G(lsc + "weights/weight"))
        self.colsum_B(spart["br"].view(B, 1), self.G(rsc + "inter2att/inter2logits/linearLayerlogits/biases/bias").view(1))
        self.colsum_B(spart["bc"].view(B, 1), self.G(lsc + "biases/bias").view(1))
        if c.writeSelfAtt:
            ssc = wsc + "inter2attselfAttention/inter2logits/linearLayerlogits/"
            self.colsum_B(part["ws"], self.G(ssc + "weights/weight"))
            self.colsum_B(spart["bs"].view(B, 1), self.G(ssc + "biases/bias").view(1))
        out = collections.OrderedDict(self.g)
        out["knowledgeBase"] = dkb
        out["questionCntxWords" if c.controlContextual else "questionWords"] = dwords
        out["vecQuestions"] = dq
        return out


def check_backward(cell, tc):
    """Refuses, before any launch, a backward `mac_backward(cell, ..., tc=tc)` cannot run: the shape rules of the tensor-core
    forms.  Needs only the constructed cell, so a caller can check before its forward."""
    if getattr(cell, "_use_tape", False):
        if tc:
            # tensor cores on the tape: the composed read unit's [B*N, .] linears (mac_linear_bwd_tc, any B*N) and the fused
            # read unit (mac_read_bwd_tc); everything else on the tape stays on its fp32 kernels
            if cell.prec != _lib.PREC["bf16"]:
                raise NotImplementedError("the tape backward runs the fp32 kernels")
            if cell._fused_read and (cell.d % 128 or (cell.B * cell.N) % 64):
                raise NotImplementedError("tensor-core backward needs d % 128 == 0 and (B*N) % 64 == 0")
        return
    tc32 = tc and cell.prec == _lib.PREC["tc32"]
    if tc32 and cell.d % 128:
        raise NotImplementedError("split-bf16 tensor-core backward needs d % 128 == 0")
    if tc and not tc32 and (cell.d % 128 or (cell.B * cell.N) % 64):
        raise NotImplementedError("tensor-core backward needs d % 128 == 0 and (B*N) % 64 == 0")


def mac_backward(cell, d_control, d_memory, bucket=None, zero_bucket=True, d_vecq=None, tc=False):
    """Gradients of sum(d_control * control_L) + sum(d_memory * memory_L) w.r.t. every cell parameter and input.
    `tc=True`: the read unit's projections on tensor cores in backward too (bf16 operands, fp32 accumulation)."""
    if not getattr(cell, "save_for_backward", False):
        raise RuntimeError("construct the MACCell with save_for_backward=True and run the forward first")
    if getattr(cell, "_tape", None) is not None:       # flags outside the hand-scheduled sweep: node-by-node (tape.py)
        check_backward(cell, tc)
        return cell._tape.run(d_control, d_memory, bucket, zero_bucket, d_vecq, tc=tc)
    return _Bwd(cell, bucket, zero_bucket, tc=tc).run(d_control, d_memory, d_vecq)
