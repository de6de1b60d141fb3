"""ORACLE (test infrastructure only): differentiable fp64 PyTorch restatement of the cell, used to check the hand-written
backward -- the scheduled sweep of `autograd._Bwd` and the tape of `tape.py` -- against `torch.autograd` (the reference
itself uses TF autodiff, model.py:626-636).

It covers every flag `oracle/mac_oracle.py` implements and is ported from it function by function: `_Cell` has one method
per `MACOracle` method, with the same scopes, the same order of operations and the same dropout calls, so that it consumes
the uniform draws in the reference's call order exactly as `MACOracle.dropout` does.  Its forward is pinned to the numpy
oracle and to the fixtures in tests/test_oracle_golden.py and tests/test_tape_autograd_bounds.py."""
import torch

PREFIX = "MACnetwork/"
INF = 1e30          # ops.py:10


class _Cell(object):
    """`MACOracle` on fp64 torch tensors: `p` maps full variable names to leaf tensors."""

    def __init__(self, cfg, p, uniforms, dropouts, train, dev):
        self.cfg, self.p, self.dev, self.train = cfg, p, dev, train
        self.uniforms = iter(uniforms or [])
        self.dropouts = {"memory": dropouts[0], "read": dropouts[1], "write": dropouts[2]}

    def t64(self, a):
        return torch.as_tensor(a, dtype=torch.float64).to(self.dev)

    def var(self, scope, name):
        return self.p[PREFIX + scope + name]

    def act(self, kind, x):
        """ops.py:161-187 (`activations` dict with the `config.relu` switch)."""
        if kind == "NON":
            return x
        if kind == "TANH":
            return torch.tanh(x)
        if kind == "SIGMOID":
            return torch.sigmoid(x)
        if kind == "ELU":
            return torch.nn.functional.elu(x)
        if kind == "RELU":
            return torch.nn.functional.elu(x) if self.cfg.relu == "ELU" else torch.relu(x)
        raise ValueError(kind)

    def dropout(self, x, keep):
        """tf.nn.dropout (TF1): x/keep*floor(keep+U); exact identity at keep == 1 (no draw)."""
        if float(keep) == 1.0:
            return x
        u = self.t64(next(self.uniforms))
        assert tuple(u.shape) == tuple(x.shape), (u.shape, x.shape)
        return x / float(keep) * torch.floor(float(keep) + u)

    def linear(self, x, scope, name, in_dim, out_dim, act="NON", dropout=1.0, bias=0.0):
        """ops.py:298-333, with the nested `name_2` layer when act != NON; out_dim == 1 -> vector weight, row-dot."""
        sc = scope + "linearLayer" + name + "/"
        W = self.var(sc, "weights/weight")
        b = self.var(sc, "biases/bias") + float(bias)
        x = self.dropout(x, dropout)
        if out_dim > 1:
            assert tuple(W.shape) == (in_dim, out_dim), (sc, W.shape, in_dim, out_dim)
            y = torch.matmul(x, W) + b
        else:
            assert tuple(W.shape) == (in_dim,), (sc, W.shape, in_dim)
            y = torch.sum(x * W, dim=-1) + b
        y = self.act(act, y)
        if act != "NON":
            y = self.linear(y, sc, name + "_2", out_dim, out_dim)
        return y

    def inter2att(self, inter, scope, dim, dropout=1.0, name=""):
        """ops.py:114-120, 140-144 (sumMod = LIN)."""
        logits = self.linear(inter, scope + "inter2att" + name + "/inter2logits/", "logits", dim, 1, dropout=dropout)
        return torch.softmax(logits, dim=-1)

    def mul(self, x, y, dim, scope, name, proj=None, inter_mod="MUL", concat=None):
        """ops.py:668-725; returns (out, outDim, projectedX)."""
        sc = scope + "mul" + name + "/"
        orig_x, orig_dim = x, dim
        proj_x = None
        if proj is not None:
            x = self.dropout(x, proj["dropout"])
            y = self.dropout(y, proj["dropout"])
            xn, yn = ("proj", "proj") if proj["shared"] else ("projX", "projY")
            x = self.linear(x, sc, xn, dim, proj["dim"])
            y = self.linear(y, sc, yn, dim, proj["dim"])
            dim = proj["dim"]
            proj_x = x
        yb = y.unsqueeze(-2)
        if inter_mod == "MUL":
            mb = float(self.cfg.mulBias)
            out = (x + mb) * (yb + mb)
        elif inter_mod == "BL":
            out = torch.matmul(x, self.var(sc, "weights/weight")) * yb + self.var(sc, "biases/bias")
        elif inter_mod == "ADD":
            out = torch.tanh(x + yb)
        else:
            raise NotImplementedError(inter_mod)
        if concat and concat.get("x"):
            cx, cd = (proj_x, dim) if concat.get("proj", False) else (orig_x, orig_dim)
            out = torch.cat([out, cx], dim=-1)
            dim += cd
        return out, dim, proj_x

    # -------------------------------------------------------------- state init
    def init_state(self, name, dim, init_type, B):
        """mac_cell.py:496-505."""
        if init_type == "PRM":
            return self.var("", name).unsqueeze(0).expand(B, dim)
        if init_type == "ZERO":
            return torch.zeros((B, dim), dtype=torch.float64, device=self.dev)
        return self.vecQuestions

    def zero_state(self, vecQuestions, questionWords, questionCntxWords, questionLengths, knowledgeBase):
        """mac_cell.py:59-79 + 539-592."""
        c = self.cfg
        self.vecQuestions, self.knowledgeBase = vecQuestions, knowledgeBase
        B = vecQuestions.shape[0]
        c0 = self.init_state("initCtrl", c.ctrlDim, c.initCtrl, B)
        m0 = self.init_state("initMem", c.memDim, c.initMem, B)
        self.controls, self.memories = c0.unsqueeze(1), m0.unsqueeze(1)
        self.contControl = c0
        words = questionCntxWords if c.controlContextual else questionWords
        self.inWords = self.outWords = words
        if c.controlInWordsProj or c.controlOutWordsProj:
            pw = self.linear(words, "", "wordsProj", c.ctrlDim, c.ctrlDim)
            self.inWords = pw if c.controlInWordsProj else words
            self.outWords = pw if c.controlOutWordsProj else words
        S = words.shape[1]
        valid = (torch.arange(S, device=self.dev).unsqueeze(0) < questionLengths.unsqueeze(1)).double()
        self.mask = (1 - valid) * (-INF)                                           # ops.py:243-247
        if c.memoryVariationalDropout:
            keep = float(self.dropouts["memory"])                                    # ops.py:1054-1059
            self.memDpMask = (torch.ones((B, c.memDim), dtype=torch.float64, device=self.dev) if keep == 1.0
                              else torch.floor(keep + self.t64(next(self.uniforms))))
        return c0, m0

    # -------------------------------------------------------------- units
    def control(self, controlInput, inWords, outWords, control, contControl, name=""):
        """mac_cell.py:133-187."""
        c = self.cfg
        sc = "MACCell/control" + name + "/"
        dim = c.ctrlDim
        new_cont = controlInput
        if c.controlFeedPrev:
            new_cont = control if c.controlFeedPrevAtt else contControl
            if c.controlFeedInputs:
                new_cont = torch.cat([new_cont, controlInput], dim=-1)
                dim += c.ctrlDim
            new_cont = self.linear(new_cont, sc, "contControl", dim, c.ctrlDim, act=c.controlContAct)
            dim = c.ctrlDim
        inter = new_cont.unsqueeze(1) * inWords
        if c.controlConcatWords:
            inter = torch.cat([inter, inWords], dim=-1)
            dim += c.ctrlDim
        if c.controlProj:
            inter = self.linear(inter, sc, "", dim, c.ctrlDim, act=c.controlProjAct)
            dim = c.ctrlDim
        logits = self.linear(inter, sc + "inter2logits/", "logits", dim, 1)
        att = torch.softmax(logits + self.mask, dim=-1)
        self.att_question = att
        new_control = (att.unsqueeze(-1) * outWords).sum(-2)
        if c.controlContinuous:
            new_control = new_cont
        return new_control, new_cont

    def read(self, knowledgeBase, memory, control, name=""):
        """mac_cell.py:209-277."""
        c = self.cfg
        sc = "MACCell/read" + name + "/"
        dim = c.memDim
        if c.memoryVariationalDropout:
            memory = memory / float(self.dropouts["memory"]) * self.memDpMask     # ops.py:1065-1067
        else:
            memory = self.dropout(memory, self.dropouts["memory"])
        proj = None
        if c.readProjInputs:
            proj = {"dim": c.attDim, "shared": c.readProjShared, "dropout": self.dropouts["read"]}
            dim = c.attDim
        inter, inter_dim, projectedKB = self.mul(
            knowledgeBase, memory, c.memDim, sc, "memInter", proj=proj, inter_mod=c.readMemAttType,
            concat={"x": c.readMemConcatKB, "proj": c.readMemConcatProj})
        if c.readMemProj:
            inter = self.linear(inter, sc, "memKbProj", inter_dim, dim, act=c.readMemAct)
        else:
            dim = inter_dim
        if c.readCtrl:
            inter, _, _ = self.mul(inter, control, dim, sc, "ctrlInter", inter_mod=c.readCtrlAttType, concat={"x": False})
            if c.readCtrlConcatKB:
                if c.readCtrlConcatProj:
                    added, added_dim = projectedKB, c.attDim
                else:
                    added, added_dim = knowledgeBase, c.memDim
                inter = torch.cat([inter, added], dim=-1)
                dim += added_dim
            inter = self.act(c.readCtrlAct, inter)
        att = self.inter2att(inter, sc, dim, dropout=self.dropouts["read"])
        self.att_kb = att
        if c.readSmryKBProj:
            knowledgeBase = projectedKB
        return (att.unsqueeze(-1) * knowledgeBase).sum(-2)

    def write(self, memory, info, control, contControl, name=""):
        """mac_cell.py:305-375."""
        c = self.cfg
        sc = "MACCell/write" + name + "/"
        if c.writeInfoProj:
            info = self.linear(info, sc, "info", c.memDim, c.memDim)
        info = self.act(c.writeInfoAct, info)
        if c.writeSelfAtt:
            self_control = contControl if c.writeSelfAttMod == "CONT" else control
            self_control = self.linear(self_control, sc, "ctrlProj", c.ctrlDim, c.ctrlDim)
            inter = self.controls * self_control.unsqueeze(1)
            att = self.inter2att(inter, sc, c.ctrlDim, name="selfAttention")
            self_smry = (att.unsqueeze(-1) * self.memories).sum(-2)
        new_mem, dim = memory, c.memDim
        if c.writeInputs == "INFO":
            new_mem = info
        elif c.writeInputs == "SUM":
            new_mem = new_mem + info
        elif c.writeInputs == "BOTH":
            parts = [new_mem, info] + ([new_mem * info] if c.writeConcatMul else [])
            new_mem = torch.cat(parts, dim=-1)
            dim = dim * len(parts)
        if c.writeSelfAtt:
            new_mem = torch.cat([new_mem, self_smry], dim=-1)
            dim += c.memDim
        if c.writeMergeCtrl:
            new_mem = torch.cat([new_mem, control], dim=-1)
            dim += c.memDim
        if c.writeMemProj or dim != c.memDim:
            new_mem = self.linear(new_mem, sc, "newMemory", dim, c.memDim)
        new_mem = self.act(c.writeMemAct, new_mem)
        if c.writeGate:
            z = torch.sigmoid(self.linear(control, sc, "gate", c.ctrlDim, c.memDim, bias=c.writeGateBias))
            new_mem = new_mem * z + memory * (1 - z)
        if c.memoryBN:
            new_mem = self.batch_norm(new_mem, sc + "BatchNorm/")
        return new_mem

    def batch_norm(self, x, scope):
        """mac_cell.py:370-373 (TF 1.x batch_norm, epsilon 0.001): batch mean and biased variance in training, the stored
        statistics otherwise.  The stored statistics are not trainable (no gradient); their moving update in training is
        not restated, since nothing in one forward reads it."""
        c, eps = self.cfg, 1e-3
        P = PREFIX + scope
        beta = self.p[P + "beta"] if c.bnCenter else 0.0
        gamma = self.p[P + "gamma"] if c.bnScale else 1.0
        if self.train:
            mean = x.mean(dim=0)
            var = ((x - mean) ** 2).mean(dim=0)
        else:
            mean, var = self.p[P + "moving_mean"], self.p[P + "moving_variance"]
        return (x - mean) / torch.sqrt(var + eps) * gamma + beta

    # -------------------------------------------------------------- one step
    def step(self, i, control, memory):
        """mac_cell.py:420-480."""
        c = self.cfg
        in_name_u = ("qInput%d" % i) if c.controlInputUnshared else "qInputU"
        cell_name = str(i) if c.unsharedCells else ""
        ci = self.linear(self.vecQuestions, "MACCell/", "qInput", c.ctrlDim, c.ctrlDim)
        ci = self.act(c.controlInputAct, ci)
        ci = self.linear(ci, "MACCell/", in_name_u, c.ctrlDim, c.ctrlDim)
        new_control, self.contControl = self.control(ci, self.inWords, self.outWords, control, self.contControl,
                                                     name=cell_name)
        if c.controlWholeQ:
            new_control = self.vecQuestions
        info = self.read(self.knowledgeBase, memory, new_control, name=cell_name)
        if c.writeDropout < 1.0:          # python-level test on the *config* value (mac_cell.py:461)
            info = self.dropout(info, self.dropouts["write"])
        new_memory = self.write(memory, info, new_control, self.contControl, name=cell_name)
        self.controls = torch.cat([self.controls, new_control.unsqueeze(1)], dim=1)
        self.memories = torch.cat([self.memories, new_memory.unsqueeze(1)], dim=1)
        return new_control, new_memory, info


def graph(cfg, p, x, lengths, L, dropouts=(1.0, 1.0, 1.0), uniforms=None, train=False, trace=None):
    """The cell's L steps as a differentiable graph: `p` maps full variable names to fp64 tensors, `x` holds the fp64
    "vecQuestions", "questionWords", "questionCntxWords" and "knowledgeBase", `lengths` the question lengths (long), all on
    one device.  Returns (control_L, memory_L) tensors; every uniform of `uniforms` must be consumed.  `trace`: a list that
    receives, per step, numpy copies of the control, memory and retrieved info and of the question and knowledge-base
    attention maps ("att_question" [B, S], "att_kb" [B, N])."""
    cell = _Cell(cfg, p, uniforms, dropouts, train, x["knowledgeBase"].device)
    control, memory = cell.zero_state(x["vecQuestions"], x["questionWords"], x["questionCntxWords"], lengths,
                                      x["knowledgeBase"])
    for i in range(L):
        control, memory, info = cell.step(i, control, memory)
        if trace is not None:
            trace.append({k: v.detach().cpu().numpy() for k, v in (("control", control), ("memory", memory),
                                                                    ("info", info), ("att_question", cell.att_question),
                                                                    ("att_kb", cell.att_kb))})
    assert next(cell.uniforms, None) is None, "uniform draws left over: the dropout calls differ from the reference's"
    return control, memory


def run(cfg, params_np, inputs_np, L, dropouts=(1.0, 1.0, 1.0), uniforms=None, d_control=None, d_memory=None,
        train=False, device="cpu", trace=None):
    """Returns (control_L, memory_L, grads) as numpy arrays, with grads keyed like the product's `mac_backward` output:
    every parameter (zeros for the stored batch-norm statistics), "knowledgeBase", the words key ("questionCntxWords" with
    controlContextual, else "questionWords") and "vecQuestions".  `train`: the cell's train argument (memoryBN only);
    `device`: where the fp64 arithmetic runs; `trace`: a list that receives each step's control, memory, info and attention
    maps (see `graph`)."""
    dev = torch.device(device)
    t64 = lambda a: torch.as_tensor(a, dtype=torch.float64).to(dev)
    p = {k: t64(v).requires_grad_("/BatchNorm/moving_" not in k) for k, v in params_np.items()}
    words_key = "questionCntxWords" if cfg.controlContextual else "questionWords"
    x = {k: t64(inputs_np[k]) for k in ("vecQuestions", "questionWords", "questionCntxWords", "knowledgeBase")}
    for k in ("vecQuestions", words_key, "knowledgeBase"):
        x[k].requires_grad_(True)
    lengths = torch.as_tensor(inputs_np["questionLengths"]).long().to(dev)
    control, memory = graph(cfg, p, x, lengths, L, dropouts, uniforms, train, trace)
    grads = {}
    if d_control is not None or d_memory is not None:
        loss = 0.0
        if d_control is not None:
            loss = loss + (control * t64(d_control)).sum()
        if d_memory is not None:
            loss = loss + (memory * t64(d_memory)).sum()
        leaves = list(p.items()) + [(k, x[k]) for k in ("knowledgeBase", words_key, "vecQuestions")]
        need = [(k, v) for k, v in leaves if v.requires_grad]
        got = torch.autograd.grad(loss, [v for _, v in need], allow_unused=True)
        by_name = {k: g for (k, _), g in zip(need, got)}
        for k, v in leaves:
            g = by_name.get(k)
            grads[k] = (g if g is not None else torch.zeros_like(v)).detach().cpu().numpy()
    return control.detach().cpu().numpy(), memory.detach().cpu().numpy(), grads
