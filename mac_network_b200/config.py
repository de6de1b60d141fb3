"""Cell configuration: the slice of the reference's global `config` that the MAC cell reads.

Field names, defaults and choices follow `/root/reference/config.py:292-387` (network / control /
read / write flags), `config.py:202-213` (dropouts), `config.py:219-223` (relu, mulBias).  The
reference parses argparse flags *into a module-global singleton* (`config.py:92, 424`) that
`mac_cell.py`/`ops.py` read at graph-build time; `MACConfig` is that object for this package and
`from_args_file` accepts the reference's own `configs/args*.txt` (`@file` syntax, `config.py:96`).
"""
import dataclasses
from dataclasses import dataclass

# flags of the reference that crash in the reference itself (SURVEY.md Appendix C): rejected, not emulated
_BROKEN = {
    "addNullWord": "mac_cell.py:519,574 (method lacks self; questionLengths undefined)",
    "readCtrlConcatInter": "mac_cell.py:248-266 (dim not updated -> shape mismatch)",
    "writeGateShared": "mac_cell.py:359-367 ([B,d]*[B] does not broadcast)",
}


@dataclass
class MACConfig:
    # network (config.py:292-297)
    netLength: int = 16
    memDim: int = 512
    ctrlDim: int = 512
    attDim: int = 512
    unsharedCells: bool = False
    # initialization (config.py:300-303)
    initCtrl: str = "PRM"
    initMem: str = "PRM"
    initKBwithQ: str = "NON"
    addNullWord: bool = False
    # control unit (config.py:307-326)
    controlWholeQ: bool = False
    controlContinuous: bool = False
    controlContextual: bool = False
    controlInWordsProj: bool = False
    controlOutWordsProj: bool = False
    controlInputUnshared: bool = False
    controlInputAct: str = "TANH"
    controlFeedPrev: bool = False
    controlFeedPrevAtt: bool = False
    controlFeedInputs: bool = False
    controlContAct: str = "NON"
    controlConcatWords: bool = False
    controlProj: bool = False
    controlProjAct: str = "NON"
    # read unit (config.py:343-362)
    readProjInputs: bool = False
    readProjShared: bool = False
    readMemAttType: str = "MUL"
    readMemConcatKB: bool = False
    readMemConcatProj: bool = False
    readMemProj: bool = False
    readMemAct: str = "RELU"
    readCtrl: bool = False
    readCtrlAttType: str = "MUL"
    readCtrlConcatKB: bool = False
    readCtrlConcatProj: bool = False
    readCtrlConcatInter: bool = False
    readCtrlAct: str = "RELU"
    readSmryKBProj: bool = False
    # write unit (config.py:369-387)
    writeInputs: str = "BOTH"
    writeConcatMul: bool = False
    writeInfoProj: bool = False
    writeInfoAct: str = "NON"
    writeSelfAtt: bool = False
    writeSelfAttMod: str = "NON"
    writeMergeCtrl: bool = False
    writeMemProj: bool = False
    writeMemAct: str = "NON"
    writeGate: bool = False
    writeGateShared: bool = False
    writeGateBias: float = 1.0
    memoryBN: bool = False        # batch normalisation of the new memory (mac_cell.py:369-373; config.py:194-199)
    bnDecay: float = 0.999
    bnCenter: bool = False
    bnScale: bool = False
    # dropouts (config.py:202-213) and nonlinearity (config.py:219-223)
    memoryDropout: float = 0.85
    readDropout: float = 0.85
    writeDropout: float = 1.0
    memoryVariationalDropout: bool = False
    relu: str = "STD"
    mulBias: float = 0.0

    # ------------------------------------------------------------------ construction
    @classmethod
    def from_flags(cls, flags, **overrides):
        """`flags`: iterable of argparse tokens ("--relu=ELU", "--readCtrl", "--netLength", "4")."""
        fields = {f.name: f for f in dataclasses.fields(cls)}
        kw, ignored = {}, []
        toks = [t.strip() for t in flags if t.strip()]
        i = 0
        while i < len(toks):
            t = toks[i]
            i += 1
            if not t.startswith("--"):
                continue
            key, eq, val = t[2:].partition("=")
            if key not in fields:
                ignored.append(t)        # non-cell flag (--adam, --clip, --encBi ...)
                continue
            f = fields[key]
            if f.type in (bool, "bool") and key != "unsharedCells":
                kw[key] = True           # action="store_true"
                continue
            if not eq:
                val = toks[i]
                i += 1
            if key == "unsharedCells":   # type=bool in the reference: any non-empty string is True
                kw[key] = bool(val)
            else:
                kw[key] = type(f.default)(val)
        kw.update(overrides)
        cfg = cls(**kw)
        cfg.ignored_flags = ignored
        cfg.validate()
        return cfg

    @classmethod
    def from_args_file(cls, path, **overrides):
        with open(path) as fh:
            return cls.from_flags(fh.read().split(), **overrides)

    @classmethod
    def args(cls, variant="args", **overrides):
        """The shipped flag files (`/root/reference/configs/args{,1,2,3,4}.txt`), cell-relevant part."""
        common = ["--memoryVariationalDropout", "--relu=ELU", "--controlContextual", "--readProjInputs",
                  "--readMemConcatKB", "--readMemConcatProj", "--readMemProj", "--readCtrl", "--writeMemProj"]
        extra = {
            "args": ["--initCtrl=Q", "--controlInputUnshared"],
            "args2": ["--initCtrl=Q", "--controlInputUnshared"],
            "args1": ["--initCtrl=PRM", "--controlFeedPrev", "--controlFeedPrevAtt", "--controlFeedInputs",
                      "--controlContAct=TANH"],
            "args3": ["--initCtrl=Q", "--controlInputUnshared", "--writeSelfAtt", "--writeSelfAttMod=CONT"],
            "args4": ["--initCtrl=Q", "--controlInputUnshared", "--writeGate"],
            # BASELINE.json configs[4]: args3 U args4 on a 7x7 grid
            "gqa": ["--initCtrl=Q", "--controlInputUnshared", "--writeSelfAtt", "--writeSelfAttMod=CONT",
                    "--writeGate"],
        }[variant]
        return cls.from_flags(common + extra, **overrides)

    # ------------------------------------------------------------------ checks
    def validate(self):
        for k, why in _BROKEN.items():
            if getattr(self, k):
                raise NotImplementedError("--%s is broken/unsupported in the reference: %s" % (k, why))
        if self.initKBwithQ != "NON":
            raise NotImplementedError("--initKBwithQ crashes in the reference (mac_cell.py:564, ops.py:65)")
        if self.relu not in ("STD", "ELU"):
            raise NotImplementedError("--relu=%s: PRM adds per-call variables, LKY/SELU crash (ops.py:171-175)"
                                      % self.relu)
        for k in ("readMemAttType", "readCtrlAttType"):
            if getattr(self, k) not in ("MUL", "BL", "ADD"):
                raise NotImplementedError("--%s=DIAG crashes in the reference (ops.py:704-707)" % k)
        if self.readCtrl:
            dim = self.attDim if self.readProjInputs else self.memDim
            if not self.readMemProj and self.readMemConcatKB:
                dim += self.attDim if self.readMemConcatProj else self.memDim
            if dim != self.ctrlDim:
                raise NotImplementedError("readCtrl with interaction dim != ctrlDim: NameError in mac_cell.py:246")
        if self.readMemConcatKB and self.readMemConcatProj and not self.readProjInputs:
            raise NotImplementedError("concat.proj without proj: projVals unbound (ops.py:716)")
        if self.readSmryKBProj and not self.readProjInputs:
            raise NotImplementedError("readSmryKBProj needs readProjInputs (mac_cell.py:233, 271-272)")
        if self.readCtrlConcatKB and self.readCtrlConcatProj and not self.readProjInputs:
            raise NotImplementedError("readCtrlConcatProj needs readProjInputs (mac_cell.py:254-255)")
        if self.writeSelfAtt and self.writeSelfAttMod not in ("NON", "CONT"):
            raise ValueError("writeSelfAttMod")
        if not (self.memDim == self.ctrlDim):
            raise NotImplementedError("memDim != ctrlDim is outside the shipped configs")
        return self

    @property
    def is_fast_path(self):
        """True when the flag set is one the fused sm_90a kernels cover (the shipped args*.txt family)."""
        return (self.readProjInputs and not self.readProjShared and self.readMemConcatKB and self.readMemConcatProj
                and self.readMemProj and self.readCtrl and self.readMemAttType == "MUL"
                and self.readCtrlAttType == "MUL" and self.readMemAct == "RELU" and self.readCtrlAct == "RELU"
                and self.relu == "ELU" and not self.readCtrlConcatKB and not self.readSmryKBProj
                and self.mulBias == 0.0 and self.attDim == self.memDim)
