"""Generate tests/golden/output_<layout>_<widths>_<mode>.npz: the UNMODIFIED reference's `MACnet.outputOp`, `MACnet.classifier`
and `addAnswerLossOp` (model.py:512-596) on the numpy TF1 shim, with --outQuestion on or off, --outQuestionMul and
--outputBN (batchNorm={"decay": bnDecay, "train": train}, model.py:96).

    python oracle/gen_output_options.py            # needs the reference checkout (build container only)

Layouts: q0 (question off), q1 (question on: the shipped flag files'), qmul (question and its product), each with and
without batch norm; classifier widths (), (8,) and (8, 6); at eval and in training (the reference's outputDropout 0.85).
With batch norm the fixture also holds each layer's stored statistics before ("initial/<name>") and after ("final/<name>")
the call: moved by the training call, untouched at eval.  The inputs and parameter values are drawn as
`gen_golden.run_output_case` draws them, so the q1_h8 fixtures carry the same values as output_eval / output_train."""
import importlib
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import gen_golden as gg                      # noqa: E402  (puts the shim and the reference on sys.path)

tf = gg.tf

LAYOUTS = {"q0": (False, False), "q1": (True, False), "qmul": (True, True)}
WIDTHS = {"h0": (), "h8": (8,), "h8_6": (8, 6)}
BN_DECAY = 0.9               # far enough from 1 that one update moves the statistics visibly


def cases():
    for lname, (question, mul) in LAYOUTS.items():
        for bn in (False, True):
            for wname, hidden in WIDTHS.items():
                for train in (False, True):
                    name = "output_%s%s_%s_%s" % (lname, "_bn" if bn else "", wname, "train" if train else "eval")
                    yield name, dict(train=train, hidden=hidden, question=question, mul=mul, bn=bn)


def run_case(name, train, hidden, question, mul, bn, seed=17, B=6, d=16, A=12, decay=BN_DECAY):
    ref_model = importlib.import_module("model")
    gg.set_reference_config("@args.txt", ["--outClassifierDims"] + [str(h) for h in hidden], dict(L=1, d=d), train)
    rc = gg._ref_config.config
    rc.answerWordsNum = A
    rc.outQuestion, rc.outQuestionMul, rc.outputBN, rc.bnDecay = question, mul, bn, decay
    from mac_network_b200.output_unit import init_output_params, output_specs
    specs = output_specs(d, d, list(hidden), A, question=question, mul=mul, bn=bn)
    params = init_output_params(specs, seed=seed, dtype=np.float64)
    rng = np.random.RandomState(seed + 1)
    memory, vecq = rng.standard_normal((B, d)), 0.5 * np.tanh(rng.standard_normal((B, d)))
    answers = rng.randint(0, A, size=(B,)).astype(np.int32)
    keep = rc.outputDropout if train else 1.0
    store = tf.reset_shim(values=params, seed=seed + 2, dtype=np.float64)
    me = types.SimpleNamespace(dropouts={"output": keep}, answerLossList=[],
                               batchNorm={"decay": rc.bnDecay, "train": train})          # model.py:96
    feats, dim = ref_model.MACnet.outputOp(me, tf.constant(memory), tf.constant(vecq), None, None)
    logits = ref_model.MACnet.classifier(me, feats, dim)
    loss, losses = ref_model.MACnet.addAnswerLossOp(me, logits, answers)
    created = {k: list(v.shape) for k, v in store.vars.items()}
    assert created == {k: list(v[0]) for k, v in specs.items()}, (created, specs)
    out = {"logits": np.asarray(logits), "losses": np.asarray(losses), "loss": np.asarray(loss),
           "memory": memory, "vecQuestions": vecq, "answers": answers}
    for i, u in enumerate(store.uniform_draws):
        out["uniform_%03d" % i] = u.astype(np.float64)
    for k, v in store.vars.items():
        if "/BatchNorm/moving_" in k:
            out["initial/" + k] = np.asarray(params[k], np.float64)
            out["final/" + k] = np.asarray(v, np.float64)
    meta = {"case": name, "train": train, "keep": keep, "B": B, "d": d, "A": A, "hidden": list(hidden), "param_seed": seed,
            "relu": rc.relu, "variables": created, "n_uniform": len(store.uniform_draws), "question": question, "mul": mul,
            "bn": bn, "bnDecay": rc.bnDecay}
    out["meta_json"] = np.frombuffer(json.dumps(meta, sort_keys=True).encode(), dtype=np.uint8)
    return out


def main():
    outdir = os.path.join(gg.ROOT, "tests", "golden")
    only = sys.argv[1:]
    for name, kw in cases():
        if only and name not in only:
            continue
        out = run_case(name, **kw)
        path = os.path.join(outdir, name + ".npz")
        np.savez_compressed(path, **out)
        print("%-28s %8.1f KB  draws=%d" % (name, os.path.getsize(path) / 1024.0,
                                             sum(k.startswith("uniform_") for k in out)))


if __name__ == "__main__":
    main()
