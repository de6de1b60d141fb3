"""Every form of the read unit's backward (mac_read_bwd, mac_read_bwd_tc, mac_read_bwd_tc32: csrc/backward.cu) through this
tree's library and an earlier commit's, on the same inputs and pre-filled accumulators, compared bit for bit, with the
number of kernel launches per call.
Usage:  python profiles/read_bwd_forms_equal.py OUT_DIR --base-lib PATH

  --base-lib   the earlier commit's libmac_b200.so; the library this tree's build() made is the other side.  Both are loaded
               into one process.
Shapes: the headline (B=64, N=196, d=512) and the GQA shape (B*N = 3136) for every form, (5, 49, 128) for tc32 (B*N = 245 is
not a multiple of 64) and (3, 7, 20) for fp32 (d not a multiple of 128).  Each form runs at keep_read 1 and 0.85, and at 0.85
with dkb = NULL (the products of dKB skipped) and, for fp32, with dWm2 = NULL (its weight gradient skipped).  `save` and the
attention come from one fp32 mac_read_fwd of this tree's library.  The 13 outputs (the gradients into the pre-filled
accumulators, dmem_in into a NaN-filled buffer) are compared byte for byte, and each library runs every case twice, which
tells a difference between them from run-to-run variation.  Writes OUT_DIR/read_bwd_forms_equal.json."""
import argparse
import ctypes
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mac_network_b200 import _lib as L_  # noqa: E402
from profiles.read_fwd_forms_equal import open_lib  # noqa: E402
from profiles.read_step_128 import device_info  # noqa: E402

SHAPES = {"headline": ((64, 196, 512), ("fp32", "tc", "tc32")), "gqa": ((64, 49, 512), ("fp32", "tc", "tc32")),
          "tc32_bn245": ((5, 49, 128), ("tc32",)), "fp32_d20": ((3, 7, 20), ("fp32",))}
NAME = {"fp32": "mac_read_bwd", "tc": "mac_read_bwd_tc", "tc32": "mac_read_bwd_tc32"}
OUTS = ["dkb", "dmem_in", "dcontrol", "dWx", "dbx_part", "dWy", "dby", "dWm", "dbm_part", "dWm2", "dbm2_part", "dwr_part",
        "dbr_part"]


def inputs(lib, B, N, d, keep, seed):
    """Seeded weights, knowledge base, memory and control, the forward's `save` and attention at `keep`, dinfo, and the
    accumulators' initial values."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *s, scale=1.0: (torch.randn(*s, device="cuda", generator=g) * scale).contiguous()
    M = B * N
    w = {"Wx": r(d, d, scale=d ** -0.5), "Wy": r(d, d, scale=d ** -0.5), "Wm": r(2 * d, d, scale=(2 * d) ** -0.5),
         "Wm2": r(d, d, scale=d ** -0.5), "wr": r(d, scale=4 * d ** -0.5)}
    for b in ("bx", "by", "bm", "bm2"):
        w[b] = r(d, scale=0.1)
    wt = {k: w[k].t().contiguous() for k in ("Wx", "Wy", "Wm", "Wm2")}
    rw = L_.ReadWeights(*[L_.ptr(w[k]) for k in ("Wx", "bx", "Wy", "by", "Wm", "bm", "Wm2", "bm2", "wr")], 0.25)
    x = {"kb": torch.nn.functional.elu(r(B, N, d)), "mem": r(B, d), "ctrl": r(B, d), "dinfo": r(B, d)}
    x["save"] = torch.full((3 * M * d + B * d,), float("nan"), device="cuda")
    x["att"], info = torch.empty(B, N, device="cuda"), torch.empty(B, d, device="cuda")
    wsb = lib.mac_read_workspace_bytes(B, N, d, 0)
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    p = L_.ptr
    L_.check(lib.mac_read_fwd(p(x["kb"]), None, p(x["mem"]), p(x["ctrl"]), ctypes.byref(rw), keep, 11, 3, 0, p(info),
                              p(x["att"]), p(x["save"]), p(ws), wsb, B, N, d, L_.stream_ptr()), "mac_read_fwd")
    size = {"dkb": (B, N, d), "dWx": (d, d), "dWy": (d, d), "dby": (d,), "dWm": (2 * d, d), "dWm2": (d, d), "dbr_part": (B,)}
    pre = {k: r(*size.get(k, (B, d))) for k in OUTS}
    torch.cuda.synchronize()
    return w, wt, rw, x, pre


def run_case(lib, form, keep, skip, x, w, wt, rw, pre, B, N, d):
    """One call of `form`; returns the outputs (None for a skipped one) and the launches it made."""
    p, s = L_.ptr, L_.stream_ptr()
    outs = {k: None if k in skip else (torch.full_like(pre[k], float("nan")) if k == "dmem_in" else pre[k].clone())
            for k in OUTS}
    wsb = getattr(lib, NAME[form] + "_workspace_bytes")(B, N, d)
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    # the fills above run in torch's runtime, the call below in the library's: let them finish first
    torch.cuda.synchronize()
    wts = [p(wt[k]) for k in (("Wx", "Wy", "Wm", "Wm2") if form == "fp32" else ("Wy",))]
    before = lib.mac_b200_launch_count()
    L_.check(getattr(lib, NAME[form])(p(x["kb"]), p(x["mem"]), p(x["ctrl"]), ctypes.byref(rw), *wts, p(x["att"]), p(x["save"]),
                                      p(x["dinfo"]), keep, 11, 3, *[p(outs[k]) for k in OUTS], p(ws), wsb, B, N, d, s),
             NAME[form])
    launches = lib.mac_b200_launch_count() - before
    torch.cuda.synchronize()
    return {k: v for k, v in outs.items() if v is not None}, launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--base-lib", required=True)
    args = ap.parse_args()
    libs = {"base": open_lib(os.path.abspath(args.base_lib)), "new": L_.load()}
    out, all_same = {}, True
    for sname, ((B, N, d), forms) in SHAPES.items():
        res = {}
        for keep in (1.0, 0.85):
            w, wt, rw, x, pre = inputs(libs["new"], B, N, d, keep, seed=B * 1000 + N + int(keep * 100))
            variants = [()] if keep == 1.0 else [(), ("dkb",)]
            for form in forms:
                for skip in variants + ([("dWm2",)] if form == "fp32" and keep < 1 else []):
                    name = "%s_keep%g%s" % (form, keep, "".join("_no_" + k for k in skip))
                    # base, new, and each once more: a form that is not deterministic run to run shows up as base != base
                    got, launches = {}, {}
                    for side in ("base", "new", "base_again", "new_again"):
                        got[side], launches[side] = run_case(libs[side.split("_")[0]], form, keep, skip, x, w, wt, rw, pre,
                                                             B, N, d)
                    cmp = {"launches": launches, "launches_equal": len(set(launches.values())) == 1}
                    all_same &= cmp["launches_equal"]
                    for k in got["new"]:
                        eq = lambda u, v: bool(torch.equal(got[u][k].view(torch.uint8), got[v][k].view(torch.uint8)))
                        c = {"base_new": eq("base", "new"), "base_rerun": eq("base", "base_again"),
                             "new_rerun": eq("new", "new_again"), "finite": bool(got["new"][k].isfinite().all())}
                        all_same &= c["base_new"] and c["finite"]
                        cmp[k] = c
                    res[name] = cmp
                    bad = [k for k in got["new"] if not (cmp[k]["base_new"] and cmp[k]["finite"])]
                    print("%-11s %-24s launches %s; %s" % (
                        sname, name, launches["new"] if cmp["launches_equal"] else "DIFFERENT %s" % launches,
                        "DIFFERENT or not finite: " + ",".join(bad) if bad else "%d outputs same" % len(got["new"])),
                        flush=True)
        out[sname] = {"B": B, "N": N, "d": d, "cases": res}
    out["all_bit_identical_finite_and_same_launches"] = all_same
    out["device"] = device_info()
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "read_bwd_forms_equal.json"), "w") as f:
        json.dump(out, f, indent=1)
    print("all bit-identical, finite and with the same launches:", all_same)
    return 0 if all_same else 1


if __name__ == "__main__":
    sys.exit(main())
