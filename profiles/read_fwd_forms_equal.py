"""Every form of the read unit's forward (csrc/read_fwd.cuh) through this tree's library and an earlier commit's, on the same
inputs, compared bit for bit.
Usage:  python profiles/read_fwd_forms_equal.py OUT_DIR --base-lib PATH

  --base-lib   the earlier commit's libmac_b200.so; the library this tree's build() made is the other side.  Both are loaded
               into one process.
Shapes: the headline (B=64, N=196, d=512), the GQA shape (B*N = 3136) and one the fused read step refuses (N = 300).  Forms:
fp32, bf16 and tc32 training (mac_read_fwd with `save`, keep_read 1 and 0.85), and the inference forms (mac_read_invariant +
mac_read_fwd_inv) of fp32, bf16 (the fused step where the shape allows it, the four-launch chain with and without kb_bf16),
tc32 and fp8 (where the shape allows it).  info, att, save and inv (region by region of its layout) are compared byte for
byte, and each library runs every form twice, which tells a difference between them from run-to-run variation.  Before
`save` became fp32 for every precision the caller widened the bf16 training chain's P, H and I1 from the workspace itself
(mac_widen_bf16 on slabs 0, 2 and 3 behind the fp32 part): the base side does that here, so both sides give the backward
the same `save`.
Writes OUT_DIR/read_fwd_forms_equal.json."""
import argparse
import ctypes
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mac_network_b200 import _lib as L_  # noqa: E402
from profiles.read_step_128 import device_info  # noqa: E402

FP32, BF16, TC32, FP8 = 0, 1, 2, 3
SHAPES = {"headline": (64, 196, 512), "gqa": (64, 49, 512), "step_refused": (4, 300, 512)}


def open_lib(path):
    lib = ctypes.CDLL(path)
    for name, (res, args) in L_.PROTOTYPES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    return lib


def inputs(lib, B, N, d, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *s, scale=1.0: (torch.randn(*s, device="cuda", generator=g) * scale).contiguous()
    x = {"kb": torch.nn.functional.elu(r(B, N, d)), "mem": r(B, d), "ctrl": r(B, d)}
    x["kb16"] = x["kb"].to(torch.bfloat16)
    w = {"Wx": r(d, d, scale=d ** -0.5), "Wy": r(d, d, scale=d ** -0.5), "Wm": r(2 * d, d, scale=(2 * d) ** -0.5),
         "Wm2": r(d, d, scale=d ** -0.5), "wr": r(d, scale=d ** -0.5)}
    for b in ("bx", "by", "bm", "bm2"):
        w[b] = r(d, scale=0.1)
    s = L_.stream_ptr()

    def pack(fn, W, K, n, dtype, cols):
        out = torch.empty(n * cols, dtype=dtype, device="cuda")
        L_.check(fn(L_.ptr(W), L_.ptr(out), K, n, s), "pack")
        return out
    pk = {"Wx_bf16": pack(lib.mac_pack_weight_bf16, w["Wx"], d, d, torch.bfloat16, d),
          "Wm_bf16": pack(lib.mac_pack_weight_bf16, w["Wm"], 2 * d, d, torch.bfloat16, 2 * d),
          "Wm2_bf16": pack(lib.mac_pack_weight_bf16, w["Wm2"], d, d, torch.bfloat16, d),
          "Wx_s3": pack(lib.mac_pack_weight_split3, w["Wx"], d, d, torch.bfloat16, 3 * d),
          "Wma_s3": pack(lib.mac_pack_weight_split3, w["Wm"][:d].contiguous(), d, d, torch.bfloat16, 3 * d),
          "Wmb_s3": pack(lib.mac_pack_weight_split3, w["Wm"][d:].contiguous(), d, d, torch.bfloat16, 3 * d),
          "Wm2_s3": pack(lib.mac_pack_weight_split3, w["Wm2"], d, d, torch.bfloat16, 3 * d),
          "Wm_s3": pack(lib.mac_pack_weight_split3, w["Wm"], 2 * d, d, torch.bfloat16, 6 * d)}
    for name, W in (("Wm_fp8", w["Wm"][:d].contiguous()), ("Wm2_fp8", w["Wm2"])):
        pk[name] = torch.empty(d * d, dtype=torch.uint8, device="cuda")
        pk[name + "_scale"] = torch.empty(d, device="cuda")
        L_.check(lib.mac_pack_weight_fp8(L_.ptr(W), L_.ptr(pk[name]), L_.ptr(pk[name + "_scale"]), d, d, s), "pack fp8")
    rw = L_.ReadWeights(*[L_.ptr(w[k]) for k in ("Wx", "bx", "Wy", "by", "Wm", "bm", "Wm2", "bm2", "wr")], 0.25,
                        *[L_.ptr(pk[k]) for k in ("Wx_bf16", "Wm_bf16", "Wm2_bf16", "Wx_s3", "Wma_s3", "Wmb_s3", "Wm2_s3",
                                                  "Wm_fp8", "Wm_fp8_scale", "Wm2_fp8", "Wm2_fp8_scale", "Wm_s3")])
    torch.cuda.synchronize()
    return x, w, pk, rw


def run_form(lib, side, form, x, rw, B, N, d):
    """One call of `form` through `lib`; returns the tensors to compare."""
    prec, kind, keep, kb16 = form
    M, s, p = B * N, L_.stream_ptr(), L_.ptr
    nan = lambda n: torch.full((n,), float("nan"), device="cuda")
    info, att = nan(B * d), nan(M)
    wsb = lib.mac_read_workspace_bytes(B, N, d, prec)
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    k16 = p(x["kb16"]) if kb16 else None
    save = nan(3 * M * d + B * d) if kind == "train" else None
    # the fills above run in torch's runtime, the call below in the library's: let them finish first
    torch.cuda.synchronize()
    if kind == "train":
        L_.check(lib.mac_read_fwd(p(x["kb"]), k16, p(x["mem"]), p(x["ctrl"]), ctypes.byref(rw), keep, 11, 3, prec, p(info),
                                  p(att), p(save), p(ws), wsb, B, N, d, s), "mac_read_fwd")
        if side == "base" and prec == BF16:
            base, n = ws.data_ptr(), M * d
            fp32 = int(lib.mac_read_workspace_bytes(B, N, d, FP32))
            off = ((base + fp32 + 1023) & ~1023) - base
            slab = (M * d * 2 + 1023) & ~1023
            srcs = (ctypes.c_void_p * 3)(*[base + off + k * slab for k in (0, 2, 3)])
            dsts = (ctypes.c_void_p * 3)(*[save.data_ptr() + 4 * k * n for k in range(3)])
            L_.check(lib.mac_widen_bf16(srcs, dsts, 3, n, s), "mac_widen_bf16")
        torch.cuda.synchronize()
        return {"info": info, "att": att, "save": save}
    nb = lib.mac_read_invariant_bytes(B, N, d, prec)
    inv = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    kb = None if prec in (BF16, FP8) and kb16 else p(x["kb"])
    # the bf16 and fp8 step-invariant parts are computed from kb_bf16; kb16 = False runs the step on the fp32 knowledge base
    inv_k16 = p(x["kb16"]) if prec in (BF16, FP8) else None
    L_.check(lib.mac_read_invariant(kb, inv_k16, ctypes.byref(rw), prec, p(inv), nb, B, N, d, s), "mac_read_invariant")
    L_.check(lib.mac_read_fwd_inv(kb, k16, p(inv), None, p(x["mem"]), p(x["ctrl"]), ctypes.byref(rw), prec, p(info), p(att),
                                  p(ws), wsb, B, N, d, s), "mac_read_fwd_inv")
    torch.cuda.synchronize()
    # the bf16 and fp8 layouts start at the first 1 KB boundary of the buffer, the tc32 scratch at the first one behind
    # [P | Q]: compare the laid-out regions, wherever the allocator put the buffer
    base, f32 = inv.data_ptr(), M * d * 4
    al = lambda o: ((base + o + 1023) & ~1023) - base
    if prec in (BF16, FP8):
        regions = {"inv": inv[al(0):al(0) + nb - 1024]}
    elif prec == TC32:
        regions = {"inv": inv[:2 * f32], "inv_split": inv[al(2 * f32):al(2 * f32) + f32]}
    else:
        regions = {"inv": inv}
    return {"info": info, "att": att, **regions}


def describe(a, b, M, d):
    """Where two differing tensors differ: count of differing elements, largest difference, and for `save` which part."""
    if a.dtype == torch.uint8:
        return "%d of %d bytes" % (int((a != b).sum()), a.numel())
    diff = (a != b) & ~(a.isnan() & b.isnan())
    out = "%d of %d elements, NaN %d / %d, max |diff| %.3g" % (int(diff.sum()), a.numel(), int(a.isnan().sum()),
                                                               int(b.isnan().sum()), float((a - b)[diff].abs().max()))
    if a.numel() > 3 * M * d:
        out += ", parts " + ",".join(n for k, n in enumerate(("P", "H", "I1", "y")) if bool(diff[k * M * d:(k + 1) * M * d].any()))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--base-lib", required=True)
    args = ap.parse_args()
    libs = {"base": open_lib(os.path.abspath(args.base_lib)), "new": L_.load()}
    out, all_same = {}, True
    device = device_info()
    for sname, (B, N, d) in SHAPES.items():
        step = bool(libs["new"].mac_read_step_fused_supported(B, N, d))
        forms = [(FP32, "train", 1.0, False), (FP32, "train", 0.85, False), (BF16, "train", 1.0, True),
                 (BF16, "train", 0.85, True), (TC32, "train", 1.0, False), (TC32, "train", 0.85, False),
                 (FP32, "inv", 1.0, False), (BF16, "inv", 1.0, True), (BF16, "inv", 1.0, False), (TC32, "inv", 1.0, False)]
        if step:
            forms.append((FP8, "inv", 1.0, True))
        x, w, packs, rw = inputs(libs["new"], B, N, d, seed=B * 1000 + N)     # rw points into w and packs: keep them
        res = {}
        for form in forms:
            prec, kind, keep, kb16 = form
            name = "%s_%s%s%s" % (["fp32", "bf16", "tc32", "fp8"][prec], kind, "_keep%g" % keep if keep < 1 else "",
                                  "" if prec in (FP32, TC32) or kind == "train" else ("_kb_bf16" if kb16 else "_kb_fp32"))
            # base, new, and each once more: a form that is not deterministic run to run shows up as base != base
            got = {side: run_form(libs[side.split("_")[0]], side.split("_")[0], form, x, rw, B, N, d)
                   for side in ("base", "new", "base_again", "new_again")}
            cmp = {}
            for k in got["new"]:
                eq = lambda u, v: bool(torch.equal(got[u][k].view(torch.uint8), got[v][k].view(torch.uint8)))
                cmp[k] = {"base_new": eq("base", "new"), "base_rerun": eq("base", "base_again"),
                          "new_rerun": eq("new", "new_again"), "base_rerun_new": eq("base_again", "new")}
                if got["new"][k].is_floating_point():        # every element written, nothing left NaN
                    cmp[k]["finite"] = bool(got["new"][k].isfinite().all())
                    all_same &= cmp[k]["finite"]
                if not cmp[k]["base_new"]:
                    cmp[k]["where"] = describe(got["base"][k], got["new"][k], B * N, d)
                all_same &= cmp[k]["base_new"]
            res[name] = cmp
            print("%-13s %-26s %s" % (sname, name, "; ".join(
                "%s %s%s%s%s" % (k, "same" if v["base_new"] else "DIFFERENT (%s)" % v["where"],
                                 "" if v.get("finite", True) else " NOT FINITE",
                                 "" if v["base_rerun"] else ", base rerun differs (rerun %s new)" % (
                                     "equals" if v["base_rerun_new"] else "differs from"),
                                 "" if v["new_rerun"] else ", new rerun differs")
                for k, v in cmp.items())), flush=True)
        out[sname] = {"B": B, "N": N, "d": d, "fused_step_shape": step, "forms": res}
    out["all_bit_identical_and_finite"] = all_same
    out["device"] = device
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "read_fwd_forms_equal.json"), "w") as f:
        json.dump(out, f, indent=1)
    print("all bit-identical and finite:", all_same)
    return 0 if all_same else 1


if __name__ == "__main__":
    sys.exit(main())
