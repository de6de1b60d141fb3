"""Generate tests/golden/stem_geom_*.npz: the UNMODIFIED reference's `MACnet.stem` (model.py:165-204) on the numpy TF1 shim
for the stem's geometry flags (--stemKernelSize, --stemKernelSizes, --stemStrideSizes, --stemLinear).

    python oracle/gen_stem_geometry.py            # needs the reference checkout (build container only)

The shim's `tf.nn.conv2d` covers stride 1 with odd kernels, what the default stem uses; this script adds TF's SAME
padding for strides and even kernels around it (`_conv2d_same`), leaving that branch and the fixtures it pinned as they
are.  Variable values come from `mac_network_b200.stem.init_stem_params`; names and shapes are whatever the reference
creates, stored in the fixture so `stem_specs` can be checked against them."""
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import gen_golden as gg        # noqa: E402  (puts the shim and the reference on sys.path)

tf = gg.tf
_shim_conv2d = tf.nn.conv2d

# name -> extra reference flags; each case is generated at eval and in training (the reference's stemDropout, 0.82)
CASES = {
    "k1": ["--stemKernelSize", "1"],
    "k53_s21": ["--stemKernelSizes", "5", "3", "--stemStrideSizes", "2", "1"],
    "k42": ["--stemKernelSizes", "4", "2"],
    "linear": ["--stemLinear"],
}


def _conv2d_same(inp, filter=None, strides=None, padding="SAME", **kwargs):
    """tf.nn.conv2d, NHWC / HWIO, padding SAME, any stride: Ho = ceil(H / s), pad_total = max((Ho - 1) s + k - H, 0), the
    odd padding row on the bottom (TF's conv_ops)."""
    k = np.asarray(filter)
    kh, kw = k.shape[0], k.shape[1]
    if tuple(strides) == (1, 1, 1, 1) and kh % 2 and kw % 2:
        return _shim_conv2d(inp, filter=filter, strides=strides, padding=padding, **kwargs)
    assert padding == "SAME" and strides[0] == strides[3] == 1
    x = np.asarray(inp)
    B, H, W, _ = x.shape
    sh, sw = strides[1], strides[2]
    Ho, Wo = -(-H // sh), -(-W // sw)
    ph, pw = max((Ho - 1) * sh + kh - H, 0), max((Wo - 1) * sw + kw - W, 0)
    xp = np.zeros((B, H + ph, W + pw, x.shape[3]), dtype=x.dtype)
    xp[:, ph // 2:ph // 2 + H, pw // 2:pw // 2 + W, :] = x
    out = np.zeros((B, Ho, Wo, k.shape[3]), dtype=x.dtype)
    for i in range(kh):
        for j in range(kw):
            out += np.einsum("bhwc,co->bhwo", xp[:, i:i + (Ho - 1) * sh + 1:sh, j:j + (Wo - 1) * sw + 1:sw, :], k[i, j])
    return tf._t(out)


def run_case(name, flags, train, seed=41, B=2, H=5, W=4, cin=8, cout=8):
    """The stem as `MACnet.build` calls it (model.py:165-204), through the reference's own method."""
    import importlib
    ref_model = importlib.import_module("model")
    gg.set_reference_config("@args.txt", ["--stemDim", str(cout)] + flags, dict(L=1, d=cout), train)
    rc = gg._ref_config.config
    from mac_network_b200.stem import stem_specs, init_stem_params
    specs = stem_specs(cin, cout, rc.stemNumLayers, rc.stemKernelSize, ksizes=rc.stemKernelSizes, linear=rc.stemLinear)
    params = init_stem_params(specs, seed=seed, dtype=np.float64)
    images = np.maximum(np.random.RandomState(seed + 1).standard_normal((B, H, W, cin)), 0)    # post-ReLU ResNet features
    keep = rc.stemDropout if train else 1.0
    store = tf.reset_shim(values=params, seed=seed + 2, dtype=np.float64)
    me = types.SimpleNamespace(dropouts={"stem": keep}, batchNorm=None, batchSize=B, H=H, W=W)
    kb = ref_model.MACnet.stem(me, tf.constant(images), cin, cout)
    created = {k: list(v.shape) for k, v in store.vars.items()}
    assert created == {k: list(v[0]) for k, v in specs.items()}, (created, specs)
    out = {"images": images, "kb": np.asarray(kb)}
    for i, u in enumerate(store.uniform_draws):
        out["uniform_%03d" % i] = u.astype(np.float64)
    strides = rc.stemStrideSizes or [1] * rc.stemNumLayers
    meta = {"case": name, "flags": flags, "train": train, "keep": keep, "shape": [B, H, W, cin, cout],
            "layers": rc.stemNumLayers, "ksize": rc.stemKernelSize, "ksizes": rc.stemKernelSizes, "strides": strides,
            "linear": bool(rc.stemLinear), "param_seed": seed, "relu": rc.relu, "variables": created,
            "n_uniform": len(store.uniform_draws)}
    out["meta_json"] = np.frombuffer(json.dumps(meta, sort_keys=True).encode(), dtype=np.uint8)
    return out


def main():
    tf.nn.conv2d = staticmethod(_conv2d_same)
    outdir = os.path.join(gg.ROOT, "tests", "golden")
    only = sys.argv[1:]
    for case, flags in CASES.items():
        for train in (False, True):
            name = "stem_geom_%s_%s" % (case, "train" if train else "eval")
            if only and name not in only:
                continue
            out = run_case(name, flags, train)
            path = os.path.join(outdir, name + ".npz")
            np.savez_compressed(path, **out)
            print("%-28s %8.1f KB  draws=%d" % (name, os.path.getsize(path) / 1024.0,
                                                 sum(k.startswith("uniform_") for k in out)))


if __name__ == "__main__":
    main()
