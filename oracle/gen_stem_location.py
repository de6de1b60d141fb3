"""Generate tests/golden/stem_loc_*.npz: the UNMODIFIED reference's `MACnet.stem` (model.py:165-204) on the numpy TF1 shim
with --locationAware (ops.addLocation, ops.py:440-559).

    python oracle/gen_stem_location.py            # needs the reference checkout (build container only)

The location code calls TF ops the shim does not define (`linspace`, `meshgrid`, `sin`, `cos`, `pow`, `range`); this
script adds them to the shim module at run time, as `gen_stem_geometry.py` adds strided SAME convolutions, so the shim
and the fixtures it pinned are unchanged.  The grid is 5 x 4 (H != W), so the axis order is pinned."""
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import gen_golden as gg                      # noqa: E402  (puts the shim and the reference on sys.path)
from oracle import gen_stem_geometry as geom             # noqa: E402

tf = gg.tf

# name -> extra reference flags; each case is generated at eval and in training (the reference's stemDropout, 0.82)
CASES = {
    "L": ["--locationAware"],
    "PE_d4_b05": ["--locationAware", "--locationType", "PE", "--locationDim", "4", "--locationBias", "0.5"],
    "PE_k53_s21": ["--locationAware", "--locationType", "PE", "--locationDim", "3", "--stemKernelSizes", "5", "3",
                   "--stemStrideSizes", "2", "1"],
}


def _add_shim_ops():
    tf.linspace = lambda start, stop, num: tf._t(np.linspace(float(start), float(stop), int(num)))
    tf.meshgrid = lambda *xs, **kw: [tf._t(m) for m in np.meshgrid(*[np.asarray(x) for x in xs],
                                                                    indexing=kw.get("indexing", "xy"))]
    tf.sin = lambda x: tf._t(np.sin(np.asarray(x)))
    tf.cos = lambda x: tf._t(np.cos(np.asarray(x)))
    tf.pow = lambda a, b: tf._t(np.power(np.asarray(a, np.float64), np.asarray(b, np.float64)))
    tf.range = lambda n: tf._t(np.arange(int(n)))


def run_case(name, flags, train, seed=43, B=2, H=5, W=4, cin=8, cout=8):
    import importlib
    ref_model = importlib.import_module("model")
    gg.set_reference_config("@args.txt", ["--stemDim", str(cout)] + flags, dict(L=1, d=cout), train)
    rc = gg._ref_config.config
    ref_ops = importlib.import_module("ops")
    from mac_network_b200.stem import stem_specs, init_stem_params
    location = (rc.locationType, rc.locationBias, rc.locationDim)
    specs = stem_specs(cin, cout, rc.stemNumLayers, rc.stemKernelSize, ksizes=rc.stemKernelSizes, location=location)
    params = init_stem_params(specs, seed=seed, dtype=np.float64)
    images = np.maximum(np.random.RandomState(seed + 1).standard_normal((B, H, W, cin)), 0)
    keep = rc.stemDropout if train else 1.0
    grid, l = ref_ops.locations[rc.locationType](H, W, rc.locationDim)         # the reference's own grid, for the record
    store = tf.reset_shim(values=params, seed=seed + 2, dtype=np.float64)
    me = types.SimpleNamespace(dropouts={"stem": keep}, batchNorm=None, batchSize=B, H=H, W=W)
    kb = ref_model.MACnet.stem(me, tf.constant(images), cin, cout)
    created = {k: list(v.shape) for k, v in store.vars.items()}
    assert created == {k: list(v[0]) for k, v in specs.items()}, (created, specs)
    out = {"images": images, "kb": np.asarray(kb), "grid": np.asarray(grid, np.float64)}
    for i, u in enumerate(store.uniform_draws):
        out["uniform_%03d" % i] = u.astype(np.float64)
    strides = rc.stemStrideSizes or [1] * rc.stemNumLayers
    meta = {"case": name, "flags": flags, "train": train, "keep": keep, "shape": [B, H, W, cin, cout],
            "layers": rc.stemNumLayers, "ksize": rc.stemKernelSize, "ksizes": rc.stemKernelSizes, "strides": strides,
            "location": [rc.locationType, float(rc.locationBias), int(rc.locationDim)], "l": int(l),
            "param_seed": seed, "relu": rc.relu, "variables": created, "n_uniform": len(store.uniform_draws)}
    out["meta_json"] = np.frombuffer(json.dumps(meta, sort_keys=True).encode(), dtype=np.uint8)
    return out


def main():
    tf.nn.conv2d = staticmethod(geom._conv2d_same)
    _add_shim_ops()
    outdir = os.path.join(gg.ROOT, "tests", "golden")
    only = sys.argv[1:]
    for case, flags in CASES.items():
        for train in (False, True):
            name = "stem_loc_%s_%s" % (case, "train" if train else "eval")
            if only and name not in only:
                continue
            out = run_case(name, flags, train)
            path = os.path.join(outdir, name + ".npz")
            np.savez_compressed(path, **out)
            print("%-28s %8.1f KB  draws=%d" % (name, os.path.getsize(path) / 1024.0,
                                                 sum(k.startswith("uniform_") for k in out)))


if __name__ == "__main__":
    main()
