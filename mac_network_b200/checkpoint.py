"""Checkpoint interchange and attention-map export (SURVEY.md section 8(f) rank 4).

* Weights are exchanged under the reference's TensorFlow variable names (`macModel/MACnetwork/MACCell/...`,
  `main.py:163-201`, Appendix B), including the EMA shadows `<name>/ExponentialMovingAverage` (`model.py:659-667`).
  `save_tf_checkpoint` / `load_tf_checkpoint` read and write TensorFlow's own checkpoint format (the `.index` +
  `.data-00000-of-00001` pair of `tf.train.Saver`, `main.py:163-201`) without TensorFlow (`tf_bundle.py`), so trained
  `weights{epoch}.ckpt` files of the reference load directly; the flat `.npz` container with the same names as keys stays
  as the light-weight form.
* `save_training_state` / `load_training_state` add what `tf.train.Saver()` with no variable list also writes
  (`main.py:163-165`): the Adam slots under TF's slot names `<variable>/Adam` (m) and `<variable>/Adam_1` (v), and the
  `beta1_power` / `beta2_power` accumulators (= beta^step), so a run resumes with the same optimizer trajectory
  (`main.py:185-201`: `--restore`).
* `attention_maps` lays the per-step maps out the way `MACnet.buildPredsList` does (`model.py:693-710`):
  `attMap[key][step][sample]`, keys `kb` (length H*W, reshaped to the image grid by `visualization.py:121`),
  `question`, `self`, `gate`, so the reference's visualisation script can consume them unchanged.
"""
import collections
import json

import numpy as np

MODEL_SCOPE = "macModel/"          # model.py:774
EMA_SUFFIX = "/ExponentialMovingAverage"


def _untracked(name):
    """Variables the reference's optimizer and EMA never see (`ema.apply(tf.trainable_variables())`, model.py:658-667):
    the output unit's stored batch-norm statistics.  No EMA shadow or Adam slot is written or expected for them."""
    from .output_unit import is_moving_stat
    return is_moving_stat(name)


def save_checkpoint(path, params, ema_flat=None):
    """Write parameters (and optionally the EMA shadow buffer laid out like `params.flat`) under TF variable names."""
    out = collections.OrderedDict()
    for name, t in params.t.items():
        shape = params.specs[name][0]
        out[MODEL_SCOPE + name] = t.detach().cpu().numpy().reshape(shape)
    if ema_flat is not None:
        ema = ema_flat.detach().cpu().numpy()
        for name, (shape, _) in params.specs.items():
            if _untracked(name):
                continue
            n = int(np.prod(shape)) if shape else 1
            o = params.offsets[name]
            out[MODEL_SCOPE + name + EMA_SUFFIX] = ema[o:o + n].reshape(shape)
    np.savez(path, **out)
    return list(out)


def save_tf_checkpoint(prefix, values, ema_values=None, extra=None):
    """Write {variable name without the model scope: array} (+ EMA shadows, + extra entries such as global_step) as a real
    TensorFlow checkpoint `<prefix>.index` / `<prefix>.data-00000-of-00001`, plus the `checkpoint` state file
    `tf.train.latest_checkpoint` reads (`main.py:171-178`).  `ema_values` entries of the output unit's stored batch-norm
    statistics are skipped: the reference keeps no shadow of them."""
    import os
    from .tf_bundle import write_tensor_bundle
    out = {MODEL_SCOPE + k: np.asarray(v, dtype=np.float32) for k, v in values.items()}
    if ema_values is not None:
        out.update({MODEL_SCOPE + k + EMA_SUFFIX: np.asarray(v, dtype=np.float32) for k, v in ema_values.items()
                    if not _untracked(k)})
    if extra:
        out.update(extra)
    names = write_tensor_bundle(prefix, out)
    base = os.path.basename(prefix)
    with open(os.path.join(os.path.dirname(prefix) or ".", "checkpoint"), "w") as fh:
        fh.write('model_checkpoint_path: "%s"\nall_model_checkpoint_paths: "%s"\n' % (base, base))
    return names


def load_tf_checkpoint(prefix, use_ema=False, verify=True):
    """{variable name without the model scope: array} from a TensorFlow checkpoint written by the reference (or by
    `save_tf_checkpoint`), ready for `MACParams(values=...)`; `use_ema=True` substitutes the EMA shadows (`main.py:717-719`).
    Optimizer slots, power accumulators and variables outside the model scope are skipped."""
    from .tf_bundle import read_tensor_bundle
    raw = read_tensor_bundle(prefix, verify=verify)
    vals = {}
    for k, v in raw.items():
        if not k.startswith(MODEL_SCOPE) or k.endswith((EMA_SUFFIX, "/Adam", "/Adam_1")):
            continue
        src = k + EMA_SUFFIX if (use_ema and k + EMA_SUFFIX in raw) else k
        vals[k[len(MODEL_SCOPE):]] = np.asarray(raw[src], dtype=np.float32)
    return vals


ADAM_M, ADAM_V = "/Adam", "/Adam_1"          # tf.train.AdamOptimizer slot names


def save_training_state(path, trainer):
    """Weights + EMA shadows + Adam slots + step of a `DPTrainer` (replicated state: rank 0 writes it)."""
    p = trainer.params
    out = collections.OrderedDict()
    flats = {"": p.flat, EMA_SUFFIX: trainer.ema, ADAM_M: trainer.adam_m, ADAM_V: trainer.adam_v}
    host = {suffix: t.detach().cpu().numpy() for suffix, t in flats.items()}
    for name, (shape, _) in p.specs.items():
        n = int(np.prod(shape)) if shape else 1
        o = p.offsets[name]
        for suffix, buf in host.items():
            if suffix and _untracked(name):
                continue
            out[MODEL_SCOPE + name + suffix] = buf[o:o + n].reshape(shape)
    step = int(trainer.step_id)
    out["beta1_power"] = np.float32(trainer.hp["b1"] ** step)
    out["beta2_power"] = np.float32(trainer.hp["b2"] ** step)
    out["mac_b200/step"] = np.int64(step)
    np.savez(path, **out)                 # numpy appends ".npz" to a path without it; load_training_state looks for both
    return list(out)


def load_training_state(path, trainer):
    """Restore what `save_training_state` wrote into an identically configured `DPTrainer` (every rank calls it)."""
    import os
    import torch
    if not os.path.exists(path) and os.path.exists(path + ".npz"):
        path = path + ".npz"
    z = np.load(path)
    p = trainer.params
    flats = {"": p.flat, EMA_SUFFIX: trainer.ema, ADAM_M: trainer.adam_m, ADAM_V: trainer.adam_v}
    for suffix, dst in flats.items():
        host = np.zeros(p.numel, dtype=np.float32)
        for name, (shape, _) in p.specs.items():
            if suffix and _untracked(name):
                continue
            key = MODEL_SCOPE + name + suffix
            if key not in z.files:
                raise KeyError("checkpoint %s has no %s" % (path, key))
            v = np.asarray(z[key], dtype=np.float32)
            if tuple(v.shape) != tuple(shape):
                raise ValueError("%s: checkpoint shape %s, model shape %s" % (key, v.shape, tuple(shape)))
            o = p.offsets[name]
            host[o:o + v.size] = v.reshape(-1)
        dst.copy_(torch.from_numpy(host))
    trainer.step_id = int(z["mac_b200/step"])
    p.touch()                      # packed / transposed / bf16 copies of the old weights are stale
    return trainer.step_id


def load_checkpoint(path, use_ema=False):
    """Returns {variable name without the model scope: array}, ready for `MACParams(values=...)`.
    `use_ema=True` substitutes the EMA shadows, like the reference's evaluation swap (`main.py:717-719`)."""
    z = np.load(path)
    vals = {}
    for k in z.files:
        if not k.startswith(MODEL_SCOPE) or k.endswith((EMA_SUFFIX, ADAM_M, ADAM_V)):
            continue
        name = k[len(MODEL_SCOPE):]
        src = k + EMA_SUFFIX if (use_ema and k + EMA_SUFFIX in z.files) else k
        vals[name] = np.asarray(z[src], dtype=np.float32)
    return vals


def attention_maps(cell, image_dims=None):
    """`attMap[key][step][sample]` as nested python lists (what model.py:703-705 indexes)."""
    out = {}
    for key in ("kb", "question", "self", "gate"):
        steps = []
        for a in cell.attentions[key]:
            arr = a.detach().cpu().numpy()
            if key == "kb" and image_dims is not None:
                arr = arr.reshape(arr.shape[0], image_dims[0], image_dims[1])
            steps.append(arr.tolist())
        out[key] = steps
    return out


def write_preds(path, cell, predictions=None, image_dims=None):
    """One JSON record per sample with its per-step attention maps (`model.py:693-710`, `preprocess.py:263-272`).
    `image_dims`: the knowledge base's grid (`Stem.grid(H, W)`) the `kb` maps are reshaped to; None takes the reference's
    14 x 14 (`visualization.py:121`) for a 196-cell knowledge base and leaves any other flat."""
    if image_dims is None:
        image_dims = (14, 14) if cell.N == 196 else None
    elif int(image_dims[0]) * int(image_dims[1]) != cell.N:
        raise ValueError("image_dims %s do not hold the %d knowledge-base cells" % (tuple(image_dims), cell.N))
    att = attention_maps(cell, image_dims)
    B = cell.B
    recs = []
    for i in range(B):
        rec = {"index": i, "attentions": {k: [step[i] for step in v] for k, v in att.items() if v}}
        if predictions is not None:
            rec["prediction"] = int(predictions[i])
        recs.append(rec)
    with open(path, "w") as fh:
        json.dump(recs, fh)
    return recs
