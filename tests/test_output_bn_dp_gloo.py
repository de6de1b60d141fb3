"""Data-parallel training of the batch-normalised output unit (--outputBN) on CPU: 2 ranks over gloo.  The gradient function is
the fp64 torch-autograd oracle (the CUDA kernels need a GPU); under test are the flat layout with the stored statistics
last, the one all-reduce that carries them in the bucket's tail (`dp.allreduce_sum_with_stats_`), and the averaging rule.

Each rank normalises with its own batch statistics, so the objective of a step is the sum over shards of the per-shard
losses / global batch; the all-reduced gradient of the trainable variables must equal that objective's gradient computed
in one process, and the stored statistics must be identical on both ranks and equal to the update by the mean over ranks
of the per-rank batch statistics."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORLD, B, D, A, DECAY = 2, 8, 16, 12, 0.9


def _problem():
    from mac_network_b200.output_unit import init_output_params, is_moving_stat, output_specs
    from mac_network_b200.mac_cell import flat_layout
    import collections
    specs = output_specs(D, D, [8], A, question=True, mul=True, bn=True)
    specs = collections.OrderedDict([kv for kv in specs.items() if not is_moving_stat(kv[0])]
                                    + [kv for kv in specs.items() if is_moving_stat(kv[0])])
    params = init_output_params(specs, seed=71, dtype=np.float64)
    rng = np.random.RandomState(72)
    memory, vecq = rng.standard_normal((B, D)), np.tanh(rng.standard_normal((B, D)))
    answers = rng.randint(0, A, size=(B,))
    offsets = flat_layout(specs)
    start = min(offsets[k] for k in specs if is_moving_stat(k))
    return specs, params, memory, vecq, answers, offsets, start


def _shard_grads(params, memory, vecq, answers, rows):
    """fp64 gradients of sum(losses of the shard) / B and the shard's stored statistics after its training forward."""
    from oracle.output_options import output_graph
    p = {k: torch.from_numpy(v).requires_grad_("/moving_" not in k) for k, v in params.items()}
    moving = {}
    _, losses = output_graph("ELU", p, torch.from_numpy(memory[rows]), torch.from_numpy(vecq[rows]),
                             torch.from_numpy(answers[rows]).long(), question=True, mul=True, bn=True, train=True,
                             decay=DECAY, moving=moving)
    names = [k for k in p if p[k].requires_grad]
    g = torch.autograd.grad(losses.sum() / B, [p[k] for k in names])
    return dict(zip(names, g)), moving


def _flat(values, specs, offsets):
    buf = torch.zeros(offsets["__total__"], dtype=torch.float64)
    for name in specs:
        if name in values:
            v = torch.as_tensor(values[name]).reshape(-1)
            buf[offsets[name]:offsets[name] + v.numel()] = v
    return buf


def _worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from mac_network_b200.dp import allreduce_sum_with_stats_, shard_rows
    specs, params, memory, vecq, answers, offsets, start = _problem()
    g, moving = _shard_grads(params, memory, vecq, answers, shard_rows(B, rank, world))
    bucket = _flat(g, specs, offsets)
    flat = _flat(dict(params, **moving), specs, offsets)       # this rank's parameters after its own forward
    allreduce_sum_with_stats_(bucket, flat, start)
    np.save(os.path.join(out_dir, "bucket%d.npy" % rank), bucket.numpy())
    np.save(os.path.join(out_dir, "flat%d.npy" % rank), flat.numpy())
    dist.destroy_process_group()


def test_two_rank_output_batch_norm(tmp_path):
    from mac_network_b200.dp import shard_rows
    port = 29500 + ((os.getpid() + 977) % 2000)
    mp.spawn(_worker, args=(WORLD, port, str(tmp_path)), nprocs=WORLD, join=True)
    specs, params, memory, vecq, answers, offsets, start = _problem()
    f0, f1 = (np.load(os.path.join(str(tmp_path), "flat%d.npy" % r)) for r in range(WORLD))
    b0, b1 = (np.load(os.path.join(str(tmp_path), "bucket%d.npy" % r)) for r in range(WORLD))
    assert np.array_equal(f0, f1) and np.array_equal(b0[:start], b1[:start])      # replicas stay identical
    # trainable variables: the sum over shards of the per-shard gradients, computed in one process
    shards = [_shard_grads(params, memory, vecq, answers, shard_rows(B, r, WORLD)) for r in range(WORLD)]
    full = sum(_flat(g, specs, offsets) for g, _ in shards).numpy()
    assert np.max(np.abs(b0[:start] - full[:start])) <= 1e-12 * max(1.0, np.max(np.abs(full)))
    assert np.array_equal(f0[:start], _flat(params, specs, offsets).numpy()[:start])   # no weight touched by the exchange
    # stored statistics: moved by the mean over ranks of the per-rank batch mean and Bessel-corrected variance
    for name in (k for k in specs if "/moving_" in k):
        per = []
        for r in range(WORLD):
            x = _features(params, memory, vecq, shard_rows(B, r, WORLD), name)
            per.append(x.mean(0) if name.endswith("moving_mean") else x.var(0, ddof=1))
        want = params[name] - (params[name] - np.mean(per, axis=0)) * (1.0 - DECAY)
        o = offsets[name]
        assert np.max(np.abs(f0[o:o + want.size] - want)) <= 1e-12, name
        assert not np.allclose(want, params[name])


def _features(params, memory, vecq, rows, name):
    """The input of the batch norm that owns `name`, for the shard `rows` (layer 0: [m, q', m * q']; layer 1: the hidden
    activation after layer 0 with the shard's own batch statistics)."""
    from oracle.model_torch_autograd import _act
    from oracle.output_options import batch_norm
    p = {k: torch.from_numpy(v) for k, v in params.items()}
    m, q = torch.from_numpy(memory[rows]), torch.from_numpy(vecq[rows])
    eq = q @ p["outputUnit/linearLayeroutQuestion/weights/weight"] + p["outputUnit/linearLayeroutQuestion/biases/bias"]
    x = torch.cat([m, eq, m * eq], -1)
    if "fc_0/" in name:
        return x.numpy()
    sc = "classifier/linearLayerfc_0/"
    x = batch_norm(x, p, sc + "BatchNorm/", True, DECAY, None)
    return _act("ELU", x @ p[sc + "weights/weight"] + p[sc + "biases/bias"]).numpy()
