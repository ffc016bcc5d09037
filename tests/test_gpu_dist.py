"""-m gpu, one GPU, several processes: BASELINE configs[3] (DeepLab-v3+ sharded over 4 ranks) as a test the driver runs.

Four worker processes share cuda:0 (gloo for the rendezvous and the collectives - NCCL refuses several ranks on one device;
the collectives' payloads are staged through the host in that case, dfq_b200/dist.py::_all_gather_flat), every rank runs the
REAL kernels on its shard: chain-sharded equalization in `exact` mode + ONE all-gather (scale vectors and, replicas="exact",
the owners' equalized tensors), then sharded bias correction.  Every rank must end with the model a single process computes
on the same GPU: S, weights bit for bit, biases / fake_bias within 1e-5.  (With replicas="replay" the weights of non-owned
chains are within ~3e-6 and - bias correction being ill-conditioned in the last bit of the weights, DESIGN.md section 4 - the
biases only within 5e-2: the second test.)
The NCCL flavour of the same check (one process per GPU) is tools/dist_check.py."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


def _nw(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)


def _calibrate(sharded, name="deeplab", replicas="exact"):
    import torch.nn as nn
    from dfq_b200 import dfq, workload, dist as ddist
    from dfq_b200.utils import layer_transform as LT
    from dfq_b200.utils.relation import create_relation
    targ = [nn.Conv2d, nn.Linear]
    topo = workload.load_topology(os.path.join(GOLD, "topology_%s.json" % name))
    graph, bottoms, _ = workload.build_graph(topo, seed=0)
    LT.merge_batchnorm(None, graph, bottoms, targ)
    rels = create_relation(graph, bottoms, targ)
    info = {}
    if sharded:
        info = ddist.sharded_cross_layer_equalization(graph, rels, targ, mode="exact", replicas=replicas)
        info["bc"] = ddist.sharded_bias_correction(graph, bottoms, targ, replicate_below=1 << 18)
    else:
        dfq.cross_layer_equalization(graph, rels, targ)
        info["sweeps"] = dfq.cross_layer_equalization.last_result.n_sweeps
        dfq.bias_correction(graph, bottoms, targ)
    out = {"sweeps": np.array(info["sweeps"])}
    for i, k in enumerate(graph):
        m = graph[k]
        if type(m) in targ:
            out["w%d" % i] = m.weight.detach().numpy().copy()
            out["b%d" % i] = m.bias.detach().numpy().copy()
        elif hasattr(m, "fake_bias") and not isinstance(m, str):
            out["f%d" % i] = m.fake_bias.numpy().copy()
    for i, r in enumerate(rels):
        out["S%d" % i] = r.S.numpy().copy()
    return out, info


def _worker(rank, world, port, out_dir, replicas):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=world)
    try:
        out, info = _calibrate(True, replicas=replicas)
        out["owner"] = np.array(info["owner"])
        out["bc_sharded_levels"] = np.array(info["bc"]["sharded_levels"])
        np.savez(os.path.join(out_dir, "rank%d.npz" % rank), **out)
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(900)
@pytest.mark.parametrize("replicas", ["exact", "replay"])
def test_deeplab_sharded_over_four_ranks_equals_one_process(replicas, tmp_path):
    world = 4
    single, _ = _calibrate(False)
    port = 29500 + (os.getpid() % 2000) + (61 if replicas == "exact" else 67)
    mp.spawn(_worker, args=(world, port, str(tmp_path), replicas), nprocs=world, join=True)
    worst_w = worst_b = 0.0
    for r in range(world):
        d = np.load(tmp_path / ("rank%d.npz" % r))
        assert set(d["owner"].tolist()) == set(range(world)), "chains must be spread over all ranks"
        assert int(d["sweeps"]) == int(single["sweeps"]), (int(d["sweeps"]), int(single["sweeps"]))
        for k, v in single.items():
            if k[0] == "S":
                assert np.array_equal(d[k], v), ("S differs on rank %d" % r, k)
            elif k[0] == "w":
                worst_w = max(worst_w, _nw(d[k], v))
            elif k[0] in "bf":
                worst_b = max(worst_b, _nw(d[k], v))
    print("DeepLab, 4 ranks, replicas=%s: S bit-identical on every rank, worst weight %.3g, worst bias/fake_bias %.3g (normwise)"
          % (replicas, worst_w, worst_b))
    if replicas == "exact":
        assert worst_w == 0.0 and worst_b <= 1e-5, (worst_w, worst_b)
    else:
        assert worst_w <= 1e-5 and worst_b <= 5e-2, (worst_w, worst_b)
