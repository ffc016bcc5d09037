"""dfq_b200.int8.chain_int8 / chain_affine on seeded random graphs (tests/chain_graphs.py), on the CPU through the host
twins of the library: every rule and its near misses combined, at every legal flag set - for the affine scheme with and
without the reference's evaluation state - each chained module bit for bit against the per-layer model, its records
consistent with its graph, the base edge rule's edges all fused, and the same outputs after int8.save / load.  A last
test checks that the corpus exercises every record kind and every near miss.  DFQ_CHAIN_SEEDS sets the seed count of a
longer run."""
import collections
import os

import pytest
import torch

import chain_graphs as CG
import fakelib_int8_affine_pool_heads
import int8_layout_oracle as LO
from test_int8_upsample_host import _gpu_interpolate

SEEDS = range(int(os.environ.get("DFQ_CHAIN_SEEDS", 100)))
RECORD_FLOOR, NEAR_FLOOR = 10, 5
_counts = {}


def _verify(scheme, seed, tmp_path):
    """The records of program `seed`, verified (chain_graphs.verify) through the twins; memoized for the coverage test."""
    if (scheme, seed) in _counts:
        return _counts[scheme, seed]
    prog = CG.program(seed, scheme)
    with pytest.MonkeyPatch.context() as mp:
        (LO if scheme == "ncnn" else fakelib_int8_affine_pool_heads).install(mp)
        model = CG.build(prog)
        x = CG.inputs(prog)

        def patch():
            mp.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
            if scheme == "ncnn":
                _gpu_interpolate(mp)
        try:
            counts = CG.verify(prog, model, x, tmp_path, mp, patch)
        except BaseException:
            print(CG.describe(prog))
            raise
    _counts[scheme, seed] = counts, collections.Counter(prog["near"])
    return _counts[scheme, seed]


@pytest.mark.parametrize("seed", SEEDS)
def test_ncnn_random_graph(seed, tmp_path):
    _verify("ncnn", seed, tmp_path)


@pytest.mark.parametrize("seed", SEEDS)
def test_affine_random_graph(seed, tmp_path):
    _verify("affine", seed, tmp_path)


def test_corpus_covers_every_rule_and_near_miss(tmp_path):
    """Over all seeds, every record kind a scheme has appears at least RECORD_FLOOR times and every near miss at least
    NEAR_FLOOR times: the generator keeps exercising the rules."""
    records, near = collections.Counter(), collections.Counter()
    for scheme in ("ncnn", "affine"):
        for seed in SEEDS:
            d = tmp_path / ("%s%d" % (scheme, seed))
            d.mkdir()
            r, n = _verify(scheme, seed, d)
            records.update({(scheme, k): v for k, v in r.items()})
            near.update(n)
    rows = ["%-26s %8s %8s" % ("record", "ncnn", "affine")]
    rows += ["%-26s %8d %8d" % (k, records[("ncnn", k)], records[("affine", k)]) for k in CG.RECORD_KINDS]
    rows += ["%-26s %8d" % ("near miss " + k, near[k]) for k in CG.NEAR_MISSES]
    print("\n".join(rows))
    ncnn_kinds = [k for k in CG.RECORD_KINDS if not k.startswith("obs_")]
    low = [(s, k) for s, kinds in (("ncnn", ncnn_kinds), ("affine", CG.RECORD_KINDS)) for k in kinds
           if records[(s, k)] < RECORD_FLOOR and not (s == "affine" and k == "up_codes")]
    low += [("near", k) for k in CG.NEAR_MISSES if near[k] < NEAR_FLOOR]
    assert not low, low
