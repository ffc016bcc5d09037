"""CPU guards of the GPU boundary tests.

* The kernel constants the boundary cases of tests/test_gpu_engine.py, tests/test_gpu_int8.py and
  tests/test_gpu_activation.py were built around: a
  retune must fail here, loudly, instead of quietly moving every case off its boundary.
* The per-row acceptance bound of bias correction (oracle.dfq_oracle.bias_delta_bound) accepts the oracle's own deltas and
  rejects errors that a normwise gate over the whole layer lets through."""
import os
import re

import numpy as np
import pytest

from oracle import dfq_oracle as O

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "dfq_b200", "csrc")

# name -> (source file, value the boundary cases assume)
CONSTANTS = {
    "kStageFloats": ("rowpipe.cuh", 4608),
    "DFQ_PIPE_MAX_ROWS": ("rowpipe.cuh", 32),
    "DFQ_INV_CACHE": ("cle_engine.cu", 2044),
    "kRescanCols": ("cle_engine.cu", 1024),
    "kTableCacheBytes": ("cle_engine.cu", 9 * 1024),
    "DFQ_SUB_ITEMS": ("cle_engine.cu", 8),
    "kExpectCache": ("passes.cu", 2048),
    "kBcExCols": ("bc_stream.cuh", 512),
    # k_i8_conv_mma's CTA tile and ring (tests/test_gpu_int8.py TILES)
    "BM": ("int8_conv.cu", 128),
    "BN": ("int8_conv.cu", 64),
    "BK": ("int8_conv.cu", 64),
    "STAGES": ("int8_conv.cu", 3),
    "THREADS": ("int8_conv.cu", 128),
    # the launch formulas of the activation kernels (tests/test_gpu_activation.py)
    "kThreads": ("tensor_ops.cu", 256),
    "kItemFloats": ("tensor_ops.cu", 16),
    "kRangeCtaRow": ("tensor_ops.cu", 2048),
    "kDThreads": ("distill.cu", 256),
    "kBnstatCtaRow": ("distill.cu", 2048),
}


def _source_value(fname, name):
    with open(os.path.join(CSRC, fname)) as f:
        src = f.read()
    m = (re.search(r"^\s*#define\s+%s\s+([^\s/]+)" % name, src, re.M)
         or re.search(r"constexpr\s+[\w:]+\s+%s\s*=\s*([^;]+);" % name, src))
    expr = m.group(1) if m else None
    if expr is None or "," in expr:                 # one name of a list: constexpr int BM = 128, BN = 64, ...;
        for decl in re.findall(r"constexpr\s+[\w:]+\s+([^;]+);", src):
            items = [i.split("=", 1) for i in decl.split(",")]
            if all(len(i) == 2 for i in items):
                expr = {k.strip(): v for k, v in items}.get(name, expr)
    assert expr is not None, "%s not found in %s" % (name, fname)
    expr = expr.strip()
    assert re.fullmatch(r"[0-9 *+()]+", expr), "%s = %r is not a plain integer expression" % (name, expr)
    return eval(expr)


@pytest.mark.parametrize("name", sorted(CONSTANTS))
def test_kernel_constants_match_the_boundary_cases(name):
    fname, want = CONSTANTS[name]
    assert _source_value(fname, name) == want, \
        "%s changed: move the boundary cases of tests/test_gpu_engine.py that are built from it, then update this table" % name


def test_source_value_reads_one_name_of_a_constexpr_list():
    with open(os.path.join(CSRC, "int8_conv.cu")) as f:
        assert "constexpr int BM = 128, BN = 64, BK = 64, STAGES = 3, THREADS = 128;" in f.read()
    assert [_source_value("int8_conv.cu", n) for n in ("BN", "STAGES")] == [64, 3]


def test_int8_tile_cases_cover_both_sides_of_every_tile_size():
    """tests/test_gpu_int8.py TILES: M = N*OH*OW around BM, O around BN and 2 BN, C around 16 and BK, KT = 1 to STAGES + 1,
    and an image boundary inside an M tile."""
    import test_gpu_int8 as G
    bm, bn, bk, stages = (CONSTANTS[k][1] for k in ("BM", "BN", "BK", "STAGES"))
    assert G.TILE_EDGES == dict(M={1, 31, bm - 1, bm, bm + 1}, O={1, 7, 9, bn - 1, bn, bn + 1, 2 * bn + 1},
                                C={1, 15, 16, 17, bk, bk + 1}, KT=set(range(1, stages + 2)))
    geo = [G.tile_geometry(c) for c in G.TILES]
    for i, key in enumerate(("M", "O", "C", "KT")):
        assert G.TILE_EDGES[key] <= {g[i] for g in geo}, key
    # an M tile holding the last pixels of one image and the first of the next
    assert any(c[0] > 1 and any((m0 // (g[0] // c[0])) != ((min(m0 + bm, g[0]) - 1) // (g[0] // c[0]))
                                for m0 in range(0, g[0], bm)) for c, g in zip(G.TILES, geo))


def test_scan_columns_derive_from_the_inverse_cache():
    """kScanCols (initial column scan in shared memory) is derived from DFQ_INV_CACHE; the scan boundary cases use 1024."""
    with open(os.path.join(CSRC, "cle_engine.cu")) as f:
        src = f.read()
    assert "constexpr int kScanCols = (kInvCache + 4) / 2 < 1024 ? (kInvCache + 4) / 2 : 1024;" in src
    inv = CONSTANTS["DFQ_INV_CACHE"][1]
    assert min((inv + 4) // 2, 1024) == 1024


def _layer(shape, seed, scale=0.1):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal(shape) * scale).astype(np.float32)


def _expect(n, seed):
    rng = np.random.default_rng(seed)
    return O.relu_expectation((rng.random(n) + 0.4).astype(np.float32), (rng.standard_normal(n) * 0.5).astype(np.float32))


BOUND_LAYERS = [((48, 64, 3, 3), 64), ((36, 640, 1, 1), 640), ((16, 3, 3, 3), 3), ((6, 1200, 2, 2), 1200),
                ((64, 1, 3, 3), 64), ((24, 96, 5, 5), 96), ((12, 32, 3, 3), 64)]


@pytest.mark.parametrize("signed", [False, True])
@pytest.mark.parametrize("shape,n", BOUND_LAYERS)
def test_bias_bound_accepts_the_oracle(shape, n, signed):
    w, ex = _layer(shape, 1), _expect(n, 2)
    exact, bound = O.bias_delta_bound(w, ex, signed=signed)
    assert O.rows_outside_bound(O.bias_delta(w, ex, signed=signed), exact, bound).size == 0
    exact, bound = O.bias_delta_bound(w, ex, raw=True)
    assert O.rows_outside_bound(O.bias_absorb_wc(w, ex, n), exact, bound).size == 0


def test_bias_bound_rejects_a_dropped_last_column():
    w, ex = _layer((48, 64, 3, 3), 3), _expect(64, 4)
    exact, bound = O.bias_delta_bound(w, ex)
    E = O.quantize_error(w).reshape(48, 64, -1).sum(axis=-1, dtype=np.float32)
    E[:, -1] = 0
    got = (E.astype(np.float64) @ ex.astype(np.float64)).astype(np.float32)
    assert O.rows_outside_bound(got, exact, bound).size == 48


@pytest.mark.parametrize("shape,n", [((48, 64, 3, 3), 64), ((36, 640, 1, 1), 640)])
def test_bias_bound_rejects_half_a_percent_in_the_smallest_row(shape, n):
    """Rows with gains over two decades (as the GPU tests draw them): the smallest delta is far below the layer's largest."""
    rng = np.random.default_rng(5)
    gain = 10 ** rng.uniform(-1, 1, (shape[0],) + (1,) * (len(shape) - 1))
    w, ex = (_layer(shape, 5) * gain).astype(np.float32), _expect(n, 6)
    d = O.bias_delta(w, ex)
    exact, bound = O.bias_delta_bound(w, ex)
    assert O.rows_outside_bound(d, exact, bound).size == 0
    i = int(np.argmin(np.abs(d)))
    d[i] = np.float32(d[i] * np.float32(1.005))
    assert list(O.rows_outside_bound(d, exact, bound)) == [i]


def test_bias_bound_rejects_the_wrong_groups_expectation():
    """Grouped layer (G = 2: 12 rows x 32 columns, E[x] of 64 channels): rows of group 0 read group 1's slice."""
    w, ex = _layer((12, 32, 3, 3), 7), _expect(64, 8)
    exact, bound = O.bias_delta_bound(w, ex)
    swapped = np.concatenate([ex[32:], ex[:32]])
    got = O.bias_delta(w, ex)
    got[:6] = O.bias_delta(w, swapped)[:6]
    assert list(O.rows_outside_bound(got, exact, bound)) == list(range(6))
