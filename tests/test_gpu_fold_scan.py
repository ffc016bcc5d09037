"""The read-only scan of deferred BN folds (DFQ_FOLD_DEFER with a column scan, scan_go > 0, or a row scan, scan_rows) on both
of its kernels: the streaming k_fold_scan (DFQ_FOLD_SCAN_STREAM=1, the default where it applies) and the RowPipe k_bn_fold<false>
(DFQ_FOLD_SCAN_STREAM=0).  Both run on the same arena bits and must leave the same arena bits: column extrema (buffer 0), row
extrema, fold factors, biases and BN vectors; the weights are read only.  The fixtures are built here directly on the C ABI."""
import numpy as np
import pytest
import torch

from stack_cases import SUBNORMAL

pytestmark = pytest.mark.gpu


def _lib():
    from dfq_b200 import _lib
    _lib.require_cuda()
    return _lib


def _align4(n):
    return (n + 3) & ~3


def _build(specs, seed):
    """specs: dicts(shape=(O, J, kh, kw), go=rows per group (0: no column scan), rows=row scan, prefix=row_prefix,
    edit=f(w, gamma)).  Returns (arena on the GPU, layer table, fold table)."""
    L = _lib()
    g = torch.Generator().manual_seed(seed)
    chunks, off = [], 0
    lt = np.zeros(len(specs), dtype=L.LAYER_DT)
    ft = np.zeros(len(specs), dtype=L.FOLD_DT)

    def put(t):
        nonlocal off
        t = t.reshape(-1).float()
        pad = _align4(t.numel()) - t.numel()
        chunks.append(torch.cat([t, torch.zeros(pad)]))
        o = off
        off += t.numel() + pad
        return o

    for i, sp in enumerate(specs):
        O, J, kh, kw = sp["shape"]
        w = torch.randn(O, J, kh, kw, generator=g) * (10 ** torch.empty(O, 1, 1, 1).uniform_(-1, 1, generator=g))
        gamma = torch.rand(O, generator=g) + 0.5
        if sp.get("edit"):
            sp["edit"](w, gamma, g)
        go = sp.get("go", 0)
        nch = (O // go) * J if go else 0
        l, f = lt[i], ft[i]
        l["w_off"] = put(w)
        l["bias_off"] = put(torch.randn(O, generator=g) * 0.1)
        l["rows"], l["cols"], l["kk"] = O, J, kh * kw
        l["rel_in"] = l["rel_out"] = -1
        l["cmin_off"] = put(torch.full((2 * max(nch, 1),), 7.0))
        l["cmax_off"] = put(torch.full((2 * max(nch, 1),), -7.0))
        l["rext_off"] = put(torch.full((2 * O,), 3.0))
        l["fold_off"] = -1
        f["layer"], f["bn_eps"], f["mode"] = i, 1e-5, 1                 # DFQ_FOLD_DEFER
        f["gamma_off"] = put(gamma)
        f["beta_off"] = put(torch.randn(O, generator=g) * 0.2)
        f["mean_off"] = put(torch.randn(O, generator=g) * 0.1)
        f["var_off"] = put(torch.rand(O, generator=g) + 0.5)
        f["fake_w_off"] = put(torch.zeros(O))
        f["fake_b_off"] = put(torch.zeros(O))
        f["fac_off"] = put(torch.zeros(O))
        f["scan_go"], f["scan_gi"] = go, (J if go else 0)
        f["scan_rows"] = 1 if sp.get("rows") else 0
        f["row_prefix"] = sp.get("prefix", 0)
    arena = torch.cat(chunks).cuda()
    return arena, lt, ft


def _fold(arena, lt, ft, stream, monkeypatch):
    L = _lib()
    if stream is None:
        monkeypatch.delenv("DFQ_FOLD_SCAN_STREAM", raising=False)
    else:
        monkeypatch.setenv("DFQ_FOLD_SCAN_STREAM", str(stream))
    a = arena.clone()
    L.check(L.load().dfq_bn_fold(a.data_ptr(), a.numel(), L.table_ptr(lt), len(lt), L.table_ptr(ft), len(ft), L.stream_ptr()),
            "dfq_bn_fold")
    torch.cuda.synchronize()
    return a


def _assert_same_bits(a, b):
    diff = (a.view(torch.int32) != b.view(torch.int32)).nonzero().flatten()
    assert diff.numel() == 0, "arenas differ at %d floats, first %s: %s vs %s" % (
        diff.numel(), diff[:4].tolist(), a[diff[:4]].tolist(), b[diff[:4]].tolist())


def _both(specs, monkeypatch, seed=5):
    arena, lt, ft = _build(specs, seed)
    new = _fold(arena, lt, ft, 1, monkeypatch)
    old = _fold(arena, lt, ft, 0, monkeypatch)
    _assert_same_bits(new, old)
    _assert_same_bits(_fold(arena, lt, ft, None, monkeypatch), new)      # the default takes the streaming kernel
    return arena, lt, ft, new


# ---- edits: (w, gamma, generator) in place ------------------------------------------------------------------------------
def _degenerate(w, gamma, g):
    """a zero row, a row of -0.0, a NaN row, a row with one NaN, a row of subnormals, a constant row; a zero column"""
    w[1] = 0.0
    w[2] = -0.0
    w[3] = float("nan")
    w[4].view(-1)[5] = float("nan")
    w[5] = torch.randn(w[5].shape, generator=g) * SUBNORMAL
    w[6] = 0.5
    w[:, 1] = 0.0
    w.view(-1)[::97] = SUBNORMAL


def _negative_zero_gamma(w, gamma, g):
    """about 30 % negative BN scales (extrema swap) and a few zero ones (folded rows of +-0.0)"""
    flip = torch.rand(gamma.shape, generator=g) < 0.3
    gamma.copy_(torch.where(flip, -gamma, gamma))
    gamma[torch.randperm(gamma.numel(), generator=g)[:max(2, gamma.numel() // 16)]] = 0.0


def _all_edits(w, gamma, g):
    _negative_zero_gamma(w, gamma, g)
    _degenerate(w, gamma, g)


# ---- cases ---------------------------------------------------------------------------------------------------------------
COLUMN_CASES = {
    "kk9": [dict(shape=(256, 128, 3, 3), go=256)],
    "kk1": [dict(shape=(200, 96, 1, 1), go=200)],
    "full_stage_rows": [dict(shape=(64, 512, 3, 3), go=64)],                        # 4608-float rows, one per tile
    "grouped_kk9": [dict(shape=(96, 40, 3, 3), go=32)],                            # 3 groups, 120 columns
    "grouped_kk1": [dict(shape=(64, 48, 1, 1), go=16)],                            # 4 groups, 192 columns
    "grouped_at_scratch": [dict(shape=(64, 256, 1, 1), go=16)],                    # 1024 columns: a warp's whole scratch
    "short_rows": [dict(shape=(100, 4, 3, 3), go=100), dict(shape=(24, 100, 1, 1), go=24)],
    "odd_rows": [dict(shape=(21, 5, 3, 3), go=21), dict(shape=(37, 44, 3, 3), go=37)],   # 45-float rows: plain-copy tails
}


@pytest.mark.parametrize("edit", [None, _negative_zero_gamma, _degenerate, _all_edits],
                         ids=["plain", "neg_zero_gamma", "degenerate", "all"])
@pytest.mark.parametrize("case", sorted(COLUMN_CASES))
def test_column_scan_same_bits(case, edit, monkeypatch):
    specs = [dict(sp, edit=edit) for sp in COLUMN_CASES[case]]
    _both(specs, monkeypatch)


def test_column_scan_values(monkeypatch):
    """the streaming kernel's extrema are those of fl(w * f) computed here (every row finite)"""
    arena, lt, ft = _build([dict(shape=(96, 40, 3, 3), go=32, edit=_negative_zero_gamma)], 9)
    a = _fold(arena, lt, ft, 1, monkeypatch)
    l, f = lt[0], ft[0]
    O, J, kk = int(l["rows"]), int(l["cols"]), int(l["kk"])
    w = arena[int(l["w_off"]):int(l["w_off"]) + O * J * kk].view(O, J, kk)
    fac = a[int(f["fac_off"]):int(f["fac_off"]) + O]
    v = (w * fac.view(O, 1, 1)).view(3, 32, J, kk)                                 # 3 groups of 32 rows
    mn = v.amin(dim=(1, 3)).reshape(-1)
    mx = v.amax(dim=(1, 3)).reshape(-1)
    assert torch.equal(a[int(l["cmin_off"]):int(l["cmin_off"]) + 3 * J], mn)
    assert torch.equal(a[int(l["cmax_off"]):int(l["cmax_off"]) + 3 * J], mx)


@pytest.mark.parametrize("prefix", [0, 1, 16, 1000])
@pytest.mark.parametrize("shape", [(512, 256, 1, 1), (128, 64, 3, 3), (44, 16, 3, 3), (21, 5, 3, 3)],
                         ids=["1x1_256", "kk9_576", "kk9_144", "kk9_45"])
def test_row_scan_same_bits(shape, prefix, monkeypatch):
    _both([dict(shape=shape, rows=True, prefix=prefix, edit=_all_edits)], monkeypatch)


def test_row_and_column_scan_of_one_layer(monkeypatch):
    _both([dict(shape=(128, 64, 3, 3), go=128, rows=True, edit=_all_edits),
           dict(shape=(96, 40, 1, 1), go=32, rows=True, edit=_degenerate)], monkeypatch)


def test_ring_tails_across_layers(monkeypatch):
    """many layers of different tile counts and row lengths in one launch: a consumer warp meets layer changes at every
    position of its ring sequence, flushes its column scratch mid-stream and ends on partial tiles"""
    shapes = [(37, 44, 3, 3), (24, 100, 1, 1), (100, 4, 3, 3), (21, 5, 3, 3), (512, 512, 3, 3), (44, 16, 3, 3),
              (64, 48, 1, 1), (200, 96, 1, 1), (13, 7, 1, 1)]
    specs = []
    for i in range(27):
        s = shapes[i % len(shapes)]
        if i % 3 == 2:        # a row scan with a prefix (no column scan)
            specs.append(dict(shape=s, rows=True, prefix=(0, 1, 16, 1000)[i % 4]))
        else:
            go = s[0] // 2 if (s[0] % 2 == 0 and i % 2) else s[0]
            specs.append(dict(shape=s, go=go, rows=(i % 4 == 0), edit=_negative_zero_gamma if i % 5 == 0 else None))
    _both(specs, monkeypatch, seed=11)


def test_more_columns_than_the_scratch(monkeypatch):
    """a column-scanned layer of more than 1024 columns: the launch stays on k_bn_fold<false> (its global-atomic path), and
    forcing the streaming kernel is refused rather than silently served by the other one"""
    L = _lib()
    specs = [dict(shape=(16, 1100, 1, 1), go=16, edit=_negative_zero_gamma), dict(shape=(64, 64, 3, 3), go=64)]
    arena, lt, ft = _build(specs, 3)
    _assert_same_bits(_fold(arena, lt, ft, None, monkeypatch), _fold(arena, lt, ft, 0, monkeypatch))
    with pytest.raises(L.DfqError, match="DFQ_FOLD_SCAN_STREAM"):
        _fold(arena, lt, ft, 1, monkeypatch)
