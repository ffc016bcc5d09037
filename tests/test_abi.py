"""The C-ABI library builds, loads without a GPU and exports exactly what include/dfq_b200.h declares."""
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_functions():
    src = open(os.path.join(ROOT, "include", "dfq_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(dfq_[a-z0-9_]+)\s*\(", src)))


def test_library_builds_and_exports_every_declared_symbol():
    from dfq_b200 import _build, _lib
    _build.build()
    lib = _lib.load(build_if_missing=False)
    names = _declared_functions()
    assert len(names) >= 18
    for n in names:
        assert hasattr(lib, n), "libdfq_sm90.so does not export %s" % n
    # and the binding covers every declared function (dfq_last_error is bound separately)
    for n in names:
        assert n in _lib.SIGNATURES or n == "dfq_last_error", "dfq_b200/_lib.py has no signature for %s" % n
    assert lib.dfq_abi_version() == _lib.ABI_VERSION


def test_struct_mirrors_match_compiled_sizes():
    from dfq_b200 import _lib
    lib = _lib.load()
    for i, (name, (dt, size)) in enumerate(_lib.EXPECTED_SIZES.items()):
        assert dt.itemsize == size, name
        assert lib.dfq_struct_size(i) == size, name
    assert lib.dfq_struct_size(99) == -1


def test_struct_field_offsets_follow_the_header_order():
    """numpy's aligned layout must equal the C layout: check a few load-bearing offsets."""
    from dfq_b200 import _lib
    assert _lib.LAYER_DT.fields["rows"][1] == 16 and _lib.LAYER_DT.fields["cmin_off"][1] == 48 and _lib.LAYER_DT.fields["group"][1] == 40
    assert _lib.RELATION_DT.fields["bn_w_off"][1] == 24 and _lib.RELATION_DT.fields["inv_off"][1] == 56
    assert _lib.CLE_PARAMS_DT.fields["converge_thres"][1] == 24 and _lib.CLE_PARAMS_DT.fields["max_sweeps"][1] == 36
    assert _lib.BC_LAYER_DT.fields["flags"][1] == 20 and _lib.BC_LAYER_DT.fields["expect_off"][1] == 24
    assert _lib.QUANT_TASK_DT.fields["minmax_off"][1] == 24


def test_product_refuses_to_run_without_cuda():
    import pytest
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from dfq_b200 import _lib, dfq
    with pytest.raises(_lib.DfqError):
        dfq._layer_equalization(torch.randn(4, 2, 3, 3), torch.randn(4, 4, 3, 3), torch.zeros(4))


def test_product_never_imports_the_oracle():
    """oracle/ is test infrastructure: nothing under dfq_b200/ or dropin/ may reference it."""
    for base in ("dfq_b200", "dropin"):
        for dirpath, _, files in os.walk(os.path.join(ROOT, base)):
            for f in files:
                if f.endswith(".py"):
                    text = open(os.path.join(dirpath, f)).read()
                    assert "import oracle" not in text and "from oracle" not in text, os.path.join(dirpath, f)


def test_host_copy_segments_gathers_and_scatters_ragged_tensors():
    """dfq_host_copy_segments (host helper, no CUDA call): a threaded gather into the staging image and the scatter back
    reproduce per-tensor copies exactly - empty segments, odd sizes, staging gaps and a multi-MB tensor that several
    threads split."""
    import ctypes as C
    from dfq_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(5)
    sizes = [0, 1, 7, 1000, 3, 2_500_001, 64, 0, 999_999, 12]
    src = [rng.standard_normal(n).astype(np.float32) for n in sizes]
    offs, o = [], 16
    for n in sizes:
        offs.append(o); o += 4 * n + 4 * int(rng.integers(0, 5))      # gaps between mirrors (alignment padding in the arena)
    staging = np.full(o // 4 + 8, -7.0, dtype=np.float32)
    ptrs = np.array([a.ctypes.data for a in src], dtype=np.uint64)
    nbytes = np.array([4 * n for n in sizes], dtype=np.uint64)
    offa = np.array(offs, dtype=np.uint64)
    for threads in (0, 1, 3, 8):
        staging[...] = -7.0
        rc = lib.dfq_host_copy_segments(C.c_void_p(staging.ctypes.data), _lib.table_ptr(ptrs), _lib.table_ptr(nbytes),
                                        _lib.table_ptr(offa), len(sizes), 0, threads)
        assert rc == 0
        expect = np.full_like(staging, -7.0)
        for a, off in zip(src, offs):
            expect[off // 4: off // 4 + a.size] = a
        assert np.array_equal(staging, expect)
        dst = [np.zeros_like(a) for a in src]
        dptr = np.array([a.ctypes.data for a in dst], dtype=np.uint64)
        rc = lib.dfq_host_copy_segments(C.c_void_p(staging.ctypes.data), _lib.table_ptr(dptr), _lib.table_ptr(nbytes),
                                        _lib.table_ptr(offa), len(sizes), 1, threads)
        assert rc == 0
        for a, b in zip(src, dst):
            assert np.array_equal(a, b)
    assert lib.dfq_host_copy_segments(None, None, None, None, 0, 0, 0) == 0
    assert lib.dfq_host_copy_segments(None, None, None, None, 3, 0, 0) == _lib.load().dfq_host_copy_segments(None, None, None, None, 3, 1, 0) != 0
    assert lib.dfq_host_copy_segments(C.c_void_p(staging.ctypes.data), _lib.table_ptr(ptrs), _lib.table_ptr(nbytes),
                                      _lib.table_ptr(offa), len(sizes), 2, 0) != 0


def test_host_copy_pool_survives_a_fork():
    """The helper threads do not exist in a forked child (DataLoader workers fork): the child starts its own pool."""
    import ctypes as C
    from dfq_b200 import _lib
    lib = _lib.load()

    def roundtrip():
        src = np.arange(3_000_000, dtype=np.float32)
        staging = np.zeros(src.size + 4, dtype=np.float32)
        ptrs = np.array([src.ctypes.data], dtype=np.uint64)
        nbytes = np.array([4 * src.size], dtype=np.uint64)
        offs = np.array([16], dtype=np.uint64)
        rc = lib.dfq_host_copy_segments(C.c_void_p(staging.ctypes.data), _lib.table_ptr(ptrs), _lib.table_ptr(nbytes),
                                        _lib.table_ptr(offs), 1, 0, 4)
        return rc == 0 and np.array_equal(staging[4:], src)

    assert roundtrip()                 # the parent's pool exists now
    pid = os.fork()
    if pid == 0:
        ok = False
        try:
            ok = roundtrip()
        finally:
            os._exit(0 if ok else 1)
    _, status = os.waitpid(pid, 0)
    assert os.WIFEXITED(status) and os.WEXITSTATUS(status) == 0
    assert roundtrip()
