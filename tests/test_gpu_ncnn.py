"""ncnn.load / ncnn.write and their kernels on the GPU: every blob of the reference's int8 model against the interpreter
with the integer oracle and the oracle's plane mean, the code packers, dfq_i8_plane_mean against the oracle, the chained
and saved model, and a seeded ResNet-18 written and read back."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import ncnn_int8_case as case
import ncnn_oracle

pytestmark = pytest.mark.gpu
needs_model = pytest.mark.skipif(case.paths() is None, reason="the reference's int8 ncnn model is not staged")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _batch(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, 3, 224, 224, generator=g)


@needs_model
def test_every_blob_equals_the_oracle_interpreter_through_the_inner_product():
    from dfq_b200 import ncnn
    x = _batch(2)
    net = case.Int8Net()
    ref = net.forward(x, case.oracle_executor, upto="779")
    pooled = torch.from_numpy(ncnn_oracle.plane_mean(ref["779"].numpy(), False))
    ip = next(l for l in net.layers if l["name"] == "781")
    ref["780"] = pooled
    ref["781"] = case.oracle_executor(ip["spec"], pooled.reshape(2, -1, 1, 1)).reshape(2, -1)
    layers = ncnn.parse_param(case.paths()[0])
    blobs = [l["tops"][0] for l in layers if l["type"] not in ("Split", "Softmax")]
    gm = ncnn.load(*case.paths(), outputs=blobs + ["782"])
    got = gm(x.cuda())
    for name, y in zip(blobs, got):
        assert torch.equal(y.cpu(), ref[name]), name
    torch.testing.assert_close(got[-1].cpu(), torch.softmax(ref["781"], 1), rtol=1e-6, atol=1e-7)


@needs_model
def test_unpacked_codes_equal_the_file():
    from dfq_b200 import int8 as I, ncnn
    gm = ncnn.load(*case.paths())
    convs = [m for m in gm.modules() if isinstance(m, I.Int8Conv2d)]
    recs = case.parse()
    assert len(convs) == len(recs) == 53
    for m, r in zip(convs, recs):
        assert np.array_equal(m.unpack_codes().cpu().numpy().reshape(-1), r["codes"]), r["name"]


@pytest.mark.parametrize("O,C_in,k,groups", [(64, 3, 3, 1), (40, 40, 3, 40), (33, 17, 1, 1), (16, 256, 5, 1),
                                             (1000, 1280, 1, 1), (96, 96, 5, 96)])
def test_pack_then_unpack_is_the_identity(O, C_in, k, groups):
    from dfq_b200 import int8 as I
    g = torch.Generator().manual_seed(O + C_in + k)
    codes = torch.randint(-127, 128, (O, C_in // groups, k, k), generator=g, dtype=torch.int8)
    m = I.Int8Conv2d.from_codes(codes.numpy(), None, 8.0, 16.0, 1, k // 2, 1, groups)
    assert torch.equal(m.unpack_codes().cpu(), codes)
    w = codes.float() / 16.0                                    # the fp32 packer gives the same bytes, pads included
    assert torch.equal(I.Int8Conv2d(w, None, 8.0, 16.0, 1, k // 2, 1, groups).weight_codes, m.weight_codes)


def _bits(v):
    """fp32 bit patterns with every NaN as one pattern (the device's NaN payload is not the host's)."""
    v = np.array(v, np.float32)
    v[np.isnan(v)] = np.nan
    return v.view(np.int32)


def _plane(N, C_, P, seed, edges):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, C_, P, generator=g) * 3
    if edges:
        flat = x.view(-1)
        vals = torch.tensor([float("nan"), float("inf"), -float("inf"), -0.0, 1e-45, -3e-42, 1e30, -1e30])
        idx = torch.randint(0, flat.numel(), (min(64, flat.numel()),), generator=g)
        flat[idx] = vals[torch.arange(idx.numel()) % vals.numel()]
        x[0, 0] = -0.0
    return x


PLANES = [(1, 1, 1), (7, 17, 49), (256, 1280, 49), (1, 16, 263169), (7, 4096, 1), (3, 17, 4225), (256, 1280, 1),
          (1, 4096, 49)]


def _mean_call(xd, N, C_, P, divide, scale, want_y, want_q):
    """One dfq_i8_plane_mean call into fresh sentinel-filled buffers: (rc, y | None, yq | None)."""
    from dfq_b200 import _lib
    cp = (C_ + 15) // 16 * 16
    y = torch.full((N, C_), 7.0, device="cuda") if want_y else None
    yq = torch.full((N, cp), 99, dtype=torch.int8, device="cuda") if want_q else None
    ptr = lambda t: None if t is None else C.c_void_p(t.data_ptr())     # noqa: E731
    rc = _lib.load().dfq_i8_plane_mean(ptr(xd), ptr(y), ptr(yq), N, C_, P, divide, C.c_float(scale), _lib.stream_ptr())
    return rc, y, yq


@pytest.mark.parametrize("N,C_,P", PLANES)
@pytest.mark.parametrize("edges", [False, True])
def test_plane_mean_equals_the_oracle(N, C_, P, edges):
    x = _plane(N, C_, P, N * 31 + C_ * 7 + P, edges)
    xd = x.cuda()
    cp = (C_ + 15) // 16 * 16
    for divide in (0, 1):
        want = ncnn_oracle.plane_mean(x.numpy(), bool(divide))
        for scale in (0.0, 0.37, 1e30):
            codes = np.zeros((N, cp), np.int8)
            codes[:, :C_] = ncnn_oracle.q8(want, np.float32(scale))
            for want_y, want_q in ((True, True), (True, False), (False, True)):     # together, then each alone
                rc, y, yq = _mean_call(xd, N, C_, P, divide, scale, want_y, want_q)
                assert rc == 0
                if y is not None:
                    assert np.array_equal(_bits(y.cpu().numpy()), _bits(want)), (divide, scale, want_y, want_q)
                if yq is not None:
                    assert np.array_equal(yq.cpu().numpy(), codes), (divide, scale, want_y, want_q)


def test_plane_mean_and_packers_do_not_synchronise_the_host():
    from dfq_b200 import int8 as I, ncnn
    x = _plane(256, 1280, 49, 11, False).cuda()
    mean, codes_mean = ncnn.PlaneMean(False), ncnn.PlaneMean(True, out_scale=0.5)
    codes = torch.randint(-127, 128, (64, 32, 3, 3), dtype=torch.int8)
    layer = I.Int8Conv2d.from_codes(codes.numpy(), None, 8.0, 16.0, 1, 1)
    y, q = mean(x), codes_mean(x)                               # first calls: library load, allocator warm-up
    layer.unpack_codes()
    torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(3):
            y2, q2 = mean(x), codes_mean(x)
            back = layer.unpack_codes()
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    assert torch.equal(y, y2) and torch.equal(q, q2) and torch.equal(back.cpu(), codes)


def test_device_refusals_name_the_condition():
    from dfq_b200 import _lib
    lib = _lib.load()
    x = torch.zeros(2, 16, 4, device="cuda")
    y = torch.zeros(2, 16, device="cuda")
    q = torch.zeros(64, dtype=torch.int8, device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr())                      # noqa: E731
    st = _lib.stream_ptr()
    cases = [((None, p(y), None, 2, 16, 4, 0, 1.0), "null input"),
             ((p(x), None, None, 2, 16, 4, 0, 1.0), "no output"),
             ((p(x), p(y), None, 2, 16, 0, 0, 1.0), "empty dimension"),
             ((p(x), p(y), None, 2, 16, 4, 2, 1.0), "divide must be"),
             ((p(x), None, C.c_void_p(q.data_ptr() + 1), 2, 16, 4, 0, 1.0), "16-byte aligned"),
             ((p(x), None, p(q), 2, 16, 4, 0, float("nan")), "out_scale"),
             ((p(x), p(x), None, 2, 16, 4, 0, 1.0), "overlap")]
    for args, msg in cases:
        assert lib.dfq_i8_plane_mean(*args[:7], C.c_float(args[7]), st) == -1
        err = lib.dfq_last_error().decode()
        assert err.startswith("dfq_i8_plane_mean: ") and msg in err, err
    from dfq_b200 import int8 as I
    m = I.Int8Conv2d.from_codes(np.ones((32, 16, 3, 3), np.int8), None, 8.0, 16.0, 1, 1)
    g = _lib.table_ptr(m._pack_geometry())
    codes = torch.zeros(32 * 16 * 9, dtype=torch.int8, device="cuda")
    before = m.weight_codes.clone()
    for fn in ("dfq_i8_pack_codes", "dfq_i8_unpack_codes"):
        src, dst = (codes, m.weight_codes) if fn == "dfq_i8_pack_codes" else (m.weight_codes, codes)
        assert getattr(lib, fn)(None, p(dst), g, st) == -1
        assert fn + ": null pointer" in lib.dfq_last_error().decode()
        assert getattr(lib, fn)(p(src), None, g, st) == -1
        assert fn + ": null pointer" in lib.dfq_last_error().decode()
        assert getattr(lib, fn)(p(m.weight_codes), C.c_void_p(m.weight_codes.data_ptr() + 64), g, st) == -1
        assert fn + ": codes and packed overlap" in lib.dfq_last_error().decode()
        assert getattr(lib, fn)(p(src), p(dst), None, st) == -1
        assert "null geometry" in lib.dfq_last_error().decode()
    assert torch.equal(m.weight_codes, before)


@needs_model
def test_chained_model_equals_the_per_layer_model_and_saves(tmp_path):
    from dfq_b200 import int8 as I, ncnn
    gm = ncnn.load(*case.paths())
    ch = I.chain_int8(gm, residual=True, pool_cat=True)
    convs = [m for m in ch.modules() if isinstance(m, I.Int8Conv2d)]
    assert len(ch.requantized_edges) == 52 and len(ch.fused_adds) == 10
    assert sum(m.codes_in for m in convs) == 52 and ch.requantized_edges[-1][0] == "_780_mean"
    for n in (1, 7, 256):
        x = _batch(n, n).cuda()
        assert torch.equal(gm(x), ch(x)), n
    path = str(tmp_path / "m.pt")
    I.save(ch, path)
    back = I.load(path)
    x = _batch(7, 3).cuda()
    assert torch.equal(back(x), ch(x))
    torch.save(x.cpu(), str(tmp_path / "x.pt"))
    torch.save(ch(x).cpu(), str(tmp_path / "y.pt"))
    code = ("import sys, torch; sys.path.insert(0, %r); from dfq_b200 import int8; m = int8.load(%r); "
            "x = torch.load(%r).cuda(); assert torch.equal(m(x).cpu(), torch.load(%r)); "
            "assert not any(k.startswith(('ncnn_int8_case', 'oracle')) for k in sys.modules)"
            % (ROOT, path, str(tmp_path / "x.pt"), str(tmp_path / "y.pt")))
    subprocess.run([sys.executable, "-c", code], check=True, cwd=str(tmp_path))


def test_resnet18_write_then_load(tmp_path):
    from dfq_b200 import ncnn
    import ncnn_models
    m, graph, targ = ncnn_models.resnet18_int8()
    p, b = str(tmp_path / "r.param"), str(tmp_path / "r.bin")
    written = ncnn.write(m, graph, targ, p, b)
    pool = next(w for w in written if w[0] == "Pooling" and (4, 1) in w[4])
    gm = ncnn.load(p, b, outputs=[pool[2][0], pool[3][0], written[-1][3][0]])
    x = _batch(7, 5).cuda()
    trunk = torch.nn.Sequential(*list(m.children())[:-2])
    feat, pooled, logits = gm(x)
    assert torch.equal(feat, trunk(x))
    assert torch.equal(pooled, torch.from_numpy(ncnn_oracle.plane_mean(feat.flatten(2).cpu().numpy(), True)).cuda())
    assert torch.equal(logits, m.fc(pooled))


@needs_model
def test_mobilenetv2_write_then_load_equals_the_converted_model_in_the_interpreter(monkeypatch, tmp_path):
    """This package's GPU calibration of the bundled checkpoint (BN fold, signed equalization), converted at the table's
    activation scales and written by ncnn.write: the loaded file equals, blob for blob, the same converted layers run in
    the interpreter on the written .param (its Reduction through ncnn's plane mean), and the converted model itself."""
    import ncnn_models
    import ncnn_table_case
    from dfq_b200 import int8 as I, ncnn
    if ncnn_table_case.checkpoint_path() is None:
        pytest.skip("the bundled checkpoint is not staged in oracle/_ref")
    graph, targ = case.calibrated_graph(monkeypatch)
    rows = np.load(os.path.join(ROOT, "tests", "golden", "ncnn_table_rows.npz"))
    model, _, _ = ncnn_models.mobilenetv2_int8(graph, targ, rows["activation_scales"])
    p, b = str(tmp_path / "m.param"), str(tmp_path / "m.bin")
    ncnn.write(model, graph, targ, p, b)
    monkeypatch.setattr(case, "paths", lambda: [p, b])
    net = case.Int8Net()
    layers = [m for m in model.modules() if isinstance(m, I._Int8Layer)]
    execute = lambda s, x: layers[s["index"]].run(x)[0]         # noqa: E731
    mean = next(l for l in net.layers if l["type"] == "Reduction")
    fc = next(l for l in net.layers if l["type"] == "InnerProduct")
    blobs = [l["tops"][0] for l in net.layers if l["type"] not in ("Split", "Softmax")]
    gm = ncnn.load(p, b, outputs=blobs)
    x = _batch(7, 9).cuda()
    ref = net.forward(x, execute, upto=net.layers[net.layers.index(mean) - 1]["name"])     # through the Reshape
    got = dict(zip(blobs, gm(x)))
    for name in blobs[:blobs.index(mean["tops"][0])]:
        assert torch.equal(got[name], ref[name]), name
    pooled = ncnn.PlaneMean(False)(ref[mean["bottoms"][0]])
    assert torch.equal(got[mean["tops"][0]], pooled)
    assert torch.equal(got[fc["tops"][0]], execute(fc["spec"], pooled.reshape(7, -1, 1, 1)).reshape(7, -1))
    assert torch.equal(got[fc["tops"][0]], model.classifier(pooled))
    assert torch.equal(got[mean["bottoms"][0]], model.features(x).view(7, 1280, -1))
