"""ncnn.load / ncnn.write without a GPU: the reader against tests/ncnn_int8_case.py's parser on the reference's model, every
refusal on mutated copies of its files (before any library call), a writer -> reader round trip of a seeded ResNet-18
through tests/fakelib_ncnn.py, and the plane-mean oracle against an explicit loop."""
import os

import numpy as np
import pytest
import torch

import ncnn_int8_case as case
import ncnn_oracle

needs_model = pytest.mark.skipif(case.paths() is None, reason="the reference's int8 ncnn model is not staged")


@pytest.fixture
def fake(monkeypatch):
    import fakelib_ncnn
    return fakelib_ncnn.install(monkeypatch)


@needs_model
def test_reader_matches_the_interpreter_parser_field_for_field():
    from dfq_b200 import ncnn
    pp, bp = case.paths()
    assert os.path.getsize(bp) == 3614632
    layers = ncnn.parse_param(pp)
    ref = case.parse_param()
    assert len(layers) == len(ref) == 112
    for a, b in zip(layers, ref):
        assert (a["type"], a["name"], a["bottoms"], a["tops"]) == (b["type"], b["name"], b["bottoms"], b["tops"])
        assert all(a["params"][k] == v for k, v in b["params"].items())
    recs = ncnn.parse_bin(bp, layers)
    want = case.parse()
    assert list(recs) == [r["name"] for r in want]
    for r in want:
        got = recs[r["name"]]
        assert np.array_equal(got["codes"], r["codes"])
        assert np.array_equal(got["bias"], r["bias"])
        assert np.array_equal(got["w_scales"], r["w_scales"])
        assert got["in_scale"].tobytes() == np.float32(r["in_scale"]).tobytes()


@needs_model
def test_loaded_graph_is_named_by_blob(fake):
    from dfq_b200 import ncnn
    gm = ncnn.load(*case.paths())
    names = [n.name for n in gm.graph.nodes if n.op != "output"]
    layers = ncnn.parse_param(case.paths()[0])
    want = [ncnn.ident(l["tops"][0]) for l in layers if l["type"] != "Split"]
    # every layer but the Splits is a node named by its top; an InnerProduct adds its two reshapes' nodes
    assert [n for n in names if not n.endswith(("_in", "_fc"))] == want
    assert len(want) == 112 - 10
    assert names.count("_781_in") == names.count("_781_fc") == 1


def _mutated(tmp_path, param_edit=None, bin_edit=None):
    pp, bp = case.paths()
    p2, b2 = str(tmp_path / "m.param"), str(tmp_path / "m.bin")
    text = open(pp).read()
    open(p2, "w").write(param_edit(text) if param_edit else text)
    data = open(bp, "rb").read()
    open(b2, "wb").write(bin_edit(data) if bin_edit else data)
    return p2, b2


def _line(text, name, edit):
    lines = text.split("\n")
    i = next(i for i, l in enumerate(lines) if len(l.split()) > 1 and l.split()[1] == name)
    lines[i] = edit(lines[i])
    return "\n".join(lines)


REFUSALS = [
    ("type", lambda t: _line(t, "621", lambda l: l.replace("ReLU ", "Sigmoid", 1)), None, "621 (Sigmoid)"),
    ("key", lambda t: _line(t, "619", lambda l: l + " 9=1"), None, "key 9 is not implemented"),
    ("value", lambda t: _line(t, "643", lambda l: l + " 0=2"), None, "only op_type 0"),
    ("fp32-record", lambda t: _line(t, "619", lambda l: l.replace("8=2", "8=0")), None, "int8_scale_term"),
    ("reduction", lambda t: _line(t, "780", lambda l: l.replace("0=3", "0=0")), None, "operation 3"),
    ("pad", lambda t: _line(t, "619", lambda l: l.replace("4=1", "4=-233")), None, "non-negative padding"),
    ("order", lambda t: _line(t, "621", lambda l: l.replace(" 619 621", " 999 621")), None,
     "bottom blob 999 is used before it is produced"),
    ("split", lambda t: _line(t, "splitncnn_0", lambda l: l.replace("1 2 633", "1 3 633")), None, "splitncnn_0"),
    ("tag", None, lambda d: b"\0\0\0\0" + d[4:], "record tag"),
    ("truncated", None, lambda d: d[:-8], "ends at byte"),
    ("long", None, lambda d: d + b"\0\0\0\0", "account for"),
]


@needs_model
@pytest.mark.parametrize("what,pe,be,msg", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_refusals_by_name_before_any_library_call(fake, tmp_path, what, pe, be, msg):
    from dfq_b200 import ncnn
    p, b = _mutated(tmp_path, pe, be)
    with pytest.raises(ncnn.NcnnError, match=msg.replace("(", r"\(").replace(")", r"\)")):
        ncnn.load(p, b)
    assert fake.calls == []


def test_write_read_round_trip_resnet18(fake, tmp_path):
    from dfq_b200 import int8 as I, ncnn
    import ncnn_models
    m, graph, targ = ncnn_models.resnet18_int8()
    p, b, t = (str(tmp_path / ("r." + e)) for e in ("param", "bin", "table"))
    written = ncnn.write(m, graph, targ, p, b, t)
    types = [w[0] for w in written]
    assert types.count("Convolution") == 20 and types.count("InnerProduct") == 1 and types.count("BinaryOp") == 8
    assert types.count("Pooling") == 2 and "Flatten" in types and types.count("Split") == 8
    gm = ncnn.load(p, b)
    src = [mod for mod in m.modules() if isinstance(mod, I._Int8Layer)]
    got = [mod for mod in gm.modules() if isinstance(mod, I.Int8Conv2d)]
    assert len(src) == len(got) == 21
    for a, c in zip(src, got):
        assert torch.equal(a.weight_codes, c.weight_codes) and torch.equal(a.bias, c.bias)
        assert torch.equal(a.w_scale, c.w_scale) and a.act_scale == c.act_scale
        assert (a.kernel_size, a.stride, a.padding, a.groups) == (c.kernel_size, c.stride, c.padding, c.groups)
    table = open(t).read().split("\n")
    assert table[0].startswith(written[1][1] + "_param_0 ")


def test_write_refuses_a_node_it_cannot_read_back(fake, tmp_path):
    from dfq_b200 import ncnn
    import ncnn_models

    class Sig(torch.nn.Module):
        def __init__(self, m):
            super().__init__()
            self.m = m

        def forward(self, x):
            return torch.sigmoid(self.m(x))
    m, graph, targ = ncnn_models.resnet18_int8()
    with pytest.raises(ncnn.NcnnError, match="sigmoid"):
        ncnn.write(Sig(m), graph, targ, str(tmp_path / "a.param"), str(tmp_path / "a.bin"))
    assert not os.path.exists(tmp_path / "a.param")


def test_plane_mean_oracle_is_the_left_to_right_loop():
    f = np.float32
    rows = [[np.nan, 1, 2], [np.inf, -np.inf, 1], [-0.0, -0.0, -0.0], [1e-45, 1e-45, 3e-45], [1e8, 1, -1e8],
            [3e38, 3e38, -3e38], [0.1, 0.2, 0.3]]
    x = np.array(rows, f)[None]
    for divide in (False, True):
        got = ncnn_oracle.plane_mean(x, divide)[0]
        for i, r in enumerate(rows):
            s = f(0)
            with np.errstate(over="ignore", invalid="ignore"):
                for v in r:
                    s = f(s + f(v))
                want = f(s / f(3)) if divide else f(s * f(f(1) / f(3)))
            assert np.array_equal(np.array(got[i]).view(np.int32), np.array(want).view(np.int32), equal_nan=False) or \
                (np.isnan(got[i]) and np.isnan(want)), (i, got[i], want)
    assert not np.signbit(ncnn_oracle.plane_mean(x, True)[0, 2])     # the sum starts at +0.f: -0.0 planes give +0.0


def _structure(layers):
    """(type, params, bottoms as (producer index, top index)) per layer: a .param with its names aside."""
    where = {t: (i, j) for i, l in enumerate(layers) for j, t in enumerate(l["tops"])}
    return [(l["type"], l["params"], [where[b] for b in l["bottoms"]]) for l in layers]


@needs_model
def test_written_mobilenetv2_is_the_reference_file_names_aside(monkeypatch, tmp_path):
    """The bundled checkpoint, oracle-calibrated (BN fold + signed CLE) and converted at the table's activation scales,
    written by ncnn.write: the reference's 112 layer types, keys and wiring, a .bin of its 3,614,632 bytes whose codes equal
    the reference's wherever the oracle's codes of this calibration do, a .table named by the written blobs, and a reader
    that gives back every code, bias and scale."""
    import fakelib
    import fakelib_ncnn
    import ncnn_models
    import int8_oracle as O
    from dfq_b200 import int8 as I, ncnn
    fakelib_ncnn.install(monkeypatch, fakelib.torch_sqrt)
    graph, targ = case.calibrated_graph(monkeypatch)
    rows = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ncnn_table_rows.npz"))
    model, _, _ = ncnn_models.mobilenetv2_int8(graph, targ, rows["activation_scales"])
    p, b, t = (str(tmp_path / ("m." + e)) for e in ("param", "bin", "table"))
    ncnn.write(model, graph, targ, p, b, t)                     # the table from the calibration's observers
    mine, ref = ncnn.parse_param(p), ncnn.parse_param(case.paths()[0])
    assert _structure(mine) == _structure(ref)
    assert os.path.getsize(b) == os.path.getsize(case.paths()[1]) == 3614632
    recs, want = ncnn.parse_bin(b, mine), case.parse()
    layers = [graph[k] for k in graph if type(graph[k]) in targ]
    same = 0
    for lay, r, src, ws in zip([l for l in mine if l["type"] in ncnn.WEIGHTED], want, layers, rows["weight_scales"]):
        got = recs[lay["name"]]
        oracle = O.i8_quantize(src.weight.detach().numpy().reshape(-1), np.float32(ws))
        eq = oracle == r["codes"]
        assert np.array_equal(got["codes"][eq], r["codes"][eq]), lay["name"]
        same += int((got["codes"] == r["codes"]).sum())
    assert same >= 3_469_750
    table = open(t).read().split("\n")
    weighted = [l["name"] for l in mine if l["type"] in ncnn.WEIGHTED]
    assert [ln.split()[0] for ln in table[:53]] == [n + "_param_0" for n in weighted]
    assert [ln.split()[0] for ln in table[53:106]] == weighted
    types = [l["type"] for l in mine]
    assert types.count("Split") == 10 and types[-3:] == ["Reduction", "InnerProduct", "Softmax"]
    gm = ncnn.load(p, b)
    src = [m for m in model.modules() if isinstance(m, I._Int8Layer)]
    got = [m for m in gm.modules() if isinstance(m, I.Int8Conv2d)]
    assert len(src) == len(got) == 53
    for a, c in zip(src, got):
        assert torch.equal(a.weight_codes, c.weight_codes) and torch.equal(a.bias, c.bias)
        assert torch.equal(a.w_scale, c.w_scale) and a.act_scale == c.act_scale
        assert (a.kernel_size, a.stride, a.padding, a.groups) == (c.kernel_size, c.stride, c.padding, c.groups)
    assert sum(isinstance(m, ncnn.PlaneMean) and not m.divide for m in gm.modules()) == 1


READER_DIMS = [
    ("reduction-not-after-reshape", lambda t: _line(_line(t, "779", lambda l: l.replace("Reshape ", "ReLU    ", 1)
                                                          .replace(" 0=-1 1=1280", "")), "780", lambda l: l),
     "blob 779 is 3-D"),
    ("reshape-of-a-vector", lambda t: _line(t, "779", lambda l: l.replace(" 767 779", " 780x 779")), "used before"),
    ("depthwise-term-2", lambda t: _line(t, "622", lambda l: l.replace("8=1", "8=2")), "int8_scale_term must be 1"),
]


@needs_model
@pytest.mark.parametrize("what,pe,msg", READER_DIMS, ids=[r[0] for r in READER_DIMS])
def test_reader_refuses_layouts_it_does_not_read(fake, tmp_path, what, pe, msg):
    from dfq_b200 import ncnn
    p, b = _mutated(tmp_path, pe)
    with pytest.raises(ncnn.NcnnError, match=msg):
        ncnn.load(p, b)
    assert fake.calls == []
