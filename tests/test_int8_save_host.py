"""dfq_b200.int8.save / load on the CPU, through the host twins of the library: chained models of both schemes at every
flag round-trip to equal node lists, module states, shared storages and records and compute the same outputs; the file
loads under torch.load(weights_only=True); and every refusal leaves no file behind and the model unchanged."""
import os

import numpy as np
import pytest
import torch
import torch.fx as fx
import torch.nn as nn

import fakelib_int8_affine_pool_heads
import int8_layout_oracle as LO
from deeplab_mobilenet_padded import DeepLabMobileNetPadded
from ssd_lite_like import SSDLiteLike
from test_int8_affine_layout_host import CatNet
from test_int8_affine_layout_host import _chain as _affine_layout_chain
from test_int8_affine_pool_heads_host import CatPoolNet, PoolNet, fixed_range_model
from test_int8_affine_pool_heads_host import _chain as _affine_chain
from test_int8_chain_host import _identity_bns
from test_int8_pool_cat_host import _scales_through_pools
from test_int8_upsample_host import _convert

NCNN_FLAGS = [dict(), dict(residual=True), dict(residual=True, pool_cat=True),
              dict(residual=True, pool_cat=True, upsample=True),
              dict(residual=True, pool_cat=True, upsample=True, layout=True)]
AFFINE_FLAGS = [dict(), dict(residual=True), dict(residual=True, concat=True), dict(residual=True, pools=True),
                dict(residual=True, concat=True, fold_pads=True), dict(residual=True, concat=True, fold_pads=True, heads=True)]


def _called(gm):
    """{path: module} of what save() keeps: the graph's call_module targets and the chained layers."""
    from dfq_b200 import int8_io
    mods = {n.target: gm.get_submodule(n.target) for n in gm.graph.nodes if n.op == "call_module"}
    mods.update((p, gm.get_submodule(p)) for p in int8_io._uncalled_layers(gm, mods))
    return mods


def _attrs(m):
    from dfq_b200 import int8_io
    if isinstance(m, int8_io._LAYERS):
        keys = m._copied + m._modes
    elif type(m) in int8_io._CONSTRUCTED:
        keys = int8_io._CONSTRUCTED[type(m)]
    else:
        keys = [k for k in vars(m) if not k.startswith("_")]
    return {k: (getattr(m, k).tolist() if isinstance(getattr(m, k), np.ndarray) else getattr(m, k)) for k in keys}


def _node_list(gm):
    return [(n.op, n.name, n.target, fx.node.map_arg(n.args, lambda a: ("node", a.name)),
             fx.node.map_arg(n.kwargs, lambda a: ("node", a.name))) for n in gm.graph.nodes]


def _storage_groups(gm):
    """The partition of (path, tensor name) by the storage it lives in."""
    groups = {}
    for p, m in _called(gm).items():
        for k, t in list(m._buffers.items()) + list(m._parameters.items()):
            if t is not None:
                groups.setdefault(t.untyped_storage().data_ptr(), set()).add((p, k))
    return sorted(sorted(g) for g in groups.values())


def assert_round_trip(gm, m):
    """m equals gm in everything save() keeps."""
    from dfq_b200 import int8_io
    assert _node_list(m) == _node_list(gm)
    assert type(m).__name__ == type(gm).__name__
    a, b = _called(gm), _called(m)
    assert a.keys() == b.keys()
    for p in a:
        assert type(a[p]) is type(b[p]), p
        assert _attrs(a[p]) == _attrs(b[p]), p
        for k in list(a[p]._buffers) + list(a[p]._parameters):
            x, y = getattr(a[p], k), getattr(b[p], k)
            assert x.dtype == y.dtype and torch.equal(x, y), (p, k)
        for ha, hb in zip(getattr(a[p], "heads", ()), getattr(b[p], "heads", ())):   # the same modules as at their paths
            assert hb is b[next(q for q in a if a[q] is ha)], p
    assert _storage_groups(m) == _storage_groups(gm)
    for k in int8_io.RECORDS:
        assert hasattr(m, k) == hasattr(gm, k), k
        if hasattr(gm, k):
            assert getattr(m, k) == getattr(gm, k), k


def _same(a, b):
    if isinstance(a, (tuple, list)):
        return len(a) == len(b) and all(_same(u, v) for u, v in zip(a, b))
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


def _round_trip(gm, x, tmp_path, name="m.pt"):
    from dfq_b200 import int8
    path = tmp_path / name
    int8.save(gm, path)
    m = int8.load(path)
    assert_round_trip(gm, m)
    if x is not None:
        with torch.no_grad():
            assert _same(m(x), gm(x))
    return m, path


def _ncnn_round_trips(monkeypatch, tmp_path, model, x, flag_sets):
    """[(gm, loaded)] of `model` converted through the ncnn twins and chained at each of flag_sets, both run on x.  Saved
    and loaded before the CPU tensors pass for GPU ones (the chains trace the real F.interpolate)."""
    from dfq_b200 import int8
    LO.install(monkeypatch)
    _convert(model.eval(), _scales_through_pools(model))
    pairs = [(gm, _round_trip(gm, None, tmp_path, "m%d.pt" % i)[0])
             for i, gm in enumerate(int8.chain_int8(model, **flags) for flags in flag_sets)]
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    for gm, m in pairs:
        with torch.no_grad():
            assert _same(m(x), gm(x))
    return pairs


# ---- both schemes at every flag -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("net", ["ssd", "deeplab"])
def test_ncnn_chains_round_trip(monkeypatch, tmp_path, net):
    model = _identity_bns(SSDLiteLike(num_classes=5, is_test=True) if net == "ssd" else DeepLabMobileNetPadded(num_classes=5))
    x = torch.randn(1, 3, 65, 65, generator=torch.Generator().manual_seed(2))
    pairs = _ncnn_round_trips(monkeypatch, tmp_path, model, x, NCNN_FLAGS)
    assert len(pairs[-1][1].fused_heads if net == "ssd" else pairs[-1][1].folded_pads) == (2 if net == "ssd" else 17)


@pytest.mark.parametrize("observed", [False, True])
def test_affine_ssd_chains_round_trip(monkeypatch, tmp_path, observed):
    """SSD-Lite with its heads written in place, at two input sizes (the head offsets follow the input)."""
    from dfq_b200 import int8
    from test_int8_affine_observe_host import _state
    import affine_observed_state
    fakelib_int8_affine_pool_heads.install(monkeypatch)
    model = fixed_range_model(SSDLiteLike(21, is_test=True))
    x = torch.randn(1, 3, 64, 64).clamp_(-2.5, 2.5)
    _affine_chain(monkeypatch, model, x, concat=True, fold_pads=True, heads=True)
    records = affine_observed_state.record_ops(model, x)
    for i, flags in enumerate(AFFINE_FLAGS):
        if observed:
            with _state(model, records):
                gm = int8.chain_affine(model, **flags)
        else:
            gm = int8.chain_affine(model, **flags)
        m, _ = _round_trip(gm, x, tmp_path, "m%d.pt" % i)
        if flags.get("heads"):
            assert len(m.fused_heads) == 2 and len({o for o, _, _ in m.fused_observers}) == (33 if observed else 0)
            x2 = torch.randn(2, 3, 48, 80).clamp_(-2.5, 2.5)
            with torch.no_grad():
                assert _same(m(x2), gm(x2))


@pytest.mark.parametrize("observed", [False, True])
@pytest.mark.parametrize("net", ["pool_stem", "cat_pool", "cat_upsample"])
def test_affine_pools_and_upsamples_round_trip(monkeypatch, tmp_path, net, observed):
    from dfq_b200 import int8
    if net == "cat_upsample":
        x = torch.randn(2, 3, 8, 8)
        gm, _ = _affine_layout_chain(monkeypatch, CatNet(upsample="size"), x, observed=observed, concat=True)
        assert any(isinstance(m, int8.AffineInt8UpsampleBilinear) for m in gm.modules())
    else:
        x = torch.randn(2, 3, 12, 12)
        gm, _, _ = _affine_chain(monkeypatch, PoolNet(stem=True) if net == "pool_stem" else CatPoolNet(), x,
                                 observed=observed, concat=net == "cat_pool", pools=True)
        assert any(isinstance(m, int8.AffineInt8MaxPool2d) for m in gm.modules())
    _round_trip(gm, x, tmp_path)


def test_file_loads_as_plain_containers_and_stores_each_buffer_once(monkeypatch, tmp_path):
    """torch.load(weights_only=True) reads the file; a buffer several modules hold (a detection head's layer, held by its
    concatenation too) is one tensor in it and one tensor again after loading."""
    from dfq_b200 import int8, int8_io
    model = _identity_bns(SSDLiteLike(num_classes=5, is_test=True))
    x = torch.randn(1, 3, 64, 64, generator=torch.Generator().manual_seed(2))
    (gm, m), = _ncnn_round_trips(monkeypatch, tmp_path, model, x, NCNN_FLAGS[-1:])
    path = tmp_path / "m0.pt"
    st = torch.load(path, weights_only=True)
    assert st["format"] == int8_io.FORMAT and st["version"] == int8_io.VERSION
    storages = {t.untyped_storage().data_ptr() for p, mod in _called(gm).items() for t in mod._buffers.values()}
    assert len(st["tensors"]) == len(storages)
    heads = next(mod for mod in m.modules() if isinstance(mod, int8.Int8HeadConcat))
    for h in heads.heads:
        assert m.get_submodule(h.layer_name) is h
    codes = sum(t.numel() for t in st["tensors"] if t.dtype == torch.int8)
    assert codes == sum(mod.weight_codes.numel() for mod in _called(gm).values() if isinstance(mod, int8_io._LAYERS))
    assert os.path.getsize(path) < 1.25 * sum(t.numel() * t.element_size() for t in st["tensors"]) + 200_000


# ---- refusals ----------------------------------------------------------------------------------------------------------------
@fx.wrap
def _user_scale(x):
    return x * 2


class ReLU(nn.ReLU):
    """A model's own class under a torch.nn name."""


def _small(monkeypatch):
    from dfq_b200 import int8
    x = torch.randn(2, 3, 12, 12)
    gm, _, _ = _affine_chain(monkeypatch, PoolNet(stem=True), x, pools=True)
    return gm, x


def _snapshot(gm):
    return gm.code, _node_list(gm), {p: (_attrs(m), {k: t.clone() for k, t in m._buffers.items()})
                                     for p, m in _called(gm).items()}


def _unchanged(gm, snap, tmp_path):
    code, nodes, mods = _snapshot(gm)
    assert (code, nodes) == snap[:2]
    assert mods.keys() == snap[2].keys()
    for p, (a, bufs) in mods.items():
        assert a == snap[2][p][0] and all(torch.equal(t, snap[2][p][1][k]) for k, t in bufs.items()), p
    assert os.listdir(tmp_path) == []


def _refused(gm, tmp_path, match):
    from dfq_b200 import _lib, int8
    snap = _snapshot(gm) if isinstance(gm, fx.GraphModule) else None
    with pytest.raises(_lib.DfqError, match=match):
        int8.save(gm, tmp_path / "m.pt")
    if snap is not None:
        _unchanged(gm, snap, tmp_path)
    assert os.listdir(tmp_path) == []


def test_a_per_layer_model_is_refused(monkeypatch, tmp_path):
    from dfq_b200 import int8
    x = torch.randn(2, 3, 12, 12)
    model = PoolNet()
    _affine_chain(monkeypatch, model, x, pools=True)
    before = {k: t.clone() for k, t in model.state_dict().items()}
    _refused(model, tmp_path, r"chain_int8\(model\) or chain_affine\(model\) with no flags")
    assert all(torch.equal(t, before[k]) for k, t in model.state_dict().items())
    gm = int8.chain_affine(model)                               # the documented way
    _round_trip(gm, x, tmp_path)


def test_a_function_off_the_allowlist_is_refused(monkeypatch, tmp_path):
    gm, _ = _small(monkeypatch)
    out = next(n for n in gm.graph.nodes if n.op == "output")
    with gm.graph.inserting_before(out):
        y = gm.graph.call_function(_user_scale, (out.args[0],))
    out.args = (y,)
    gm.recompile()
    _refused(gm, tmp_path, r"node _user_scale calls .*_user_scale, which is not on the allowlist")


def test_a_tensor_method_off_the_allowlist_is_refused(monkeypatch, tmp_path):
    gm, _ = _small(monkeypatch)
    out = next(n for n in gm.graph.nodes if n.op == "output")
    with gm.graph.inserting_before(out):
        y = gm.graph.call_method("sigmoid", (out.args[0],))
    out.args = (y,)
    gm.recompile()
    _refused(gm, tmp_path, r"tensor method 'sigmoid'")


@pytest.mark.parametrize("mod, name", [(ReLU(), "test_int8_save_host.ReLU"), (nn.Conv2d(16, 16, 1), "Conv2d")])
def test_a_module_class_off_the_allowlist_is_refused(monkeypatch, tmp_path, mod, name):
    """A model's own class, even under a torch.nn name, and a torch.nn layer the chains never leave (an unconverted
    convolution)."""
    gm, _ = _small(monkeypatch)
    gm.add_submodule("extra", mod)
    out = next(n for n in gm.graph.nodes if n.op == "output")
    with gm.graph.inserting_before(out):
        y = gm.graph.call_module("extra", (out.args[0],))
    out.args = (y,)
    gm.recompile()
    _refused(gm, tmp_path, r"module extra is a .*%s, which a chained int8 model does not hold" % name)


def _saved(monkeypatch, tmp_path):
    from dfq_b200 import int8
    gm, x = _small(monkeypatch)
    int8.save(gm, tmp_path / "m.pt")
    return torch.load(tmp_path / "m.pt", weights_only=True)


def _load_refused(tmp_path, st, match):
    from dfq_b200 import _lib, int8
    torch.save(st, tmp_path / "bad.pt")
    with pytest.raises(_lib.DfqError, match=match):
        int8.load(tmp_path / "bad.pt")


@pytest.mark.parametrize("key, value, match", [
    ("format", "something.else", "not a chained int8 model file"), ("version", 2, "format version 2"),
    ("version", "1", "format version '1'")])
def test_a_tampered_tag_or_version_is_refused(monkeypatch, tmp_path, key, value, match):
    st = _saved(monkeypatch, tmp_path)
    st[key] = value
    _load_refused(tmp_path, st, match)


@pytest.mark.parametrize("where", ["records", "nodes", "requantized_edges", "module_attr", "node_args"])
def test_a_missing_key_is_refused(monkeypatch, tmp_path, where):
    st = _saved(monkeypatch, tmp_path)
    if where in ("records", "nodes"):
        del st[where]
    elif where == "requantized_edges":
        del st["records"]["requantized_edges"]
    elif where == "module_attr":
        del next(r for r in st["modules"] if r["type"] == "AffineInt8Conv2d")["attrs"]["constants"]
    else:
        del st["nodes"][1]["args"]
    _load_refused(tmp_path, st, "missing|has no")


@pytest.mark.parametrize("edit, match", [
    (lambda st: st["modules"][0].update(type="Conv2d"), "module type 'Conv2d' is not on the allowlist"),
    (lambda st: next(n for n in st["nodes"] if n["op"] == "call_function").update(target="os.system"),
     "calls 'os.system', which is not on the allowlist"),
    (lambda st: next(n for n in st["nodes"] if n["op"] == "call_method" or n["op"] == "call_function").update(
        op="call_method", target="__reduce__"), "tensor method '__reduce__'"),
    (lambda st: st["nodes"][1].update(op="get_attr"), "is a 'get_attr' node"),
    (lambda st: st["nodes"][-1].update(args={"tuple": [{"node": "nowhere"}]}), "'nowhere', which no earlier node")])
def test_load_checks_the_allowlist_again(monkeypatch, tmp_path, edit, match):
    st = _saved(monkeypatch, tmp_path)
    edit(st)
    _load_refused(tmp_path, st, match)


def test_a_pickled_object_is_refused(monkeypatch, tmp_path):
    """A file holding anything but plain containers and tensors does not load: no code of it runs."""
    from dfq_b200 import _lib, int8
    gm, _ = _small(monkeypatch)
    torch.save(gm, tmp_path / "gm.pt")
    with pytest.raises(_lib.DfqError, match="does not load as plain containers"):
        int8.load(tmp_path / "gm.pt")


def test_load_without_a_cuda_device_raises_dfq_error(monkeypatch, tmp_path):
    from dfq_b200 import _lib, int8
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(_lib.DfqError, match="requires a CUDA device"):
        int8.load(tmp_path / "m.pt")


# ---- names the generated forward spells as code, and the layers' geometry ---------------------------------------------------
def _node(st, op):
    return next(n for n in st["nodes"] if n["op"] == op)


def _inject_path(st, payload):
    n = _node(st, "call_module")
    st["paths"][payload] = st["paths"][n["target"]]
    n["target"] = payload


def _inject_plain(st, attrs=None, buffers=None):
    st["modules"].append({"type": "ReLU", "attrs": dict(training=False, inplace=False, **(attrs or {})),
                          "buffers": buffers or {}, "params": {}})
    st["paths"]["extra"] = len(st["modules"]) - 1


def _layer(st):
    return next(r for r in st["modules"] if r["type"] == "AffineInt8Conv2d")


def _shrink_codes(st):
    i = _layer(st)["buffers"]["weight_codes"]
    st["tensors"][i] = st["tensors"][i][:-16].clone()


@pytest.mark.parametrize("edit, match", [
    (lambda st, f: _node(st, "placeholder").update(target='x=open(%r,"w").write("1")' % f), "is not an identifier"),
    (lambda st, f: _node(st, "placeholder").update(args={"tuple": ["default"]}), "takes no default value"),
    (lambda st, f: _node(st, "call_module").update(kwargs={'inplace=bool(open(%r,"w").write("1")) and False, _u' % f: 1}),
     "keyword .* is not an identifier"),
    (lambda st, f: _inject_path(st, 'a")or open(%r,"w").write("1")or getattr(self,"b' % f),
     "is not a dotted path of identifiers and indices"),
    (lambda st, f: _node(st, "output").update(args={"tuple": [{"dict": [['x": open(%r,"w").write("1"), "' % f,
                                                                          None]]}]}), "dict key .* is not an identifier"),
    (lambda st, f: st.update(class_name='M(): pass\nopen(%r,"w")' % f), "class name .* is not an identifier"),
    (lambda st, f: _node(st, "output").update(name="output; import os"), "node name .* is not an identifier"),
], ids=["placeholder", "default", "keyword", "path", "dict_key", "class_name", "node_name"])
def test_names_that_would_be_code_are_refused(monkeypatch, tmp_path, edit, match):
    """The generated forward spells node names, parameters, module paths, keywords and dict keys as source: anything but an
    identifier (or an index in a path) is refused before fx generates code, so a crafted file runs nothing."""
    st = _saved(monkeypatch, tmp_path)
    pwned = str(tmp_path / "PWNED")
    edit(st, pwned)
    _load_refused(tmp_path, st, match)
    assert not os.path.exists(pwned)


@pytest.mark.parametrize("edit, match", [
    (_shrink_codes, "buffer weight_codes is torch.int8"),
    (lambda st: st["tensors"].__setitem__(_layer(st)["buffers"]["bias"],
                                          st["tensors"][_layer(st)["buffers"]["bias"]].double()), "buffer bias is torch.float64"),
    (lambda st: _layer(st)["attrs"].update(cpad=_layer(st)["attrs"]["cpad"] + 16), "do not fit together"),
    (lambda st: _layer(st)["attrs"].update(kernel_size=(3, 0)), "geometry"),
    (lambda st: _layer(st)["buffers"].pop("tap_table"), "buffers"),
    (lambda st: _layer(st)["attrs"].update(out_slice=(8, 16)), "channel slice"),
    (lambda st: _inject_plain(st, attrs={"_forward_hooks": 0}), "'_forward_hooks' is not a stored attribute"),
    (lambda st: _inject_plain(st, attrs={"forward": 1}), "'forward' is not a stored attribute"),
    (lambda st: _inject_plain(st, buffers={"train": 0}), "'train' is not a stored attribute"),
], ids=["codes_short", "bias_dtype", "cpad", "kernel", "no_tap_table", "slice", "private_attr", "method_attr", "buffer"])
def test_state_that_does_not_fit_its_module_is_refused(monkeypatch, tmp_path, edit, match):
    """A layer's buffers must be what its stored geometry makes (the kernels would read past them otherwise), and a torch.nn
    leaf takes only the public attributes save() writes."""
    st = _saved(monkeypatch, tmp_path)
    edit(st)
    _load_refused(tmp_path, st, match)


@pytest.mark.parametrize("device", ["cpu", "cuda:1"])
def test_a_device_other_than_the_current_one_is_refused(monkeypatch, tmp_path, device):
    from dfq_b200 import _lib, engine, int8
    _saved(monkeypatch, tmp_path)
    monkeypatch.setattr(engine, "_default_device", lambda: torch.device("cuda", 0))
    with pytest.raises(_lib.DfqError, match="is not the current CUDA device"):
        int8.load(tmp_path / "m.pt", device=device)
