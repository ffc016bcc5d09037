"""The launch context of the package (DESIGN.md, "Launch context") without a GPU: every library call that takes a stream is
made inside `_lib.launch(...)` and passes the stream it yields - checked on the source, so an entry point added later
cannot launch on the current device's stream while its tensors are on another - and launch()'s refusals by name."""
import ast
import os
import re

import pytest
import torch

from dfq_b200 import _lib

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
PKG = os.path.join(ROOT, "dfq_b200")


def _stream_entries():
    """Names of the C ABI functions whose last parameter is the stream (include/dfq_b200.h)."""
    with open(os.path.join(ROOT, "include", "dfq_b200.h")) as f:
        header = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    decls = re.findall(r"\bint\s+(dfq_\w+)\s*\(([^;]*?)\)\s*;", header, flags=re.S)
    return {name for name, params in decls if re.search(r"\bstream\s*$", params.strip())}


STREAM_ENTRIES = _stream_entries()


def _sources():
    for d, _, files in os.walk(PKG):
        for f in sorted(files):
            if f.endswith(".py"):
                path = os.path.join(d, f)
                with open(path) as fh:
                    yield os.path.relpath(path, ROOT), ast.parse(fh.read(), path)


def _is_launch(expr):
    """`_lib.launch(...)`, or `launch(...)` inside _lib.py."""
    if not isinstance(expr, ast.Call):
        return False
    f = expr.func
    return (isinstance(f, ast.Attribute) and f.attr == "launch" and isinstance(f.value, ast.Name) and f.value.id == "_lib") \
        or (isinstance(f, ast.Name) and f.id == "launch")


def _entry_of(node, aliases):
    """The library function a call's callee names: `<x>.dfq_name`, or a local name bound to one."""
    f = node.func
    if isinstance(f, ast.Attribute) and f.attr in STREAM_ENTRIES:
        return f.attr
    if isinstance(f, ast.Name):
        return aliases.get(f.id)
    return None


def _aliases(fn):
    """Local names bound to a stream-taking library function in `fn`: `n = lib.dfq_x` or `n = getattr(lib, "dfq_x", ..)`."""
    out = {}
    for node in ast.walk(fn):
        if isinstance(node, ast.Assign) and len(node.targets) == 1 and isinstance(node.targets[0], ast.Name):
            v = node.value
            if isinstance(v, ast.Attribute) and v.attr in STREAM_ENTRIES:
                out[node.targets[0].id] = v.attr
            elif isinstance(v, ast.Call) and isinstance(v.func, ast.Name) and v.func.id == "getattr" and len(v.args) >= 2 \
                    and isinstance(v.args[1], ast.Constant) and v.args[1].value in STREAM_ENTRIES:
                out[node.targets[0].id] = v.args[1].value
    return out


def _launch_calls(tree):
    """(call node, library function, stream names bound by the launch contexts around the call, in its own function)."""
    found = []

    def visit(node, bound, aliases):
        if isinstance(node, (ast.FunctionDef, ast.AsyncFunctionDef, ast.Lambda)):
            bound, aliases = (), _aliases(node)
        if isinstance(node, (ast.With, ast.AsyncWith)):
            names = tuple(it.optional_vars.id for it in node.items
                          if _is_launch(it.context_expr) and isinstance(it.optional_vars, ast.Name))
            for it in node.items:
                visit(it, bound, aliases)
            for stmt in node.body:
                visit(stmt, bound + names, aliases)
            return
        if isinstance(node, ast.Call):
            entry = _entry_of(node, aliases)
            if entry is not None:
                found.append((node, entry, bound))
        for child in ast.iter_child_nodes(node):
            visit(child, bound, aliases)

    visit(tree, (), {})
    return found


def test_the_header_scan_finds_the_stream_entries():
    # every kernel entry takes the stream last; the two host-only entries do not
    assert {"dfq_cls_count", "dfq_seg_argmax", "dfq_pre_resample", "dfq_jpeg_decode", "dfq_png_decode", "dfq_ssd_nms",
            "dfq_map_curve", "dfq_i8_conv", "dfq_i8_plane_mean", "dfq_cle_run", "dfq_cle_run_bc"} <= STREAM_ENTRIES
    assert not {"dfq_host_copy_segments", "dfq_cle_takes_stack", "dfq_abi_version"} & STREAM_ENTRIES
    assert STREAM_ENTRIES <= set(_lib.SIGNATURES)


def test_every_library_launch_is_inside_the_launch_context():
    bad, seen = [], set()
    for path, tree in _sources():
        for node, entry, bound in _launch_calls(tree):
            seen.add(entry)
            last = node.args[-1] if node.args else None
            if not bound:
                bad.append("%s:%d %s outside `with _lib.launch(...) as st`" % (path, node.lineno, entry))
            elif not (isinstance(last, ast.Name) and last.id in bound and not node.keywords):
                bad.append("%s:%d %s does not pass the launch context's stream last" % (path, node.lineno, entry))
    assert not bad, "\n".join(bad)
    # the walk sees the package's launches: every evaluation entry point, the int8 layers and the calibration engine
    assert {"dfq_cls_count", "dfq_seg_argmax", "dfq_pre_resample", "dfq_jpeg_decode", "dfq_png_decode", "dfq_ssd_decode",
            "dfq_ssd_nms", "dfq_ssd_compact", "dfq_ssd_soft_nms", "dfq_ssd_soft_compact", "dfq_map_match", "dfq_map_curve",
            "dfq_i8_plane_mean", "dfq_i8_conv", "dfq_i8_affine_conv", "dfq_cle_run", "dfq_cle_run_bc", "dfq_bias_correct",
            "dfq_quantize_tensors"} <= seen


def test_only_launch_reads_the_current_stream():
    bad = []
    for path, tree in _sources():
        for node in ast.walk(tree):
            name = node.attr if isinstance(node, ast.Attribute) else node.id if isinstance(node, ast.Name) else None
            if name == "stream_ptr" and not (path.endswith("_lib.py") and isinstance(node, ast.Name)):
                bad.append("%s:%d" % (path, node.lineno))
            if name == "current_stream" and isinstance(node, ast.Attribute):
                call = next((c for c in ast.walk(tree) if isinstance(c, ast.Call) and c.func is node), None)
                if call is not None and not call.args and not path.endswith("_lib.py"):
                    bad.append("%s:%d current_stream() of the current device" % (path, node.lineno))
    assert not bad, "\n".join(bad)


def test_the_walk_catches_a_launch_outside_the_context():
    src = '''
def good(x):
    with _lib.launch(x) as st:
        _lib.check(lib.dfq_cls_count(a, b, c, d, 1, 2, st), "w")

def outside(x):
    _lib.check(lib.dfq_cls_count(a, b, c, d, 1, 2, _lib.stream_ptr()), "w")

def wrong_stream(x):
    with _lib.launch(x) as st:
        _lib.check(lib.dfq_seg_argmax(a, b, c, d, e, other), "w")

def aliased(self, x):
    run = getattr(self.lib, "dfq_cle_run_bc", None)
    run(x)

def nested(x):
    with _lib.launch(x) as st:
        def later():
            lib.dfq_minmax(a, 1, b, st)
'''
    calls = _launch_calls(ast.parse(src))
    assert [(e, bool(b)) for _, e, b in calls] == [("dfq_cls_count", True), ("dfq_cls_count", False),
                                                   ("dfq_seg_argmax", True), ("dfq_cle_run_bc", False),
                                                   ("dfq_minmax", False)]
    assert calls[2][0].args[-1].id not in calls[2][2]


# ---- launch()'s refusals and its host path ---------------------------------------------------------------------------

@pytest.mark.parametrize("on, named", [
    ((torch.device("cuda", 0), torch.device("cuda", 1)), "cuda:0 and cuda:1"),
    ((torch.device("cuda", 1), None, "cuda:0"), "cuda:1 and cuda:0"),
    ((torch.zeros(2), torch.device("cuda", 3)), "cpu and cuda:3"),
    ((torch.device("cuda", 2), torch.zeros(1), "cuda:2"), "cuda:2 and cpu"),
    ((), "none"),
    ((None, None), "none"),
])
def test_launch_refuses_tensors_on_two_devices_by_name(on, named):
    # refused before any device is entered: on this host torch.cuda.device() could not run
    with pytest.raises(_lib.DfqError, match="a library call takes its tensors on one device, got %s$" % named):
        with _lib.launch(*on):
            raise AssertionError("the body must not run")


def test_launch_on_host_tensors_enters_no_device(monkeypatch):
    sentinel = object()
    monkeypatch.setattr(_lib, "stream_ptr", lambda: sentinel)
    monkeypatch.setattr(torch.cuda, "device", lambda *a: (_ for _ in ()).throw(AssertionError("entered a device")))
    with _lib.launch(torch.zeros(3), None, torch.zeros(1, dtype=torch.int64), "cpu") as st:
        assert st is sentinel


def test_launch_enters_the_tensors_device_and_restores_it(monkeypatch):
    """The device entered and the stream read inside it, with torch.cuda's device switch and stream query stood in."""
    current, log = [0], []

    class Dev:
        def __init__(self, i):
            self.i = i

        def __enter__(self):
            log.append(("enter", self.i))
            self.prev, current[0] = current[0], self.i

        def __exit__(self, *exc):
            current[0] = self.prev
            log.append(("exit", self.i))
            return False

    monkeypatch.setattr(torch.cuda, "device", Dev)
    monkeypatch.setattr(torch.cuda, "current_device", lambda: current[0])
    monkeypatch.setattr(_lib, "stream_ptr", lambda: ("stream of", current[0]))
    with _lib.launch(torch.device("cuda", 1), "cuda:1", None) as st:
        assert st == ("stream of", 1) and current[0] == 1
    assert current == [0] and log == [("enter", 1), ("exit", 1)]
    with _lib.launch("cuda") as st:                 # no index: the current device
        assert st == ("stream of", 0)
    with pytest.raises(ValueError, match="boom"):   # an error inside the call still restores the device
        with _lib.launch(torch.device("cuda", 2)):
            assert current[0] == 2
            raise ValueError("boom")
    assert current == [0]


def test_entry_points_refuse_mixed_devices_through_the_host_twins(monkeypatch):
    """Mixed devices reach launch() through classify.predict's and segment.predict's host twins: the fakes stand tensors
    on the CPU in for GPU tensors, and one tensor reporting another GPU is refused by launch() before the library runs."""
    import fakelib_classify
    fake = fakelib_classify.install(monkeypatch)
    from dfq_b200 import classify
    x = torch.randn(4, 5)
    assert torch.equal(classify.predict(x), torch.max(x, 1)[1])
    real_get_device = torch.Tensor.get_device
    monkeypatch.setattr(torch.Tensor, "get_device", lambda self: 1 if self.dtype == torch.int64 else real_get_device(self))
    n = fake.calls.count("dfq_cls_count")
    with pytest.raises(_lib.DfqError, match="one device, got cpu and cuda:1"):
        classify.predict(x)
    assert fake.calls.count("dfq_cls_count") == n


# ---- the GPU suite's programs run in fresh interpreters ------------------------------------------------------------------
def test_the_subprocess_bodies_resolve_every_name():
    """tests/test_gpu_context.py runs some checks in a fresh interpreter (a second GPU needs cuda:0 to be used first): the
    program imports the module and calls one of its functions.  Every global name those functions read must exist in the
    module, so a body cannot fail with a NameError on a machine where it first runs."""
    import builtins
    import dis
    import sys
    import types
    import test_gpu_context as T
    for name in T.SUBPROCESS_BODIES:
        missing, stack = set(), [getattr(T, name).__code__]
        while stack:
            co = stack.pop()
            stack.extend(c for c in co.co_consts if isinstance(c, types.CodeType))
            for ins in dis.get_instructions(co):
                if ins.opname in ("LOAD_GLOBAL", "LOAD_NAME") and ins.argval not in vars(T) \
                        and not hasattr(builtins, ins.argval):
                    missing.add(ins.argval)
        assert not missing, (name, missing)
        # the program itself: everything up to its last statement runs here, and that statement calls the body
        tree = ast.parse(T._subprocess_code(name, "x"))
        call = tree.body[-1].value
        assert isinstance(call, ast.Call) and ast.unparse(call.func) == "test_gpu_context." + name
        path, ns = list(sys.path), {}
        try:
            exec(compile(ast.Module(tree.body[:-1], []), "<program>", "exec"), ns)
        finally:
            sys.path[:] = path
        assert getattr(ns["test_gpu_context"], name) is getattr(T, name)
