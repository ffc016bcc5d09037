"""Import helper for the UNMODIFIED reference tree (jakc4103/DFQ), wherever a checkout exists.

Test/fixture infrastructure only.  Nothing in the product package (``dfq_b200``), ``bench.py``,
``__graft_entry__.smoke()`` or the ``-m gpu`` tests imports this file: none of them needs the reference
tree.  It is used by

* ``tools/make_golden.py``  - generates ``tests/golden/*`` by running the reference here, and
* ``oracle/ref_data.py`` (``REF_ROOT`` only), which stages the reference's data files for the tests.

The shims are the ones SURVEY.md section 8(b) lists for torch 2.11 / python 3.12: stub the optional
visualisation deps *after* ``import torch``, alias ``collections.Mapping``.
"""
import collections
import collections.abc
import importlib
import os
import sys
import types

REF_ROOT = os.environ.get("DFQ_REFERENCE_ROOT", "/root/reference")

_STUBS = [
    "pydot", "graphviz", "tensorboardX", "matplotlib", "matplotlib.pyplot",
    "pytorchcv", "pytorchcv.models", "pytorchcv.models.common",
    "pytorchcv.models.shufflenetv2", "pytorchcv.model_provider",
]


def available() -> bool:
    return os.path.isfile(os.path.join(REF_ROOT, "dfq.py"))


def install():
    """Put the reference on sys.path (read-only tree: no bytecode) and return its hot-path modules."""
    if not available():
        raise RuntimeError("reference tree not found at %s" % REF_ROOT)
    import torch  # noqa: F401  (must precede the stubs: torch.fx probes pydot)
    for name in _STUBS:
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["graphviz"].Digraph = object
    sys.modules["tensorboardX"].SummaryWriter = object
    sys.modules["pytorchcv.models.common"].ConvBlock = object
    for n in ("ShuffleUnit", "ShuffleInitBlock"):
        setattr(sys.modules["pytorchcv.models.shufflenetv2"], n, object)
    collections.Mapping = collections.abc.Mapping
    sys.dont_write_bytecode = True
    # our own drop-in dirs must NOT shadow the reference here
    sys.path[:] = [p for p in sys.path if not p.rstrip("/").endswith("dropin")]
    for mod in ("dfq", "utils", "utils.quantize", "utils.layer_transform", "utils.relation", "improve_dfq"):
        if mod in sys.modules and not getattr(sys.modules[mod], "__file__", "").startswith(REF_ROOT):
            del sys.modules[mod]
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)
    ref = types.SimpleNamespace()
    ref.dfq = importlib.import_module("dfq")
    ref.quantize = importlib.import_module("utils.quantize")
    ref.layer_transform = importlib.import_module("utils.layer_transform")
    ref.relation = importlib.import_module("utils.relation")
    return ref


def tracer():
    from PyTransformer.transformers.torchTransformer import TorchTransformer
    return TorchTransformer
