#!/usr/bin/env python
"""Run the reference's UNMODIFIED main_cls.py / main_seg.py / main_ssd.py on top of dfq_b200.

    python tools/run_main.py cls --quantize --relu --equalize --correction

`dropin/` is placed ahead of the reference tree on sys.path, so `from dfq import ...`, `from utils.quantize import ...`,
`from utils.layer_transform import ...`, `from utils.relation import ...` and `from improve_dfq import ...` bind to the
H100 implementation while models, datasets, the tracer (PyTransformer) and the evaluation code stay the reference's.
Needs the reference checkout (DFQ_REFERENCE_ROOT, default /root/reference), a CUDA device and - for the evaluation the
scripts run at the end - the datasets at the paths hard-coded in those scripts.

`tests/test_run_main.py` drives exactly this entry (through `tests/main_harness.py`, which adds synthetic datasets and the
oracle-backed executor on a GPU-less machine) and compares the calibrated model and its outputs with fixtures produced by
the same unmodified scripts running on the reference's own modules.
"""
import collections
import collections.abc
import os
import runpy
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.environ.get("DFQ_REFERENCE_ROOT", "/root/reference")

# optional third-party modules the reference imports for visualisation / model zoos / image IO; none is on the path
_OPTIONAL = ("pydot", "graphviz", "tensorboardX", "matplotlib", "matplotlib.pyplot", "pytorchcv", "pytorchcv.models",
             "pytorchcv.models.common", "pytorchcv.models.shufflenetv2", "pytorchcv.model_provider", "cv2")


def prepare_environment(use_dropin=True):
    """The shims SURVEY.md section 8(b) lists for torch 2.x / python 3.12, then sys.path: dropin/ (optional), repo, reference."""
    import torch  # noqa: F401  (before the stubs: torch.fx probes pydot)
    for name in _OPTIONAL:
        try:
            __import__(name)
        except Exception:
            sys.modules.setdefault(name, types.ModuleType(name))
    if not hasattr(sys.modules["graphviz"], "Digraph"):
        sys.modules["graphviz"].Digraph = object
    if not hasattr(sys.modules["tensorboardX"], "SummaryWriter"):
        sys.modules["tensorboardX"].SummaryWriter = object
    for mod, names in (("pytorchcv.models.common", ("ConvBlock",)), ("pytorchcv.models.shufflenetv2", ("ShuffleUnit", "ShuffleInitBlock"))):
        for n in names:
            if not hasattr(sys.modules[mod], n):
                setattr(sys.modules[mod], n, object)
    collections.Mapping = collections.abc.Mapping            # PyTransformer/transformers/utils.py:491
    import torch.optim.lr_scheduler as sched                 # ZeroQ/distill_data.py:160-163 passes verbose=
    if not getattr(sched.ReduceLROnPlateau, "_dfq_shim", False):
        _orig = sched.ReduceLROnPlateau

        class _Plateau(_orig):
            _dfq_shim = True

            def __init__(self, *a, verbose=None, **kw):
                super().__init__(*a, **kw)
        sched.ReduceLROnPlateau = _Plateau
    sys.dont_write_bytecode = True
    sys.path[:0] = ([os.path.join(ROOT, "dropin")] if use_dropin else []) + [ROOT, REF]
    os.chdir(REF)                                             # relative checkpoint paths in the scripts


def run(which, flags, use_dropin=True):
    script = os.path.join(REF, "main_%s.py" % which)
    if not os.path.isfile(script):
        sys.exit("reference script not found: %s" % script)
    prepare_environment(use_dropin)
    sys.argv = [script] + list(flags)
    return runpy.run_path(script, run_name="__main__")


def main():
    if len(sys.argv) < 2 or sys.argv[1] not in ("cls", "seg", "ssd"):
        sys.exit("usage: run_main.py cls|seg|ssd [flags of the reference script]")
    run(sys.argv[1], sys.argv[2:])


if __name__ == "__main__":
    main()
