#!/usr/bin/env python
"""Run the reference's UNMODIFIED main_cls.py / main_seg.py / main_ssd.py end to end on a machine without datasets
(and, in the build container, without a GPU), capture what they calibrated and what the calibrated model computes.

    python tests/main_harness.py --impl dropin    --out /tmp/a.npz cls --quantize --relu --equalize --correction
    python tests/main_harness.py --impl reference --out tests/golden/main_cls.npz cls --quantize --relu --equalize --correction

--impl dropin      tools/run_main.py exactly as a user would start it: `dropin/` shadows the reference's dfq / utils.* /
                   improve_dfq modules with dfq_b200.  With a CUDA device the real libdfq_sm90.so runs; without one the
                   oracle-backed executor of tests/fakelib.py stands in for the library (test infrastructure).
--impl reference   the same script on the reference's own modules (fixture generation, build container only).

Test infrastructure (it imports tests/fakelib.py and therefore oracle/): only tests/test_run_main.py and the fixture
generation use it.  What it adds on top of tools/run_main.py, none of which touches the calibration path:

* synthetic datasets in place of the hard-coded ImageNet / VOC paths (main_cls.py:46, main_seg.py:92, main_ssd.py:154):
  seeded clamp(N(0,1)) images, so the scripts' own inference loop (with `replace_op()` active, i.e. the patched
  Tensor.__add__/torch.cat/torch.mean/F.interpolate observers) runs over a few images;
* `torch.load(..., map_location='cpu', weights_only=False)` when no GPU is visible (the DeepLab checkpoint holds CUDA
  storages, main_seg.py:107), `.cuda()` as a no-op there, DataLoader without worker processes;
* global forward hooks that remember the outermost module of the inference phase and its outputs.
"""
import argparse
import hashlib
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (HERE, ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

N_IMAGES = {"cls": 8, "seg": 2, "ssd": 2}


class _State:
    inference = False
    depth = 0
    top = None
    outputs = []
    observer_calls = 0      # QuantMeasure.forward calls during the inference phase (layer inputs + patched functional ops)
    op_observer_calls = 0   # ... of which through CustomTensorOP (the observers replace_op() attaches to add/cat/mean/...)


def _flatten(out, acc):
    if isinstance(out, torch.Tensor):
        acc.append(out.detach().float().cpu().numpy().copy())
    elif isinstance(out, (list, tuple)):
        for o in out:
            _flatten(o, acc)
    elif isinstance(out, dict):
        for k in sorted(out):
            _flatten(out[k], acc)


def _install_capture():
    import torch.nn.modules.module as M

    def pre(mod, args):
        _State.depth += 1
        if _State.inference:
            name = type(mod).__name__
            if name == "QuantMeasure":
                _State.observer_calls += 1
            elif name == "CustomTensorOP":
                _State.op_observer_calls += 1

    def post(mod, args, output):
        _State.depth -= 1
        if _State.depth == 0 and _State.inference:
            _State.top = mod
            acc = []
            _flatten(output, acc)
            _State.outputs.append(acc)
    M.register_module_forward_pre_hook(pre)
    M.register_module_forward_hook(post)


def _images(n, size, lo=-2.11790393, hi=2.64, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, 3, size, size, generator=g).clamp_(lo, hi)


def _install_synthetic_data(which):
    import torch.utils.data as tud
    _DL = tud.DataLoader

    class DataLoader(_DL):
        def __init__(self, dataset, *a, **kw):
            kw["num_workers"] = 0
            kw["pin_memory"] = False
            super().__init__(dataset, *a, **kw)
    tud.DataLoader = DataLoader
    n = N_IMAGES[which]
    if which == "cls":
        import torchvision.datasets as tvd

        class ImageFolder(tud.Dataset):
            def __init__(self, root, transform=None, **kw):
                _State.inference = True
                self.x = _images(n, 224)

            def __len__(self):
                return len(self.x)

            def __getitem__(self, i):
                return self.x[i], i % 1000
        tvd.ImageFolder = ImageFolder
    elif which == "seg":
        import dataset.segmentation.pascal as pascal

        class VOCSegmentation(tud.Dataset):
            NUM_CLASSES = 21

            def __init__(self, args, base_dir=None, split="val", label=None):
                _State.inference = True
                self.x = _images(n, 513)

            def __len__(self):
                return len(self.x)

            def __getitem__(self, i):
                return {"image": self.x[i], "label": torch.zeros(513, 513)}
        pascal.VOCSegmentation = VOCSegmentation
    else:
        import dataset.detection.voc_dataset as voc

        class VOCDataset:
            def __init__(self, root, transform=None, target_transform=None, is_test=False, keep_difficult=False, label_file=None):
                self.ids = ["%06d" % i for i in range(n)]
                self.class_names = ("BACKGROUND", "aeroplane")
                g = np.random.RandomState(0)
                self.imgs = [g.randint(0, 255, (300, 300, 3)).astype(np.uint8) for _ in range(n)]

            def __len__(self):
                return n

            def get_image(self, i):
                _State.inference = True
                return self.imgs[i]

            def get_annotation(self, i):
                return self.ids[i], (np.array([[10., 10., 100., 100.]], np.float32), np.array([1], np.int64), np.array([0], np.uint8))
        voc.VOCDataset = VOCDataset
        # torch >= 2 keeps the strides of the permuted HWC image through `.to(device)` (predictor.py:33-34) and the
        # reference's observer then fails on `.view(B, -1)` (quantize.py:106); torch 1.1 made that copy contiguous
        import modeling.detection.transforms.transforms as TT
        _call = TT.ToTensor.__call__
        TT.ToTensor.__call__ = lambda self, cvimage, boxes=None, labels=None: (
            _call(self, cvimage, boxes, labels)[0].contiguous(), boxes, labels)


def _cpu_only_shims():
    """No GPU (build container): checkpoints load on the CPU and `.cuda()` keeps tensors where they are."""
    _load = torch.load

    def load(f, *a, **kw):
        kw.setdefault("map_location", "cpu")
        kw.setdefault("weights_only", False)
        return _load(f, *a, **kw)
    torch.load = load
    torch.Tensor.cuda = lambda self, *a, **kw: self
    torch.nn.Module.cuda = lambda self, *a, **kw: self
    _to = torch.nn.Module.to

    def to(self, *a, **kw):
        a = tuple(x for x in a if not (isinstance(x, torch.device) and x.type == "cuda") and x != "cuda")
        return _to(self, *a, **kw) if (a or kw) else self
    torch.nn.Module.to = to


def _reference_eps_shim():
    """torch >= 2.x rejects the eps=0 the reference's merge_batchnorm leaves on the identity BN (layer_transform.py:272);
    1e-12 is bit-identical for var=1 (SURVEY.md 8(b) item 3).  Only needed when the REFERENCE's modules run."""
    import torch.nn.functional as F
    _bn = F.batch_norm

    def batch_norm(input, running_mean, running_var, weight=None, bias=None, training=False, momentum=0.1, eps=1e-5):
        return _bn(input, running_mean, running_var, weight, bias, training, momentum, eps if eps > 0 else 1e-12)
    F.batch_norm = batch_norm


def _gpu_shims():
    _load = torch.load

    def load(f, *a, **kw):
        kw.setdefault("weights_only", False)
        return _load(f, *a, **kw)
    torch.load = load


def snapshot(model):
    """Calibration state of a model as plain arrays, keyed by position among the modules of each kind."""
    out = {}
    convs = [m for m in model.modules() if isinstance(m, (torch.nn.Conv2d, torch.nn.Linear))]
    dig = []
    for i, m in enumerate(convs):
        w = np.ascontiguousarray(m.weight.detach().cpu().numpy())
        dig.append((hashlib.sha256(w.tobytes()).hexdigest(), float(np.abs(w).max()), float(w.astype(np.float64).sum())))
        if m.bias is not None:
            out["bias_%d" % i] = m.bias.detach().cpu().numpy().copy()
        q = getattr(m, "quant", None)
        if q is not None:
            out["qrange_%d" % i] = np.array([float(q.running_min), float(q.running_max)])
    out["w_sha"] = np.array([d[0] for d in dig])
    out["w_absmax"] = np.array([d[1] for d in dig])
    out["w_sum"] = np.array([d[2] for d in dig])
    out["w_class"] = np.array([type(m).__name__ for m in convs])
    j = 0
    for m in model.modules():
        if hasattr(m, "fake_bias"):
            out["fb_%d" % j] = m.fake_bias.detach().cpu().numpy().copy()
            out["fw_%d" % j] = m.fake_weight.detach().cpu().numpy().copy()
            j += 1
    # the functional-op observers: CustomTensorOP registered on the model by switch_layers (layer_transform.py:176)
    ops = getattr(model, "custom_tensor_op", None)
    if ops is not None:
        for k, q in enumerate(ops.children()):
            out["oprange_%d" % k] = np.array([float(q.running_min), float(q.running_max)])
    out["observer_calls"] = np.array([_State.observer_calls, _State.op_observer_calls])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--impl", choices=("dropin", "reference"), default="dropin")
    ap.add_argument("--out", required=True)
    ap.add_argument("which", choices=("cls", "seg", "ssd"))
    args, flags = ap.parse_known_args()
    import run_main
    have_gpu = torch.cuda.is_available()
    run_main.prepare_environment(use_dropin=(args.impl == "dropin"))
    fake = None
    if args.impl == "dropin" and not have_gpu:
        import fakelib
        fake = fakelib.install_plain(fakelib.torch_sqrt)
    (_gpu_shims if have_gpu else _cpu_only_shims)()
    if args.impl == "reference":
        _reference_eps_shim()
    _install_synthetic_data(args.which)
    _install_capture()
    script = os.path.join(run_main.REF, "main_%s.py" % args.which)
    sys.argv = [script] + flags
    import runpy
    err = None
    try:
        runpy.run_path(script, run_name="__main__")
    except BaseException as e:  # the scripts' evaluation code may choke on the synthetic annotations; calibration is done by then
        if _State.top is None:
            raise
        err = repr(e)
    assert _State.top is not None, "the script never ran its model over the synthetic data"
    out = snapshot(_State.top)
    n_out = max(len(o) for o in _State.outputs)
    for k in range(n_out):
        parts = [o[k].reshape(o[k].shape[0], -1) if o[k].ndim > 1 else o[k].reshape(1, -1) for o in _State.outputs if len(o) > k]
        width = max(set(p.shape[1] for p in parts), key=lambda w: sum(1 for p in parts if p.shape[1] == w))
        out["output_%d" % k] = np.concatenate([p for p in parts if p.shape[1] == width], axis=0)
    out["meta"] = np.array(repr(dict(impl=args.impl, which=args.which, flags=flags, gpu=have_gpu, tail_error=err,
                                     library_calls=sorted(set(fake.calls)) if fake is not None else None)))
    np.savez_compressed(args.out, **out)
    print("main_harness: %s %s -> %s (%d forward calls captured%s)" % (args.impl, args.which, args.out, len(_State.outputs),
                                                                       ", tail error " + err if err else ""))


if __name__ == "__main__":
    main()
