"""dfq_b200.int8.save / load on the H100: every network the chain tests build, under both schemes, loads back to a model
whose outputs are torch.equal to the saved one's, with equal records - SSD-Lite at two input sizes, one model loaded in a
fresh process that cannot import torchvision, the test helpers or the reference's code - and the file sizes."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import affine_distilled_state as D
import affine_observed_state
from test_int8_save_host import assert_round_trip

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def no_tf32():
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def _equal(a, b):
    if isinstance(a, (tuple, list)):
        return len(a) == len(b) and all(_equal(u, v) for u, v in zip(a, b))
    return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


def _check(gm, xs, tmp_path, name):
    """Save gm, load it, and check the loaded model against it on every input in xs; returns (loaded, file size)."""
    from dfq_b200 import int8
    path = tmp_path / (name + ".pt")
    int8.save(gm, path)
    m = int8.load(path)
    assert_round_trip(gm, m)
    with torch.no_grad():
        for x in xs:
            assert _equal(m(x), gm(x)), (name, tuple(x.shape))
    size = os.path.getsize(path)
    from dfq_b200 import int8_io
    print("%s: %d bytes, records %s" % (name, size, {k: len(getattr(m, k)) for k in int8_io.RECORDS if hasattr(m, k)}))
    return m, size


# ---- the ncnn scheme ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("net", ["mobilenet_v2", "resnet18"])
def test_ncnn_classifiers(tmp_path, net):
    """Per layer (no flags) and with residual=True; MobileNetV2's file against its fp32 state dict."""
    from dfq_b200 import int8
    import test_gpu_int8_chain as GC
    model, x = GC._folded_and_converted(net)
    codes = sum(m.weight_codes.numel() for m in model.modules() if isinstance(m, int8._Int8Layer))
    _, plain = _check(int8.chain_int8(model), [x], tmp_path, net + "_plain")
    _, size = _check(int8.chain_int8(model, residual=True), [x], tmp_path, net)
    import torchvision
    weights = sum(p.numel() for n, p in getattr(torchvision.models, net)(num_classes=1000).state_dict().items()
                  if n.endswith("weight") and p.dim() > 1)
    print("%s: %d weights, fp32 state dict of the weights %d bytes, chained int8 file %d bytes (%.2f bytes per weight), "
          "packed codes %d bytes" % (net, weights, 4 * weights, size, size / weights, codes))
    if net == "mobilenet_v2":
        assert max(size, plain) < 1.6 * weights


@pytest.mark.parametrize("net", ["squeezenet1_1", "googlenet"])
def test_ncnn_pool_cat_networks(tmp_path, net):
    from dfq_b200 import int8
    import test_gpu_int8_pool_cat as GP
    model, x = GP._model(net)
    m, _ = _check(int8.chain_int8(model, residual=True, pool_cat=True), [x], tmp_path, net)
    assert m.fused_cats and m.fused_pools


def test_ncnn_deeplab_with_fixed_padding(tmp_path):
    from dfq_b200 import int8
    import test_gpu_int8_layout as GL
    model, x = GL._net("deeplab", 2, 129)
    m, _ = _check(int8.chain_int8(model, residual=True, pool_cat=True, upsample=True, layout=True), [x], tmp_path, "deeplab")
    assert len(m.folded_pads) == 17 and len(m.fused_cats) == 2 and m.fused_upsamples


def test_ncnn_ssd_lite_at_two_sizes(tmp_path):
    from dfq_b200 import int8
    import test_gpu_int8_layout as GL
    model, x = GL._net("ssd", 2, 300, is_test=True)
    x2 = torch.randn(3, 3, 240, 320, device="cuda")
    m, _ = _check(int8.chain_int8(model, residual=True, pool_cat=True, upsample=True, layout=True), [x, x2], tmp_path,
                  "ssd")
    assert [(c, len(p), k) for c, p, k in m.fused_heads] == [("cat", 6, 21), ("cat_1", 6, 4)]


# ---- the affine scheme, in the reference's evaluation state -------------------------------------------------------------------
AFFINE = {"mobilenet_v2": (224, dict(residual=True)), "resnet18": (224, dict(residual=True, pools=True)),
          "googlenet": (224, dict(residual=True, concat=True, pools=True)),
          "deeplab": (129, dict(residual=True, concat=True, fold_pads=True)),
          "ssd": (300, dict(residual=True, concat=True, fold_pads=True, heads=True))}


@pytest.mark.parametrize("net", list(AFFINE))
def test_affine_evaluation_state(no_tf32, tmp_path, net):
    """Saved while replace_op() is active, loaded and run with it active (as the mains evaluate) and, for SSD-Lite, in a
    fresh process where it never ran."""
    from dfq_b200 import int8
    size, flags = AFFINE[net]
    g = torch.Generator(device="cuda").manual_seed(2)
    with affine_observed_state.evaluation_state(net, size=size, batch=4) as (model, qgraph, qtarg):
        int8.convert_affine(model, qgraph, qtarg)
        gm = int8.chain_affine(model, **flags)
        x = torch.randn(2, 3, size, size, device="cuda", generator=g).clamp_(-2.5, 2.5)
        xs = [x] + ([torch.randn(3, 3, 240, 320, device="cuda", generator=g).clamp_(-2.5, 2.5)] if net == "ssd" else [])
        m, _ = _check(gm, xs, tmp_path, "affine_" + net)
        assert m.fused_observers == gm.fused_observers and m.fused_observers
        if net == "ssd":
            _in_a_fresh_process(gm, xs, tmp_path)


def test_affine_distilled_range(no_tf32, tmp_path):
    from dfq_b200 import int8
    with D.distilled_state("resnet18", "distill_range", size=224, batch=4) as (model, qgraph, qtarg):
        int8.convert_affine(model, qgraph, qtarg)
        gm = int8.chain_affine(model, residual=True, pools=True)
        x = D.inputs("resnet18", 2, 224, torch.Generator(device="cuda").manual_seed(2))
        _check(gm, [x], tmp_path, "affine_distilled_resnet18")


_CHILD = r"""
import importlib.abc, sys
BLOCKED = {"torchvision", "dropin", "oracle", "tests", "utils", "modeling", "ssd_lite_like", "deeplab_mobilenet_padded",
           "affine_observed_state", "affine_distilled_state", "conftest", "dfq", "improve_dfq", "ZeroQ"}

class Blocker(importlib.abc.MetaPathFinder):
    def find_spec(self, name, path=None, target=None):
        if name.split(".")[0] in BLOCKED:
            raise ImportError("blocked: " + name)
        return None

sys.meta_path.insert(0, Blocker())
sys.path = [p for p in sys.path if not p.rstrip("/").endswith("tests")]
import numpy as np, torch
from dfq_b200 import int8, int8_io
from dfq_b200.utils import layer_transform as LT
assert not LT.raw_torch_op, "replace_op() ran"
m = int8.load(sys.argv[1])
with torch.no_grad():
    for i, f in enumerate(sys.argv[2:]):
        y = m(torch.from_numpy(np.load(f)).cuda())
        for j, t in enumerate(y if isinstance(y, tuple) else (y,)):
            np.save(f[:-4] + "_got%d.npy" % j, t.cpu().numpy())
print("records", sorted(k for k in int8_io.RECORDS if hasattr(m, k)), "torchvision" in sys.modules)
"""


def _in_a_fresh_process(gm, xs, tmp_path):
    """The saved model loaded by a `python -c` that blocks torchvision, the tests' and the reference's modules: its outputs
    equal the parent's, saved as .npy."""
    from dfq_b200 import int8
    path = tmp_path / "child.pt"
    int8.save(gm, path)
    files = []
    with torch.no_grad():
        for i, x in enumerate(xs):
            f = str(tmp_path / ("x%d.npy" % i))
            np.save(f, x.cpu().numpy())
            for j, t in enumerate(y if isinstance(y := gm(x), tuple) else (y,)):
                np.save(f[:-4] + "_want%d.npy" % j, t.cpu().numpy())
            files.append(f)
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-c", _CHILD, str(path)] + files, cwd=ROOT, env=env, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    print(r.stdout.strip())
    for f in files:
        j = 0
        while os.path.exists(f[:-4] + "_want%d.npy" % j):
            want, got = np.load(f[:-4] + "_want%d.npy" % j), np.load(f[:-4] + "_got%d.npy" % j)
            assert want.shape == got.shape and np.array_equal(want.view(np.int32), got.view(np.int32)), (f, j)
            j += 1
        assert j > 0
