"""The drop-in boundary, end to end: the reference's UNMODIFIED main_cls.py / main_seg.py / main_ssd.py run through
tools/run_main.py's environment (dropin/ ahead of the reference on sys.path) and must calibrate the bundled checkpoints to
the same model the same scripts produce on the reference's own modules.

How: tests/main_harness.py starts the script in a subprocess (synthetic datasets instead of the hard-coded ImageNet/VOC
paths; without a GPU the oracle-backed executor stands in for libdfq_sm90.so and is given the host's torch.sqrt, as the
fixture's reference run used it) and dumps (a) every Conv/Linear weight digest, bias, BN fake_weight/fake_bias, every
observer range, (b) how many observers fired during the script's own inference loop (layer inputs and - through
replace_op() - the patched Tensor.__add__/torch.cat/torch.mean/F.interpolate calls), (c) the model outputs.  The expected
values (tests/golden/main_<which>.npz) were produced by `main_harness.py --impl reference`, i.e. by the reference.

Needs the reference checkout (skipped where it is absent).
"""
import ast
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = os.path.join(HERE, "golden")
REF = os.environ.get("DFQ_REFERENCE_ROOT", "/root/reference")

FLAGS = {
    "cls": ["--quantize", "--relu", "--equalize", "--correction"],
    "seg": ["--quantize", "--relu", "--equalize", "--correction"],
    "ssd": ["--quantize", "--relu", "--equalize", "--correction"],
}


def _nw(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)


def _run(which, tmp_path, extra=()):
    out = str(tmp_path / ("%s.npz" % which))
    cmd = [sys.executable, os.path.join(HERE, "main_harness.py"), "--impl", "dropin", "--out", out, which] + FLAGS[which] + list(extra)
    env = dict(os.environ, PYTHONDONTWRITEBYTECODE="1")
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, env=env, cwd=ROOT)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    return np.load(out), res.stdout


@pytest.mark.skipif(not os.path.isfile(os.path.join(REF, "main_cls.py")), reason="reference checkout not present")
@pytest.mark.parametrize("which", ["cls", "seg", "ssd"])
def test_unmodified_main_script_calibrates_like_the_reference(which, tmp_path):
    gold_path = os.path.join(GOLD, "main_%s.npz" % which)
    if not os.path.isfile(gold_path):
        pytest.skip("no fixture for main_%s.py" % which)
    gold = np.load(gold_path)
    got, log = _run(which, tmp_path)
    meta = ast.literal_eval(str(got["meta"]))
    if not meta["gpu"]:
        # every stage went through the library's entry points (here: their oracle-backed stand-ins)
        assert {"dfq_bn_fold", "dfq_cle_run", "dfq_bias_correct", "dfq_quantize_tensors"} <= set(meta["library_calls"])
    for marker in ("Start cross layer equalization", "Start bias correction", "Quantizing Layer parameters", "SET QUANT MIN MAX"):
        assert marker in log, marker
    assert list(got["w_class"]) == list(gold["w_class"])
    # the observers fired exactly as often as in the reference run: layer inputs + functional ops patched by replace_op()
    assert list(got["observer_calls"]) == list(gold["observer_calls"]) and gold["observer_calls"][1] > 0
    # weights: the 8-bit codes of the calibrated model.  On the fixture's machine the executor reproduces the reference's
    # fold + equalization bit for bit (host sqrt injected) -> identical digests; elsewhere / on the GPU (IEEE sqrt) the last
    # bit of S may differ (DESIGN.md section 4) -> per-tensor max|w| and sum within 1e-5
    same = np.asarray(got["w_sha"] == gold["w_sha"])
    if not meta["gpu"]:
        assert same.all(), "weights differ from the reference run in layers %s" % np.nonzero(~same)[0].tolist()
    assert np.allclose(got["w_absmax"], gold["w_absmax"], rtol=1e-5, atol=0)
    tol = 1e-5 if same.all() else 5e-2
    for k in gold.files:
        kind = k.split("_")[0]
        if kind in ("bias", "fb", "fw"):
            assert _nw(got[k], gold[k]) < tol, (k, _nw(got[k], gold[k]))
        elif kind in ("qrange", "oprange"):
            # set_quant_minmax: rectified-Gaussian moments cancel (layer_transform.py:411-422), 3e-4 as in test_host_logic
            assert _nw(got[k], gold[k]) < max(3e-4, tol), (k, got[k], gold[k])
    # the calibrated 8-bit model computes the same function (activation codes may flip where a range moved by 1e-4)
    for k in gold.files:
        if k.startswith("output_"):
            assert got[k].shape == gold[k].shape
            assert _nw(got[k], gold[k]) < 0.15, (k, _nw(got[k], gold[k]))
    if which == "cls":
        assert np.array_equal(got["output_0"].argmax(1), gold["output_0"].argmax(1))


@pytest.mark.skipif(not os.path.isfile(os.path.join(REF, "main_cls.py")), reason="reference checkout not present")
def test_launcher_imports_every_name_the_scripts_need():
    """tools/run_main.py's environment alone (no test shims): the import block of all three scripts resolves against
    dropin/ - the round-1 failure (`from improve_dfq import GradHook`, ZeroQ/distill_data.py:28) stays fixed."""
    code = (
        "import sys; sys.path.insert(0, %r); import run_main; run_main.prepare_environment()\n"
        "import dfq, improve_dfq, utils.quantize, utils.layer_transform, utils.relation\n"
        "assert 'dropin' in dfq.__file__ and 'dropin' in improve_dfq.__file__, dfq.__file__\n"
        "from ZeroQ.distill_data import getDistilData\n"
        "from improve_dfq import GradHook, ModuleHook, update_scale, transform_quant_layer, set_scale, update_quant_range, set_update_stat, bias_correction_distill\n"
        "from dfq import cross_layer_equalization, bias_absorption, bias_correction, _quantize_error, clip_weight\n"
        "from utils.layer_transform import switch_layers, replace_op, restore_op, set_quant_minmax, merge_batchnorm, quantize_targ_layer\n"
        "from utils.quantize import QuantConv2d, QuantLinear, QuantNConv2d, QuantNLinear, QuantMeasure, QConv2d, QLinear, set_layer_bits, quantize\n"
        "from utils.relation import create_relation\n"
        "from utils.metrics import Evaluator\n"
        "import torch; h = GradHook(torch.nn.Parameter(torch.randn(4, 3, 3, 3))); assert h.mask.shape == (4, 3, 3, 3)\n"
        "try:\n    update_scale()\nexcept NotImplementedError as e:\n    assert 'learned-scale' in str(e)\nelse:\n    raise SystemExit('update_scale must raise')\n"
        "print('imports ok')\n" % os.path.join(ROOT, "tools"))
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert res.returncode == 0 and "imports ok" in res.stdout, res.stdout[-2000:] + res.stderr[-3000:]
