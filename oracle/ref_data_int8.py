"""The reference's int8 ncnn model, modeling/ncnn/model_quant_relu_equal.{param,bin} (3.6 MB): the bundled MobileNetV2
after `--quantize --relu --equalize` in ncnn's int8 format (tests/ncnn_int8_case.py parses it).  Data, never sources, staged
next to the checkpoint oracle/ref_data.py stages, into the git-ignored oracle/_ref/; where the reference checkout is absent or
unreadable nothing is staged and the tests that need the model skip.
"""
import os
import shutil

from oracle.ref_data import OUT

FILES = [os.path.join("modeling", "ncnn", "model_quant_relu_equal." + ext) for ext in ("param", "bin")]


def stage() -> list:
    """Copy every file of FILES that exists in the reference checkout and is not staged yet; returns the staged paths."""
    from tools.refenv import REF_ROOT as ref_root
    done = []
    for rel in FILES:
        src, dst = os.path.join(ref_root, rel), os.path.join(OUT, os.path.basename(rel))
        if not os.path.isfile(dst):
            if not os.access(src, os.R_OK):
                continue
            os.makedirs(OUT, exist_ok=True)
            shutil.copyfile(src, dst + ".part")
            os.replace(dst + ".part", dst)
        done.append(dst)
    return done
