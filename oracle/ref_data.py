"""Data of the reference checkout (jakc4103/DFQ) that tests read, staged into the git-ignored oracle/_ref/.

Only data is staged, never sources: the bundled MobileNetV2 checkpoint (14 MB) behind the golden ncnn calibration table
(tests/ncnn_table_case.py).  The reference checkout is the one tools/refenv.py imports (DFQ_REFERENCE_ROOT); where it is
absent or unreadable nothing is staged and the tests that need the checkpoint skip.
"""
import os
import shutil

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
FILES = [os.path.join("modeling", "classification", "mobilenetv2_1.0-f2a8633.pth.tar")]


def stage() -> list:
    """Copy every file of FILES that exists in the reference checkout and is not staged yet; returns the staged paths."""
    from tools.refenv import REF_ROOT as ref_root
    done = []
    for rel in FILES:
        src, dst = os.path.join(ref_root, rel), os.path.join(OUT, os.path.basename(rel))
        if os.path.isfile(dst):
            done.append(dst)
            continue
        if not os.access(src, os.R_OK):
            continue
        os.makedirs(OUT, exist_ok=True)
        shutil.copyfile(src, dst + ".part")
        os.replace(dst + ".part", dst)
        done.append(dst)
    return done
