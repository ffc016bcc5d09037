"""dfq_b200.int8.chain_int8 / chain_affine on seeded random graphs (tests/chain_graphs.py) with the library's kernels: the
host suite's checks (tests/test_int8_chain_random_host.py) - bit for bit against the per-layer model at every flag set,
the affine scheme also in the reference's evaluation state, the records consistent with the graph, each layer launched
once, and int8.save / load - on the H100, so the chained epilogues (dfq_i8_conv_fused, _slice, _nhwc; the affine _fused,
_observed, _layout, _rows, max pool and upsample entries) run at shapes and combinations the networks never give them.
Batch 1 and 3, inputs up to 13 x 13."""
import pytest
import torch

import chain_graphs as CG

pytestmark = pytest.mark.gpu
SEEDS = range(40)


@pytest.fixture(autouse=True)
def _no_tf32():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    flags = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = flags


@pytest.mark.parametrize("scheme", ["ncnn", "affine"])
@pytest.mark.parametrize("seed", SEEDS)
def test_random_graph_on_the_gpu(seed, scheme, tmp_path, monkeypatch):
    """Even seeds at batch 1, odd ones at batch 3."""
    batch = (1, 3)[seed % 2]
    prog = CG.program(seed, scheme)
    if prog["batch"] != batch and any(p["n"] == "const" for op in prog["ops"] if op["k"] == "heads"
                                      for p in op["parts"]):
        prog = dict(prog, ops=[dict(op, batch=batch) if op["k"] == "heads" else op for op in prog["ops"]])
    model = CG.build(prog).cuda()
    x = CG.inputs(prog, batch).cuda()
    try:
        CG.verify(prog, model, x, tmp_path, monkeypatch)
    except BaseException:
        print(CG.describe(prog))
        raise
