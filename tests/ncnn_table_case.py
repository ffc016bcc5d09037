"""The reference's only checked-in numeric artefact - modeling/ncnn/model_quant_relu_equal.table (`--quantize --relu
--equalize` on the bundled MobileNetV2 checkpoint, written by convert_ncnn.py:178-201) - reproduced through THIS package's
entry points: merge_batchnorm, create_relation, signed cross_layer_equalization, set_quant_minmax, export.ncnn_scales.

Shared by the CPU test (oracle-backed executor, tests/test_host_logic.py) and the -m gpu test (libdfq_sm90.so,
tests/test_gpu_pipeline.py).  Data: the 53 + 53 expected rows are committed (tests/golden/ncnn_table_rows.npz, extracted
from the reference's table by tools/make_golden.py); the checkpoint (14 MB) is DATA of the reference, staged by
`__graft_entry__.build()` (oracle/ref_data.py) into the git-ignored oracle/_ref/ where a reference checkout is readable.
"""
import os

import numpy as np
import torch
import torch.nn as nn

from dfq_b200 import workload

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
CKPT_NAME = "mobilenetv2_1.0-f2a8633.pth.tar"


def checkpoint_path():
    p = os.path.join(os.path.dirname(HERE), "oracle", "_ref", CKPT_NAME)
    return p if os.path.isfile(p) else None


def run(monkeypatch):
    """Returns (got_w, gold_w, got_a, gold_a): weight and activation scale rows, computed and expected."""
    from dfq_b200 import dfq, export
    from dfq_b200.utils import layer_transform as LT
    from dfq_b200.utils import quantize as Q
    from dfq_b200.utils.relation import create_relation
    rows = np.load(os.path.join(GOLD, "ncnn_table_rows.npz"))
    topo = workload.load_topology(os.path.join(GOLD, "topology_mobilenetv2.json"))
    graph, bottoms, modules = workload.build_graph(topo, seed=0, conv_cls=Q.QuantNConv2d, linear_cls=Q.QuantNLinear)
    sd = torch.load(checkpoint_path(), map_location="cpu")
    it = iter([v for k, v in sd.items() if "num_batches_tracked" not in k])
    with torch.no_grad():
        for m in modules:
            if isinstance(m, (nn.Conv2d, nn.Linear)):
                m.weight.copy_(next(it))
                if m.bias is not None:
                    m.bias.copy_(next(it))
            elif isinstance(m, nn.BatchNorm2d):
                m.weight.copy_(next(it)); m.bias.copy_(next(it)); m.running_mean.copy_(next(it)); m.running_var.copy_(next(it))
    targ = [Q.QuantNConv2d, Q.QuantNLinear]
    record = [tuple(x) for x in topo["tensor_ops"]]
    ops = []
    for _, op_name in record:
        ops.extend(Q.QuantMeasure(num_bits=8, momentum=0.1) for _ in range(int(op_name.split('_')[-1])))
    monkeypatch.setattr(LT, "module_tensor_op", LT.CustomTensorOP(ops, record))
    Q.set_layer_bits(graph, 8, 8, 8, targ)
    LT.merge_batchnorm(None, graph, bottoms, targ)
    rels = create_relation(graph, bottoms, targ)
    dfq.cross_layer_equalization(graph, rels, targ, converge_thres=2e-7, signed=True)
    LT.set_quant_minmax(graph, bottoms, verbose=False)
    scales = export.ncnn_scales(graph, targ)
    return (np.array([s[0] for s in scales]), rows["weight_scales"], np.array([s[2] for s in scales]), rows["activation_scales"])
