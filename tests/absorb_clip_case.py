"""Inputs shared by the absorption / clip tests and tools/make_golden.py absorb_clip: a chain over the cases the
absorption distinguishes, and the seeded models of the reference fixture tests/golden/ref_absorb_clip.npz."""
from dfq_b200 import workload


def _conv(i, o, k=3, groups=1):
    return dict(in_channels=i, out_channels=o, kernel_size=[k, k], stride=[1, 1], padding=[k // 2, k // 2], dilation=[1, 1],
                groups=groups, bias=False)


def edge_topology():
    """One chain over the cases the absorption distinguishes: a ReLU before a depthwise and before a grouped second layer
    (absorb), no activation and a ReLU6 between two layers (do not absorb), a Data-fed first layer (clipped, never
    corrected) and a Linear head no relation reaches."""
    n = [dict(key="Data", type="Data", bottoms=None)]
    prev = "Data"

    def add(key, typ, args, act=None):
        nonlocal prev
        n.append(dict(key=key, type=typ, args=args, bottoms=[prev]))
        prev = key
        if typ == "Conv2d":
            n.append(dict(key=key + "_bn", type="BatchNorm2d", args=dict(num_features=args["out_channels"], eps=1e-5),
                          bottoms=[prev]))
            prev = key + "_bn"
        if act:
            n.append(dict(key=key + "_act", type=act, args={}, bottoms=[prev]))
            prev = key + "_act"
    add("c0", "Conv2d", _conv(3, 32), "ReLU")
    add("c1", "Conv2d", _conv(32, 32, groups=32), "ReLU")      # depthwise second of (c0, c1)
    add("c2", "Conv2d", _conv(32, 32, groups=2), "ReLU")       # grouped second of (c1, c2)
    add("c3", "Conv2d", _conv(32, 48, k=1))                    # no activation between c3 and c4
    add("c4", "Conv2d", _conv(48, 16, k=1), "ReLU6")           # ReLU6 between c4 and c5
    add("c5", "Conv2d", _conv(16, 24, k=1), "ReLU")
    add("pool", "AdaptiveAvgPool2d", dict(output_size=1))
    add("flat", "Flatten", {})
    add("fc", "Linear", dict(in_features=24, out_features=10))
    return dict(name="absorb_edges", input=[1, 3, 8, 8], nodes=n)


# the fixture: (model name, seed, absorption N, clip range).  N <= 0 because the seeded BNs (beta ~ N(0, 0.2), gamma in
# [0.5, 1.5]) make the mains' N = 3 absorb nothing.
FIXTURE_CASES = [("edges", 11, 0.0, (-0.05, 0.05)), ("stack", 12, -0.25, (-0.08, 0.08))]


def topology(name):
    return edge_topology() if name == "edges" else workload.stack_topology(2, channels=32)
