"""Edge cases of the soft NMS as data: one-image scenes (scores [1, P, C], decoded boxes [1, P, 4]) whose segments hold
ties, NaN and +-inf scores and boxes, zero-area and identical boxes, a single candidate, scores at the threshold and one
ulp above it, and a class in which every prior is a candidate.  Shared by the CPU tests (the oracle against box_utils)
and the GPU tests (the kernel against the oracle on CUDA tensors)."""
import numpy as np
import torch

THR = 0.01
SIGMA = 0.3
NAN, INF = float("nan"), float("inf")


def _up(x):
    return float(np.nextafter(np.float32(x), np.float32(1)))


def _random_boxes(g, P, spread=1.0):
    c = torch.rand(P, 2, generator=g) * spread
    wh = torch.rand(P, 2, generator=g) * 0.3 + 0.01
    return torch.cat([c - wh / 2, c + wh / 2], 1)


def scenes():
    """[(name, scores [1, P, C], boxes [1, P, 4])]."""
    out = []
    g = torch.Generator().manual_seed(3)

    # ties: equal scores on overlapping and on disjoint boxes, -0.0 and +0.0 below a negative threshold elsewhere
    P, C = 64, 4
    s = torch.zeros(1, P, C)
    b = _random_boxes(g, P).unsqueeze(0)
    s[0, :, 1] = torch.tensor([0.5, 0.25] * (P // 2))
    s[0, :, 2] = 0.125
    s[0, 10:20, 3] = 0.75
    b[0, 10:20] = b[0, 10]                         # identical boxes with identical scores
    out.append(("ties", s, b))

    # non-finite scores: NaN never a candidate, +inf one (it decays to NaN against itself-like boxes), -inf never
    P, C = 40, 3
    s = torch.rand(1, P, C, generator=g) * 0.5
    b = _random_boxes(g, P, 0.5).unsqueeze(0)
    s[0, 0:4, 1] = torch.tensor([NAN, INF, -INF, INF])
    s[0, 5, 2] = INF
    s[0, 6, 2] = NAN
    out.append(("nonfinite_scores", s, b))

    # non-finite boxes: NaN coordinates, +-inf coordinates (inf areas and inf - inf)
    P, C = 32, 3
    s = torch.rand(1, P, C, generator=g) * 0.5 + 0.02
    b = _random_boxes(g, P, 0.4).unsqueeze(0)
    b[0, 0] = torch.tensor([NAN, 0.1, 0.2, 0.3])
    b[0, 1] = torch.tensor([-INF, -INF, INF, INF])
    b[0, 2] = torch.tensor([0.1, 0.1, INF, 0.2])
    b[0, 3] = torch.tensor([0.1, NAN, NAN, 0.2])
    s[0, 1, 1] = 0.99                               # the infinite box is picked first in class 1
    s[0, 0, 2] = 0.99                               # the NaN box first in class 2
    out.append(("nonfinite_boxes", s, b))

    # zero-area, inverted and identical boxes
    P, C = 48, 2
    s = torch.rand(1, P, C, generator=g) * 0.5 + 0.02
    b = _random_boxes(g, P, 0.3).unsqueeze(0)
    b[0, 0:8] = torch.tensor([0.2, 0.2, 0.2, 0.2])               # points
    b[0, 8:12] = torch.tensor([0.3, 0.3, 0.1, 0.5])              # inverted in x: clamped to zero area
    b[0, 12:24] = b[0, 30]                                       # identical to another box
    out.append(("degenerate_boxes", s, b))

    # one candidate in a class; a class without; scores at the threshold and one ulp above
    P, C = 16, 4
    s = torch.zeros(1, P, C)
    b = _random_boxes(g, P).unsqueeze(0)
    s[0, 3, 1] = 0.4
    s[0, :, 3] = THR
    s[0, 2, 3] = _up(THR)
    s[0, 9, 3] = _up(THR)
    b[0, 9] = b[0, 2]                               # decays below the threshold at once
    out.append(("single_and_threshold", s, b))

    # every prior a candidate, boxes crowded so that many rows decay out at every step
    P, C = 700, 2
    s = torch.rand(1, P, C, generator=g) * 0.9 + 0.05
    b = _random_boxes(g, P, 0.2).unsqueeze(0)
    out.append(("all_candidates_crowded", s, b))

    # rows rescored to exactly the threshold and to values that tie after the decay
    P, C = 24, 2
    s = torch.full((1, P, C), 0.5)
    b = torch.tensor([0.0, 0.0, 1.0, 1.0]).repeat(1, P, 1)
    b[0, 1:, 0] = torch.linspace(0.05, 0.95, P - 1)
    out.append(("shifted_copies", s, b))
    return out
