"""dfq_b200.int8.chain_int8(..., residual=True, pool_cat=True, upsample=True) on the CPU: which bilinear upsamples are fused
and how, and that the chained module computes what the per-layer one does - through the host twins of the library
(tests/int8_upsample_oracle.py), with torch told that CPU tensors are on the GPU and F.interpolate computing what torch's
CUDA kernel computes (the oracle).  Also the oracle's fused multiply-add against exact rationals."""
import math
from collections import OrderedDict

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import int8_upsample_oracle as UO
from deeplab_v3plus_like import DeepLabV3PlusLike
from test_int8_chain_host import _identity_bns, _x
from test_int8_pool_cat_host import _scales_through_pools

f32 = np.float32
INF = math.inf
NONE = (-INF, INF)
_TORCH_INTERPOLATE = F.interpolate


# ---- the oracle's fma -----------------------------------------------------------------------------------------------------
def _fma_cases():
    rng = np.random.default_rng(0)
    a = (rng.standard_normal(3000) * np.exp2(rng.integers(-30, 30, 3000))).astype(f32)
    b = (rng.standard_normal(3000) * np.exp2(rng.integers(-30, 30, 3000))).astype(f32)
    c = (-(a.astype(np.float64) * b) * (1 + rng.standard_normal(3000) * 1e-6)).astype(f32)   # heavy cancellation
    c[::3] = (rng.standard_normal(1000) * 4).astype(f32)
    one, ulp = f32(1), np.spacing(f32(1))
    edge = [(one + ulp, one + ulp, -one),                                    # exact product has bits beyond fp32
            (one + ulp, one - ulp / 2, f32(0)),
            (f32(1.5), f32(2 ** -24), one),
            (one + 2 * ulp, f32(2 ** -25), one),                             # just above a tie
            (f32(3), f32(2 ** -25) * (1 + ulp), one),
            (f32(2 ** -75), f32(2 ** -75), f32(2 ** -149)),                  # subnormal results
            (f32(2 ** -70), f32(-(2 ** -70)), f32(2 ** -126)),
            (f32(3.4e38), f32(2), f32(-3.4e38)),                             # overflowing product, finite result
            (f32(3.4e38), f32(1.5), f32(0)),                                 # overflow
            (f32(0.1), f32(10), f32(-1)), (f32(-0.0), f32(5), f32(0.0)), (f32(0.75), f32(0.5), f32(-0.375))]
    ea, eb, ec = (np.array(v, f32) for v in zip(*edge))
    return np.concatenate([a, ea]), np.concatenate([b, eb]), np.concatenate([c, ec])


def test_fma32_rounds_once_like_exact_rationals():
    a, b, c = _fma_cases()
    got = UO.fma32(a, b, c)
    want = np.array([UO.fma32_exact(*t) for t in zip(a, b, c)], f32)
    assert np.array_equal(got == 0, want == 0)
    nz = want != 0
    assert np.array_equal(got[nz].view(np.uint32), want[nz].view(np.uint32))


def test_oracle_copies_an_unchanged_size_and_keeps_special_values():
    x = np.array([np.nan, np.inf, -0.0, 1e-40, 1.0, -2.0], f32).reshape(1, 1, 2, 3)
    y = UO.i8_upsample_bilinear(x, 2, 3, False)
    assert np.array_equal(y.view(np.uint32), x.view(np.uint32))
    y = UO.i8_upsample_bilinear(np.full((1, 1, 1, 1), -0.0, f32), 3, 2, True)
    assert np.all(y.view(np.uint32) == 0x80000000)                          # fma(1, -0, fl(0 * -0)) = -0 + -0
    y = UO.i8_upsample_bilinear(np.array([[[[-0.0, 0.0]]]], f32), 1, 3, False)
    assert y.view(np.uint32).tolist() == [[[[0, 0, 0]]]]                    # fma(1, -0, fl(0 * +0)): +0, not x's -0


# ---- chain_int8 -----------------------------------------------------------------------------------------------------------
def _convert(model, acts):
    from dfq_b200 import int8
    graph = OrderedDict((id(m), m) for m in model.modules() if isinstance(m, (nn.Conv2d, nn.Linear)))
    names = {id(m): n for n, m in model.named_modules()}
    int8.convert_to_int8(model, graph, [nn.Conv2d, nn.Linear], act_scales=[acts[names[k]] for k in graph])


def _gpu_interpolate(monkeypatch):
    """F.interpolate computing, for bilinear with a size, what torch's CUDA kernel computes (the oracle)."""
    orig = F.interpolate

    def interpolate(input, size=None, scale_factor=None, mode="nearest", align_corners=None, recompute_scale_factor=None,
                    antialias=False):
        if mode == "bilinear" and size is not None and scale_factor is None and not antialias:
            return torch.from_numpy(UO.i8_upsample_bilinear(input.numpy(), int(size[0]), int(size[1]), bool(align_corners)))
        return orig(input, size, scale_factor, mode, align_corners, recompute_scale_factor, antialias)
    monkeypatch.setattr(F, "interpolate", interpolate)


def _chain(monkeypatch, model, x, acts):
    """The chained module (upsample=True) of `model` converted at `acts`, checked bit for bit against the per-layer model on
    x through the twins."""
    from dfq_b200 import int8
    fake = UO.install(monkeypatch)
    torch.manual_seed(0)
    model = model.eval()
    _convert(model, acts)
    gm = int8.chain_int8(model, residual=True, pool_cat=True, upsample=True)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    _gpu_interpolate(monkeypatch)
    with torch.no_grad():
        fake.calls.clear()
        y = gm(x)
        ref = model(x)
    y, ref = (t["out"] if isinstance(t, dict) else t for t in (y, ref))
    assert y.dtype == torch.float32 and np.array_equal(y.numpy().view(np.int32), ref.numpy().view(np.int32))
    return gm, fake


class _Branches(nn.Module):
    """a -> relu (9x11), p -> relu -> upsample (5x6 -> 9x11) -> `after`, cat -> z; `how` picks the size (a shape query on
    the other cat operand, as the reference's DeepLab; a constant; the input's shape) or an fp32 user."""

    def __init__(self, how="slice", after=None, align_corners=True, **interp):
        super().__init__()
        self.a, self.p = nn.Conv2d(3, 16, 3, 1, 1), nn.Conv2d(3, 24, 3, 2, 1)
        self.z, self.z2 = nn.Conv2d(40, 8, 1), nn.Conv2d(24, 8, 1)
        self.how, self.after, self.ac = how, after or nn.Identity(), align_corners
        self.interp = interp or dict(mode="bilinear")

    def forward(self, x):
        a = F.relu(self.a(x))
        kw = dict(self.interp)
        if "scale_factor" not in kw:
            kw["size"] = {"const": (9, 11), "input": x.shape[-2:]}.get(self.how, a.size()[2:])
        u = self.after(F.interpolate(F.relu(self.p(x)), align_corners=self.ac, **kw))
        if self.how == "fp32_user":
            return self.z2(u).mean((2, 3)) + u.mean()
        return self.z(torch.cat([a, u], 1)).mean((2, 3))


ACTS = {"a": 7.0, "p": 7.0, "z": 3.0, "z2": 5.0}


@pytest.mark.parametrize("how", ["slice", "const", "input"])
def test_upsample_writes_its_slice_of_the_cat(monkeypatch, how):
    gm, fake = _chain(monkeypatch, _Branches(how), _x(), ACTS)
    assert gm.fused_upsamples == [("interpolate", "p", "slice", True)]
    assert gm.fused_cats == [("cat", ["a", "interpolate"], [0, 16])]
    assert ("cat", "z", NONE) in gm.requantized_edges
    assert gm.get_submodule("p").epilogue == (None, (0.0, INF), NONE, False, True)
    up = gm.get_submodule("int8_up_interpolate")
    assert up.out_slice == (16, 48) and up.clamp == NONE and up.out_scale == 3.0
    assert fake.calls.count("dfq_i8_upsample_bilinear") == 1 and fake.calls.count("dfq_i8_conv_slice") == 1


@pytest.mark.parametrize("query", ["size_slice", "shape", "size_dims", "on_producer"])
def test_shape_queries_on_cat_operands_read_the_slice_writers_shape(monkeypatch, query):
    """Sizes read off a cat operand (the reference's `size=x4.size()[2:]`), off its producer, and off the upsample's own
    output: those users only read shapes, the cat still fuses, and each query gets [N, C, H, W] of its operand."""
    from dfq_b200 import int8

    class M(_Branches):
        def forward(self, x):
            pa = self.a(x)
            a = F.relu(pa)
            src = pa if query == "on_producer" else a
            size = {"size_slice": lambda: src.size()[2:], "shape": lambda: src.shape[-2:],
                    "size_dims": lambda: (src.size(2), src.size(3)), "on_producer": lambda: src.size()[-2:]}[query]()
            u = F.interpolate(F.relu(self.p(x)), size=size, mode="bilinear", align_corners=True)
            return self.z(torch.cat([a, u], 1)).mean((2, 3)) * (u.size(1) - 23) * (src.shape[1] - 15)
    model = M()
    gm, _ = _chain(monkeypatch, model, _x(), ACTS)
    assert gm.fused_upsamples == [("interpolate", "p", "slice", True)]
    assert gm.fused_cats == [("cat", ["a", "interpolate"], [0, 16])]
    views = [n for n in gm.graph.nodes if n.op == "call_function" and n.target is int8._nchw_view]
    assert len(views) == (4 if query == "size_dims" else 3)
    monkeypatch.setattr(F, "interpolate", _TORCH_INTERPOLATE)                        # trace with torch's again
    assert int8.chain_int8(model, residual=True, pool_cat=True).fused_cats == []     # without upsample=True: as before


def test_clamp_after_the_upsample_is_composed_with_the_cat_tail(monkeypatch):
    class M(_Branches):
        def forward(self, x):
            a = F.relu(self.a(x))
            u = F.hardtanh(F.interpolate(self.p(x), size=x.shape[-2:], mode="bilinear", align_corners=False), -1.0, 2.0)
            return self.z(F.relu6(torch.cat([a, u], 1))).mean((2, 3))
    gm, _ = _chain(monkeypatch, M(), _x(), ACTS)
    assert gm.fused_upsamples == [("interpolate", "p", "slice", False)]
    assert gm.get_submodule("int8_up_interpolate").clamp == (0.0, 2.0)
    assert gm.get_submodule("a").requant == (3.0, 0.0, 6.0)
    assert gm.get_submodule("p").epilogue == (None, NONE, NONE, False, True)


def test_upsample_whose_users_take_codes(monkeypatch):
    class M(_Branches):
        def forward(self, x):
            u = F.relu(F.interpolate(F.relu(self.p(x)), size=(9, 11), mode="bilinear", align_corners=False))
            return self.z2(u).mean((2, 3)) + self.z3(u).mean((2, 3))

        def __init__(self):
            super().__init__()
            self.z3 = nn.Conv2d(24, 8, 1)
    gm, fake = _chain(monkeypatch, M(), _x(), dict(ACTS, z3=5.0))
    assert gm.fused_upsamples == [("interpolate", "p", "codes", False)]
    assert {e for e in gm.requantized_edges if e[0] == "interpolate"} == {("interpolate", "z2", (0.0, INF)),
                                                                           ("interpolate", "z3", (0.0, INF))}
    assert gm.get_submodule("int8_up_interpolate").out_slice is None
    assert not any(n.op == "call_function" and n.target is torch.relu for n in gm.graph.nodes)


@pytest.mark.parametrize("what", ["fp32_user", "scales_apart", "nearest", "bicubic", "scale_factor", "antialias",
                                  "align_none", "nn_nearest"])
def test_upsamples_that_stay_in_torch(monkeypatch, what):
    acts = dict(ACTS)
    if what == "fp32_user":
        model = _Branches("fp32_user")
    elif what == "scales_apart":
        class M(_Branches):
            def __init__(self):
                super().__init__()
                self.z3 = nn.Conv2d(24, 8, 1)

            def forward(self, x):
                u = F.interpolate(F.relu(self.p(x)), size=(9, 11), mode="bilinear", align_corners=True)
                return self.z2(u).mean((2, 3)) + self.z3(u).mean((2, 3))
        model = M()
        acts["z3"] = float(np.nextafter(f32(5.0), f32(9)))
    elif what == "nn_nearest":
        class M(_Branches):
            def __init__(self):
                super().__init__()
                self.up = nn.Upsample(size=(9, 11), mode="nearest")

            def forward(self, x):
                return self.z(torch.cat([F.relu(self.a(x)), self.up(F.relu(self.p(x)))], 1)).mean((2, 3))
        model = M()
    else:
        interp = {"nearest": dict(mode="nearest"), "bicubic": dict(mode="bicubic"),
                  "scale_factor": dict(mode="bilinear", scale_factor=(9 / 5, 11 / 6)),
                  "antialias": dict(mode="bilinear", antialias=True), "align_none": dict(mode="bilinear")}[what]
        model = _Branches("slice", align_corners=None if what in ("align_none", "nearest") else False, **interp)
    from dfq_b200 import int8
    UO.install(monkeypatch)
    _convert(model.eval(), acts)
    gm = int8.chain_int8(model, residual=True, pool_cat=True, upsample=True)
    assert gm.fused_upsamples == [] and gm.fused_cats == []
    if what in ("fp32_user", "scales_apart"):
        _chain(monkeypatch, model, _x(), acts)                  # converted again: bit-identical with the upsample in torch


def test_nn_upsample_module_fuses(monkeypatch):
    class M(_Branches):
        def __init__(self):
            super().__init__()
            self.up = nn.Upsample(size=(9, 11), mode="bilinear", align_corners=True)

        def forward(self, x):
            return self.z(torch.cat([F.relu(self.a(x)), self.up(F.relu(self.p(x)))], 1)).mean((2, 3))
    gm, _ = _chain(monkeypatch, M(), _x(), ACTS)
    assert gm.fused_upsamples == [("up", "p", "slice", True)]


def test_upsample_needs_pool_cat():
    from dfq_b200 import _lib, int8
    with pytest.raises(_lib.DfqError, match="upsample=True builds on pool_cat=True"):
        int8.chain_int8(_Branches(), residual=True, upsample=True)


def test_size_checked_at_run_time_naming_the_node(monkeypatch):
    from dfq_b200 import _lib, int8
    UO.install(monkeypatch)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    m = int8.Int8UpsampleBilinear(24, True, 3.0, name="interpolate_7")
    x = torch.randn(1, 24, 5, 6)
    for bad in [(0, 4), (3,), (3, 4, 5), 7, (3.0, 4), (True, 4), (-1, 4)]:
        with pytest.raises(_lib.DfqError, match="interpolate_7: size must be a pair of positive ints"):
            m(x, bad)
    assert tuple(m(x, torch.Size([9, 11])).shape) == (1, 9, 11, 32)


# ---- the two segmentation networks -----------------------------------------------------------------------------------------
def _deeplab_like_scales(model):
    return _scales_through_pools(model)


def test_deeplab_v3plus_like_fuses_both_cats_and_runs_bit_identically(monkeypatch):
    from dfq_b200 import int8
    model = _identity_bns(DeepLabV3PlusLike(num_classes=5))
    gm, fake = _chain(monkeypatch, model, torch.randn(1, 3, 49, 45, generator=torch.Generator().manual_seed(2)),
                      _deeplab_like_scales(model))
    assert [c[0] for c in gm.fused_cats] == ["cat", "cat_1"]
    assert gm.fused_cats[0][1][-1] == "interpolate" and gm.fused_cats[1][1][0] == "interpolate_1"
    assert gm.fused_upsamples == [("interpolate", "aspp.pool.1", "slice", True),
                                  ("interpolate_1", "aspp.project.0", "slice", True)]
    assert {"aspp.project.0", "last_conv.0"} <= {q for _, q, _ in gm.requantized_edges}
    assert [n.name for n in gm.graph.nodes if n.op == "call_function" and "interpolate" in str(n.target)] == \
        ["interpolate_2"]                                                   # the logits' upsample stays in torch
    assert sum(n.op == "call_function" and n.target is int8._nchw_view for n in gm.graph.nodes) == 2   # x3's and r's sizes
    assert fake.calls.count("dfq_i8_upsample_bilinear") == 2


def test_torchvision_deeplabv3_resnet50_fuses_its_aspp_cat(monkeypatch):
    import torchvision
    from dfq_b200 import int8
    UO.install(monkeypatch)
    torch.manual_seed(0)
    model = _identity_bns(torchvision.models.segmentation.deeplabv3_resnet50(
        weights=None, weights_backbone=None, aux_loss=False, num_classes=5))
    _convert(model, _scales_through_pools(model))
    gm = int8.chain_int8(model, residual=True, pool_cat=True, upsample=True)
    base = int8.chain_int8(model, residual=True, pool_cat=True)
    assert base.fused_cats == [] and gm.fused_upsamples == [("interpolate", "classifier.0.convs.4.1", "slice", False)]
    assert [c[0] for c in gm.fused_cats] == ["cat"] and len(gm.fused_cats[0][1]) == 5
    carried, before = ({q for _, q, _ in m.requantized_edges} for m in (gm, base))
    assert carried == before | {"classifier.0.project.0"}
