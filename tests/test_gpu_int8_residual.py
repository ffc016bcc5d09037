"""The residual int8 epilogue on the H100: dfq_i8_conv_fused against the oracle byte for byte and bit for bit, and
dfq_b200.int8.chain_int8(..., residual=True) on whole models bit for bit against the per-layer path."""
import ctypes as C
import math
from collections import Counter

import numpy as np
import pytest
import torch
import torch.nn as nn

import int8_chain_oracle as CO
import int8_oracle as O
import int8_residual_oracle as RO
import test_gpu_int8 as G
import test_gpu_int8_chain as GC

pytestmark = pytest.mark.gpu
f32 = np.float32
INF = math.inf
NONE = (-INF, INF)
SENTINEL, TAIL = -128, 64                        # never a code (the clamp is +-127); elements checked past each output's end
Y_SENTINEL = np.uint32(0x7FBADBAD)               # a NaN payload no fp32 op produces
CLAMPS = {"none": (NONE, NONE), "relu_after": (NONE, (0.0, INF)), "pre_post": ((-1.0, 2.5), (0.0, 6.0)),
          "both_relu6": ((0.0, 6.0), (0.0, 6.0))}
OUTS = {"codes": (False, True), "fp32": (True, False), "both": (True, True)}


def _vp(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _epilogue(r=0, y=0, yq=0, out_scale=1.0, pre=NONE, post=NONE):
    from dfq_b200 import _lib
    d = np.zeros(1, _lib.I8_EPILOGUE_DT)
    d[0] = (r, y, yq, out_scale) + tuple(pre) + tuple(post)
    return d


class _Bufs:
    """Sentinel-filled y (fp32) and yq (int8) buffers with sentinel tails for an [N, O, OH, OW] output."""

    def __init__(self, N, O_, OH, OW):
        self.n = N * O_ * OH * OW
        self.nq = N * OH * OW * ((O_ + 15) // 16 * 16)
        self.y = torch.from_numpy(np.full(self.n + TAIL, Y_SENTINEL, np.uint32).view(np.float32)).cuda()
        self.yq = torch.full((self.nq + TAIL + 16,), SENTINEL, dtype=torch.int8, device="cuda")

    def read(self):
        torch.cuda.synchronize()
        return self.y.cpu().numpy().view(np.uint32), self.yq.cpu().numpy()

    def untouched(self):
        y, yq = self.read()
        return bool(np.all(y == Y_SENTINEL) and np.all(yq == SENTINEL))


def _fused_abi(layer, xq_nhwc, g, r, bufs, y_on, yq_on, out_scale, pre, post):
    from dfq_b200 import _lib
    d = _epilogue(r.data_ptr() if r is not None else 0, bufs.y.data_ptr() if y_on else 0,
                  bufs.yq.data_ptr() if yq_on else 0, out_scale, pre, post)
    return _lib.load().dfq_i8_conv_fused(_vp(xq_nhwc), _vp(layer.weight_codes), _vp(layer.dq), _vp(layer.bias),
                                         _lib.table_ptr(d), _lib.table_ptr(g), _lib.stream_ptr())


def _special_residual(y_pre, seed):
    """A residual of y's shape: random values, with NaN, +-inf, -0.0, the exact negation of some pre-clamped outputs and 3e38
    where the output is 3e38 (bias channel 0 is set to it)."""
    rng = np.random.default_rng(seed)
    r = (rng.standard_normal(y_pre.shape) * 2).astype(f32)
    flat, pre = r.reshape(-1), y_pre.reshape(-1)
    k = flat.size
    idx = rng.permutation(k)
    parts = np.array_split(idx[: max(6, k // 4)], 6)
    flat[parts[0]] = np.nan
    flat[parts[1]] = np.inf
    flat[parts[2]] = -np.inf
    flat[parts[3]] = -0.0
    flat[parts[4]] = -pre[parts[4]]                             # exact cancellation (finite values)
    r[:, 0] = f32(3e38)                                         # 3e38 + 3e38 = inf in fp32
    return r


def _check_fused(conv, x, a, ws, out, res, clamps, cpad_in=None, seed=0):
    """dfq_i8_conv_fused of `conv` on the oracle's codes of x, compared with i8_epilogue: every byte of yq (pad channels
    included) and every bit of y, sentinel tails untouched, the buffers not asked for untouched."""
    from dfq_b200 import _lib, int8
    y_on, yq_on = OUTS[out]
    pre, post = CLAMPS[clamps]
    if conv.bias is not None:
        with torch.no_grad():
            conv.bias[0] = 3e38
    layer = int8.Int8Conv2d.from_conv(conv, a, ws)
    N, Cn, H, W = x.shape
    g = layer._geometry(N, H, W)
    cpad = cpad_in or layer.cpad
    if cpad_in:
        g[0]["Cpad"] = cpad_in
        wq = torch.zeros(((conv.out_channels if conv.groups == 1 else 1) * conv.kernel_size[0] * conv.kernel_size[1] * cpad,),
                         dtype=torch.int8, device="cuda")
        _lib.check(_lib.load().dfq_i8_pack_weights(_vp(conv.weight.detach().contiguous()), _vp(layer.w_scale), _vp(wq),
                                                   _lib.table_ptr(g), _lib.stream_ptr()), "pack")
        layer.weight_codes = wq
    xq = np.zeros((N, H, W, cpad), np.int8)
    xq[..., :Cn] = O.i8_quantize(x.detach().cpu().numpy(), a).transpose(0, 2, 3, 1)
    acc, _ = G._oracle(x, conv, a, ws)
    wsb = np.broadcast_to(np.asarray(ws, f32), (conv.out_channels,))
    b = None if conv.bias is None else conv.bias.detach().cpu().numpy()
    y0 = O.i8_dequant(acc, a, wsb, b)
    r = _special_residual(CO.i8_clamp(y0, *pre), seed) if res else None
    v = RO.i8_epilogue_value(y0, r, pre, post, gpu_nan=True)
    rest = v[:, 1:] if v.shape[1] > 1 else v                   # channel 0 carries the 3e38 bias: scale from the others
    fin = np.abs(rest[np.isfinite(rest)])
    out_scale = f32(160.0 / fin.max()) if fin.size and fin.max() > 0 else f32(1.0)
    want_y, want_q = RO.i8_epilogue(acc, a, wsb, b, r, pre, post, out_scale)
    if yq_on and v.shape[1] > 1 and fin.size and fin.max() > 0:
        assert np.abs(want_q[:, 1:]).max() == 127, "the codes of the other channels reach the full range"
    assert np.array_equal(want_y.view(np.uint32), v.view(np.uint32))
    bufs = _Bufs(N, conv.out_channels, *acc.shape[2:])
    r_d = torch.from_numpy(r).cuda() if res else None
    _lib.check(_fused_abi(layer, torch.from_numpy(xq).cuda(), g, r_d, bufs, y_on, yq_on, out_scale, pre, post),
               "dfq_i8_conv_fused")
    got_y, got_q = bufs.read()
    if y_on:
        assert np.array_equal(got_y[:bufs.n], want_y.reshape(-1).view(np.uint32)), "y"
    assert np.all(got_y[bufs.n if y_on else 0:] == Y_SENTINEL), "y written past its end or when not asked for"
    if yq_on:
        assert np.array_equal(got_q[:bufs.nq], CO.to_nhwc_codes(want_q).reshape(-1)), "codes"
    assert np.all(got_q[bufs.nq if yq_on else 0:] == SENTINEL), "yq written past its end or when not asked for"
    if res:
        assert torch.equal(r_d.cpu().view(torch.int32), torch.from_numpy(r).view(torch.int32)), "the residual changed"
    return want_y


def _clamps(out, res):
    """The clamp pair of one (output, residual) combination: the six combinations of a case cover all four pairs."""
    return list(CLAMPS)[(list(OUTS).index(out) * 2 + (not res)) % len(CLAMPS)]


def _dense(case, out, res, clamps):
    N, Cn, H, W, Oc, k, s, p, d = case
    torch.manual_seed(G._seed(case))
    conv = nn.Conv2d(Cn, Oc, k, s, p, d).cuda()
    x = torch.randn(N, Cn, H, W, device="cuda") * 2
    _check_fused(conv, x, G._ascale(x), G._channel_scales(conv.weight, G._seed(case)), out, res, clamps, seed=G._seed(case))


@pytest.mark.parametrize("res", [True, False], ids=["residual", "no_residual"])
@pytest.mark.parametrize("out", list(OUTS))
@pytest.mark.parametrize("case", G.DENSE, ids=G._case_id)
def test_dense_fused_bit_exact(case, out, res):
    _dense(case, out, res, _clamps(out, res))


@pytest.mark.parametrize("res", [True, False], ids=["residual", "no_residual"])
@pytest.mark.parametrize("out", list(OUTS))
@pytest.mark.parametrize("case", G.TILES, ids=G._case_id)
def test_dense_fused_tile_edges_bit_exact(case, out, res):
    _dense(case, out, res, "pre_post")


@pytest.mark.parametrize("res", [True, False], ids=["residual", "no_residual"])
@pytest.mark.parametrize("out", list(OUTS))
@pytest.mark.parametrize("case", G.DW, ids=G._case_id)
def test_depthwise_fused_bit_exact(case, out, res):
    clamps = _clamps(out, res)
    N, Cn, H, W, k, s, p, d = case
    torch.manual_seed(G._seed(case))
    conv = nn.Conv2d(Cn, Cn, k, s, p, d, Cn).cuda()
    x = torch.randn(N, Cn, H, W, device="cuda") * 2
    _check_fused(conv, x, G._ascale(x), G._channel_scales(conv.weight, G._seed(case)), out, res, clamps, seed=G._seed(case))


@pytest.mark.parametrize("groups, C_, cpad_in", [(16, 16, 32), (24, 24, 64), (1, 16, 32), (1, 5, 48)])
def test_fused_input_cpad_wider_than_the_output(groups, C_, cpad_in):
    torch.manual_seed(60 + cpad_in + groups)
    conv = nn.Conv2d(C_, C_ if groups > 1 else 24, 3, 1, 1, groups=groups).cuda()
    x = torch.randn(2, C_, 7, 9, device="cuda") * 2
    _check_fused(conv, x, G._ascale(x), G._channel_scales(conv.weight, 60), "both", True, "pre_post", cpad_in=cpad_in)


def test_depthwise_fused_grid_stride_loop_covers_every_item():
    N, Cn, H, W = 48, 144, 56, 56
    assert N * (Cn // 16) * H * W > G._launch_cap(), "the case no longer takes a second trip through the loop"
    torch.manual_seed(8)
    conv = nn.Conv2d(Cn, Cn, 3, 1, 1, groups=Cn).cuda()
    x = torch.randn(N, Cn, H, W, device="cuda")
    _check_fused(conv, x, G._ascale(x), G._channel_scales(conv.weight, 8), "both", True, "relu_after")


def test_fused_refusals_leave_the_buffers_untouched():
    from dfq_b200 import _lib, int8
    lib = _lib.load()
    torch.manual_seed(41)
    layer = int8.Int8Conv2d.from_conv(nn.Conv2d(16, 16, 3, 1, 1).cuda(), 1.0, 1.0)
    N, H, W = 1, 5, 5
    g = layer._geometry(N, H, W)
    xq = torch.zeros(N * H * W * 16, dtype=torch.int8, device="cuda")
    bufs = _Bufs(N, 16, H, W)
    r = torch.zeros(bufs.n, device="cuda")
    y, yq = bufs.y.data_ptr(), bufs.yq.data_ptr()
    nan = float("nan")
    cases = [
        (dict(), "no output"),
        (dict(y=y, yq=yq + 1), "yq"),
        (dict(yq=yq, pre=(nan, 6.0)), "bounds"), (dict(yq=yq, pre=(0.0, nan)), "bounds"), (dict(yq=yq, pre=(6.0, 0.0)), "bounds"),
        (dict(y=y, post=(nan, 6.0)), "bounds"), (dict(y=y, post=(1.0, -1.0)), "bounds"),
        (dict(yq=yq, out_scale=INF), "out_scale"), (dict(yq=yq, out_scale=nan), "out_scale"),
        (dict(yq=yq, out_scale=-1.0), "out_scale"),
        (dict(r=y + 4 * (bufs.n - 1), y=y), "residual overlaps"), (dict(r=yq - 4 * bufs.n + 4, yq=yq), "residual overlaps"),
        (dict(r=r.data_ptr(), y=yq - 4 * bufs.n + 16, yq=yq), "y overlaps yq"),
        (dict(r=r.data_ptr() + 2, y=y), "4-byte aligned"), (dict(y=y + 1), "4-byte aligned"),
    ]
    for kw, what in cases:
        d = _epilogue(**kw)
        rc = lib.dfq_i8_conv_fused(_vp(xq), _vp(layer.weight_codes), _vp(layer.dq), _vp(layer.bias), _lib.table_ptr(d),
                                   _lib.table_ptr(g), _lib.stream_ptr())
        assert rc == -1 and what.encode() in lib.dfq_last_error(), (kw, lib.dfq_last_error())
        assert bufs.untouched(), kw
    d = _epilogue(y=y, out_scale=nan)                           # out_scale is not read without yq
    assert lib.dfq_i8_conv_fused(_vp(xq), _vp(layer.weight_codes), _vp(layer.dq), _vp(layer.bias), _lib.table_ptr(d),
                                 _lib.table_ptr(g), _lib.stream_ptr()) == 0
    g2 = np.zeros(1, _lib.I8_CONV_DT)
    for k, v in dict(N=1, C=8, H=4, W=4, O=8, kh=1, kw=1, stride_h=1, stride_w=1, dil_h=1, dil_w=1, groups=2, OH=4, OW=4,
                     Cpad=16).items():
        g2[0][k] = v
    rc = lib.dfq_i8_conv_fused(_vp(xq), _vp(xq), _vp(r), None, _lib.table_ptr(_epilogue(y=y)), _lib.table_ptr(g2),
                               _lib.stream_ptr())
    assert rc == -2 and b"groups=2" in lib.dfq_last_error()


# ---- whole models -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("net, relu6, edges, adds", [("mobilenet_v2", True, 51, 10), ("mobilenet_v2", False, 51, 10),
                                                     ("resnet18", True, 18, 8)],
                         ids=["mobilenet_v2", "mobilenet_v2_relu", "resnet18"])
def test_residual_chained_model_is_bit_identical_to_the_per_layer_path(net, relu6, edges, adds):
    from dfq_b200 import int8
    model, x = GC._folded_and_converted(net, relu6)
    with torch.no_grad():
        before = model(x)
        gm = int8.chain_int8(model, residual=True)
        assert len(gm.requantized_edges) == edges and len(gm.fused_adds) == adds
        seen_fp32, seen_codes = {}, {}
        mods = dict(model.named_modules())
        consumers = sorted({q for _, q, _ in gm.requantized_edges})
        hooks = [mods[q].register_forward_pre_hook(lambda m, i, q=q: seen_fp32.__setitem__(q, i[0].clone())) for q in consumers]
        hooks += [gm.get_submodule(q).register_forward_pre_hook(lambda m, i, q=q: seen_codes.__setitem__(q, i[0].clone()))
                  for q in consumers]
        ref = model(x)
        got = gm(x)
        for h in hooks:
            h.remove()
        after = model(x)
    assert G._same_bits(got.cpu().numpy(), ref.cpu().numpy()), "chained logits"
    assert torch.equal(before, ref) and torch.equal(after, ref), "the converted model changed"
    for q in consumers:
        want = CO.to_nhwc_codes(O.i8_quantize(seen_fp32[q].cpu().numpy(), f32(mods[q].act_scale)))
        assert np.array_equal(seen_codes[q].cpu().numpy(), want), q


# ---- the reference's int8 MobileNetV2, blob by blob --------------------------------------------------------------------
CONVS = GC.CONVS


def _residual_plan(net, mods):
    """producer conv name -> dict(pre, add, r, post, tail, codes: [consumer names], fp32: bool, skipped: layer names) for the
    .param's (mods: the converted layers, by spec index) Conv -> [ReLU] -> [BinaryOp add -> [ReLU]] -> [Split] -> consumers structure, by chain_int8's rule."""
    users = Counter(b for l in net.layers for b in l["bottoms"])
    consumers = {}
    for l in net.layers:
        for b in l["bottoms"]:
            consumers.setdefault(b, []).append(l)
    producer_of = {l["tops"][0]: l for l in net.layers if l["type"] in CONVS}

    def single(blob):
        return consumers[blob][0] if users[blob] == 1 else None

    def forward_relu(blob, skipped):
        nxt = single(blob)
        if nxt is not None and nxt["type"] == "ReLU":
            skipped.append(nxt["name"])
            return nxt["tops"][0], (0.0, INF)
        return blob, NONE

    def back_to_conv(blob):
        l = next(l for l in net.layers if blob in l["tops"])
        if l["type"] == "ReLU" and users[blob] == 1:
            blob = l["bottoms"][0]
            l = producer_of.get(blob)
        return l if l is not None and l["type"] in CONVS and users[blob] == 1 else None

    plan = {}
    for l in net.layers:
        if l["type"] not in CONVS:
            continue
        skipped = []
        end, pre = forward_relu(l["tops"][0], skipped)
        add, r, post, tail = None, None, NONE, end
        a = single(end)
        if a is not None and a["type"] == "BinaryOp" and a["params"].get(0, 0) == 0 and len(set(a["bottoms"])) == 2:
            fused = next((b for b in a["bottoms"] if back_to_conv(b) is not None), None)
            if fused == end:
                add, r = a["name"], next(b for b in a["bottoms"] if b != end)
                skipped.append(add)
                tail, post = forward_relu(a["tops"][0], skipped)
        outs = [tail]
        s = single(tail)
        if s is not None and s["type"] == "Split":
            skipped.append(s["name"])
            outs = list(s["tops"])
        users_of = [u for o in outs for u in consumers.get(o, [])]
        codes, scale = [], None
        for u in users_of:
            if u["type"] in CONVS and \
                    mods[u["spec"]["index"]].in_channels == mods[l["spec"]["index"]].out_channels:
                sc = f32(u["spec"]["in_scale"])
                if scale is None or sc.view(np.int32) == scale.view(np.int32):
                    scale = sc
                    codes.append(u["name"])
        if add is None and not codes:
            continue
        plan[l["name"]] = dict(pre=pre, add=add, r=r, post=post, tail=tail, outs=outs, codes=codes, scale=scale,
                               fp32=len(codes) < len(users_of), skipped=skipped)
    return plan


def test_reference_int8_mobilenetv2_residual_chained_blob_by_blob():
    """The reference's deployed int8 model (tests/ncnn_int8_case.py) walked with its Split and BinaryOp layers fused as
    chain_int8(residual=True) fuses them: 51 of 52 convolution inputs carried, 10 BinaryOps fused; every fp32 blob up to the
    last ReLU and the logits equal the per-layer GPU run's bit for bit, and every carried code blob equals i8_quantize of
    the per-layer blob at the consumer's input scale."""
    from dfq_b200 import int8
    case, net = G._ref_net()
    mods = []
    for s in net.specs:
        w = torch.from_numpy(case.spec_weight(s)).cuda()
        b = None if s["bias"] is None else torch.from_numpy(s["bias"]).cuda()
        mods.append(int8.Int8Linear(w, b, s["in_scale"], s["w_scales"]) if s["type"] == "InnerProduct" else
                    int8.Int8Conv2d(w, b, s["in_scale"], s["w_scales"], s["stride"], s["pad"], s["dilation"], s["groups"]))
    plan = _residual_plan(net, mods)
    carried = {q for p in plan.values() for q in p["codes"]}
    skipped = {n for p in plan.values() for n in p["skipped"]}
    n_convs = sum(l["type"] in CONVS for l in net.layers)
    assert len(carried) == 51 and n_convs == 52, (len(carried), n_convs)
    assert sum(p["add"] is not None for p in plan.values()) == 10
    x = G._ref_images().cuda()
    blobs, codes = {}, {}
    with torch.no_grad():
        ref = net.forward(x, lambda s, v: mods[s["index"]].run(v)[0])
        for l in net.layers:
            t, p, name = l["type"], l["params"], l["name"]
            if name in skipped:
                continue
            if t in CONVS:
                m = mods[l["spec"]["index"]]
                v = codes[name] if name in carried else blobs[l["bottoms"][0]]
                m = m.chained(codes_in=name in carried) if name in carried else m
                if name not in plan:
                    blobs[l["tops"][0]] = m.run(v)[0]
                    continue
                pl = plan[name]
                e = int8.Epilogue(None if pl["scale"] is None else float(pl["scale"]), pl["pre"], pl["post"],
                                  pl["add"] is not None, pl["fp32"])
                out = m.chained(codes_in=name in carried, epilogue=e, name=name).run(
                    v, residual=blobs[pl["r"]] if pl["add"] else None)[0]
                q_out, y_out = out if (e.out_scale is not None and e.fp32) else \
                    ((out, None) if e.out_scale is not None else (None, out))
                for q in pl["codes"]:
                    codes[q] = q_out
                if y_out is not None:
                    for o in [pl["tail"]] + pl["outs"]:
                        blobs[o] = y_out
                continue
            ins = [blobs[b] for b in l["bottoms"]]
            if t == "Input":
                outs = [x]
            elif t == "InnerProduct":
                outs = [mods[l["spec"]["index"]].run(ins[0].reshape(ins[0].shape[0], -1, 1, 1))[0].reshape(ins[0].shape[0], -1)]
            elif t == "ReLU":
                outs = [torch.relu(ins[0])]
            elif t == "Split":
                outs = [ins[0]] * len(l["tops"])
            elif t == "BinaryOp":
                outs = [ins[0] + ins[1]]
            elif t == "Reshape":
                outs = [ins[0].reshape(ins[0].shape[0], p[1], p[0])]
            elif t == "Reduction":
                outs = [ins[0].mean(dim=[a % (ins[0].dim() - 1) + 1 for a in p[3]])]
            elif t == "Softmax":
                outs = [torch.softmax(ins[0], dim=1)]
            for b, o in zip(l["tops"], outs):
                blobs[b] = o
    names = list(ref)
    last_relu = [l for l in net.layers if l["type"] == "ReLU"][-1]["tops"][0]
    for n in names[:names.index(last_relu) + 1]:
        if n in blobs:
            assert G._same_bits(blobs[n].cpu().numpy(), ref[n].cpu().numpy()), n
    logits = [l for l in net.layers if l["type"] == "InnerProduct"][0]["tops"][0]
    assert G._same_bits(blobs[logits].cpu().numpy(), ref[logits].cpu().numpy())
    by_name = {l["name"]: l for l in net.layers}
    for q in carried:
        want = CO.to_nhwc_codes(O.i8_quantize(ref[by_name[q]["bottoms"][0]].cpu().numpy(),
                                              f32(mods[by_name[q]["spec"]["index"]].act_scale)))
        assert np.array_equal(codes[q].cpu().numpy(), want), q
    print("reference int8 MobileNetV2: %d of %d convolution inputs carried as int8 codes, %d BinaryOps fused"
          % (len(carried), n_convs, sum(p["add"] is not None for p in plan.values())))
