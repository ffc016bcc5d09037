"""Seeded random graphs for the int8 chaining rewriters (dfq_b200.int8.chain_int8 / chain_affine)  --  TEST SUPPORT.

program(seed, scheme) draws a small op list - convolutions, pass-throughs, fan-outs, residual adds, max pools, channel
concatenations, bilinear upsamples, zero pads, SSD-style heads and a Linear tail, each wired onto earlier tensors of
consistent shapes, plus the near misses of every rule - and build(program) returns the nn.Module whose forward interprets
it.  torch.fx traces that forward into a flat graph, and every functional op is called directly from `forward`, so the
reference's patched ops (tests/affine_observed_state.record_ops) see it as the model's own.  describe(program) prints the
program as Python, to reproduce and cut down a failing seed by hand.

The consumers' keys (an ncnn act_scale, an affine (act_min, act_max, act_bits)) come from small pools, shared per tensor
so that the fan-out, pool and cat rules fire, and are sometimes nudged by one ulp or redrawn to make their near misses.
`program["near"]` counts the near misses a program holds."""
import collections
import random

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

f32 = np.float32
CHANNELS = (1, 3, 5, 16, 17, 24, 32, 48)
NCNN_KEYS = (4.0, 9.5, 21.0, 40.0, 127.0 / 3.0)
AFFINE_KEYS = ((-1.5, 2.5, 8), (0.0, 6.0, 8), (-0.75, 1.25, 4), (0.0, 1.0, 1), (-3.0, 3.0, 6), (-2.0, 0.5, 2),
               (0.0, 2.0, 3), (-4.0, 4.0, 5), (-1.0, 3.5, 7))
OBSERVER_RANGES = ((-1.5, 1.7), (-0.5, 2.5), (0.0, 6.0), (-3.0, 3.0), (-2.0, 0.25))
NEAR_MISSES = ("two_sites", "bn_not_identity", "dropout_training", "clamp_two_users", "ulp_key", "first_user_other_key",
               "add_self", "add_alpha", "add_shapes_differ", "clamp_after_pool", "cat_unaligned", "cat_same_node",
               "cat_user_other_key", "cat_dim2", "up_scale_factor", "up_nearest", "pad_asymmetric", "pad_nonzero",
               "pad_reflect", "pad_two_users", "zeropad2d", "head_not_a_head")


class _Gen:
    def __init__(self, seed, scheme):
        self.rng = random.Random(seed * 2 + (scheme == "affine"))
        self.scheme, self.seed = scheme, seed
        r = self.rng
        self.batch = r.choice((1, 3)) if r.random() < 0.3 else r.choice((1, 2))
        H, W = r.randint(5, 13), r.randint(5, 13)
        self.t = [dict(C=3, H=H, W=W, kid=None, uses=0)]     # tensors: NCHW shape, key group, users so far
        self.ops, self.mods, self.kids, self.near = [], {}, [], collections.Counter()

    # ---- keys ------------------------------------------------------------------------------------------------------
    def _draw_key(self):
        r = self.rng
        return float(f32(r.choice(NCNN_KEYS))) if self.scheme == "ncnn" else r.choice(AFFINE_KEYS)

    def _nudge(self, key):
        if self.scheme == "ncnn":
            return float(np.nextafter(f32(key), f32(np.inf)))
        lo, hi, bits = key
        return (lo, float(np.nextafter(f32(hi), f32(np.inf))), bits)

    def key(self, i, exact=False):
        """A consumer's key for tensor i: the tensor's shared key, at times one ulp away or another one."""
        t = self.t[i]
        if t["kid"] is None:
            t["kid"] = len(self.kids)
            self.kids.append(self._draw_key())
        k = self.kids[t["kid"]]
        u = self.rng.random()
        if exact or u < 0.75:
            return k
        if u < 0.87:
            self.near["ulp_key"] += 1
            return self._nudge(k)
        return self._draw_key()

    # ---- tensors and modules ---------------------------------------------------------------------------------------
    def new(self, C, H, W, kid=None):
        self.t.append(dict(C=C, H=H, W=W, kid=kid, uses=0))
        return len(self.t) - 1

    def use(self, *idx):
        for i in idx:
            self.t[i]["uses"] += 1

    def spatial(self, min_hw=1):
        return [i for i, t in enumerate(self.t) if "C" in t and t["H"] >= min_hw and t["W"] >= min_hw and not t.get("head")]

    def pick(self, min_hw=1, fresh=0.6):
        cands = self.spatial(min_hw)
        if not cands:
            cands = [0]
        if self.rng.random() < fresh:
            return cands[-1]
        return self.rng.choice(cands)

    def name(self, stem):
        n = "%s%d" % (stem, len(self.mods))
        return n

    def conv(self, src, cout=None, k=None, s=None, d=None, pad=None, dw=None, key=None, same=False):
        """A conv module on tensor src, called once; returns its output's index."""
        r, t = self.rng, self.t[src]
        C, H, W = t["C"], t["H"], t["W"]
        k = k if k is not None else r.choice((1, 3))
        s = s if s is not None else (1 if same else r.choice((1, 1, 2)))
        d = d if d is not None else (1 if k == 1 else r.choice((1, 1, 2)))
        if pad is None:
            pad = d * (k // 2) if same or r.random() < 0.7 else 0
        dw = dw if dw is not None else (C > 1 and r.random() < 0.25 and cout is None)
        cout = C if dw else (cout if cout is not None else r.choice(CHANNELS))
        OH, OW = ((n + 2 * pad - d * (k - 1) - 1) // s + 1 for n in (H, W))
        if OH < 1 or OW < 1:
            pad = d * (k // 2)
            OH, OW = ((n + 2 * pad - d * (k - 1) - 1) // s + 1 for n in (H, W))
        m = self.name("conv")
        self.mods[m] = dict(type="conv", cin=C, cout=cout, k=k, s=s, d=d, p=pad, groups=C if dw else 1,
                            key=key if key is not None else self.key(src))
        return self.call(m, src, cout, OH, OW)

    def call(self, m, src, C, H, W, kid=None):
        self.use(src)
        self.ops.append(dict(k="mod", m=m, x=src))
        return self.new(C, H, W, kid)

    def fn(self, f, src, kid="same", **kw):
        """A functional op / tensor method of one tensor that keeps its shape."""
        t = self.t[src]
        self.use(src)
        self.ops.append(dict(k=f, x=src, **kw))
        return self.new(t["C"], t["H"], t["W"], t["kid"] if kid == "same" else kid)

    def pass_through(self, src, near=True):
        r, t = self.rng, self.t[src]
        forms = ["relu_mod", "relu_f", "relu_t", "relu_m", "relu6", "hardtanh", "identity", "dropout", "bn"]
        if near:
            forms += ["bn_bad", "dropout_train"]
        f = r.choice(forms)
        if f in ("relu_f", "relu_t", "relu_m", "relu6"):
            return self.fn(f, src)
        if f == "hardtanh" and r.random() < 0.5:
            lo = r.choice((-1.0, 0.0, 0.5))
            return self.fn("hardtanh", src, lo=lo, hi=lo + r.choice((0.75, 2.0, 6.0)))
        m = self.name(f)
        spec = dict(type=f, C=t["C"])
        if f == "hardtanh":
            lo = r.choice((-2.0, 0.0))
            spec.update(lo=lo, hi=lo + r.choice((1.0, 4.0)))
        if f == "bn_bad":
            self.near["bn_not_identity"] += 1
        if f == "dropout_train":
            self.near["dropout_training"] += 1
        self.mods[m] = spec
        return self.call(m, src, t["C"], t["H"], t["W"], t["kid"])

    def chain(self, src, n=None):
        for _ in range(n if n is not None else self.rng.choice((0, 0, 1, 1, 2))):
            src = self.pass_through(src)
        return src

    def pool_params(self, H, W):
        r = self.rng
        for _ in range(20):
            k, s, d, ceil = r.choice((1, 2, 3)), r.choice((1, 2, 3)), r.choice((1, 1, 2)), r.random() < 0.4
            p = r.randint(0, min(k // 2, (d * (k - 1) + 1) // 2))
            try:
                y = F.max_pool2d(torch.zeros(1, 1, H, W), k, s, p, d, ceil_mode=ceil)
            except RuntimeError:
                continue
            if y.shape[2] >= 1 and y.shape[3] >= 1:
                return (k, s, p, d, ceil), y.shape[2], y.shape[3]
        return (1, 1, 0, 1, False), H, W

    def pool(self, src):
        r, t = self.rng, self.t[src]
        (k, s, p, d, ceil), OH, OW = self.pool_params(t["H"], t["W"])
        shared = [m for m, v in self.mods.items() if v["type"] == "maxpool"]
        if r.random() < 0.5:
            if shared and r.random() < 0.5:                     # an nn.MaxPool2d called at several sites
                m = r.choice(shared)
                v = self.mods[m]
                try:
                    y = F.max_pool2d(torch.zeros(1, 1, t["H"], t["W"]), v["k"], v["s"], v["p"], v["d"], ceil_mode=v["ceil"])
                except RuntimeError:
                    y = None
                if y is not None and min(y.shape[2:]) >= 1:
                    return self.call(m, src, t["C"], y.shape[2], y.shape[3], t["kid"])
            m = self.name("pool")
            self.mods[m] = dict(type="maxpool", k=k, s=s, p=p, d=d, ceil=ceil)
            return self.call(m, src, t["C"], OH, OW, t["kid"])
        self.use(src)
        self.ops.append(dict(k="pool", x=src, ks=k, s=s, p=p, d=d, ceil=ceil))
        return self.new(t["C"], OH, OW, t["kid"])

    def consumers(self, src, n):
        """n users of tensor src: convs (at the shared key, one ulp away, another key), a mean or a pool."""
        r = self.rng
        first_other = n >= 3 and r.random() < 0.2
        if first_other:
            self.near["first_user_other_key"] += 1
        for j in range(n):
            u = r.random()
            if first_other and j == 0:
                self.conv(src, key=self._nudge(self.key(src, exact=True)))
            elif u < 0.6:
                self.chain(self.conv(src), r.choice((0, 1)))
            elif u < 0.75:
                self.mean_tail(src)
            elif u < 0.9:
                p = self.pool(src)
                self.conv(p)
            else:
                self.conv(src, key=self._draw_key())

    def mean_tail(self, src):
        t = self.t[src]
        self.use(src)
        self.ops.append(dict(k="mean", x=src))
        i = self.new(None, None, None)
        self.t[i] = dict(vec=t["C"], uses=0, kid=None)
        if self.rng.random() < 0.6:
            m = self.name("fc")
            self.mods[m] = dict(type="linear", cin=t["C"], cout=self.rng.choice((3, 10)), key=self.key(i))
            self.use(i)
            self.ops.append(dict(k="mod", m=m, x=i))
            self.t.append(dict(vec=self.mods[m]["cout"], uses=0, kid=None))
        return i

    # ---- motifs ------------------------------------------------------------------------------------------------------
    def m_conv(self):
        r = self.rng
        y = self.conv(self.pick())
        if r.random() < 0.15:                                   # a conv called at two sites
            self.near["two_sites"] += 1
            op, t = self.ops[-1], self.t[y]
            self.conv(self.chain(self.call(op["m"], op["x"], t["C"], t["H"], t["W"]), 1))
        self.chain(y)
        if r.random() < 0.15:                                 # a clamp with a second user
            self.near["clamp_two_users"] += 1
            c = self.fn("relu6", self.conv(self.pick()))
            self.conv(c)
            self.mean_tail(c)

    def m_fanout(self):
        src = self.chain(self.conv(self.pick()))
        self.consumers(src, self.rng.randint(2, 4))

    def m_residual(self):
        r = self.rng
        s = self.pick(min_hw=2)
        t = self.t[s]
        stride = r.choice((1, 1, 2))
        cout = t["C"] if stride == 1 and r.random() < 0.5 else r.choice(CHANNELS)
        bad = r.random() < 0.08
        early = r.random() < 0.4 and not bad
        res = None
        if early or (stride == 1 and cout == t["C"] and r.random() < 0.5):
            res = s if stride == 1 and cout == t["C"] else self.conv(s, cout=cout, k=1, s=stride, pad=0, dw=False)
        mid = self.chain(self.conv(s, cout=cout, k=3, s=stride, d=1, pad=1, dw=False), r.choice((0, 1)))
        p = self.conv(mid, cout=cout, k=r.choice((1, 3)), s=1, d=1, pad=None, same=True, dw=False) \
            if r.random() < 0.6 else mid
        a = self.chain(p, r.choice((0, 0, 1)))
        if bad:
            self.near["add_shapes_differ"] += 1
            res = self.conv(s, cout=1, k=1, s=stride, pad=0, dw=False)
        elif res is None:                                       # the downsample, computed after the block
            res = self.conv(s, cout=cout, k=1, s=stride, pad=0, dw=False)
        if r.random() < 0.3:
            res = self.pass_through(res, near=False) if r.random() < 0.5 else self._identity(res)
        form = r.choice(("op", "op", "torch", "method", "alpha", "self"))
        if form == "alpha":
            self.near["add_alpha"] += 1
        if form == "self":
            self.near["add_self"] += 1
        a_, b_ = (a, a) if form == "self" else ((a, res) if r.random() < 0.7 else (res, a))
        self.use(a_, b_)
        self.ops.append(dict(k="add", form=form, a=a_, b=b_))
        ta = self.t[a]
        y = self.new(ta["C"], ta["H"], ta["W"])
        y = self.chain(y, r.choice((0, 1, 1)))
        if r.random() < 0.5:
            self.consumers(y, r.randint(1, 3))

    def _identity(self, src):
        t = self.t[src]
        f = self.rng.choice(("identity", "dropout", "bn"))
        m = self.name(f)
        self.mods[m] = dict(type=f, C=t["C"])
        return self.call(m, src, t["C"], t["H"], t["W"], t["kid"])

    def m_pool(self):
        r = self.rng
        place = r.choice(("producer", "producer", "cat", "pool", "stem"))
        if place == "cat":
            src = self.m_cat(consume=False)
        else:
            src = self.chain(self.conv(self.pick()), r.choice((0, 1)))
        p = self.pool(src)
        if place == "pool":
            p = self.pool(p)
            if r.random() < 0.5:                                # pool -> pool -> cat
                c1 = self.conv(p, cout=16, same=True, dw=False)
                self.use(p, c1)
                self.ops.append(dict(k="cat", xs=[c1, p], dim=1))
                tp = self.t[p]
                y = self.new(16 + tp["C"], tp["H"], tp["W"])
                self.conv(y)
                return
        if r.random() < 0.15:
            self.near["clamp_after_pool"] += 1
            p = self.fn("relu6", p)
        if r.random() < 0.3:
            p = self._identity(p)
        if place == "stem":                                     # the pooled tensor is a residual
            t = self.t[p]
            b = self.chain(self.conv(p, cout=t["C"], k=3, s=1, d=1, pad=1, dw=False), 1)
            c = self.conv(b, cout=t["C"], k=3, s=1, d=1, pad=1, dw=False)
            self.use(c, p)
            self.ops.append(dict(k="add", form="op", a=c, b=p))
            y = self.new(t["C"], t["H"], t["W"])
            self.conv(self.fn("relu_f", y))
            return
        self.consumers(p, r.randint(1, 3))

    def operand(self, H, W, C, last):
        """A cat operand [C, H, W]: a producer's chain, or an upsample of one."""
        r = self.rng
        srcs = [i for i in self.spatial() if (self.t[i]["H"], self.t[i]["W"]) == (H, W)]
        low = [i for i in self.spatial() if self.t[i]["H"] < H or self.t[i]["W"] < W]
        if low and r.random() < 0.5:
            u = self.chain(self.conv(r.choice(low), cout=C, same=True, dw=False), r.choice((0, 1)))
            return u, "up"
        src = r.choice(srcs) if srcs and r.random() < 0.8 else self.pick()
        if (self.t[src]["H"], self.t[src]["W"]) != (H, W):
            return self.upsample(self.conv(src, cout=C, same=True, dw=False), (H, W)), None
        return self.chain(self.conv(src, cout=C, same=True, dw=False), r.choice((0, 0, 1))), None

    def upsample(self, src, size, ref=None, near=False):
        r, t = self.rng, self.t[src]
        ac = r.random() < 0.5
        mode = "bilinear"
        form = "const" if ref is None else r.choice(("shape", "size"))
        op = dict(k="up", x=src, size=list(size), ref=ref, form=form, ac=ac, mode=mode)
        if near and r.random() < 0.25:
            if near == "nearest" or r.random() < 0.5:
                self.near["up_nearest"] += 1
                op.update(mode="nearest", ac=None)
            else:
                self.near["up_scale_factor"] += 1
                op.update(form="scale", sf=2)
                size = (t["H"] * 2, t["W"] * 2)
        self.use(src)
        if ref is not None and form != "scale":
            self.use(ref)
        self.ops.append(op)
        return self.new(t["C"], size[0], size[1])

    def m_cat(self, consume=True):
        r = self.rng
        base = self.pick()
        H, W = self.t[base]["H"], self.t[base]["W"]
        n = r.randint(2, 4)
        chans = [r.choice((16, 32, 48)) for _ in range(n - 1)] + [r.choice(CHANNELS)]
        if r.random() < 0.1:
            self.near["cat_unaligned"] += 1
            chans[0] = r.choice((5, 17, 24))
        xs, ups = [], []
        for j, C in enumerate(chans):
            x, up = self.operand(H, W, C, j == n - 1)
            xs.append(x)
            ups.append(up)
        for j, up in enumerate(ups):                            # upsample to a constant size or to another operand's
            if up:
                others = [x for jj, x in enumerate(xs) if jj != j and not ups[jj]]
                ref = r.choice(others) if others and r.random() < 0.7 else None
                xs[j] = self.upsample(xs[j], (H, W), ref, near="nearest")
        dim = r.choice((1, 1, -3))
        if r.random() < 0.08:
            self.near["cat_same_node"] += 1
            if self.t[xs[0]]["C"] % 16 == 0:
                xs.insert(0, xs[0])
            else:
                xs.append(xs[-1])
        if r.random() < 0.06:                                   # along the height: a cat of equal-channel operands
            self.near["cat_dim2"] += 1
            xs = [xs[0], self.conv(xs[0], cout=self.t[xs[0]]["C"], same=True, dw=False)]
            dim = 2
        self.use(*xs)
        self.ops.append(dict(k="cat", xs=xs, dim=dim))
        C = sum(self.t[x]["C"] for x in xs) if dim != 2 else self.t[xs[0]]["C"]
        y = self.new(C, H * (2 if dim == 2 else 1), W)
        y = self.chain(y, r.choice((0, 0, 1)))
        if not consume:
            return y
        if r.random() < 0.12:
            self.near["cat_user_other_key"] += 1
            self.conv(y)
            self.conv(y, key=self._nudge(self.key(y, exact=True)))
        else:
            for _ in range(r.choice((1, 1, 2))):
                self.conv(y, key=self.key(y, exact=True))
        return y

    def m_up_codes(self):
        r = self.rng
        src = self.chain(self.conv(self.pick()), r.choice((0, 1)))
        t = self.t[src]
        size = (t["H"] + r.randint(1, 5), t["W"] + r.randint(0, 4))
        refs = [i for i in self.spatial() if (self.t[i]["H"], self.t[i]["W"]) == size]
        u = self.upsample(src, size, r.choice(refs) if refs and r.random() < 0.5 else None, near=True)
        u = self.chain(u, r.choice((0, 1)))
        for _ in range(r.choice((1, 1, 2))):
            self.conv(u, key=self.key(u, exact=r.random() < 0.8))

    def m_pad(self):
        r = self.rng
        src = self.pick()
        if r.random() < 0.4 and self.t[src]["uses"] == 0:      # a fan-out, one of whose users is the pad
            self.conv(src)
        t = self.t[src]
        l, tp = r.choice((0, 1, 2)), r.choice((0, 1, 2))
        op = dict(k="pad", x=src, pad=[l, l, tp, tp] if r.random() < 0.7 else [l, l], mode="constant", value=None)
        near = r.random()
        if near < 0.12:
            self.near["pad_asymmetric"] += 1
            op["pad"] = [l, l + 1, tp, tp]
        elif near < 0.22:
            self.near["pad_nonzero"] += 1
            op["value"] = 0.5
        elif near < 0.3 and min(t["H"], t["W"]) > 2:
            self.near["pad_reflect"] += 1
            op.update(mode="reflect", pad=[1, 1, 1, 1])
        elif near < 0.4:
            self.near["zeropad2d"] += 1
            m = self.name("zeropad")
            self.mods[m] = dict(type="zeropad", p=1)
            y = self.call(m, src, t["C"], t["H"] + 2, t["W"] + 2)
            self.conv(y, pad=0, s=1)
            return
        pad = op["pad"] + [0, 0]
        self.use(src)
        self.ops.append(op)
        y = self.new(t["C"], t["H"] + pad[2] + pad[3], t["W"] + pad[0] + pad[1])
        k = r.choice((1, 3))
        pad_own = 0 if self.scheme == "affine" or r.random() < 0.7 else 1
        if k == 3 and self.t[y]["H"] + 2 * pad_own < 3 or self.t[y]["W"] + 2 * pad_own < 3:
            k = 1
        self.conv(y, k=k, d=1, pad=pad_own)
        if near >= 0.4 and r.random() < 0.3:
            self.near["pad_two_users"] += 1
            self.mean_tail(y)

    def m_heads(self):
        r = self.rng
        k = r.choice((2, 4, 6))
        n = r.randint(2, 3)
        parts, bad = [], r.random() < 0.15
        for j in range(n):
            src = self.pick()
            h = self.conv(src, cout=k * r.choice((1, 2, 3)), same=True, dw=False)
            if r.random() < 0.3:
                h = self.fn("relu6", h)
            if bad and j == n - 1:
                self.near["head_not_a_head"] += 1
                h = self.pool(h)
            self.t[h]["head"] = True                            # no other user: a head's operand chain is single-user
            form = r.choice(("contiguous_view", "contiguous_reshape", "reshape"))
            nform = "const" if r.random() < 0.3 else r.choice(("size0", "shape0"))
            parts.append(dict(x=h, k=k, form=form, n=nform))
            self.use(h)
        self.ops.append(dict(k="heads", parts=parts, batch=self.batch))
        i = self.new(None, None, None)
        self.t[i] = dict(rows=k, uses=0, kid=None)
        if self.rng.random() < 0.7:
            self.use(i)
            self.ops.append(dict(k="softmax", x=i))
            self.t.append(dict(rows=k, uses=0, kid=None))

    def run(self):
        r = self.rng
        motifs = [(self.m_conv, 3), (self.m_fanout, 3), (self.m_residual, 3), (self.m_pool, 3), (self.m_cat, 4),
                  (self.m_up_codes, 2), (self.m_pad, 3), (self.m_heads, 4)]
        self.conv(0, cout=r.choice((16, 24, 32)), k=3, same=True, dw=False)
        for _ in range(r.randint(3, 6)):
            f = r.choices([m for m, _ in motifs], [w for _, w in motifs])[0]
            f()
        if self.scheme == "affine" and r.random() < 0.3:        # an ncnn layer, opaque to chain_affine
            src = self.pick()
            m = self.name("ncnn")
            self.mods[m] = dict(type="ncnn_conv", cin=self.t[src]["C"], cout=16, key=float(f32(r.choice(NCNN_KEYS))))
            y = self.call(m, src, 16, self.t[src]["H"], self.t[src]["W"])
            self.conv(y)
        if r.random() < 0.4:
            self.mean_tail(self.pick())
        outs = [i for i, t in enumerate(self.t) if t["uses"] == 0 and i > 0]
        return dict(seed=self.seed, scheme=self.scheme, batch=self.batch, input=[3, self.t[0]["H"], self.t[0]["W"]],
                    mods=self.mods, ops=self.ops, outs=outs, near=dict(self.near))


def program(seed, scheme):
    """The op list of graph `seed` under `scheme` ("ncnn" or "affine"): a dict of modules, ops, outputs and near misses."""
    assert scheme in ("ncnn", "affine")
    return _Gen(seed, scheme).run()


# ---- the module ----------------------------------------------------------------------------------------------------------
def _module(spec, scheme, gen):
    t = spec["type"]
    if t == "conv":
        if scheme == "affine":
            return _qconv(spec, gen)
        c = nn.Conv2d(spec["cin"], spec["cout"], spec["k"], spec["s"], spec["p"], spec["d"], spec["groups"])
        with torch.no_grad():
            c.bias.normal_(0, 0.3, generator=gen)
        return c
    if t == "linear":
        if scheme == "affine":
            return _qlinear(spec, gen)
        return nn.Linear(spec["cin"], spec["cout"])
    if t == "ncnn_conv":
        from dfq_b200 import int8
        c = nn.Conv2d(spec["cin"], spec["cout"], 3, 1, 1)
        return int8.Int8Conv2d.from_conv(c, spec["key"], 128. / float(c.weight.detach().abs().max()))
    if t == "relu_mod":
        return nn.ReLU()
    if t == "relu6":
        return nn.ReLU6()
    if t == "hardtanh":
        return nn.Hardtanh(spec["lo"], spec["hi"])
    if t == "identity":
        return nn.Identity()
    if t in ("dropout", "dropout_train"):
        m = nn.Dropout(0.0)
        return m.train() if t == "dropout_train" else m.eval()
    if t in ("bn", "bn_bad"):
        from dfq_b200.utils.layer_transform import _identity_bn_eps
        bn = nn.BatchNorm2d(spec["C"]).eval()
        bn.eps = _identity_bn_eps()
        if t == "bn_bad":
            with torch.no_grad():
                bn.running_mean.normal_(0, 0.2, generator=gen)
                bn.weight.uniform_(0.5, 1.5, generator=gen)
        return bn
    if t == "maxpool":
        return nn.MaxPool2d(spec["k"], spec["s"], spec["p"], spec["d"], ceil_mode=spec["ceil"])
    if t == "zeropad":
        return nn.ZeroPad2d(spec["p"])
    raise ValueError(t)


def _qconv(spec, gen):
    import int8_affine_oracle as A
    from dfq_b200.utils import quantize as Q
    c = Q.QuantNConv2d(spec["cin"], spec["cout"], spec["k"], spec["s"], spec["p"], spec["d"], spec["groups"])
    return _quantized(c, spec, gen, A)


def _qlinear(spec, gen):
    import int8_affine_oracle as A
    from dfq_b200.utils import quantize as Q
    return _quantized(Q.QuantNLinear(spec["cin"], spec["cout"]), spec, gen, A)


def _quantized(c, spec, gen, A):
    lo, hi, bits = spec["key"]
    with torch.no_grad():
        c.weight.copy_(torch.from_numpy(A.fake_quant_weights(c.weight.numpy(), 8)))
        c.bias.normal_(0, 0.2, generator=gen)
    c.quant.running_min.fill_(lo)
    c.quant.running_max.fill_(hi)
    c.quant.num_bits = bits
    return c


class ChainNet(nn.Module):
    """The model of a program: its modules as attributes, its ops interpreted by forward."""

    def __init__(self, prog):
        super().__init__()
        torch.manual_seed(prog["seed"])
        gen = torch.Generator().manual_seed(prog["seed"])
        for name, spec in prog["mods"].items():
            self.add_module(name, _module(spec, prog["scheme"], gen))
        self.ops, self.outs = prog["ops"], prog["outs"]

    def forward(self, x):
        t = [x]
        for op in self.ops:
            k = op["k"]
            if k == "heads":
                ys = []
                for p in op["parts"]:
                    y = t[p["x"]].permute(0, 2, 3, 1)
                    if p["form"] != "reshape":
                        y = y.contiguous()
                    n = op["batch"] if p["n"] == "const" else (y.size(0) if p["n"] == "size0" else y.shape[0])
                    ys.append(y.view(n, -1, p["k"]) if p["form"] == "contiguous_view" else y.reshape(n, -1, p["k"]))
                t.append(torch.cat(ys, 1))
                continue
            if k == "add":
                a, b = t[op["a"]], t[op["b"]]
                if op["form"] in ("op", "self"):
                    t.append(a + b)
                elif op["form"] == "torch":
                    t.append(torch.add(a, b))
                elif op["form"] == "method":
                    t.append(a.add(b))
                else:
                    t.append(torch.add(a, b, alpha=1))
                continue
            if k == "cat":
                t.append(torch.cat([t[i] for i in op["xs"]], op["dim"]))
                continue
            x = t[op["x"]]
            if k == "mod":
                t.append(getattr(self, op["m"])(x))
            elif k == "relu_f":
                t.append(F.relu(x))
            elif k == "relu_t":
                t.append(torch.relu(x))
            elif k == "relu_m":
                t.append(x.relu())
            elif k == "relu6":
                t.append(F.relu6(x))
            elif k == "hardtanh":
                t.append(F.hardtanh(x, op["lo"], op["hi"]))
            elif k == "pool":
                t.append(F.max_pool2d(x, op["ks"], op["s"], op["p"], op["d"], ceil_mode=op["ceil"]))
            elif k == "mean":
                t.append(torch.mean(x, (2, 3)))
            elif k == "softmax":
                t.append(F.softmax(x, -1))
            elif k == "pad":
                t.append(F.pad(x, op["pad"], mode=op["mode"], value=op["value"]))
            elif k == "up":
                if op["form"] == "scale":
                    t.append(F.interpolate(x, scale_factor=op["sf"], mode=op["mode"], align_corners=op["ac"]))
                else:
                    size = tuple(op["size"]) if op["form"] == "const" else \
                        (t[op["ref"]].shape[-2:] if op["form"] == "shape" else t[op["ref"]].size()[2:])
                    t.append(F.interpolate(x, size=size, mode=op["mode"], align_corners=op["ac"]))
            else:
                raise ValueError(k)
        outs = tuple(t[i] for i in self.outs)
        return outs[0] if len(outs) == 1 else outs


def build(prog):
    """The nn.Module (eval mode but for its training-mode near misses) of a program; the affine scheme's convolutions are
    QuantNConv2d layers with fake-quantized weights and their keys as observer ranges, ready for convert_affine."""
    net = ChainNet(prog).eval()
    for name, spec in prog["mods"].items():
        if spec["type"] == "dropout_train":
            getattr(net, name).train()
    return net


def act_scales(prog):
    """{module name: act_scale} of an ncnn program's Conv2d / Linear layers."""
    return {n: s["key"] for n, s in prog["mods"].items() if s["type"] in ("conv", "linear")}


def observer_ranges(prog, n):
    """n (min, max) ranges for the functional-op observers of the evaluation state, drawn per program."""
    r = random.Random(prog["seed"] * 7 + 3)
    return [r.choice(OBSERVER_RANGES) for _ in range(n)]


def inputs(prog, batch=None):
    """A seeded input [N, 3, H, W]: finite, some values past every range (saturation), exact zeros and -0.0."""
    g = torch.Generator().manual_seed(prog["seed"] + 11)
    x = torch.randn(batch or prog["batch"], *prog["input"], generator=g) * 2.5
    flat = x.view(-1)
    idx = torch.randperm(flat.numel(), generator=g)
    k = max(1, flat.numel() // 16)
    flat[idx[:k]] = -0.0
    flat[idx[k:2 * k]] = 0.0
    flat[idx[2 * k:3 * k]] *= 20
    return x


def describe(prog):
    """The program as readable Python: its modules and a forward, with the near misses it holds."""
    lines = ["# seed %d, scheme %s, input [%d, %s], near misses %s" % (prog["seed"], prog["scheme"], prog["batch"],
                                                                        ", ".join(map(str, prog["input"])), prog["near"])]
    for n, s in prog["mods"].items():
        lines.append("self.%s = %s(%s)" % (n, s["type"], ", ".join("%s=%r" % kv for kv in s.items() if kv[0] != "type")))
    lines.append("def forward(self, t0):")
    i = 1
    for op in prog["ops"]:
        k = op["k"]
        if k == "heads":
            parts = ["t%d.permute(0, 2, 3, 1)%s.%s(%s, -1, %d)" % (
                p["x"], "" if p["form"] == "reshape" else ".contiguous()", "view" if p["form"] == "contiguous_view"
                else "reshape", op["batch"] if p["n"] == "const" else ("_.size(0)" if p["n"] == "size0" else "_.shape[0]"),
                p["k"]) for p in op["parts"]]
            rhs = "torch.cat([%s], 1)" % ", ".join(parts)
        elif k == "add":
            rhs = {"op": "t%d + t%d", "self": "t%d + t%d", "torch": "torch.add(t%d, t%d)", "method": "t%d.add(t%d)",
                   "alpha": "torch.add(t%d, t%d, alpha=1)"}[op["form"]] % (op["a"], op["b"])
        elif k == "cat":
            rhs = "torch.cat([%s], %d)" % (", ".join("t%d" % x for x in op["xs"]), op["dim"])
        elif k == "mod":
            rhs = "self.%s(t%d)" % (op["m"], op["x"])
        elif k == "pool":
            rhs = "F.max_pool2d(t%d, %d, %d, %d, %d, ceil_mode=%s)" % (op["x"], op["ks"], op["s"], op["p"], op["d"], op["ceil"])
        elif k == "hardtanh":
            rhs = "F.hardtanh(t%d, %r, %r)" % (op["x"], op["lo"], op["hi"])
        elif k == "pad":
            rhs = "F.pad(t%d, %r, mode=%r, value=%r)" % (op["x"], tuple(op["pad"]), op["mode"], op["value"])
        elif k == "up":
            size = "scale_factor=%r" % op.get("sf") if op["form"] == "scale" else "size=%s" % (
                str(tuple(op["size"])) if op["form"] == "const" else
                "t%d.shape[-2:]" % op["ref"] if op["form"] == "shape" else "t%d.size()[2:]" % op["ref"])
            rhs = "F.interpolate(t%d, %s, mode=%r, align_corners=%r)" % (op["x"], size, op["mode"], op["ac"])
        else:
            rhs = {"relu_f": "F.relu(t%d)", "relu_t": "torch.relu(t%d)", "relu_m": "t%d.relu()", "relu6": "F.relu6(t%d)",
                   "mean": "torch.mean(t%d, (2, 3))", "softmax": "F.softmax(t%d, -1)"}[k] % op["x"]
        lines.append("    t%d = %s" % (i, rhs))
        i += 1
    lines.append("    return %s" % ", ".join("t%d" % o for o in prog["outs"]))
    return "\n".join(lines)


# ---- chaining a program and checking the result --------------------------------------------------------------------------
NCNN_FLAGS = (dict(), dict(residual=True), dict(residual=True, pool_cat=True),
              dict(residual=True, pool_cat=True, upsample=True),
              dict(residual=True, pool_cat=True, upsample=True, layout=True))
AFFINE_FLAGS = (dict(), dict(residual=True), dict(residual=True, concat=True), dict(residual=True, pools=True),
                dict(residual=True, fold_pads=True), dict(residual=True, heads=True),
                dict(residual=True, concat=True, pools=True, fold_pads=True, heads=True))
# the entries that run a convolution layer, and those of them that run a chained layer's output mode
CONV_ENTRIES = ("dfq_i8_conv", "dfq_i8_conv_requant", "dfq_i8_conv_fused", "dfq_i8_conv_slice", "dfq_i8_conv_nhwc",
                "dfq_i8_affine_conv", "dfq_i8_affine_conv_fused", "dfq_i8_affine_conv_observed",
                "dfq_i8_affine_conv_layout", "dfq_i8_affine_conv_rows")
MODE_ENTRIES = CONV_ENTRIES[1:5] + CONV_ENTRIES[6:]
RECORD_KINDS = ("edge", "add", "pool_codes", "pool_fp32", "cat", "up_slice", "up_codes", "folded_pad", "head",
                "obs_operand", "obs_residual", "obs_output", "obs_cat", "obs_head", "obs_tail")


class CountingLib:
    """The library dfq_b200._lib.load() returns, each dfq_* entry's name appended to `calls` when it is called."""

    def __init__(self, lib):
        self.lib, self.calls = lib, []

    def __getattr__(self, name):
        f = getattr(self.lib, name)
        if not name.startswith("dfq_") or not callable(f):
            return f

        def call(*a, **k):
            self.calls.append(name)
            return f(*a, **k)
        return call


def count_launches(monkeypatch):
    """Route dfq_b200._lib.load() through a CountingLib (after any host twin is installed); returns its call list."""
    from dfq_b200 import _lib
    load = _lib.load
    calls = []

    def counted(build_if_missing=True):
        lib = CountingLib(load(build_if_missing))
        lib.calls = calls
        return lib
    monkeypatch.setattr(_lib, "load", counted)
    return calls


def _is_pass_through(n, mods):
    """chain_int8's pass-throughs, restated from its docstring: identity eval BN, ReLU / ReLU6 / Hardtanh in their module and
    functional forms, Identity, eval Dropout."""
    if len(n.all_input_nodes) != 1 or not n.args or n.args[0] is not n.all_input_nodes[0]:
        return False
    if n.op == "call_module":
        m = mods[n.target]
        if type(m) is nn.BatchNorm2d:
            return not m.training and bool((m.running_mean == 0).all() and (m.running_var == 1).all() and
                                           (m.weight == 1).all() and (m.bias == 0).all()) and f32(1) + f32(m.eps) == f32(1)
        return type(m) in (nn.ReLU, nn.ReLU6, nn.Hardtanh, nn.Identity) or (type(m) is nn.Dropout and not m.training)
    if n.op == "call_function":
        return n.target in (F.relu, torch.relu, F.relu6, F.hardtanh)
    return n.op == "call_method" and n.target == "relu"


def base_edges(graph, mods, layer):
    """The edges of the first paragraph of chain_int8's docstring, from the traced per-layer graph: P -> single-user
    pass-throughs -> Q, P and Q `layer` modules called at one site, every node from P to Q with one user."""
    sites = collections.Counter(n.target for n in graph.nodes if n.op == "call_module")

    def conv(n):
        return n.op == "call_module" and isinstance(mods[n.target], layer) and sites[n.target] == 1

    edges = set()
    for q in graph.nodes:
        if not conv(q) or len(q.args) != 1 or q.kwargs or not isinstance(q.args[0], torch.fx.Node):
            continue
        n = q.args[0]
        while len(n.users) == 1:
            if conv(n):
                if len(n.args) == 1 and mods[n.target].out_channels == mods[q.target].in_channels:
                    edges.add((n.target, q.target))
                break
            if not _is_pass_through(n, mods):
                break
            n = n.args[0]
    return edges


def first_user_keys(graph, mods, layer, key):
    """{producer: key of its first consumer in graph order} for each single-site `layer` producer whose single-user
    pass-through chain ends at a fan-out of single-site `layer` convolutions and torch.mean only: the fan-out rule's key,
    at which its codes consumers must read."""
    sites = collections.Counter(n.target for n in graph.nodes if n.op == "call_module")

    def conv(n):
        return n.op == "call_module" and isinstance(mods[n.target], layer) and sites[n.target] == 1 and n.args and \
            len(n.args) == 1 and not n.kwargs

    firsts = {}
    for p in graph.nodes:
        if not conv(p):
            continue
        tail = p
        while len(tail.users) == 1 and _is_pass_through(next(iter(tail.users)), mods):
            tail = next(iter(tail.users))
        users = list(tail.users)                                # graph order
        if len(users) < 2 or not all((conv(u) and u.args[0] is tail) or (u.op == "call_function" and u.target is torch.mean)
                                     for u in users):
            continue
        first = next((u for u in users if conv(u)), None)
        if first is not None:
            firsts[p.target] = key(mods[first.target])
    return firsts


def record_counts(gm):
    """Counter of the records of a chained module, by RECORD_KINDS."""
    c = collections.Counter()
    c["edge"] += len(gm.requantized_edges)
    c["add"] += len(getattr(gm, "fused_adds", ()))
    for _, mode, _ in getattr(gm, "fused_pools", ()):
        c["pool_" + mode] += 1
    c["cat"] += len(getattr(gm, "fused_cats", ()))
    for _, _, mode, _ in getattr(gm, "fused_upsamples", ()):
        c["up_" + mode] += 1
    c["folded_pad"] += len(getattr(gm, "folded_pads", ()))
    c["head"] += len(getattr(gm, "fused_heads", ()))
    for _, kind, _ in getattr(gm, "fused_observers", ()):
        c["obs_" + kind] += 1
    return c


def check_records(gm, names, floor, flags, firsts=None, key=None):
    """Assertion 2 and 3: every recorded name is a node of the traced graph or a module of the model; the layers reading
    codes are exactly the edges' consumers; nothing deleted is left or referenced; the base edges are all there."""
    from dfq_b200 import int8
    edges = gm.requantized_edges
    recorded = [n for p, q, _ in edges for n in (p, q)]
    recorded += [n for r in getattr(gm, "fused_adds", ()) for n in r[:3]]
    recorded += [n for c, ws, _ in getattr(gm, "fused_cats", ()) for n in (c, *ws)]
    recorded += [r[0] for r in getattr(gm, "fused_pools", ())]
    recorded += [n for r in getattr(gm, "fused_upsamples", ()) for n in r[:2]]
    recorded += [n for r in getattr(gm, "folded_pads", ()) for n in r[:2]]
    recorded += [n for c, ps, _ in getattr(gm, "fused_heads", ()) for n in (c, *ps)]
    recorded += [n for o, _, p in getattr(gm, "fused_observers", ()) for n in (o, p)]
    assert set(recorded) <= names, set(recorded) - names
    consumers = {id(gm.get_submodule(q)) for _, q, _ in edges if isinstance(gm.get_submodule(q), int8._ConvLayer)}
    codes_in = {id(m) for m in gm.modules() if isinstance(m, int8._ConvLayer) and m.codes_in}
    assert consumers == codes_in
    nodes = list(gm.graph.nodes)
    present = set(nodes)
    gm.graph.lint()
    for n in nodes:
        assert all(a in present for a in n.all_input_nodes), n
    deleted = [r[1] for r in getattr(gm, "fused_adds", ())] + [r[0] for r in getattr(gm, "fused_cats", ())] + \
        [r[0] for r in getattr(gm, "folded_pads", ())] + [r[0] for r in getattr(gm, "fused_heads", ())]
    assert not set(deleted) & {n.name for n in nodes}
    got = {(p, q) for p, q, _ in edges}
    if flags.get("residual"):
        assert floor <= got, floor - got
        for p, q, _ in edges:                                   # the fan-out's codes go at its first user's key
            if p in (firsts or {}):
                assert key(gm.get_submodule(q)) == firsts[p], (p, q)
    else:
        assert got == floor


def check_launches(gm, calls):
    """Each chained layer launches once per forward, in one entry of its mode; every layer call site launches once."""
    from dfq_b200 import int8
    layers = [m for m in gm.modules() if isinstance(m, int8._ConvLayer)]
    moded = [m for m in layers if m.epilogue is not None or m.out_slice is not None or m.rows or
             getattr(m, "requant", None) is not None or getattr(m, "pad_code", None) is not None]
    sites = sum(isinstance(gm.get_submodule(n.target), int8._ConvLayer) for n in gm.graph.nodes if n.op == "call_module")
    sites += sum(len(m.heads) for m in gm.modules() if isinstance(m, int8.Int8HeadConcat))
    assert sum(calls.count(e) for e in MODE_ENTRIES) == len(moded)
    assert sum(calls.count(e) for e in CONV_ENTRIES) == sites


def same(a, b):
    """Bit identity of two outputs (tensors or tuples of them), as int32 patterns."""
    if isinstance(a, (tuple, list)):
        return isinstance(b, (tuple, list)) and len(a) == len(b) and all(same(u, v) for u, v in zip(a, b))
    return a.dtype == b.dtype == torch.float32 and a.shape == b.shape and \
        torch.equal(a.detach().cpu().view(torch.int32), b.detach().cpu().view(torch.int32))


def _shapes_differ_error(prog, gm, err):
    """True when err is the DfqError of a fused add whose operands differ in shape (a near miss the program holds)."""
    from dfq_b200 import _lib
    return isinstance(err, _lib.DfqError) and "residual must be" in str(err) and \
        prog["near"].get("add_shapes_differ") and getattr(gm, "fused_adds", None)


def _affine_graph(model):
    from dfq_b200.utils import quantize as Q
    return collections.OrderedDict((id(m), m) for m in model.modules() if isinstance(m, (Q.QuantNConv2d, Q.QuantNLinear)))


def verify(prog, model, x, save_dir, mp, patch=lambda: None, observed=True):
    """Chain the per-layer `model` of `prog` (built on x's device) at every flag set of its scheme - the affine scheme also
    in the reference's evaluation state when `observed` - save and load each chained module, then, after patch() (the host
    twins' setup; for the affine scheme before it all), check each against the per-layer model bit for bit, with its
    records (check_records), launches (check_launches) and saved copy.  mp: a pytest MonkeyPatch.  Returns the Counter of records, by RECORD_KINDS."""
    import affine_observed_state
    import pytest
    from dfq_b200 import _lib, int8
    from test_int8_affine_observe_host import _state
    affine = prog["scheme"] == "affine"
    records = None
    if affine:                                                  # an opaque ncnn layer runs in the recording forward
        patch()
        records = affine_observed_state.record_ops(model, x) if observed else None
        from dfq_b200.utils import quantize as Q
        int8.convert_affine(model, _affine_graph(model), [Q.QuantNConv2d, Q.QuantNLinear])
        chain, flag_sets, layer = int8.chain_affine, AFFINE_FLAGS, int8.AffineInt8Conv2d
    else:
        graph = collections.OrderedDict((id(m), m) for m in model.modules() if type(m) in (nn.Conv2d, nn.Linear))
        names = {id(m): n for n, m in model.named_modules()}
        scales = act_scales(prog)
        int8.convert_to_int8(model, graph, [nn.Conv2d, nn.Linear], act_scales=[scales[names[k]] for k in graph])
        chain, flag_sets, layer = int8.chain_int8, NCNN_FLAGS, int8.Int8Conv2d
    traced = int8._Int8Tracer().trace(model)
    mods = dict(model.named_modules())
    floor = base_edges(traced, mods, layer)
    key = (lambda m: (f32(m.act_min).tobytes(), f32(m.act_max).tobytes(), m.act_bits)) if affine else \
        (lambda m: f32(m.act_scale).tobytes())
    firsts = first_user_keys(traced, mods, layer, key)
    before = {n: (m, m.codes_in, m.epilogue, m.out_slice, m.padding) for n, m in mods.items()
              if isinstance(m, int8._ConvLayer)}
    n_obs = sum(int(r[1].split("_")[-1]) for r in records) if records else 0
    ranges = observer_ranges(prog, n_obs)
    chained = []
    for flags in flag_sets:
        chained.append((flags, False, chain(model, **flags)))
    if records:
        with _state(model, records, ranges) as ct:
            for flags in flag_sets:
                chained.append((flags, True, chain(model, **flags)))
            assert ct.idx_name_tensor_op == 0 and ct.idx_tensor_op == 0
    names = {n.name for n in traced.nodes} | set(dict(model.named_modules()))
    loaded = []
    for i, (flags, obs, gm) in enumerate(chained):
        check_records(gm, names, floor, flags, firsts, key)
        path = save_dir / ("chain%d.pt" % i)
        if prog["near"].get("zeropad2d"):                      # a module type save() does not hold: refused
            with pytest.raises(_lib.DfqError, match="ZeroPad2d"):
                int8.save(gm, path)
            loaded.append(None)
            continue
        int8.save(gm, path)
        loaded.append(int8.load(path))
    after = {n: (m, m.codes_in, m.epilogue, m.out_slice, m.padding) for n, m in model.named_modules()
             if isinstance(m, int8._ConvLayer)}
    assert after == before                                      # the per-layer model is left as it was
    if not affine:                                              # after save / load: chain_int8 traces torch's interpolate
        patch()
    calls = count_launches(mp)
    counts = collections.Counter()

    def run_all(obs):
        with torch.no_grad():
            ref = model(x)
            for (flags, o, gm), m in zip(chained, loaded):
                if o != obs:
                    continue
                calls.clear()
                try:
                    y = gm(x)
                except Exception as e:                          # a fused add whose operands differ in shape
                    assert _shapes_differ_error(prog, gm, e), (flags, obs, e)
                    continue
                assert same(y, ref), (flags, obs)
                check_launches(gm, calls)
                assert m is None or same(m(x), y), (flags, obs, "loaded")
                counts.update(record_counts(gm))
    run_all(False)
    if records:
        with _state(model, records, ranges):
            run_all(True)
    return counts
