"""A numpy / Python restatement of libjpeg-turbo's baseline decode, as Pillow and OpenCV run it: Huffman decoding with
restart markers, dequantisation and the islow IDCT as the x86 SIMD jsimd_idct_islow computes it (16-bit dequantisation
and lane sums, pass 1 saturated to int16, the output saturated; not the C jidctint.c's masked range-limit table), "fancy"
h2v1 / h2v2 chroma upsampling (plain replication when the chroma plane is 2 samples wide or less) and ycc_rgb_convert's
16-bit fixed-point tables.  Independent of dfq_b200.jpeg: it parses the markers itself.  Test infrastructure only.

    decode(data) -> uint8 [H, W, 3], equal to np.asarray(Image.open(BytesIO(data)).convert("RGB"))
"""
import numpy as np

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,
                   7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31,
                   39, 46, 53, 60, 61, 54, 47, 55, 62, 63])        # zigzag index -> natural index


class Corrupt(Exception):
    pass


def _segments(data):
    """(markers dict, frame, scan, entropy bytes).  Only the baseline subset the product takes."""
    assert data[:2] == b"\xff\xd8"
    pos, q, h, frame, ri = 2, {}, {}, None, 0
    while True:
        while data[pos] != 0xFF:
            pos += 1
        while data[pos] == 0xFF:
            pos += 1
        m = data[pos]
        pos += 1
        ln = int.from_bytes(data[pos:pos + 2], "big")
        body = data[pos + 2:pos + ln]
        pos += ln
        if m == 0xDB:
            i = 0
            while i < len(body):
                pq, tq = body[i] >> 4, body[i] & 15
                n = 128 if pq else 64
                vals = np.frombuffer(body[i + 1:i + 1 + n], ">u2" if pq else np.uint8).astype(np.int64)
                t = np.zeros(64, np.int64)
                t[ZIGZAG] = vals
                q[tq] = t
                i += 1 + n
        elif m == 0xC4:
            i = 0
            while i < len(body):
                tc, th = body[i] >> 4, body[i] & 15
                counts = list(body[i + 1:i + 17])
                vals = list(body[i + 17:i + 17 + sum(counts)])
                h[(tc, th)] = _huff_lookup(counts, vals)
                i += 17 + sum(counts)
        elif m in (0xC0, 0xC1):
            H, W, nc = int.from_bytes(body[1:3], "big"), int.from_bytes(body[3:5], "big"), body[5]
            comps = [(body[6 + 3 * k], body[7 + 3 * k] >> 4, body[7 + 3 * k] & 15, body[8 + 3 * k]) for k in range(nc)]
            frame = (H, W, comps, q)       # the tables as SOS finds them: libjpeg latches them per scan
        elif m == 0xDD:
            ri = int.from_bytes(body[:2], "big")
        elif m == 0xDA:
            ns = body[0]
            sel = {body[1 + 2 * k]: (body[2 + 2 * k] >> 4, body[2 + 2 * k] & 15) for k in range(ns)}
            return frame, sel, h, ri, data[pos:]


def _huff_lookup(counts, vals):
    """65536-entry table: the next 16 bits -> (code length, symbol); length 0 for no code."""
    look = [(0, 0)] * 65536
    code, k = 0, 0
    for l in range(1, 17):
        for _ in range(counts[l - 1]):
            lo = code << (16 - l)
            look[lo:lo + (1 << (16 - l))] = [(l, vals[k])] * (1 << (16 - l))
            code += 1
            k += 1
        code <<= 1
    return look


def _unstuff(ent):
    """Split the entropy-coded bytes at RSTn into intervals with the stuffing removed; stop at the first other marker."""
    parts, cur, i = [], bytearray(), 0
    while i < len(ent):
        b = ent[i]
        if b == 0xFF:
            j = i + 1
            while j < len(ent) and ent[j] == 0xFF:
                j += 1
            if j < len(ent) and ent[j] == 0:
                cur.append(0xFF)
                i = j + 1
                continue
            if j < len(ent) and 0xD0 <= ent[j] <= 0xD7:
                parts.append(bytes(cur))
                cur = bytearray()
                i = j + 1
                continue
            break
        cur.append(b)
        i += 1
    parts.append(bytes(cur))
    return parts


def _decode_interval(buf, mcus, layout, tables, coef, blk0):
    """Huffman-decode `mcus` MCUs from one restart interval into coef (natural order), starting at block blk0."""
    nbits = len(buf) * 8
    buf = buf + b"\x00\x00\x00\x00"
    pos, pred, blk = 0, {}, blk0

    def peek16(p):
        b = p >> 3
        return (int.from_bytes(buf[b:b + 3], "big") >> (8 - (p & 7))) & 0xFFFF

    def bits(p, s):
        b = p >> 3
        return (int.from_bytes(buf[b:b + 4], "big") >> (32 - (p & 7) - s)) & ((1 << s) - 1)

    for _ in range(mcus):
        for ci in layout:
            dct, act = tables[ci]
            l, s = dct[peek16(pos)]
            if l == 0:
                raise Corrupt("bad DC code")
            pos += l
            diff = 0
            if s:
                r = bits(pos, s)
                pos += s
                diff = r if r >= (1 << (s - 1)) else r - (1 << s) + 1
            v = (pred.get(ci, 0) + diff)
            v = (v + 2 ** 31) % 2 ** 32 - 2 ** 31
            pred[ci] = v
            row = coef[blk]
            row[0] = (v + 32768) % 65536 - 32768
            k = 1
            while k < 64:
                l, rs = act[peek16(pos)]
                if l == 0:
                    raise Corrupt("bad AC code")
                pos += l
                r, s = rs >> 4, rs & 15
                if s:
                    k += r
                    if k > 63:
                        raise Corrupt("run past 63")
                    v = bits(pos, s)
                    pos += s
                    row[ZIGZAG[k]] = v if v >= (1 << (s - 1)) else v - (1 << s) + 1
                elif r == 15:
                    k += 15
                else:
                    break
                k += 1
            blk += 1
    if pos > nbits:
        raise Corrupt("scan ends before its last MCU")


def coefficients(data, dequantise=True):
    """(frame, int64 coefficient planes per component [by, bx, 64] in natural order, padded to whole MCUs): the int16
    block values times the quantisation table, or as the scan codes them with dequantise=False."""
    (H, W, comps, q), sel, h, ri, ent = _segments(data)
    nc = len(comps)
    if nc == 1:
        hm = vm = 1
        comps = [(comps[0][0], 1, 1, comps[0][3])]
    else:
        hm, vm = max(c[1] for c in comps), max(c[2] for c in comps)
    mx, my = -(-W // (8 * hm)), -(-H // (8 * vm))
    layout = [k for k, c in enumerate(comps) for _ in range(c[1] * c[2])]
    per = len(layout)
    coef = np.zeros((mx * my * per, 64), np.int64)
    tables = [(h[(0, sel[c[0]][0])], h[(1, sel[c[0]][1])]) for c in comps]
    total = mx * my
    parts = _unstuff(ent)
    step = ri if ri else total
    if len(parts) < -(-total // step):
        raise Corrupt("missing restart intervals")
    for k in range(-(-total // step)):
        _decode_interval(parts[k], min(step, total - k * step), layout, tables, coef, k * step * per)
    planes = []
    cm = coef.reshape(my, mx, per, 64)
    j = 0
    for c in comps:
        hv = c[1] * c[2]
        b = cm[:, :, j:j + hv].reshape(my, mx, c[2], c[1], 64).transpose(0, 2, 1, 3, 4).reshape(my * c[2], mx * c[1], 64)
        planes.append(b * q[c[3]][None, None, :] if dequantise else b.copy())
        j += hv
    return (H, W, comps, hm, vm), planes


# ---- jsimd_idct_islow ---------------------------------------------------------------------------------------------------
F = dict(c0_298=2446, c0_390=3196, c0_541=4433, c0_765=6270, c0_899=7373, c1_175=9633, c1_501=12299, c1_847=15137,
         c1_961=16069, c2_053=16819, c2_562=20995, c3_072=25172)


def wrap16(x):
    return ((x + (1 << 15)) & 0xFFFF) - (1 << 15)


def wrap32(x):
    return ((x + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)


def _idct_1d(x0, x1, x2, x3, x4, x5, x6, x7):
    """One pass of jsimd_idct_islow on int16 inputs, before the descale: the 16-bit lane sums x0 + x4, x0 - x4,
    x7 + x3 and x5 + x1 wrap (paddw / psubw), every other sum is formed in 32 bits (pmaddwd, paddd), modulo 2^32."""
    tmp3 = x2 * (F["c0_541"] + F["c0_765"]) + x6 * F["c0_541"]
    tmp2 = x2 * F["c0_541"] + x6 * (F["c0_541"] - F["c1_847"])
    tmp0 = wrap16(x0 + x4) << 13
    tmp1 = wrap16(x0 - x4) << 13
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    z3, z4 = wrap16(x7 + x3), wrap16(x5 + x1)
    z3, z4 = (z3 * (F["c1_175"] - F["c1_961"]) + z4 * F["c1_175"],
              z3 * F["c1_175"] + z4 * (F["c1_175"] - F["c0_390"]))
    tmp0 = x7 * (F["c0_298"] - F["c0_899"]) + x1 * -F["c0_899"] + z3
    tmp3 = x7 * -F["c0_899"] + x1 * (F["c1_501"] - F["c0_899"]) + z4
    tmp1 = x5 * (F["c2_053"] - F["c2_562"]) + x3 * -F["c2_562"] + z4
    tmp2 = x5 * -F["c2_562"] + x3 * (F["c3_072"] - F["c2_562"]) + z3
    return [t10 + tmp3, t11 + tmp2, t12 + tmp1, t13 + tmp0, t13 - tmp0, t12 - tmp1, t11 - tmp2, t10 - tmp3]


def _descale(v, n):
    """paddd of the rounding constant and psrad: in 32 bits, wrapping."""
    return wrap32(v + (1 << (n - 1))) >> n


def idct_islow(blocks, trace=None):
    """blocks: int64 [..., 64] dequantised (exact products), natural order -> uint8 [..., 8, 8].  A trace dict receives
    the per-block facts the crafted streams assert: "shortcut" (pass 1's DC-only path taken), "pass1" (pass 1 before its
    saturation, [n, 8, 8]) and "out" (pass 2 before the output limit, [n, 8, 8]).

    libjpeg-turbo's SIMD jsimd_idct_islow (the SSE2 and AVX2 kernels compute the same): the dequantised value is the
    low 16 bits of coefficient x quantiser (pmullw); a block whose rows 1 .. 7 are all zero takes pass 1's shortcut,
    (dc << PASS1_BITS) in 16 bits (psllw, wrapping); otherwise pass 1 saturates its results to int16 (packssdw);
    pass 2 saturates to int8 (packssdw, packsswb) and adds CENTERJSAMPLE.  Within the range of well-behaved streams
    this equals jidctint.c; outside it, jidctint.c's masked range-limit table wraps where this saturates."""
    shape = blocks.shape[:-1]
    b = blocks.reshape(-1, 8, 8)                     # [n, row(u), col]
    d = wrap16(b)
    cols = _idct_1d(*[d[:, k, :] for k in range(8)])          # pass 1 over columns: each [n, col]
    p1 = np.stack([_descale(c, 11) for c in cols], 1)         # DESCALE(, CONST_BITS - PASS1_BITS): [n, row, col]
    ws = np.clip(p1, -32768, 32767)
    dc_only = ~b[:, 1:, :].any(axis=(1, 2))
    ws[dc_only] = wrap16(d[dc_only, :1, :] << 2)
    rows = _idct_1d(*[ws[:, :, k] for k in range(8)])        # pass 2 over rows: each [n, row]
    out = np.stack([_descale(r, 18) for r in rows], 2)        # DESCALE(, CONST_BITS + PASS1_BITS + 3)
    if trace is not None:
        trace.update(shortcut=dc_only, pass1=p1, out=out)
    return (np.clip(out, -128, 127) + 128).astype(np.uint8).reshape(shape + (8, 8))


def _plane(blocks):
    by, bx = blocks.shape[:2]
    return idct_islow(blocks).transpose(0, 2, 1, 3).reshape(by * 8, bx * 8).astype(np.int64)


# ---- upsampling and colour -----------------------------------------------------------------------------------------------
def _fancy_h2v1(c, dw):
    c = c[:, :dw]
    left = np.concatenate([c[:, :1], c[:, :-1]], 1)
    right = np.concatenate([c[:, 1:], c[:, -1:]], 1)
    out = np.empty((c.shape[0], 2 * dw), np.int64)
    out[:, 0::2] = (3 * c + left + 1) >> 2
    out[:, 1::2] = (3 * c + right + 2) >> 2
    return out


def _fancy_h2v2(c, dw, dh):
    c = c[:dh, :dw]
    above = np.concatenate([c[:1], c[:-1]], 0)
    below = np.concatenate([c[1:], c[-1:]], 0)
    out = np.empty((2 * dh, 2 * dw), np.int64)
    for r, near in ((0, above), (1, below)):
        cs = 3 * c + near
        left = np.concatenate([cs[:, :1], cs[:, :-1]], 1)
        right = np.concatenate([cs[:, 1:], cs[:, -1:]], 1)
        out[r::2, 0::2] = (3 * cs + left + 8) >> 4
        out[r::2, 1::2] = (3 * cs + right + 7) >> 4
    return out


def _fix(x):
    return int(x * (1 << 16) + 0.5)


def ycc_to_rgb(y, cb, cr):
    x_cr, x_cb = cr - 128, cb - 128
    r = y + ((_fix(1.40200) * x_cr + (1 << 15)) >> 16)
    g = y + ((-_fix(0.34414) * x_cb + (1 << 15) + -_fix(0.71414) * x_cr) >> 16)
    b = y + ((_fix(1.77200) * x_cb + (1 << 15)) >> 16)
    return np.stack([np.clip(v, 0, 255) for v in (r, g, b)], -1).astype(np.uint8)


def decode(data):
    """uint8 [H, W, 3]: what Image.open(...).convert("RGB") and cv2.imdecode + cvtColor(BGR2RGB) give."""
    (H, W, comps, hm, vm), planes = coefficients(bytes(data))
    return reconstruct(H, W, hm, vm, planes)


def reconstruct(H, W, hm, vm, planes):
    """uint8 [H, W, 3] from the dequantised coefficient planes ([by, bx, 64] per component, luma sampling hm x vm)."""
    p = [_plane(b) for b in planes]
    if len(p) == 1:
        y = p[0][:H, :W]
        return np.repeat(y[:, :, None].astype(np.uint8), 3, 2)
    up = []
    for c in p[1:]:
        dw, dh = -(-W * 1 // hm), -(-H * 1 // vm)          # downsampled_width / _height of a 1x1 chroma component
        if hm == 1 and vm == 1:
            u = c
        elif dw <= 2:
            u = np.repeat(np.repeat(c[:dh, :dw], vm, 0), hm, 1)
        elif vm == 1:
            u = _fancy_h2v1(c, dw)
        else:
            u = _fancy_h2v2(c, dw, dh)
        up.append(u[:H, :W])
    return ycc_to_rgb(p[0][:H, :W], up[0], up[1])
