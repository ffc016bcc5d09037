"""A numpy / Python restatement of libjpeg-turbo's baseline decode, as Pillow and OpenCV run it: Huffman decoding with
restart markers, dequantisation, jpeg_idct_islow (CONST_BITS 13, PASS1_BITS 2, the masked range-limit table), "fancy"
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
            frame = (H, W, comps, dict(q))
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


def coefficients(data):
    """(frame, int64 coefficient planes per component [by, bx, 64] in natural order, padded to whole MCUs)."""
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
        planes.append(b * q[c[3]][None, None, :])
        j += hv
    return (H, W, comps, hm, vm), planes


# ---- jpeg_idct_islow ---------------------------------------------------------------------------------------------------
F = dict(c0_298=2446, c0_390=3196, c0_541=4433, c0_765=6270, c0_899=7373, c1_175=9633, c1_501=12299, c1_847=15137,
         c1_961=16069, c2_053=16819, c2_562=20995, c3_072=25172)


def _idct_1d(x0, x1, x2, x3, x4, x5, x6, x7):
    z2, z3 = x2, x6
    z1 = (z2 + z3) * F["c0_541"]
    tmp2 = z1 + z3 * -F["c1_847"]
    tmp3 = z1 + z2 * F["c0_765"]
    tmp0 = (x0 + x4) << 13
    tmp1 = (x0 - x4) << 13
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    tmp0, tmp1, tmp2, tmp3 = x7, x5, x3, x1
    z1, z2, z3, z4 = tmp0 + tmp3, tmp1 + tmp2, tmp0 + tmp2, tmp1 + tmp3
    z5 = (z3 + z4) * F["c1_175"]
    tmp0, tmp1, tmp2, tmp3 = tmp0 * F["c0_298"], tmp1 * F["c2_053"], tmp2 * F["c3_072"], tmp3 * F["c1_501"]
    z1, z2, z3, z4 = z1 * -F["c0_899"], z2 * -F["c2_562"], z3 * -F["c1_961"], z4 * -F["c0_390"]
    z3 += z5
    z4 += z5
    tmp0 += z1 + z3
    tmp1 += z2 + z4
    tmp2 += z2 + z3
    tmp3 += z1 + z4
    return [t10 + tmp3, t11 + tmp2, t12 + tmp1, t13 + tmp0, t13 - tmp0, t12 - tmp1, t11 - tmp2, t10 - tmp3]


def _range_limit(v):
    """range_limit[v & RANGE_MASK] of the post-IDCT table (CENTERJSAMPLE already in the table)."""
    m = v & 1023
    return np.where(m < 128, m + 128, np.where(m < 512, 255, np.where(m < 896, 0, m - 896))).astype(np.uint8)


def idct_islow(blocks):
    """blocks: int64 [..., 64] dequantised, natural order -> uint8 [..., 8, 8]."""
    b = blocks.reshape(-1, 8, 8)                     # [n, row(u), col]
    cols = _idct_1d(*[b[:, k, :] for k in range(8)])          # pass 1 over columns: each [n, col]
    ws = np.stack([(c + (1 << 10)) >> 11 for c in cols], 1)         # DESCALE(x, CONST_BITS - PASS1_BITS): [n, row, col]
    rows = _idct_1d(*[ws[:, :, k] for k in range(8)])        # pass 2 over rows: each [n, row]
    out = np.stack([_range_limit((r + (1 << 17)) >> 18) for r in rows], 2)   # DESCALE(x, CONST_BITS + PASS1_BITS + 3)
    return out.reshape(blocks.shape[:-1] + (8, 8))


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
