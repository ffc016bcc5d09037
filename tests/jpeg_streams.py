"""The crafted JPEG corpus of the decoder's tests: streams tests/jpeg_writer.py writes from chosen coefficients, each
decodable by Pillow and each reaching a path that Pillow- and OpenCV-encoded streams never reach - reconstructions far
outside 0 .. 255, Huffman codes of every length 1 .. 16, coefficient runs ending on index 63, ZRL chains, DC values that
wrap int16, restart intervals of every shape, chroma planes 1 .. 17 samples wide, and uncommon but valid headers.

    streams() -> [(name, bytes)]          # each entry asserts, as it is built, that it reaches its path

tests/golden/jpeg_crafted.npz holds the SHA-256 of Pillow's decode of every entry (`python tests/jpeg_streams.py`
rewrites it); a libjpeg-turbo build that decodes them otherwise fails as a fixture mismatch.
"""
import functools
import hashlib
import os

import numpy as np

import jpeg_oracle as O
import jpeg_writer as JW

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg_crafted.npz")
GEOMETRY = [1, 2, 3, 4, 5, 6, 15, 16, 17, 18, 31, 32, 33, 34]


def _zeros(sampling, h, w):
    hs, vs = JW.SAMPLING[sampling]
    mx, my = -(-w // (8 * hs)), -(-h // (8 * vs))
    planes = [np.zeros((my * vs, mx * hs, 64), np.int64)]
    if sampling != "gray":
        planes += [np.zeros((my, mx, 64), np.int64) for _ in range(2)]
    return planes


def _random(g, sampling, h, w, dc=60, ac=12, density=0.25):
    """Moderate random blocks: DC within +-dc, a share of AC coefficients within +-ac."""
    planes = _zeros(sampling, h, w)
    for p in planes:
        p[..., 0] = g.integers(-dc, dc + 1, p.shape[:2])
        p[..., 1:] = g.integers(-ac, ac + 1, p.shape[:2] + (63,)) * (g.random(p.shape[:2] + (63,)) < density)
    return planes


def _trace(w, planes_written=None):
    """The oracle's IDCT trace over every block of the stream: (shortcut, pass1, out), blocks of all planes stacked."""
    _, planes = O.coefficients(w.data)
    b = np.concatenate([p.reshape(-1, 64) for p in planes])
    t = {}
    O.idct_islow(b, t)
    return b, t


def _q(v):
    return np.full(64, v, np.int64)


# ---- reconstructions outside 0 .. 255 ---------------------------------------------------------------------------------
def _overshoot(sampling, seed):
    g = np.random.default_rng(seed)
    h, w = 24, 40
    planes = _random(g, sampling, h, w, dc=1100, ac=300, density=0.08)
    for p in planes:                                             # DC-only blocks, so pass 1's shortcut sees large DCs
        p.reshape(-1, 64)[::3, 1:] = 0
    wr = JW.write(planes, height=h, width=w, sampling=sampling, qtables=[_q(16), _q(12)])
    _, t = _trace(wr)
    v = t["out"]
    for lim in (384, 512, 1024):
        assert (v > lim).any() and (v < -lim).any(), (sampling, lim)
    assert (np.abs(t["pass1"]) > 32767).any()                     # pass 1 saturates
    return wr.data


def _shortcut_wrap():
    """DC-only blocks whose dc << PASS1_BITS leaves int16 (the shortcut wraps where the full pass saturates), and 16-bit
    quantisers whose products with the coefficients leave int16 (dequantisation wraps)."""
    planes = _zeros("gray", 16, 32)
    b = planes[0].reshape(-1, 64)
    b[:, 0] = [1000, -1000, 2047, -2047, 1500, 300, -700, 64]
    b[4:, 9] = [5, -3, 1, 2]
    q = np.full(64, 20, np.int64)
    q[0], q[9] = 9, 30001
    wr = JW.write(planes, height=16, width=32, qtables=[q], qbits=16)
    c, t = _trace(wr)
    assert (np.abs(c) > 32767).any()
    assert t["shortcut"][:4].all() and (np.abs(O.wrap16(c[:4, 0]) * 4) > 32767).all()
    return wr.data


# ---- Huffman codes of every length ------------------------------------------------------------------------------------
_DC_EVERY = (bytes([1] * 16), bytes(range(16)))                  # category c coded in c + 1 bits
_AC_SYMS = [0x00, 0x01, 0x02, 0x03, 0x04, 0x05, 0x06, 0x07, 0x08, 0x09, 0x0A, 0x11, 0x21, 0xF0, 0x0F, 0x3B]
_AC_EVERY = (bytes([1] * 16), bytes(_AC_SYMS))                   # _AC_SYMS[l - 1] coded in l bits


def _block_of(dc, syms):
    """A natural-order block from DC and [(run, size)] AC symbols (the value of size s: 2^(s-1), signs alternating)."""
    blk = np.zeros(64, np.int64)
    blk[0] = dc
    k = 0
    for i, (r, s) in enumerate(syms):
        k += r + 1
        blk[JW.ZIGZAG[k]] = (1 << (s - 1)) * (1 if i % 2 else -1)
    return blk


def _scan_order(p, hs, vs):
    """The (row, column) of a plane's blocks in scan order (MCU by MCU, hs x vs blocks each)."""
    my, mx = p.shape[0] // vs, p.shape[1] // hs
    return [(y * vs + dy, x * hs + dx) for y in range(my) for x in range(mx) for dy in range(vs) for dx in range(hs)]


def _every_length(sampling, seed):
    g = np.random.default_rng(seed)
    h, w = 16, 128
    hs, vs = JW.SAMPLING[sampling]
    planes = _zeros(sampling, h, w)
    ac_runs = [[(0, s)] for s in range(1, 11)] + [[(1, 1)], [(2, 1)], [(16, 1)], [(0, 15)], [(3, 11)]]
    pos = 0
    for c, p in enumerate(planes):
        prev = 0
        for r, x in _scan_order(p, hs, vs) if c == 0 else _scan_order(p, 1, 1):
            cat = (pos * 7) % 16                                  # DC differences of every category, in scan order
            diff = 0 if cat == 0 else int(g.choice([-1, 1])) * int(g.integers(1 << (cat - 1), 1 << cat))
            if abs(prev + diff) > 30000:
                diff = -diff
            prev += diff
            p[r, x] = _block_of(prev, ac_runs[pos % len(ac_runs)] + ac_runs[(pos + 3) % len(ac_runs)][:1])
            pos += 1
    huff = {(0, 0): _DC_EVERY, (1, 0): _AC_EVERY, (0, 1): _DC_EVERY, (1, 1): _AC_EVERY}
    wr = JW.write(planes, height=h, width=w, sampling=sampling, qtables=[_q(1)], huff=huff)
    for key in ((0, 0), (1, 0)):
        assert wr.lengths[key] == set(range(1, 17)), (key, sorted(wr.lengths[key]))
    return wr.data


def _optimal(maxlen, seed):
    """Tables built from the scan's statistics, folded to at most maxlen bits."""
    g = np.random.default_rng(seed)
    planes = _random(g, "420", 40, 40, dc=400, ac=200, density=0.4)
    wr = JW.write(planes, height=40, width=40, sampling="420", qtables=[_q(2), _q(3)], maxlen=maxlen)
    assert max(max(v) for v in wr.lengths.values()) == maxlen
    return wr.data


# ---- coefficient runs ---------------------------------------------------------------------------------------------------
def _runs():
    planes = _zeros("gray", 8, 8 * 48)
    b = planes[0].reshape(-1, 64)
    b[0, JW.ZIGZAG[63]] = 5                                       # 3 ZRL, then run 14 onto index 63: no EOB
    b[1, JW.ZIGZAG[[47, 63]]] = [3, -2]                           # run 15 landing on 63
    b[2, JW.ZIGZAG[1:64]] = np.arange(1, 64) % 7 - 3 + (np.arange(1, 64) % 7 == 3)   # dense up to 63
    b[3, JW.ZIGZAG[[1, 40]]] = [1, 1]                             # 2 ZRL then run 6
    b[4:, 0] = [2047 * k for k in range(44)]                      # differences of +2047 until the block value wraps
    wr = JW.write(planes, height=8, width=8 * 48, qtables=[_q(1)])
    assert 0xF0 in wr.symbols[(1, 0)] and 0x00 in wr.symbols[(1, 0)]
    c = O.coefficients(wr.data, dequantise=False)[1][0].reshape(-1, 64)
    assert (c[0] != 0).sum() == 1 and c[0, JW.ZIGZAG[63]] == 5 and c[1, JW.ZIGZAG[63]] == -2
    assert (c[5:, 1:] == 0).all()                                 # EOB right after DC
    assert (b[4:, 0] > 32767).any() and (c[:, 0] == O.wrap16(b[:, 0])).all()
    return wr.data


# ---- restart intervals ----------------------------------------------------------------------------------------------------
def _restart(sampling, h, w, ri, fill, seed):
    g = np.random.default_rng(seed)
    planes = _random(g, sampling, h, w)
    wr = JW.write(planes, height=h, width=w, sampling=sampling, qtables=[_q(4), _q(5)], ri=ri, fill=fill)
    mcus = planes[-1].shape[0] * planes[-1].shape[1]
    assert wr.intervals == -(-mcus // ri)
    assert wr.data.count(b"\xff" * (fill + 1) + b"\xd9") == 1
    return wr.data, mcus


def _restarts():
    out = []
    mcus = _restart("422", 24, 80, 1, 0, 0)[1]
    assert mcus == 15
    for ri, fill in ((1, 0), (1, 2), (15, 0), (16, 1), (40, 0), (4, 0), (7, 3), (2, 1)):
        data, _ = _restart("422", 24, 80, ri, fill, ri * 10 + fill)
        out.append(("rst_422_ri%d_fill%d" % (ri, fill), data))
    for sampling, h, w, ri in (("gray", 40, 72, 10), ("420", 33, 50, 3), ("444", 17, 70, 9)):
        data, n = _restart(sampling, h, w, ri, 1, ri)
        assert n // ri >= 1
        out.append(("rst_%s_ri%d" % (sampling, ri), data))
    return out


# ---- geometry -------------------------------------------------------------------------------------------------------------
def _geometry():
    out = []
    for sampling in ("422", "420"):
        for k, w in enumerate(GEOMETRY):
            for h in (GEOMETRY[k], GEOMETRY[-1 - k], GEOMETRY[(k + 5) % len(GEOMETRY)]):
                g = np.random.default_rng(h * 100 + w)
                planes = _random(g, sampling, h, w, dc=100, ac=20)
                out.append(("geo_%s_%dx%d" % (sampling, h, w),
                            JW.write(planes, height=h, width=w, sampling=sampling, qtables=[_q(6), _q(8)]).data))
        for h in GEOMETRY:
            for w in (2, 4, 5):                                  # chroma widths 1, 2 and 3 at every height
                g = np.random.default_rng(h * 7 + w)
                planes = _random(g, sampling, h, w, dc=100, ac=20)
                out.append(("geo_%s_%dx%d" % (sampling, h, w),
                            JW.write(planes, height=h, width=w, sampling=sampling, qtables=[_q(6), _q(8)]).data))
    return list(dict(out).items())


# ---- headers --------------------------------------------------------------------------------------------------------------
def _headers():
    out = []
    cases = {"sof1": dict(sof=0xC1), "ids_012": dict(ids=[0, 1, 2]), "split_tables": dict(group=False),
             "tables_after_sof": dict(tables_after_sof=True), "redefined": dict(redefine=True, tables_after_sof=True),
             "redefined_before_sof": dict(redefine=True), "app_com": dict(extras=True, seed=3),
             "everything": dict(sof=0xC1, ids=[0, 1, 2], group=False, tables_after_sof=True, redefine=True,
                                extras=True, ri=3, fill=1, seed=4)}
    for k, (name, kw) in enumerate(cases.items()):
        g = np.random.default_rng(50 + k)
        planes = _random(g, "420", 20, 28, dc=200, ac=40)
        wr = JW.write(planes, height=20, width=28, sampling="420", qtables=[_q(3), _q(5)], **kw)
        if kw.get("sof") == 0xC1:
            assert b"\xff\xc1" in wr.data and b"\xff\xc0" not in wr.data
        if not kw.get("group", True):
            assert wr.data.count(b"\xff\xdb") == 2 * (1 + kw.get("redefine", False))
        out.append(("hdr_" + name, wr.data))
    g = np.random.default_rng(60)
    planes = _random(g, "444", 16, 24, dc=300, ac=60)
    q16 = [np.arange(64) * 37 + 200, np.arange(64)[::-1] * 41 + 300]
    wr = JW.write(planes, height=16, width=24, sampling="444", qtables=q16, qbits=16)
    assert b"\xff\xdb" in wr.data and max(q16[0].max(), q16[1].max()) > 255
    out.append(("hdr_dqt16", wr.data))
    return out


@functools.lru_cache(maxsize=1)
def _all():
    out = [("overshoot_%s" % s, _overshoot(s, k)) for k, s in enumerate(("gray", "444", "422", "420"))]
    out.append(("shortcut_and_dequant_wrap", _shortcut_wrap()))
    out += [("codes_every_length_%s" % s, _every_length(s, k)) for k, s in enumerate(("gray", "420"))]
    out += [("codes_optimal_max%d" % m, _optimal(m, m)) for m in (8, 9, 10)]
    out.append(("runs_zrl_63_dc_wrap", _runs()))
    out += _restarts() + _geometry() + _headers()
    names = [n for n, _ in out]
    assert len(set(names)) == len(names)
    return tuple(out)


def streams():
    """[(name, bytes)] of the crafted corpus."""
    return list(_all())


def sha256(a):
    return hashlib.sha256(np.ascontiguousarray(a, np.uint8).tobytes()).hexdigest()


def fixture():
    """{name: SHA-256 of Pillow's RGB decode}."""
    z = np.load(FIXTURE)
    return dict(zip(z["names"].tolist(), z["sha256"].tolist()))


if __name__ == "__main__":
    import jpeg_corpus as JC
    s = streams()
    np.savez_compressed(FIXTURE, names=np.array([n for n, _ in s]), sha256=np.array([sha256(JC.pillow(d)) for _, d in s]))
    print("%d streams -> %s" % (len(s), FIXTURE))
