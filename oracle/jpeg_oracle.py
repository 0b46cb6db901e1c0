"""jpeg_oracle -- numpy restatement of the baseline JPEG decode that `PIL.Image.open(...).convert("RGB")` performs
(Pillow 12.2 with libjpeg-turbo, third-party code the reference reaches and does not pin). TEST INFRASTRUCTURE ONLY.

Restated from the algorithms, not from any source file: marker parsing and Huffman decoding (ITU-T T.81), the
integer "slow" inverse DCT (Loeffler-Ligtenberg-Moschytz, 13-bit constants, 2 extra bits kept between the passes),
the triangle-filter chroma upsampling and the 16-bit fixed-point YCbCr -> RGB conversion that the library's defaults
select. tests/test_jpeg_decode_cpu.py pins `decode` to Pillow bit for bit; csrc/jpeg_decode.cuh implements the same
arithmetic for the host (entropy stage) and the device (everything after it).

Rules settled here against Pillow's pixels:
* a component's "row above the first" and "row below the last" are that row itself, where "last" is the last row of
  the component's true (unpadded) downsampled size ceil(size * v / vmax); likewise the first and last *true* columns
  take the one-sided form of the filter, so samples in the MCU padding never reach the output;
* the triangle filter is used only when the downsampled width exceeds 2; narrower components are replicated;
* the shortcut the library takes for blocks / columns without AC terms gives the value of the full butterfly, so the
  restatement (and the kernel) has no data-dependent branch;
* an overshoot after the IDCT saturates to 0..255 (the library's SIMD path; seen on streams with damaged coefficients);
* the library's SIMD IDCT keeps products and the values between its passes in 16-bit lanes. `parse` therefore refuses
  (Corrupt) any block whose sum of |dequantised coefficient| over a column exceeds MAX_COLUMN_SUM, as the host stage of
  the product does: below it the 64-bit arithmetic here and the 16-bit lanes agree, above it only Pillow knows;
* Huffman tables are validated as the library does (no all-ones code of a used length, DC symbols <= 15), and the
  stream must end in EOI right after the last scan: Pillow raises on the others."""
import numpy as np

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,
                   6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38,
                   31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])           # zigzag position -> natural (row-major) index

GREY, YCBCR, RGB = 0, 1, 2
MAX_COLUMN_SUM = 2800


class Unsupported(ValueError):
    """a stream outside the supported subset (progressive, arithmetic, 12-bit, CMYK, other sampling factors)"""


class Corrupt(ValueError):
    """a truncated or damaged stream"""


def _fix(x, bits):
    return int(x * (1 << bits) + 0.5)


class _Huff(object):
    """16-bit look-ahead table: code prefix -> (length, symbol); length 0 marks an invalid code"""

    def __init__(self, counts, symbols):
        self.length = [0] * 65536
        self.symbol = [0] * 65536
        code, k = 0, 0
        maxlen = max([ln for ln in range(1, 17) if counts[ln - 1]] or [0])
        for ln in range(1, 17):
            for _ in range(counts[ln - 1]):
                if code >= (1 << ln):
                    raise Corrupt("Huffman table over-subscribed")
                lo = code << (16 - ln)
                for j in range(lo, lo + (1 << (16 - ln))):
                    self.length[j] = ln
                    self.symbol[j] = symbols[k]
                code += 1
                k += 1
            if ln <= maxlen and code >= (1 << ln):
                raise Corrupt("Huffman table uses an all-ones code")
            code <<= 1


def _segments(data, pos):
    """entropy-coded bytes from `pos`: (list of de-stuffed restart segments, list of the RSTn numbers between them,
    position of the marker that ends the scan or len(data))"""
    segs, rst, cur = [], [], bytearray()
    n = len(data)
    while True:
        j = data.find(b"\xff", pos)
        if j < 0 or j + 1 >= n:
            cur += data[pos:] if j < 0 else data[pos:j]
            segs.append(bytes(cur))
            return segs, rst, n
        cur += data[pos:j]
        m = data[j + 1]
        if m == 0:
            cur.append(0xFF)
            pos = j + 2
        elif m == 0xFF:                                   # fill byte in front of a marker
            pos = j + 1
        elif 0xD0 <= m <= 0xD7:
            segs.append(bytes(cur))
            rst.append(m - 0xD0)
            cur = bytearray()
            pos = j + 2
        else:
            segs.append(bytes(cur))
            return segs, rst, j


class _Bits(object):
    def __init__(self, seg):
        self.buf = seg + b"\0\0\0\0"
        self.nbits = len(seg) * 8
        self.p = 0

    def peek16(self):
        i = self.p >> 3
        return (int.from_bytes(self.buf[i:i + 3], "big") >> (8 - (self.p & 7))) & 0xFFFF

    def decode(self, h):
        v = self.peek16()
        ln = h.length[v]
        if ln == 0:
            raise Corrupt("invalid Huffman code")
        self.p += ln
        return h.symbol[v]

    def receive_extend(self, s):
        if s == 0:
            return 0
        i = self.p >> 3
        v = (int.from_bytes(self.buf[i:i + 4], "big") >> (32 - (self.p & 7) - s)) & ((1 << s) - 1)
        self.p += s
        return v if v >= (1 << (s - 1)) else v - (1 << s) + 1


def parse(data):
    """encoded bytes -> descriptor dict: width, height, ncomp, hmax, vmax, color, mcus_x, mcus_y and, per component,
    `h`, `v`, `dw`, `dh` (true downsampled size), `bw`, `bh` (block grid padded to whole MCUs), `quant` (uint16 [64],
    natural order, as latched when the component's scan started) and `coef` (int16 [bh * bw, 64], natural order, DC
    prediction undone)"""
    data = bytes(data)
    n = len(data)
    if n < 4 or data[0] != 0xFF or data[1] != 0xD8:
        raise Corrupt("no SOI")
    pos = 2
    qt, dc_t, ac_t = {}, {}, {}
    frame = None
    restart = 0
    jfif = False
    adobe = None
    done = set()
    while True:
        if pos >= n or data[pos] != 0xFF:                 # a marker must follow at once (fill bytes aside)
            raise Corrupt("no marker where one is due")
        while pos < n and data[pos] == 0xFF:
            pos += 1
        if pos >= n:
            raise Corrupt("stream ends before every component was decoded")
        m = data[pos]
        pos += 1
        if m == 0xD9:
            raise Corrupt("EOI before every component was decoded")
        if m < 0xC0 or m in (0xD8, 0xDE, 0xDF) or 0xD0 <= m <= 0xD7 or 0xF0 <= m < 0xFE:
            raise Corrupt("reserved or misplaced marker 0x%02X" % m)
        if pos + 2 > n:
            raise Corrupt("truncated segment")
        ln = (data[pos] << 8) | data[pos + 1]
        if ln < 2 or pos + ln > n:
            raise Corrupt("truncated segment")
        seg = data[pos + 2:pos + ln]
        pos += ln
        if m == 0xDB:
            i = 0
            while i < len(seg):
                pq, tq = seg[i] >> 4, seg[i] & 15
                i += 1
                if pq > 1 or tq > 3 or i + 64 * (pq + 1) > len(seg):
                    raise Corrupt("bad DQT")
                t = np.zeros(64, np.uint16)
                for k in range(64):
                    t[ZIGZAG[k]] = (seg[i + 2 * k] << 8 | seg[i + 2 * k + 1]) if pq else seg[i + k]
                i += 64 * (pq + 1)
                qt[tq] = t
        elif m == 0xC4:
            i = 0
            while i < len(seg):
                if i + 17 > len(seg):
                    raise Corrupt("bad DHT")
                tc, th = seg[i] >> 4, seg[i] & 15
                counts = list(seg[i + 1:i + 17])
                i += 17
                if tc > 1 or th > 3 or sum(counts) > 256 or i + sum(counts) > len(seg):
                    raise Corrupt("bad DHT")
                if not tc and any(v > 15 for v in seg[i:i + sum(counts)]):
                    raise Corrupt("DC symbol")
                (ac_t if tc else dc_t)[th] = _Huff(counts, list(seg[i:i + sum(counts)]))
                i += sum(counts)
        elif m in (0xC0, 0xC1):
            if frame is not None or len(seg) < 6:
                raise Corrupt("bad SOF")
            if seg[0] != 8:
                raise Unsupported("sample precision %d" % seg[0])
            height, width, nc = seg[1] << 8 | seg[2], seg[3] << 8 | seg[4], seg[5]
            if nc not in (1, 3):
                raise Unsupported("%d components" % nc)
            if len(seg) != 6 + 3 * nc or width == 0 or height == 0:
                raise Corrupt("bad SOF")
            comps = [{"id": seg[6 + 3 * c], "h": seg[7 + 3 * c] >> 4, "v": seg[7 + 3 * c] & 15, "tq": seg[8 + 3 * c]}
                     for c in range(nc)]
            if any(not (1 <= c["h"] <= 4 and 1 <= c["v"] <= 4) for c in comps):
                raise Corrupt("bad SOF")
            if nc == 1:
                comps[0]["h"] = comps[0]["v"] = 1             # a lone component is never interleaved
            elif ((comps[0]["h"], comps[0]["v"]) not in ((1, 1), (2, 1), (2, 2))
                  or any((c["h"], c["v"]) != (1, 1) for c in comps[1:])):
                raise Unsupported("sampling factors")
            if any(c["tq"] > 3 for c in comps) or len(set(c["id"] for c in comps)) != nc:
                raise Corrupt("bad SOF")
            hmax, vmax = comps[0]["h"], comps[0]["v"]
            mx, my = -(-width // (8 * hmax)), -(-height // (8 * vmax))
            for c in comps:
                c["dw"], c["dh"] = -(-width * c["h"] // hmax), -(-height * c["v"] // vmax)
                c["bw"], c["bh"] = mx * c["h"], my * c["v"]
                c["coef"] = np.zeros((c["bh"] * c["bw"], 64), np.int16)
            frame = {"width": width, "height": height, "ncomp": nc, "hmax": hmax, "vmax": vmax, "mcus_x": mx,
                     "mcus_y": my, "comps": comps}
        elif m in (0xC2, 0xC3, 0xC5, 0xC6, 0xC7, 0xC9, 0xCA, 0xCB, 0xCD, 0xCE, 0xCF, 0xCC, 0xC8):
            raise Unsupported("SOF / coding marker 0x%02X" % m)
        elif m == 0xDD:
            if len(seg) != 2:
                raise Corrupt("bad DRI")
            restart = seg[0] << 8 | seg[1]
        elif m == 0xE0:
            jfif = jfif or seg[:5] == b"JFIF\0"
        elif m == 0xEE:
            if seg[:5] == b"Adobe" and len(seg) >= 12:
                adobe = seg[11]
        elif m == 0xDA:
            if frame is None or len(seg) < 1:
                raise Corrupt("SOS before SOF")
            ns = seg[0]
            if ns < 1 or ns > frame["ncomp"] or len(seg) != 4 + 2 * ns:
                raise Corrupt("bad SOS")
            if (seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns]) != (0, 63, 0):
                raise Unsupported("spectral selection / successive approximation")
            scan = []
            for k in range(ns):
                cid, tt = seg[1 + 2 * k], seg[2 + 2 * k]
                idx = [i for i, c in enumerate(frame["comps"]) if c["id"] == cid]
                if not idx or idx[0] in [s[0] for s in scan] or idx[0] in done:
                    raise Corrupt("bad SOS component")
                if (tt >> 4) not in dc_t or (tt & 15) not in ac_t or frame["comps"][idx[0]]["tq"] not in qt:
                    raise Corrupt("scan uses an undefined table")
                scan.append((idx[0], dc_t[tt >> 4], ac_t[tt & 15]))
            if ns not in (1, frame["ncomp"]):
                raise Unsupported("partially interleaved scan")
            for ci, _, _ in scan:
                frame["comps"][ci]["quant"] = qt[frame["comps"][ci]["tq"]].copy()
            pos = _scan(data, pos, frame, scan, restart)
            done.update(s[0] for s in scan)
            if len(done) == frame["ncomp"]:
                while data[pos:pos + 2] == b"\xff\xff":
                    pos += 1
                if data[pos:pos + 2] != b"\xff\xd9":
                    raise Corrupt("no EOI after the last scan")
                break
        # APPn, COM and anything else with a length: skipped
    nc = frame["ncomp"]
    ids = [c["id"] for c in frame["comps"]]
    if nc == 1:
        frame["color"] = GREY
    elif jfif:
        frame["color"] = YCBCR
    elif adobe is not None:
        frame["color"] = RGB if adobe == 0 else YCBCR
    else:
        frame["color"] = RGB if ids == [ord("R"), ord("G"), ord("B")] else YCBCR
    for c in frame["comps"]:
        lim = np.abs(c["coef"].astype(np.int64) * c["quant"].astype(np.int64)[None, :]).reshape(-1, 8, 8).sum(1).max()
        if lim > MAX_COLUMN_SUM:
            raise Corrupt("coefficients beyond the range in which the library's 16-bit IDCT is reproduced")
    return frame


def _scan(data, pos, frame, scan, restart):
    comps = frame["comps"]
    segs, rst, end = _segments(data, pos)
    if len(scan) == 1:                                    # non-interleaved: the component's own block grid
        c = comps[scan[0][0]]
        mx, my = -(-c["dw"] // 8), -(-c["dh"] // 8)
        units = [(scan[0][0], 0, 0, scan[0][1], scan[0][2])]
        sx = sy = 1
    else:
        mx, my = frame["mcus_x"], frame["mcus_y"]
        units = [(ci, bx, by, d, a) for ci, d, a in scan for by in range(comps[ci]["v"]) for bx in range(comps[ci]["h"])]
        sx = sy = None
    total = mx * my
    nseg = 1 if restart == 0 else -(-total // restart)
    if len(segs) < nseg:
        raise Corrupt("entropy data ends early")
    if any(r != (i & 7) for i, r in enumerate(rst[:nseg - 1])):
        raise Corrupt("restart markers out of sequence")
    mcu = 0
    for s in range(nseg):
        bits = _Bits(segs[s])
        pred = [0, 0, 0]
        for _ in range(total - mcu if restart == 0 else min(restart, total - mcu)):
            my_, mx_ = divmod(mcu, mx)
            for ci, bx, by, dct, act in units:
                c = comps[ci]
                hh, vv = (c["h"], c["v"]) if sx is None else (1, 1)
                blk = c["coef"][(my_ * vv + by) * c["bw"] + mx_ * hh + bx]
                t = bits.decode(dct)
                if t > 15:
                    raise Corrupt("DC category")
                pred[ci] += bits.receive_extend(t)
                blk[0] = np.int16(((pred[ci] + 32768) & 0xFFFF) - 32768)
                k = 1
                while k < 64:
                    rs = bits.decode(act)
                    r, t = rs >> 4, rs & 15
                    if t:
                        k += r
                        if k > 63:
                            raise Corrupt("AC run past the block")
                        blk[ZIGZAG[k]] = bits.receive_extend(t)
                        k += 1
                    elif r == 15:
                        k += 16
                    else:
                        break
                if bits.p > bits.nbits:
                    raise Corrupt("entropy data ends inside a block")
            mcu += 1
    if len(segs) > nseg:                                  # restart markers beyond the last MCU
        raise Corrupt("extra restart markers")
    return end


# ---- everything after the entropy stage: what the device kernels do

C = {k: v for k, v in zip(
    ("c0298", "c0390", "c0541", "c0765", "c0899", "c1175", "c1501", "c1847", "c1961", "c2053", "c2562", "c3072"),
    (2446, 3196, 4433, 6270, 7373, 9633, 12299, 15137, 16069, 16819, 20995, 25172))}       # round(x * 2**13)


def _butterfly(x, shift):
    """one 1-D pass over the last axis of int64 [..., 8]; the result is descaled by `shift` bits with rounding"""
    x0, x1, x2, x3, x4, x5, x6, x7 = (x[..., i] for i in range(8))
    z1 = (x2 + x6) * C["c0541"]
    t2 = z1 - x6 * C["c1847"]
    t3 = z1 + x2 * C["c0765"]
    t0 = (x0 + x4) << 13
    t1 = (x0 - x4) << 13
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    o0, o1, o2, o3 = x7, x5, x3, x1
    z1, z2, z3, z4 = o0 + o3, o1 + o2, o0 + o2, o1 + o3
    z5 = (z3 + z4) * C["c1175"]
    o0, o1, o2, o3 = o0 * C["c0298"], o1 * C["c2053"], o2 * C["c3072"], o3 * C["c1501"]
    z1, z2 = -z1 * C["c0899"], -z2 * C["c2562"]
    z3, z4 = -z3 * C["c1961"] + z5, -z4 * C["c0390"] + z5
    o0, o1, o2, o3 = o0 + z1 + z3, o1 + z2 + z4, o2 + z2 + z3, o3 + z1 + z4
    out = np.stack([t10 + o3, t11 + o2, t12 + o1, t13 + o0, t13 - o0, t12 - o1, t11 - o2, t10 - o3], axis=-1)
    return (out + (1 << (shift - 1))) >> shift


def idct_blocks(coef, quant):
    """int16 [N, 64] natural order, uint16 [64] -> uint8 [N, 8, 8]"""
    x = (coef.astype(np.int64) * quant.astype(np.int64)[None, :]).reshape(-1, 8, 8)
    ws = _butterfly(x.transpose(0, 2, 1), 11).transpose(0, 2, 1)           # columns first, 2 extra bits kept
    return np.clip(_butterfly(ws, 18) + 128, 0, 255).astype(np.uint8)        # rows, +128, saturation


def component_plane(c):
    """uint8 [bh * 8, bw * 8] samples of one component, MCU padding included"""
    px = idct_blocks(c["coef"], c["quant"])
    return px.reshape(c["bh"], c["bw"], 8, 8).transpose(0, 2, 1, 3).reshape(c["bh"] * 8, c["bw"] * 8)


def upsample(plane, dw, dh, hs, vs, width, height):
    """true-size samples plane[:dh, :dw] expanded by (hs, vs) in {1, 2} -> int64 [height, width]"""
    p = plane[:dh, :dw].astype(np.int64)
    if hs == 1 and vs == 1:
        return p[:height, :width]
    if dw <= 2:                                           # too narrow for the triangle filter: replicated
        return np.repeat(np.repeat(p, vs, axis=0), hs, axis=1)[:height, :width]
    if vs == 1:
        left = np.concatenate([p[:, :1], p[:, :-1]], axis=1)
        right = np.concatenate([p[:, 1:], p[:, -1:]], axis=1)
        even = (3 * p + left + 1) >> 2
        odd = (3 * p + right + 2) >> 2
        even[:, 0], odd[:, -1] = p[:, 0], p[:, -1]
        out = np.empty((dh, 2 * dw), np.int64)
        out[:, 0::2], out[:, 1::2] = even, odd
        return out[:height, :width]
    above = np.concatenate([p[:1], p[:-1]], axis=0)
    below = np.concatenate([p[1:], p[-1:]], axis=0)
    rows = np.empty((2 * dh, dw), np.int64)
    rows[0::2], rows[1::2] = 3 * p + above, 3 * p + below
    left = np.concatenate([rows[:, :1], rows[:, :-1]], axis=1)
    right = np.concatenate([rows[:, 1:], rows[:, -1:]], axis=1)
    even = (3 * rows + left + 8) >> 4
    odd = (3 * rows + right + 7) >> 4
    even[:, 0], odd[:, -1] = (4 * rows[:, 0] + 8) >> 4, (4 * rows[:, -1] + 7) >> 4
    out = np.empty((2 * dh, 2 * dw), np.int64)
    out[:, 0::2], out[:, 1::2] = even, odd
    return out[:height, :width]


def ycc_to_rgb(y, cb, cr):
    cb, cr = cb - 128, cr - 128
    r = y + ((_fix(1.40200, 16) * cr + 32768) >> 16)
    g = y + ((-_fix(0.34414, 16) * cb + 32768 - _fix(0.71414, 16) * cr) >> 16)
    b = y + ((_fix(1.77200, 16) * cb + 32768) >> 16)
    return np.clip(np.stack([r, g, b], axis=-1), 0, 255).astype(np.uint8)


def pixels(frame):
    """descriptor with coefficients -> uint8 [H, W, 3], what PIL's .convert("RGB") gives"""
    w, h = frame["width"], frame["height"]
    comps = frame["comps"]
    full = [upsample(component_plane(c), c["dw"], c["dh"], frame["hmax"] // c["h"], frame["vmax"] // c["v"], w, h)
            for c in comps]
    if frame["color"] == GREY:
        return np.repeat(full[0][..., None], 3, axis=-1).astype(np.uint8)
    if frame["color"] == RGB:
        return np.stack(full, axis=-1).astype(np.uint8)
    return ycc_to_rgb(*full)


def decode(data):
    return pixels(parse(data))
