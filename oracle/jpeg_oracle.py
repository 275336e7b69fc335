"""A numpy restatement of the baseline JPEG decode that Image.open(f).convert('RGB' | 'L') performs through libjpeg-turbo, stage
by stage, without PIL: the header parse, Huffman decode to quantised coefficients, the `islow` integer IDCT with its range
limit, fancy (triangle-filter) upsampling, the fixed-point YCbCr -> RGB tables and PIL's ITU-R 601 luma.  Written from ITU-T
T.81 and the algorithm descriptions; tests/golden/jpeg.npz (oracle/gen_golden_jpeg.py) pins it to what Pillow decodes.

Each stage is a function of its own so a mismatch of csrc/jpeg.cu can be localised: parse() -> entropy() -> idct() ->
upsample() -> colour().  decode() runs them all.
"""
import numpy as np


class JpegError(ValueError):
    """An unsupported or malformed stream, refused before decoding (the reason is the library's wording)."""


# STATUS codes of a corrupt entropy-coded segment (csrc/jpeg.cu writes the same per image)
OK, TRUNCATED, BAD_CODE, BAD_RUN, BAD_RESTART = 0, 1, 2, 3, 4
STATUS_TEXT = {TRUNCATED: "entropy-coded data truncated", BAD_CODE: "invalid Huffman code",
               BAD_RUN: "AC coefficient run past the end of the block", BAD_RESTART: "restart marker missing or out of sequence"}


def _natural_order():
    out = []
    for s in range(15):
        rows = range(min(s, 7), max(0, s - 7) - 1, -1) if s % 2 == 0 else range(max(0, s - 7), min(s, 7) + 1)
        out += [r * 8 + (s - r) for r in rows]
    return np.array(out, np.int64)


NATURAL = _natural_order()          # NATURAL[k]: row-major index of the k-th coefficient in zig-zag order

_SOF_REFUSED = {0xC2: "progressive JPEG (SOF2)", 0xC3: "lossless JPEG (SOF3)", 0xC5: "hierarchical JPEG (SOF5)",
                0xC6: "hierarchical JPEG (SOF6)", 0xC7: "hierarchical JPEG (SOF7)", 0xC9: "arithmetic-coded JPEG (SOF9)",
                0xCA: "arithmetic-coded JPEG (SOF10)", 0xCB: "arithmetic-coded JPEG (SOF11)", 0xCD: "arithmetic-coded JPEG (SOF13)",
                0xCE: "arithmetic-coded JPEG (SOF14)", 0xCF: "arithmetic-coded JPEG (SOF15)", 0xDE: "hierarchical JPEG (DHP)",
                0xCC: "arithmetic-coded JPEG (DAC)"}


def parse(data):
    """Markers up to the first SOS -> dict: width, height, comps [(id, h, v, tq, td, ta)], quant {tq: int64[64] natural order},
    dc / ac {slot: (bits[16], values)}, restart (MCUs), scan (byte offset of the entropy-coded segment) and colour ('gray',
    'ycc').  Raises JpegError for everything the decoder refuses."""
    b = bytes(data)
    n = len(b)
    if n < 4 or b[0] != 0xFF or b[1] != 0xD8:
        raise JpegError("not a JPEG stream (no SOI marker)")
    pos, quant, dc, ac, restart, frame, jfif, adobe = 2, {}, {}, {}, 0, None, False, None
    while True:
        if pos >= n:
            raise JpegError("truncated header (no SOS marker)")
        if b[pos] != 0xFF:
            raise JpegError("malformed header (a marker was expected)")
        while pos < n and b[pos] == 0xFF:
            pos += 1
        if pos >= n:
            raise JpegError("truncated header (no SOS marker)")
        m = b[pos]
        pos += 1
        if m == 0xD9:
            raise JpegError("malformed header (EOI before SOS)")
        if m == 0xD8 or m == 0x01 or 0xD0 <= m <= 0xD7 or m == 0x00:
            raise JpegError("malformed header (unexpected marker 0x%02X)" % m)
        if pos + 2 > n:
            raise JpegError("truncated header")
        L = (b[pos] << 8) | b[pos + 1]
        if L < 2 or pos + L > n:
            raise JpegError("truncated header")
        seg = b[pos + 2:pos + L]
        pos += L
        if m in _SOF_REFUSED:
            raise JpegError(_SOF_REFUSED[m] + " is not supported")
        if m in (0xC0, 0xC1):
            if frame is not None:
                raise JpegError("malformed header (two SOF markers)")
            if len(seg) < 6:
                raise JpegError("malformed header (short SOF)")
            P, H, W, nf = seg[0], (seg[1] << 8) | seg[2], (seg[3] << 8) | seg[4], seg[5]
            if P != 8:
                raise JpegError("%d-bit samples are not supported" % P)
            if len(seg) != 6 + 3 * nf:
                raise JpegError("malformed header (SOF length)")
            if H == 0 or W == 0:
                raise JpegError("malformed header (zero width or height)")
            if nf == 4:
                raise JpegError("CMYK / YCCK JPEG is not supported")
            if nf not in (1, 3):
                raise JpegError("%d-component JPEG is not supported" % nf)
            comps = [(seg[6 + 3 * i], seg[7 + 3 * i] >> 4, seg[7 + 3 * i] & 15, seg[8 + 3 * i]) for i in range(nf)]
            if len({c[0] for c in comps}) != nf or any(c[3] > 3 or not 1 <= c[1] <= 4 or not 1 <= c[2] <= 4 for c in comps):
                raise JpegError("malformed header (SOF components)")
            frame = (W, H, comps)
        elif m == 0xC4:
            i = 0
            while i < len(seg):
                if i + 17 > len(seg):
                    raise JpegError("malformed header (short DHT)")
                tc, th = seg[i] >> 4, seg[i] & 15
                bits = list(seg[i + 1:i + 17])
                cnt = sum(bits)
                if tc > 1 or th > 3 or cnt > 256 or i + 17 + cnt > len(seg):
                    raise JpegError("malformed header (bad DHT)")
                vals = list(seg[i + 17:i + 17 + cnt])
                code = 0
                for l in range(16):
                    code += bits[l]
                    if code > (1 << (l + 1)):
                        raise JpegError("malformed header (bad Huffman table)")
                    code <<= 1
                if tc == 0 and any(v > 15 for v in vals):
                    raise JpegError("malformed header (bad Huffman table)")
                (ac if tc else dc)[th] = (bits, vals)
                i += 17 + cnt
        elif m == 0xDB:
            i = 0
            while i < len(seg):
                pq, tq = seg[i] >> 4, seg[i] & 15
                size = 128 if pq else 64
                if pq > 1 or tq > 3 or i + 1 + size > len(seg):
                    raise JpegError("malformed header (bad DQT)")
                raw = np.frombuffer(seg[i + 1:i + 1 + size], ">u2" if pq else np.uint8).astype(np.int64)
                q = np.zeros(64, np.int64)
                q[NATURAL] = raw
                quant[tq] = q
                i += 1 + size
        elif m == 0xDD:
            if len(seg) != 2:
                raise JpegError("malformed header (bad DRI)")
            restart = (seg[0] << 8) | seg[1]
        elif m == 0xE0:
            jfif = jfif or seg[:5] == b"JFIF\0"
        elif m == 0xEE:
            if seg[:5] == b"Adobe" and len(seg) >= 12:
                adobe = seg[11]
        elif m == 0xDA:
            if frame is None:
                raise JpegError("malformed header (SOS before SOF)")
            W, H, comps = frame
            if len(seg) < 1 or len(seg) != 4 + 2 * seg[0]:
                raise JpegError("malformed header (SOS length)")
            ns = seg[0]
            if ns != len(comps):
                raise JpegError("multi-scan sequential JPEG is not supported")
            sel = [(seg[1 + 2 * i], seg[2 + 2 * i] >> 4, seg[2 + 2 * i] & 15) for i in range(ns)]
            if [s[0] for s in sel] != [c[0] for c in comps]:
                raise JpegError("malformed header (SOS components)")
            ss, se, ahl = seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns]
            if ss != 0 or se != 63 or ahl != 0:
                raise JpegError("malformed header (sequential scan with a spectral selection)")
            if len(comps) == 3:
                samp = [(c[1], c[2]) for c in comps]
                if samp[1:] != [(1, 1), (1, 1)] or samp[0] not in ((1, 1), (2, 1), (2, 2)):
                    raise JpegError("sampling factors %s are not supported" % "x".join("%d%d" % s for s in samp))
                if jfif:
                    colour = "ycc"
                elif adobe is not None:
                    if adobe == 0:
                        raise JpegError("Adobe RGB (transform 0) JPEG is not supported")
                    colour = "ycc"
                elif [c[0] for c in comps] == [82, 71, 66]:
                    raise JpegError("RGB (component ids R, G, B) JPEG is not supported")
                else:
                    colour = "ycc"
            else:
                colour = "gray"
            out = []
            for c, s in zip(comps, sel):
                if c[3] not in quant:
                    raise JpegError("scan references undefined quantisation table %d" % c[3])
                if s[1] not in dc:
                    raise JpegError("scan references undefined DC Huffman table %d" % s[1])
                if s[2] not in ac:
                    raise JpegError("scan references undefined AC Huffman table %d" % s[2])
                h, v = (c[1], c[2]) if len(comps) == 3 else (1, 1)
                out.append((c[0], h, v, c[3], s[1], s[2]))
            return dict(width=W, height=H, comps=out, quant={k: v.copy() for k, v in quant.items()}, dc=dict(dc), ac=dict(ac),
                        restart=restart, scan=pos, colour=colour)


def geometry(hdr):
    """MCU grid and per-component block grids: (mcux, mcuy, [(bw, bh, dw, dh)]) with dw, dh the component's downsampled size"""
    W, H, comps = hdr["width"], hdr["height"], hdr["comps"]
    hmax, vmax = max(c[1] for c in comps), max(c[2] for c in comps)
    if len(comps) == 1:
        bw, bh = -(-W // 8), -(-H // 8)
        return bw, bh, [(bw, bh, W, H)]
    mcux, mcuy = -(-W // (8 * hmax)), -(-H // (8 * vmax))
    return mcux, mcuy, [(mcux * c[1], mcuy * c[2], -(-W * c[1] // hmax), -(-H * c[2] // vmax)) for c in comps]


def _lut(table):
    """16-bit lookup: for every 16-bit window, (code length << 8) | symbol, 0 where no code matches"""
    bits, vals = table
    lut = np.zeros(65536, np.int64)
    code, k = 0, 0
    for l in range(1, 17):
        for _ in range(bits[l - 1]):
            lut[code << (16 - l):(code + 1) << (16 - l)] = (l << 8) | vals[k]
            code += 1
            k += 1
        code <<= 1
    return lut.tolist()


def _intervals(b, start):
    """The entropy-coded segment from `start` split at RST markers: [(rst number or None, bytes with stuffing removed)] and the
    segment's end"""
    n = len(b)
    out, p, q, num = [], start, start, None
    while True:
        q = b.find(b"\xff", q)
        if q < 0 or q + 1 >= n:        # a last 0xFF starts a marker the bytes cut off
            end = n if q < 0 else q
            break
        nxt = b[q + 1]
        if nxt == 0x00:
            q += 2
            continue
        if 0xD0 <= nxt <= 0xD7:
            out.append((num, b[p:q]))
            num, p, q = nxt - 0xD0, q + 2, q + 2
            continue
        if nxt == 0xFF:        # fill bytes before a marker: the data ends here unless an RST follows
            r = q
            while r < n and b[r] == 0xFF:
                r += 1
            if r < n and 0xD0 <= b[r] <= 0xD7:
                out.append((num, b[p:q]))
                num, p, q = b[r] - 0xD0, r + 1, r + 1
                continue
        end = q
        break
    out.append((num, b[p:end]))
    return [(k, d.replace(b"\xff\x00", b"\xff")) for k, d in out], end


def entropy(data, hdr):
    """Huffman decode -> ([int32 [bh, bw, 64] quantised coefficients in row-major (natural) order per component], status).
    One restart interval at a time, DC prediction reset at each; a corrupt interval leaves zeros from its first bad block on,
    and the status is the largest code of any interval."""
    b = bytes(data)
    mcux, mcuy, grids = geometry(hdr)
    comps = hdr["comps"]
    coefs = [np.zeros((g[1], g[0], 64), np.int32) for g in grids]
    flat = [c.reshape(-1, 64) for c in coefs]
    luts = {}
    for c in comps:
        luts.setdefault(("dc", c[4]), _lut(hdr["dc"][c[4]]))
        luts.setdefault(("ac", c[5]), _lut(hdr["ac"][c[5]]))
    blocks = []        # (component, h, v) of an MCU's blocks in scan order
    for ci, c in enumerate(comps):
        blocks += [(ci, h, v) for v in range(c[2]) for h in range(c[1])]
    total = mcux * mcuy
    ri = hdr["restart"] or total
    n_int = -(-total // ri)
    ivs, _ = _intervals(b, hdr["scan"])
    status = OK
    nat = NATURAL.tolist()
    for it in range(n_int):
        if it >= len(ivs):
            status = max(status, TRUNCATED)
            break
        num, seg = ivs[it]
        if it > 0 and num != (it - 1) % 8:
            status = max(status, BAD_RESTART)
            continue
        real = len(seg) * 8
        bits = np.unpackbits(np.frombuffer(seg + bytes(520), np.uint8)).astype(np.int64)
        win = np.zeros(len(bits) - 16, np.int64)
        for i in range(16):
            win += bits[i:i + len(win)] << (15 - i)
        win = win.tolist()
        pred = [0] * len(comps)
        p = 0
        bad = OK
        for mcu in range(it * ri, min(total, (it + 1) * ri)):
            my, mx = divmod(mcu, mcux)
            for ci, h, v in blocks:
                c = comps[ci]
                dlut, alut = luts[("dc", c[4])], luts[("ac", c[5])]
                blk = flat[ci][(my * c[2] + v) * grids[ci][0] + mx * c[1] + h]
                e = dlut[win[p]]
                if e == 0:
                    bad = BAD_CODE
                    break
                p += e >> 8
                s = e & 255
                if s:
                    r = win[p] >> (16 - s)
                    p += s
                    if r < (1 << (s - 1)):
                        r += 1 - (1 << s)
                    s = r
                pred[ci] += s
                vals = [0] * 64
                vals[0] = pred[ci]
                k = 1
                while k < 64:
                    e = alut[win[p]]
                    if e == 0:
                        bad = BAD_CODE
                        break
                    p += e >> 8
                    rs = e & 255
                    r, s = rs >> 4, rs & 15
                    if s:
                        k += r
                        if k > 63:
                            bad = BAD_RUN
                            break
                        r = win[p] >> (16 - s)
                        p += s
                        if r < (1 << (s - 1)):
                            r += 1 - (1 << s)
                        vals[nat[k]] = r
                    elif r != 15:
                        break
                    else:
                        k += 15
                    k += 1
                if bad:
                    break
                if p > real:
                    bad = TRUNCATED
                    break
                blk[:] = np.array(vals, np.int64).astype(np.int16)      # JCOEF is 16-bit
            if bad:
                break
        status = max(status, bad)
    return coefs, status


C1, C2, PASS1 = 13, 2, 2
F = dict(f0298=2446, f0390=3196, f0541=4433, f0765=6270, f0899=7373, f1175=9633, f1501=12299, f1847=15137, f1961=16069,
         f2053=16819, f2562=20995, f3072=25172)


def _idct_1d(x0, x1, x2, x3, x4, x5, x6, x7, shift):
    """one islow butterfly over int64 arrays; the inputs of pass 2 carry no << CONST_BITS yet"""
    z1 = (x2 + x6) * F["f0541"]
    t2 = z1 - x6 * F["f1847"]
    t3 = z1 + x2 * F["f0765"]
    t0 = (x0 + x4) << C1
    t1 = (x0 - x4) << C1
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    o0, o1, o2, o3 = x7, x5, x3, x1
    z1, z2, z3, z4 = o0 + o3, o1 + o2, o0 + o2, o1 + o3
    z5 = (z3 + z4) * F["f1175"]
    o0, o1, o2, o3 = o0 * F["f0298"], o1 * F["f2053"], o2 * F["f3072"], o3 * F["f1501"]
    z1, z2, z3, z4 = -z1 * F["f0899"], -z2 * F["f2562"], -z3 * F["f1961"] + z5, -z4 * F["f0390"] + z5
    o0, o1, o2, o3 = o0 + z1 + z3, o1 + z2 + z4, o2 + z2 + z3, o3 + z1 + z4
    d = lambda v: (v + (1 << (shift - 1))) >> shift
    return [d(t10 + o3), d(t11 + o2), d(t12 + o1), d(t13 + o0), d(t13 - o0), d(t12 - o1), d(t11 - o2), d(t10 - o3)]


def range_limit(v):
    """libjpeg-turbo's post-IDCT range limit as its SIMD islow applies it: saturate to [-128, 127], then + 128"""
    return (np.clip(v, -128, 127) + 128).astype(np.uint8)


def idct(coefs, q):
    """islow IDCT of int [..., 64] quantised coefficients (natural order) with the int64[64] table q -> uint8 [..., 8, 8]"""
    x = coefs.astype(np.int64).reshape(-1, 8, 8) * q.reshape(8, 8)
    cols = _idct_1d(*[x[:, r, :] for r in range(8)], C1 - PASS1)          # pass 1: columns, rows of x indexed by r
    ws = np.stack(cols, axis=1).astype(np.int32).astype(np.int64)           # the int workspace
    rows = _idct_1d(*[ws[:, :, c] for c in range(8)], C1 + PASS1 + 3)       # pass 2: rows
    return range_limit(np.stack(rows, axis=2)).reshape(coefs.shape[:-1] + (8, 8))


def planes(coefs, hdr):
    """every component's IDCT output as a uint8 plane [bh * 8, bw * 8]"""
    out = []
    for c, k in zip(hdr["comps"], coefs):
        bh, bw = k.shape[:2]
        out.append(idct(k, hdr["quant"][c[3]]).transpose(0, 2, 1, 3).reshape(bh * 8, bw * 8))
    return out


def upsample(plane, h, v, W, H):
    """a chroma plane (downsampled size ceil(W / h) x ceil(H / v) valid) to W x H: h1v1 copies; h2v1 / h2v2 use libjpeg's
    fancy triangle filter, except that a plane at most 2 samples wide is replicated"""
    dw, dh = -(-W // h), -(-H // v)
    p = plane[:dh, :dw].astype(np.int32)
    if h == 1:
        return p[:H, :W].astype(np.uint8)
    if dw <= 2:
        rows = np.repeat(p, v, axis=0) if v == 2 else p
        return np.repeat(rows, 2, axis=1)[:H, :W].astype(np.uint8)
    left = np.concatenate([p[:, :1], p[:, :-1]], axis=1)
    right = np.concatenate([p[:, 1:], p[:, -1:]], axis=1)
    out = np.zeros((p.shape[0], 2 * dw), np.int32)
    if v == 1:
        out[:, 0::2] = (3 * p + left + 1) >> 2
        out[:, 1::2] = (3 * p + right + 2) >> 2
        return out[:H, :W].astype(np.uint8)
    up = np.concatenate([p[:1], p[:-1]], axis=0)
    dn = np.concatenate([p[1:], p[-1:]], axis=0)
    res = np.zeros((2 * dh, 2 * dw), np.int32)
    for r0, nb in ((0, up), (1, dn)):
        cs = 3 * p + nb
        csl = np.concatenate([cs[:, :1], cs[:, :-1]], axis=1)
        csr = np.concatenate([cs[:, 1:], cs[:, -1:]], axis=1)
        res[r0::2, 0::2] = (3 * cs + csl + 8) >> 4
        res[r0::2, 1::2] = (3 * cs + csr + 7) >> 4
    return res[:H, :W].astype(np.uint8)


SCALE, HALF = 16, 1 << 15


def _fix(x):
    return int(x * (1 << SCALE) + 0.5)


_X = np.arange(256, dtype=np.int64) - 128
CR_R = (_fix(1.40200) * _X + HALF) >> SCALE
CB_B = (_fix(1.77200) * _X + HALF) >> SCALE
CR_G = -_fix(0.71414) * _X
CB_G = -_fix(0.34414) * _X + HALF


def ycc_to_rgb(y, cb, cr):
    """libjpeg's fixed-point YCbCr -> RGB (16 fraction bits), clipped to 0..255"""
    y, cb, cr = y.astype(np.int64), cb.astype(np.int64), cr.astype(np.int64)
    r = y + CR_R[cr]
    g = y + ((CB_G[cb] + CR_G[cr]) >> SCALE)
    b = y + CB_B[cb]
    return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8)


def rgb_to_l(rgb):
    """PIL's RGB -> L: (R * 19595 + G * 38470 + B * 7471 + 0x8000) >> 16"""
    x = rgb.astype(np.int64)
    return ((x[..., 0] * 19595 + x[..., 1] * 38470 + x[..., 2] * 7471 + 0x8000) >> 16).astype(np.uint8)[..., None]


def colour(pl, hdr, mode):
    """the component planes -> uint8 [H, W, 3] ('RGB') or [H, W, 1] ('L')"""
    W, H = hdr["width"], hdr["height"]
    if hdr["colour"] == "gray":
        y = pl[0][:H, :W]
        return np.repeat(y[..., None], 3, -1) if mode == "RGB" else y[..., None].copy()
    hy, vy = hdr["comps"][0][1], hdr["comps"][0][2]
    rgb = ycc_to_rgb(pl[0][:H, :W], upsample(pl[1], hy, vy, W, H), upsample(pl[2], hy, vy, W, H))
    return rgb if mode == "RGB" else rgb_to_l(rgb)


def decode(data, mode="RGB", with_status=False):
    """the whole decode: bytes -> uint8 [H, W, 3 or 1] (and the entropy status when with_status)"""
    hdr = parse(data)
    coefs, status = entropy(data, hdr)
    out = colour(planes(coefs, hdr), hdr, mode)
    return (out, status) if with_status else out
