"""A numpy restatement of the baseline JPEG encode that Image.save(f, quality=q) performs through libjpeg-turbo (and that
cv2.imencode writes byte for byte), stage by stage, without PIL: 'L' as one component, 'RGB' as YCbCr 4:2:0, the Annex K
quantisation tables scaled by jpeg_quality_scaling with force_baseline, the Annex K Huffman tables, no restart interval and no
metadata.  tests/golden/jpeg_encode.npz (oracle/gen_golden_jpeg_encode.py) pins it to Pillow's bytes.

Each stage is a function of its own, named after the libjpeg-turbo function it follows, so a mismatch of csrc/jpeg_encode.cu
can be localised: rgb_ycc() -> component_planes() (edge expansion, h2v2 downsampling) -> blocks() (MCU order, dummy blocks)
-> fdct_islow() -> quantize() -> entropy() (zig-zag, DC differences, Huffman, padding, stuffing) -> header().  encode() runs
them all.
"""
import numpy as np

from oracle.jpeg_oracle import NATURAL

MODES = {"L": 1, "RGB": 3}
MAX_SIDE = 65500                    # libjpeg's JPEG_MAX_DIMENSION

# Annex K.1, natural (row-major) order
STD_QUANT = (np.array([16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29,
                       51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92, 49, 64, 78, 87, 103, 121,
                       120, 101, 72, 92, 95, 98, 112, 100, 103, 99], np.int64),
             np.array([17, 18, 24, 47] + [99] * 4 + [18, 21, 26, 66] + [99] * 4 + [24, 26, 56] + [99] * 5 + [47, 66] + [99] * 38,
                      np.int64))

# Annex K.3: (bits[1..16], vals) of DC luminance, AC luminance, DC chrominance, AC chrominance
_AC_LUM_VALS = bytes.fromhex(
    "01020300041105122131410613516107227114328191a1082342b1c11552d1f02433627282090a161718191a25262728292a3435363738393a"
    "434445464748494a535455565758595a636465666768696a737475767778797a838485868788898a92939495969798999aa2a3a4a5a6a7a8a9"
    "aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae1e2e3e4e5e6e7e8e9eaf1f2f3f4f5f6f7f8f9fa")
_AC_CHR_VALS = bytes.fromhex(
    "000102031104052131061241510761711322328108144291a1b1c109233352f0156272d10a162434e125f11718191a262728292a35363738393a"
    "434445464748494a535455565758595a636465666768696a737475767778797a82838485868788898a92939495969798999aa2a3a4a5a6a7a8a9"
    "aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae2e3e4e5e6e7e8e9eaf2f3f4f5f6f7f8f9fa")
STD_HUFF = {
    "dc0": ((0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0), bytes(range(12))),
    "ac0": ((0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7D), _AC_LUM_VALS),
    "dc1": ((0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0), bytes(range(12))),
    "ac1": ((0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77), _AC_CHR_VALS),
}


def check_args(mode, quality, height, width):
    """the library's refusals, in its wording"""
    if mode not in MODES:
        raise ValueError("mode must be 'L' or 'RGB'")
    if not 1 <= quality <= 100:
        raise ValueError("quality must be 1 .. 100")
    if not (1 <= height <= MAX_SIDE and 1 <= width <= MAX_SIDE):
        raise ValueError("height and width must be 1 .. %d" % MAX_SIDE)


# ------------------------------------------------------------------------------------------------------------- tables

def quant_tables(quality):
    """jcparam.c jpeg_set_quality(quality, force_baseline=TRUE): jpeg_quality_scaling, then jpeg_add_quant_table's
    (basic * scale + 50) / 100 clamped to 1 .. 255.  -> (luminance, chrominance), int64 [64] natural order"""
    scale = 5000 // quality if quality < 50 else 200 - 2 * quality
    return tuple(np.clip((t * scale + 50) // 100, 1, 255) for t in STD_QUANT)


def huff_codes(bits, vals):
    """jchuff.c jpeg_make_c_derived_tbl: canonical codes -> (code[256], size[256]) indexed by symbol"""
    code, size = np.zeros(256, np.int64), np.zeros(256, np.int64)
    c, k = 0, 0
    for l in range(1, 17):
        for _ in range(bits[l - 1]):
            code[vals[k]], size[vals[k]] = c, l
            c, k = c + 1, k + 1
        c <<= 1
    return code, size


# ------------------------------------------------------------------------------------------------------- sample planes

SCALEBITS, ONE_HALF, CBCR_OFFSET = 16, 1 << 15, 128 << 16


def _fix(x):
    return int(x * (1 << SCALEBITS) + 0.5)


def rgb_ycc(rgb):
    """jccolor.c rgb_ycc_convert with its rgb_ycc_tab: uint8 [H, W, 3] -> Y, Cb, Cr int64 [H, W].  Cb and Cr round with
    ONE_HALF - 1 so that 255 is never exceeded."""
    r, g, b = (rgb[..., i].astype(np.int64) for i in range(3))
    y = (_fix(0.29900) * r + _fix(0.58700) * g + _fix(0.11400) * b + ONE_HALF) >> SCALEBITS
    cb = (-_fix(0.16874) * r - _fix(0.33126) * g + _fix(0.5) * b + CBCR_OFFSET + ONE_HALF - 1) >> SCALEBITS
    cr = (_fix(0.5) * r - _fix(0.41869) * g - _fix(0.08131) * b + CBCR_OFFSET + ONE_HALF - 1) >> SCALEBITS
    return y, cb, cr


def geometry(mode, height, width):
    """-> (MCUs across, MCUs down, [(blocks across, blocks down) per component]) of jdinput-style sizing:
    a component's width_in_blocks = ceil(ceil(W * h / hmax) / 8)"""
    if mode == "L":
        bw, bh = -(-width // 8), -(-height // 8)
        return bw, bh, [(bw, bh)]
    cw, ch = -(-width // 2), -(-height // 2)
    return -(-width // 16), -(-height // 16), [(-(-width // 8), -(-height // 8))] + [(-(-cw // 8), -(-ch // 8))] * 2


def h2v2_downsample(plane, out_w):
    """jcsample.c h2v2_downsample: expand_right_edge of the full-resolution rows to 2 * out_w columns (the last column
    repeated), then each output sample (a + b + c + d + bias) >> 2 with bias 1, 2, 1, 2, ... along the row.  The rows come in
    pairs: jcprepct.c repeats the last row when the height is odd."""
    H, W = plane.shape
    p = np.pad(plane, ((0, H % 2), (0, 2 * out_w - W)), mode="edge")
    s = p[0::2, 0::2] + p[0::2, 1::2] + p[1::2, 0::2] + p[1::2, 1::2]
    bias = 1 + (np.arange(out_w) & 1)
    return (s + bias) >> 2


def component_planes(img, mode):
    """uint8 [H, W] ('L') or [H, W, 3] ('RGB') -> one int64 plane per component, expanded to whole blocks: jcsample.c's
    expand_right_edge (last column repeated) and jcprepct.c's expand_bottom_edge (last row repeated), the chroma after
    downsampling"""
    H, W = img.shape[:2]
    _, _, comp = geometry(mode, H, W)
    if mode == "L":
        bw, bh = comp[0]
        return [np.pad(img.astype(np.int64), ((0, 8 * bh - H), (0, 8 * bw - W)), mode="edge")]
    y, cb, cr = rgb_ycc(img)
    (yw, yh), (cw, chb) = comp[0], comp[1]
    out = [np.pad(y, ((0, 8 * yh - H), (0, 8 * yw - W)), mode="edge")]
    for c in (cb, cr):
        d = h2v2_downsample(c, 8 * cw)
        out.append(np.pad(d, ((0, 8 * chb - d.shape[0]), (0, 0)), mode="edge"))
    return out


# ------------------------------------------------------------------------------------------------------------------ DCT

CONST_BITS, PASS1_BITS = 13, 2
FIX_0_298631336, FIX_0_390180644, FIX_0_541196100, FIX_0_765366865 = 2446, 3196, 4433, 6270
FIX_0_899976223, FIX_1_175875602, FIX_1_501321110, FIX_1_847759065 = 7373, 9633, 12299, 15137
FIX_1_961570560, FIX_2_053119869, FIX_2_562915447, FIX_3_072711026 = 16069, 16819, 20995, 25172


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _fdct_1d(d, first):
    """one pass of jfdctint.c jpeg_fdct_islow over the last axis of d (int64 [..., 8]): the even part with its
    LEFT_SHIFT (pass 1) or DESCALE (pass 2) by PASS1_BITS, the odd part with DESCALE by CONST_BITS -/+ PASS1_BITS"""
    t0, t7 = d[..., 0] + d[..., 7], d[..., 0] - d[..., 7]
    t1, t6 = d[..., 1] + d[..., 6], d[..., 1] - d[..., 6]
    t2, t5 = d[..., 2] + d[..., 5], d[..., 2] - d[..., 5]
    t3, t4 = d[..., 3] + d[..., 4], d[..., 3] - d[..., 4]
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    o = np.empty_like(d)
    sh = CONST_BITS - PASS1_BITS if first else CONST_BITS + PASS1_BITS
    if first:
        o[..., 0], o[..., 4] = (t10 + t11) << PASS1_BITS, (t10 - t11) << PASS1_BITS
    else:
        o[..., 0], o[..., 4] = _descale(t10 + t11, PASS1_BITS), _descale(t10 - t11, PASS1_BITS)
    z1 = (t12 + t13) * FIX_0_541196100
    o[..., 2] = _descale(z1 + t13 * FIX_0_765366865, sh)
    o[..., 6] = _descale(z1 - t12 * FIX_1_847759065, sh)
    z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
    z5 = (z3 + z4) * FIX_1_175875602
    t4, t5, t6, t7 = t4 * FIX_0_298631336, t5 * FIX_2_053119869, t6 * FIX_3_072711026, t7 * FIX_1_501321110
    z1, z2 = z1 * -FIX_0_899976223, z2 * -FIX_2_562915447
    z3, z4 = z3 * -FIX_1_961570560 + z5, z4 * -FIX_0_390180644 + z5
    o[..., 7] = _descale(t4 + z1 + z3, sh)
    o[..., 5] = _descale(t5 + z2 + z4, sh)
    o[..., 3] = _descale(t6 + z2 + z3, sh)
    o[..., 1] = _descale(t7 + z1 + z4, sh)
    return o


def fdct_islow(blk):
    """jcdctmgr.c convsamp's level shift (sample - 128), then jfdctint.c: rows, then columns.  int64 [n, 8, 8] samples ->
    DCT output scaled by 8, natural order"""
    d = _fdct_1d(blk - 128, True)
    return _fdct_1d(d.swapaxes(1, 2), False).swapaxes(1, 2)


def quantize(dct, qtbl):
    """jcdctmgr.c quantize: round(|x| / (8 q)) with halves away from zero, the sign restored (libjpeg-turbo's reciprocal
    multiply gives the same integers)"""
    div = (qtbl << 3).reshape(8, 8)
    return np.sign(dct) * ((np.abs(dct) + (div >> 1)) // div)


# --------------------------------------------------------------------------------------------------------------- blocks

def blocks(img, mode, quality):
    """-> quantised coefficients int64 [blocks, 64] natural order, the component of each block and whether it is a dummy,
    in scan order: 'L' row-major; 'RGB' per MCU Y00 Y01 Y10 Y11 Cb Cr.  jccoefct.c compress_data fills the MCU's blocks
    past the component's right / bottom edge as dummy blocks: zero AC, DC copied from the block before (so their DC
    difference is 0)."""
    planes = component_planes(img, mode)
    q = quant_tables(quality)
    mx, my, comp = geometry(mode, *img.shape[:2])
    coef = []
    for c, (p, (bw, bh)) in enumerate(zip(planes, comp)):
        b = p.reshape(bh, 8, bw, 8).swapaxes(1, 2).reshape(-1, 8, 8)
        coef.append(quantize(fdct_islow(b), q[min(c, 1)]).reshape(bh, bw, 64))
    if mode == "L":
        return coef[0].reshape(-1, 64), np.zeros(mx * my, np.int64), np.zeros(mx * my, bool)
    out, cid, dummy = [], [], []
    yw, yh = comp[0]
    for j in range(my):
        for i in range(mx):
            for r in range(2):
                for s in range(2):
                    y, x = 2 * j + r, 2 * i + s
                    real = y < yh and x < yw
                    if real:
                        out.append(coef[0][y, x])
                    else:
                        d = np.zeros(64, np.int64)
                        d[0] = out[-1][0]
                        out.append(d)
                    cid.append(0)
                    dummy.append(not real)
            for c in (1, 2):
                out.append(coef[c][j, i])
                cid.append(c)
                dummy.append(False)
    return np.array(out, np.int64).reshape(-1, 64), np.array(cid, np.int64), np.array(dummy, bool)


# -------------------------------------------------------------------------------------------------------------- entropy

def _nbits(v):
    """the magnitude category: bits of |v| (0 for 0)"""
    return int(abs(int(v))).bit_length()


def entropy(coef, comp):
    """jchuff.c encode_one_block over the blocks in scan order: zig-zag order; the DC difference from the previous block of
    the same component (0 before the first), coded as its category's DC code then the category's low bits of v (v - 1 when
    negative); each non-zero AC coefficient after a run r of zeros as ZRL (0xF0) per 16 zeros, then symbol (r << 4 | size)
    and the bits; EOB (0x00) when the block ends in zeros.  jchuff.c flush_bits pads the last byte with 1-bits and
    emit_byte writes 0x00 after every 0xFF.  -> the entropy-coded bytes"""
    tabs = {k: huff_codes(*v) for k, v in STD_HUFF.items()}
    pieces, pred = [], [0, 0, 0]

    def put(code, size):
        if size:
            pieces.append(format(int(code), "0%db" % size))

    for blk, c in zip(coef, comp):
        dc_code, dc_size = tabs["dc%d" % min(c, 1)]
        ac_code, ac_size = tabs["ac%d" % min(c, 1)]
        zz = blk[NATURAL]
        diff = int(zz[0]) - pred[c]
        pred[c] = int(zz[0])
        n = _nbits(diff)
        put(dc_code[n], dc_size[n])
        put((diff - (diff < 0)) & ((1 << n) - 1), n)
        run = 0
        for k in range(1, 64):
            v = int(zz[k])
            if v == 0:
                run += 1
                continue
            while run > 15:
                put(ac_code[0xF0], ac_size[0xF0])
                run -= 16
            n = _nbits(v)
            sym = (run << 4) | n
            put(ac_code[sym], ac_size[sym])
            put((v - (v < 0)) & ((1 << n) - 1), n)
            run = 0
        if run:
            put(ac_code[0], ac_size[0])
    bits = "".join(pieces)
    bits += "1" * (-len(bits) % 8)
    raw = int(bits, 2).to_bytes(len(bits) // 8, "big") if bits else b""
    return raw.replace(b"\xff", b"\xff\x00")


# --------------------------------------------------------------------------------------------------------------- header

def _segment(marker, body):
    return bytes([0xFF, marker]) + (len(body) + 2).to_bytes(2, "big") + body


def header(mode, quality, height, width):
    """jcmarker.c write_file_header / write_frame_header / write_scan_header: SOI, APP0 JFIF 1.01 (density 1:1, units 0,
    no thumbnail), one DQT per table (8-bit, zig-zag order), SOF0, one DHT per table (DC0, AC0, then DC1, AC1 for 'RGB'), SOS"""
    nc = MODES[mode]
    q = quant_tables(quality)
    h = b"\xff\xd8" + _segment(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    for t in range(min(nc, 2)):
        h += _segment(0xDB, bytes([t]) + bytes(q[t][NATURAL].tolist()))
    comps = [(1, 0x11, 0)] if nc == 1 else [(1, 0x22, 0), (2, 0x11, 1), (3, 0x11, 1)]
    h += _segment(0xC0, bytes([8]) + height.to_bytes(2, "big") + width.to_bytes(2, "big") + bytes([nc])
                  + b"".join(bytes(c) for c in comps))
    for t in range(min(nc, 2)):
        for cls, key in ((0, "dc%d" % t), (1, "ac%d" % t)):
            bits, vals = STD_HUFF[key]
            h += _segment(0xC4, bytes([cls << 4 | t]) + bytes(bits) + bytes(vals))
    sel = [(1, 0x00)] if nc == 1 else [(1, 0x00), (2, 0x11), (3, 0x11)]
    h += _segment(0xDA, bytes([nc]) + b"".join(bytes(s) for s in sel) + b"\x00\x3f\x00")
    return h


def encode(img, mode="RGB", quality=95):
    """uint8 [H, W] or [H, W, 1] ('L'), [H, W, 3] ('RGB') -> the JPEG file's bytes, equal to Pillow's save(quality=quality)"""
    img = np.asarray(img, np.uint8)
    if mode == "L" and img.ndim == 3:
        img = img[..., 0]
    check_args(mode, quality, img.shape[0], img.shape[1])
    coef, comp, _ = blocks(img, mode, quality)
    return header(mode, quality, img.shape[0], img.shape[1]) + entropy(coef, comp) + b"\xff\xd9"


# ------------------------------------------------------------------------------------------------------------- capacity

MAX_BLOCK_BITS = 22 + 63 * 26       # a DC code of <= 11 bits + 11 value bits, then 63 AC codes of <= 16 bits + 10 value bits


def header_bytes(mode):
    return len(header(mode, 50, 1, 1))


def blocks_per_image(mode, height, width):
    mx, my, _ = geometry(mode, height, width)
    return mx * my * (1 if mode == "L" else 6)


def capacity(mode, height, width):
    """the worst-case file size the library reserves per image: header, every block at MAX_BLOCK_BITS plus 7 pad bits,
    every byte stuffed, EOI"""
    raw = (blocks_per_image(mode, height, width) * MAX_BLOCK_BITS + 7) // 8
    return header_bytes(mode) + 2 * raw + 2


# ------------------------------------------------------------------------------------------------------------- fixtures

def _hash(idx, seed):
    """splitmix64 of (index, seed), uint64: a stateless generator that stays the same across numpy versions"""
    z = idx.astype(np.uint64) + np.uint64((seed * 0x9E3779B97F4A7C15) & 0xFFFFFFFFFFFFFFFF)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def fixture(kind, height, width, channels, seed=0):
    """a test image uint8 [H, W, C]: 'const0' / 'const128' / 'const255', 'ramp' (a diagonal ramp per channel), 'noise'
    (uniform), 'checker' (0 / 255 pixel checkerboard) or 'flow' (the quantised planes of a smooth seeded flow field, by
    tvl1_oracle.planes; each channel its own plane)"""
    H, W, C = height, width, channels
    y, x, c = np.meshgrid(np.arange(H), np.arange(W), np.arange(C), indexing="ij")
    if kind.startswith("const"):
        return np.full((H, W, C), int(kind[5:]), np.uint8)
    if kind == "ramp":
        return ((x * 255 // max(W - 1, 1) + y * 3 + c * 40) % 256).astype(np.uint8)
    if kind == "noise":
        idx = (y * W + x) * C + c
        return (_hash(idx.reshape(-1), seed).reshape(H, W, C) >> np.uint64(56)).astype(np.uint8)
    if kind == "checker":
        return (((x + y) & 1) * 255).astype(np.uint8)
    if kind == "flow":
        from oracle import tvl1_oracle as T
        ph = (_hash(np.arange(8 * C), seed) >> np.uint64(11)).astype(np.float64) / float(1 << 53)
        f = np.zeros((C, H, W))
        for k in range(C):
            a = ph[8 * k:8 * k + 8]
            f[k] = (14 * np.sin(x[..., 0] * (0.01 + 0.05 * a[0]) + y[..., 0] * (0.02 * a[1]) + 6.3 * a[2])
                    + 9 * np.cos(y[..., 0] * (0.01 + 0.04 * a[3]) - x[..., 0] * (0.015 * a[4]) + 6.3 * a[5]) + 4 * (a[6] - 0.5))
        return T.planes(f.astype(np.float32)).reshape(C, H, W).transpose(1, 2, 0).copy()
    raise ValueError(kind)
