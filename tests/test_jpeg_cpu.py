"""CPU tests of the device JPEG decoder's host side: the parser's eligibility, EXIF orientation and header checks
(centerpose_b200/jpeg.py), and a numpy model of the three device stages (entropy decode, ISLOW IDCT, fancy upsampling
with integer YCbCr->BGR) pinned byte for byte against cv2.imdecode.  Fixtures are made here with cv2.imencode."""
import struct

import cv2
import numpy as np
import pytest

from centerpose_b200 import jpeg

SIZES = [(1, 1), (7, 5), (8, 8), (15, 17), (16, 16), (33, 47), (97, 131)]
QUALITIES = [10, 50, 75, 95, 100]
SAMPLINGS = {"444": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, "422": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
             "440": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440, "420": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, "gray": None}
CONTENTS = ["noise", "smooth", "smooth_noise"]


def make_image(h, w, content, seed, gray=False):
    rng = np.random.RandomState(seed)
    c = 1 if gray else 3
    if content == "noise":
        im = rng.randint(0, 256, (h, w, c))
    else:
        y, x = np.mgrid[0:h, 0:w].astype(np.float64)
        ph = rng.uniform(0, 6, 3)
        im = np.stack([127.5 + 127.5 * np.sin(x / max(w, 2) * 3 + y / max(h, 2) * 2 + ph[k]) for k in range(c)], -1)
        if content == "smooth_noise":
            im = im + rng.normal(0, 12, im.shape)
    im = np.clip(np.rint(im), 0, 255).astype(np.uint8)
    return im[:, :, 0] if gray else im


def encode(im, quality=75, sampling="420", rst=0, optimize=False, progressive=False):
    params = [cv2.IMWRITE_JPEG_QUALITY, quality]
    if sampling not in ("gray", None):
        params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, SAMPLINGS[sampling] if sampling in SAMPLINGS
                   else cv2.IMWRITE_JPEG_SAMPLING_FACTOR_411]
    if rst:
        params += [cv2.IMWRITE_JPEG_RST_INTERVAL, rst]
    if optimize:
        params += [cv2.IMWRITE_JPEG_OPTIMIZE, 1]
    if progressive:
        params += [cv2.IMWRITE_JPEG_PROGRESSIVE, 1]
    ok, buf = cv2.imencode(".jpg", im, params)
    assert ok
    return buf.tobytes()


def with_exif(data, orientation, big_endian=False):
    """The file with an APP1 Exif segment holding IFD0 {Orientation: orientation} spliced in after SOI."""
    o = ">" if big_endian else "<"
    tiff = (b"MM" if big_endian else b"II") + struct.pack(o + "HI", 42, 8) + struct.pack(o + "H", 1) + \
        struct.pack(o + "HHIHH", 0x0112, 3, 1, orientation, 0) + struct.pack(o + "I", 0)
    payload = b"Exif\x00\x00" + tiff
    return data[:2] + b"\xFF\xE1" + struct.pack(">H", len(payload) + 2) + payload + data[2:]


def cv2_decode(data):
    return cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)


# ---- the numpy model of the device stages -----------------------------------------------------------------------------

def _segment_bits(data, start, end):
    """The segment's entropy-coded bits with stuffed zero bytes removed; reading stops at a marker."""
    seg = np.frombuffer(data, np.uint8)[start:end]
    out, i = [], 0
    while i < len(seg):
        b = int(seg[i])
        if b == 0xFF:
            if i + 1 < len(seg) and seg[i + 1] == 0:
                out.append(0xFF)
                i += 2
                continue
            break
        out.append(b)
        i += 1
    return np.unpackbits(np.array(out, np.uint8)) if out else np.zeros(0, np.uint8)


class _Bits:
    def __init__(self, bits):
        self.bits = np.concatenate([bits, np.zeros(64, np.uint8)])
        self.real = len(bits)
        self.pos = 0

    def peek(self, n):
        v = 0
        for b in self.bits[self.pos:self.pos + n]:
            v = (v << 1) | int(b)
        return v

    def get(self, n):
        v = self.peek(n)
        self.pos += n
        if self.pos > len(self.bits) - 32:
            self.bits = np.concatenate([self.bits, np.zeros(64, np.uint8)])
        return v

    def symbol(self, t):
        e = int(t["lut"][self.peek(jpeg.LUT_BITS)])
        if e:
            self.pos += e >> 8
            return e & 255
        ln = jpeg.LUT_BITS + 1
        while ln <= 16 and self.peek(ln) > t["maxcode"][ln]:
            ln += 1
        if ln > 16:
            raise ValueError("code longer than 16 bits")
        v = int(t["val"][self.peek(ln) + t["valoff"][ln]])
        self.pos += ln
        return v


def _extend(v, s):
    return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v


def model_coefficients(info, data):
    """Entropy decode: per component an int64 array (block rows, blocks per row, 64) in natural order."""
    blocks = info.blocks()
    coef = [np.zeros((bh, bw, 64), np.int64) for bw, bh in blocks]
    mx, my = info.mcu
    total = mx * my
    ri = info.restart_interval or total
    units = [(0, dy, dx) for dy in range(info.vs) for dx in range(info.hs)] + [(c, 0, 0) for c in range(1, info.ncomp)]
    for s, (start, end) in enumerate(info.segments):
        r = _Bits(_segment_bits(data, start, end))
        pred = [0] * info.ncomp
        for m in range(s * ri, min((s + 1) * ri, total)):
            my_, mx_ = divmod(m, mx)
            for c, dy, dx in units:
                hs, vs = (info.hs, info.vs) if c == 0 else (1, 1)
                blk = coef[c][my_ * vs + dy, mx_ * hs + dx]
                t = info.huff[(0, info.dc[c])][2]
                n = r.symbol(t)
                pred[c] += _extend(r.get(n), n)
                blk[0] = pred[c]
                t = info.huff[(1, info.ac[c])][2]
                k = 1
                while k < 64:
                    sym = r.symbol(t)
                    run, n = sym >> 4, sym & 15
                    if n:
                        k += run
                        if k > 63:
                            raise ValueError("run past coefficient 63")
                        blk[jpeg.ZIGZAG[k]] = _extend(r.get(n), n)
                        k += 1
                    elif run == 15:
                        k += 16
                    else:
                        break
            if r.pos > r.real:
                raise ValueError("data ends before the segment's last MCU")
    return coef


def _idct_1d(x, shift):
    """One pass of libjpeg's jpeg_idct_islow over axis 0 (8 rows of int64), descaled by ``shift``."""
    F = dict(a=2446, b=3196, c=4433, d=6270, e=7373, f=9633, g=12299, h=15137, i=16069, j=16819, k=20995, l=25172)
    z2, z3 = x[2], x[6]
    z1 = (z2 + z3) * F["c"]
    tmp2 = z1 - z3 * F["h"]
    tmp3 = z1 + z2 * F["d"]
    tmp0 = (x[0] + x[4]) << 13
    tmp1 = (x[0] - x[4]) << 13
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    tmp0, tmp1, tmp2, tmp3 = x[7], x[5], x[3], x[1]
    z1, z2, z3, z4 = tmp0 + tmp3, tmp1 + tmp2, tmp0 + tmp2, tmp1 + tmp3
    z5 = (z3 + z4) * F["f"]
    tmp0, tmp1, tmp2, tmp3 = tmp0 * F["a"], tmp1 * F["j"], tmp2 * F["l"], tmp3 * F["g"]
    z1, z2, z3, z4 = -z1 * F["e"], -z2 * F["k"], -z3 * F["i"] + z5, -z4 * F["b"] + z5
    tmp0, tmp1, tmp2, tmp3 = tmp0 + z1 + z3, tmp1 + z2 + z4, tmp2 + z2 + z3, tmp3 + z1 + z4
    d = lambda v: (v + (1 << (shift - 1))) >> shift
    return np.stack([d(t10 + tmp3), d(t11 + tmp2), d(t12 + tmp1), d(t13 + tmp0),
                     d(t13 - tmp0), d(t12 - tmp1), d(t11 - tmp2), d(t10 - tmp3)])


def model_planes(info, coef):
    """Dequantise (16-bit product, as libjpeg-turbo's SIMD does) and IDCT: one uint8 plane per component, whole
    blocks."""
    planes = []
    for c, cf in enumerate(coef):
        bh, bw = cf.shape[:2]
        q = ((cf * info.qt[c] + 32768) & 0xFFFF) - 32768
        x = q.reshape(bh, bw, 8, 8).transpose(2, 3, 0, 1)          # (row u, column v, by, bx)
        ws = _idct_1d(x, 11)                                        # columns: over u
        out = _idct_1d(ws.transpose(1, 0, 2, 3), 18).transpose(1, 0, 2, 3)   # rows: over v
        out = np.clip(out + 128, 0, 255).astype(np.uint8)           # (y, x, by, bx)
        planes.append(out.transpose(2, 0, 3, 1).reshape(bh * 8, bw * 8))
    return planes


def _fancy_h(p, cw):
    """h2v1 triangle filter over the first cw columns of p (int64), edge columns repeated."""
    p = p[:, :cw]
    left = np.concatenate([p[:, :1], p[:, :-1]], 1)
    right = np.concatenate([p[:, 1:], p[:, -1:]], 1)
    return left, right


def model_upsample(info, plane, rows_scale):
    """Chroma plane (component 1 or 2) at full resolution (h, w), as libjpeg-turbo's fancy upsampler."""
    h, w = info.h, info.w
    cw, ch = -(-w // info.hs), -(-h // info.vs)
    p = plane[:ch, :cw].astype(np.int64)
    if info.hs == 1 and info.vs == 1:
        return p
    if info.hs == 2 and cw <= 2:                                     # libjpeg falls back to box for narrow planes
        return np.repeat(np.repeat(p, 2, 1), info.vs, 0)[:h, :w]
    if info.vs == 2:
        above = np.concatenate([p[:1], p[:-1]], 0)
        below = np.concatenate([p[1:], p[-1:]], 0)
        sums = np.empty((2 * ch, cw), np.int64)
        sums[0::2] = 3 * p + above
        sums[1::2] = 3 * p + below
        if info.hs == 1:
            out = np.empty_like(sums)
            out[0::2] = (sums[0::2] + 1) >> 2
            out[1::2] = (sums[1::2] + 2) >> 2
            return out[:h, :w]
        left, right = _fancy_h(sums, cw)
        out = np.empty((2 * ch, 2 * cw), np.int64)
        out[:, 0::2] = (3 * sums + left + 8) >> 4
        out[:, 1::2] = (3 * sums + right + 7) >> 4
        return out[:h, :w]
    left, right = _fancy_h(p, cw)
    out = np.empty((ch, 2 * cw), np.int64)
    out[:, 0::2] = (3 * p + left + 1) >> 2
    out[:, 1::2] = (3 * p + right + 2) >> 2
    return out[:h, :w]


def model_decode(data):
    """The three device stages on the host: BGR uint8, orientation applied."""
    info = jpeg.parse(data)
    assert info.eligible, info.reason
    planes = model_planes(info, model_coefficients(info, data))
    y = planes[0][:info.h, :info.w].astype(np.int64)
    if info.ncomp == 1:
        bgr = np.stack([y, y, y], -1)
    else:
        cb = model_upsample(info, planes[1], None) - 128
        cr = model_upsample(info, planes[2], None) - 128
        r = y + ((91881 * cr + 32768) >> 16)
        g = y + ((-46802 * cr - 22554 * cb + 32768) >> 16)
        b = y + ((116130 * cb + 32768) >> 16)
        bgr = np.stack([b, g, r], -1)
    bgr = np.clip(bgr, 0, 255).astype(np.uint8)
    o = info.orientation                        # OpenCV's ApplyExifOrientation: transpose for 5-8, then flips
    if o >= 5:
        bgr = bgr.transpose(1, 0, 2)
    if o in (2, 3, 6, 7):
        bgr = bgr[:, ::-1]
    if o in (3, 4, 7, 8):
        bgr = bgr[::-1]
    return np.ascontiguousarray(bgr)


# ---- parser -----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("sampling", ["444", "422", "440", "420", "gray"])
@pytest.mark.parametrize("variant", ["baseline", "optimize", "rst1", "rst3", "rst100"])
def test_parser_accepts_device_files(sampling, variant):
    im = make_image(40, 56, "smooth_noise", 1, gray=sampling == "gray")
    rst = int(variant[3:]) if variant.startswith("rst") else 0
    data = encode(im, 75, sampling, rst=rst, optimize=variant == "optimize")
    info = jpeg.parse(data, "x.jpg")
    assert info.eligible, info.reason
    assert (info.oh, info.ow) == (40, 56) and info.ncomp == (1 if sampling == "gray" else 3)
    mx, my = info.mcu
    assert len(info.segments) == (-(-mx * my // rst) if rst else 1)
    assert info.restart_interval == rst
    assert (info.segments[:, 0] < info.segments[:, 1]).all()


@pytest.mark.parametrize("kind", ["411", "progressive", "png"])
def test_parser_sends_other_files_to_the_host(kind):
    im = make_image(24, 40, "smooth", 2)
    if kind == "png":
        with pytest.raises(ValueError, match="a.png"):
            jpeg.parse(cv2.imencode(".png", im)[1].tobytes(), "a.png")
        return
    data = encode(im, 75, "411") if kind == "411" else encode(im, 75, "420", progressive=True)
    info = jpeg.parse(data, "a.jpg")
    assert not info.eligible and info.reason
    assert (info.oh, info.ow) == (24, 40)


@pytest.mark.parametrize("orientation", range(1, 9))
@pytest.mark.parametrize("big_endian", [False, True])
def test_parser_reads_exif_orientation(orientation, big_endian):
    im = make_image(24, 40, "smooth_noise", 3)
    data = with_exif(encode(im, 90, "420"), orientation, big_endian)
    info = jpeg.parse(data)
    assert info.orientation == orientation
    want = cv2_decode(data)
    assert (info.oh, info.ow) == want.shape[:2] == ((40, 24) if orientation >= 5 else (24, 40))
    assert np.array_equal(model_decode(data), want)


def test_parser_rejects_bad_headers_naming_the_image():
    data = encode(make_image(16, 16, "noise", 4), 75, "420")
    sos = data.index(b"\xFF\xDA")
    dqt = data.index(b"\xFF\xDB")
    dht = data.index(b"\xFF\xC4")
    bad = {
        "cut_in_header": data[:sos - 7],
        "long_segment": data[:dqt + 2] + b"\xFF\xFF" + data[dqt + 4:],
        "zero_size": data.replace(b"\xFF\xC0\x00\x11\x08\x00\x10\x00\x10", b"\xFF\xC0\x00\x11\x08\x00\x00\x00\x10"),
        "bad_prefix_code": data[:dht + 5] + bytes([3]) + data[dht + 6:],
        "undefined_table": data[:sos + 6] + bytes([0x33]) + data[sos + 7:],
        "no_soi": data[2:],
    }
    assert bad["zero_size"] != data
    for what, b in bad.items():
        with pytest.raises(ValueError, match="img_%s.jpg" % what):
            jpeg.parse(b, "img_%s.jpg" % what)


def test_truncated_entropy_data_still_parses_and_the_model_flags_it():
    data = encode(make_image(64, 64, "noise", 5), 90, "420")
    cut = data[:len(data) // 2]
    info = jpeg.parse(cut)
    assert info.eligible and info.segments[-1, 1] == len(cut)
    with pytest.raises(ValueError, match="data ends"):
        model_coefficients(info, cut)


# ---- the model against cv2.imdecode ------------------------------------------------------------------------------------

@pytest.mark.parametrize("sampling", ["444", "422", "440", "420", "gray"])
@pytest.mark.parametrize("quality", QUALITIES)
def test_model_equals_cv2_imdecode(sampling, quality):
    n = 0
    for h, w in SIZES:
        for content in CONTENTS:
            for rst in (0, 2):
                if (h * w > 1000 and quality not in (50, 95)) or (rst and h * w > 1000):
                    continue                                 # the plain-Python entropy decode is slow
                im = make_image(h, w, content, h * 1000 + w + quality, gray=sampling == "gray")
                data = encode(im, quality, sampling, rst=rst)
                got, want = model_decode(data), cv2_decode(data)
                assert got.shape == want.shape, (h, w, content, rst)
                assert np.array_equal(got, want), (h, w, content, rst, int((got != want).sum()))
                n += 1
    assert n >= 30


def test_pack_lays_out_tables_segments_and_files():
    """The launch buffer read back on the host: every entry's Huffman tables, segment ranges and file bytes sit at
    its offsets, workspace ranges do not overlap, and the quantisation tables are in natural order."""
    files = [encode(make_image(40, 56, "noise", 7), 75, "420", rst=3), encode(make_image(9, 11, "smooth", 8, True), 50,
             "gray"), encode(make_image(33, 47, "smooth_noise", 9), 95, "444", optimize=True)]
    infos = [jpeg.parse(d) for d in files]
    dst = [0, 1000, 5000]
    buf, ws = jpeg.pack(infos, files, dst)
    table = buf[:len(files) * jpeg.JPEG_IMAGE.itemsize].view(jpeg.JPEG_IMAGE)
    end = 0
    for e, info, data, d in zip(table, infos, files, dst):
        assert e["dst_offset"] == d and (e["h"], e["w"], e["ncomp"]) == (info.h, info.w, info.ncomp)
        assert e["seg_offset"] % 8 == 0 and e["huff_offset"] % 4 == 0 and e["coef_offset"] % 16 == 0
        assert e["coef_offset"] == end and e["plane_offset"] - e["coef_offset"] == info.workspace_bytes() * 2 // 3
        end = e["coef_offset"] + info.workspace_bytes()
        segs = buf[e["seg_offset"]:e["seg_offset"] + 16 * e["nseg"]].view("<i8").reshape(-1, 2)
        base = segs[0, 0] - info.segments[0, 0]
        assert np.array_equal(segs - base, info.segments)
        assert buf[base:base + len(data)].tobytes() == data
        huff = buf[e["huff_offset"]:].view(np.uint8)
        for c in range(info.ncomp):
            assert np.array_equal(e["qt"][c], info.qt[c])
            for tbl, cls, tid in ((int(e["dc_tbl"][c]), 0, info.dc[c]), (int(e["ac_tbl"][c]), 1, info.ac[c])):
                got = huff[tbl * jpeg.HUFF.itemsize:(tbl + 1) * jpeg.HUFF.itemsize].view(jpeg.HUFF)[0]
                assert got.tobytes() == info.huff[(cls, tid)][2].tobytes()
    assert ws == end
