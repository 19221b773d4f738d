"""CPU tests of progressive JPEG decoding's host side: the parser's scan list and the progressive files it sends to
the host (centerpose_b200/jpeg.py), ``pack`` with progressive and sequential entries, and a numpy model of the
progressive entropy stage (T.81 G.1.2 as libjpeg-turbo's jdphuff.c) that, followed by the IDCT and colour stages of
tests/test_jpeg_cpu.py, equals cv2.imdecode byte for byte."""
import numpy as np
import pytest

from centerpose_b200 import jpeg
from tests.test_jpeg_cpu import (CONTENTS, QUALITIES, SAMPLINGS, SIZES, _segment_bits, cv2_decode, encode, make_image,
                                 model_planes, model_upsample)

RESTARTS = [0, 1, 3, 100]


def penc(im, quality=75, sampling="420", rst=0):
    return encode(im, quality, sampling, rst=rst, progressive=True)


# ---- the numpy model of the progressive entropy stage ------------------------------------------------------------------

class _Reader:
    """MSB-first bits of one segment (stuffing removed, reading stops at a marker), zeros past its end."""

    def __init__(self, data, start, end):
        self.s = (_segment_bits(data, start, end) + 48).tobytes().decode()
        self.real = len(self.s)
        self.pos = 0

    def get(self, n):
        v = self.s[self.pos:self.pos + n].ljust(n, "0")
        self.pos += n
        return int(v, 2) if n else 0

    def symbol(self, t):
        """T.81 F.2.2.3 DECODE over the table's maxcode / valptr."""
        for ln in range(1, 17):
            code = int(self.s[self.pos:self.pos + ln].ljust(ln, "0"), 2)
            if code <= t["maxcode"][ln]:
                self.pos += ln
                return int(t["val"][code + t["valoff"][ln]])
        raise ValueError("code longer than 16 bits")


def _extend(v, s):
    return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v


def _w16(v):
    """libjpeg's JCOEF store: the low 16 bits, signed."""
    return ((v + 32768) & 0xFFFF) - 32768


def _unit_blocks(info, scan, coef, u):
    """(scan component index, block) of unit u: an MCU of every scan component, or one block of the component's own
    grid."""
    if len(scan.comps) > 1:
        my, mx = divmod(u, info.mcu[0])
        for i, c in enumerate(scan.comps):
            hs, vs = (info.hs, info.vs) if c == 0 else (1, 1)
            for dy in range(vs):
                for dx in range(hs):
                    yield i, coef[scan.comps[i]][my * vs + dy, mx * hs + dx]
    else:
        by, bx = divmod(u, info.coded_blocks(scan.comps[0])[0])
        yield 0, coef[scan.comps[0]][by, bx]


def _refine(blk, pos, r, p1, m1):
    if r.get(1) and not blk[pos] & p1:
        blk[pos] = _w16(blk[pos] + (p1 if blk[pos] >= 0 else m1))


def model_progressive_coefficients(info, data):
    """Every scan in file order into zeroed blocks: per component an int64 array (block rows, blocks per row, 64) in
    natural order, whole MCUs."""
    Z = jpeg.ZIGZAG
    coef = [np.zeros((bh, bw, 64), np.int64) for bw, bh in info.blocks()]
    for sc in info.progressive:
        total = sc.units(info)
        ri = sc.restart_interval or total
        ss, se, ah, al = sc.ss, sc.se, sc.ah, sc.al
        p1, m1 = 1 << al, -(1 << al)
        for q, (start, end) in enumerate(sc.segments):
            r = _Reader(data, start, end)
            pred, eobrun = [0] * len(sc.comps), 0
            for u in range(q * ri, min((q + 1) * ri, total)):
                for i, blk in _unit_blocks(info, sc, coef, u):
                    if ss == 0 and ah == 0:
                        s = r.symbol(info.tables[sc.dc[i]])
                        pred[i] += _extend(r.get(s), s)
                        blk[0] = _w16(pred[i] << al)
                    elif ss == 0:
                        if r.get(1):
                            blk[0] = _w16(blk[0] | p1)
                    elif ah == 0:
                        if eobrun:
                            eobrun -= 1
                            continue
                        k = ss
                        while k <= se:
                            sym = r.symbol(info.tables[sc.ac[0]])
                            run, s = sym >> 4, sym & 15
                            if s:
                                k += run
                                if k > se:
                                    raise ValueError("run past Se")
                                blk[Z[k]] = _w16(_extend(r.get(s), s) << al)
                            elif run == 15:
                                k += 15
                            else:
                                eobrun = (1 << run) - 1 + r.get(run)
                                break
                            k += 1
                    else:
                        k = ss
                        if not eobrun:
                            while k <= se:
                                sym = r.symbol(info.tables[sc.ac[0]])
                                run, s, v = sym >> 4, sym & 15, 0
                                if s:
                                    if s != 1:
                                        raise ValueError("refinement size %d" % s)
                                    v = p1 if r.get(1) else m1
                                elif run != 15:
                                    eobrun = (1 << run) + r.get(run)
                                    break
                                while k <= se:            # correction bits; the zero run counts zero-history ones
                                    if blk[Z[k]]:
                                        _refine(blk, Z[k], r, p1, m1)
                                    else:
                                        run -= 1
                                        if run < 0:
                                            break
                                    k += 1
                                if v:
                                    if k > se:
                                        raise ValueError("run past Se")
                                    blk[Z[k]] = v
                                k += 1
                        if eobrun:
                            for k in range(k, se + 1):
                                if blk[Z[k]]:
                                    _refine(blk, Z[k], r, p1, m1)
                            eobrun -= 1
                if r.pos > r.real:
                    raise ValueError("data ends before the segment's last unit")
    return coef


def model_progressive_decode(data):
    """The progressive entropy model, then the IDCT, upsampling and colour stages: BGR uint8, orientation applied."""
    info = jpeg.parse(data)
    assert info.progressive, info.reason
    planes = model_planes(info, model_progressive_coefficients(info, data))
    y = planes[0][:info.h, :info.w].astype(np.int64)
    if info.ncomp == 1:
        bgr = np.stack([y, y, y], -1)
    else:
        cb = model_upsample(info, planes[1], None) - 128
        cr = model_upsample(info, planes[2], None) - 128
        bgr = np.stack([y + ((116130 * cb + 32768) >> 16), y + ((-46802 * cr - 22554 * cb + 32768) >> 16),
                        y + ((91881 * cr + 32768) >> 16)], -1)
    bgr = np.clip(bgr, 0, 255).astype(np.uint8)
    o = info.orientation
    if o >= 5:
        bgr = bgr.transpose(1, 0, 2)
    if o in (2, 3, 6, 7):
        bgr = bgr[:, ::-1]
    if o in (3, 4, 7, 8):
        bgr = bgr[::-1]
    return np.ascontiguousarray(bgr)


# ---- an independent walk over the file's markers ------------------------------------------------------------------------

def _walk(data):
    """(marker, payload offset, payload end) of every marker segment, and (0xDA, data start, data end) after each SOS
    for its entropy-coded data (RST markers included), found byte by byte."""
    out, pos, n = [], 2, len(data)
    while pos + 1 < n:
        m = data[pos + 1]
        if m == 0xD9:
            break
        ln = (data[pos + 2] << 8) | data[pos + 3]
        out.append((m, pos + 4, pos + 2 + ln))
        pos += 2 + ln
        if m == 0xDA:
            start = pos
            while pos + 1 < n and not (data[pos] == 0xFF and data[pos + 1] not in (0,) + tuple(range(0xD0, 0xD8))):
                pos += 1
            out.append((None, start, pos))
    return out


# ---- parser -----------------------------------------------------------------------------------------------------------

# libjpeg's jpeg_simple_progression (what cv2 writes with IMWRITE_JPEG_PROGRESSIVE): (components, Ss, Se, Ah, Al)
SIMPLE_YCC = [([0, 1, 2], 0, 0, 0, 1), ([0], 1, 5, 0, 2), ([2], 1, 63, 0, 1), ([1], 1, 63, 0, 1), ([0], 6, 63, 0, 2),
              ([0], 1, 63, 2, 1), ([0, 1, 2], 0, 0, 1, 0), ([2], 1, 63, 1, 0), ([1], 1, 63, 1, 0), ([0], 1, 63, 1, 0)]
SIMPLE_GRAY = [([0], 0, 0, 0, 1), ([0], 1, 5, 0, 2), ([0], 6, 63, 0, 2), ([0], 1, 63, 2, 1), ([0], 0, 0, 1, 0),
               ([0], 1, 63, 1, 0)]


@pytest.mark.parametrize("sampling", ["444", "422", "440", "420", "gray"])
@pytest.mark.parametrize("rst", RESTARTS)
def test_parser_reads_the_scan_list(sampling, rst):
    """Scans, Ss / Se / Ah / Al, the tables each scan binds (those of the DHT segments before its SOS) and the
    segments of each scan, against a byte-by-byte walk of the file."""
    im = make_image(40, 56, "smooth_noise", 1, gray=sampling == "gray")
    data = penc(im, 75, sampling, rst)
    info = jpeg.parse(data, "p.jpg")
    assert not info.eligible and info.reason and info.progressive, info.reason
    assert (info.oh, info.ow) == (40, 56)
    want = SIMPLE_GRAY if sampling == "gray" else SIMPLE_YCC
    assert [(s.comps, s.ss, s.se, s.ah, s.al) for s in info.progressive] == want
    cids = list(data[data.index(b"\xFF\xC2") + 10::3][:info.ncomp])
    huff, k = {}, 0
    walk = _walk(data)
    for (m, a, b), nxt in zip(walk, walk[1:] + [None]):
        if m == 0xC4:
            jpeg._read_dht(data[a:b], huff, "p.jpg")
        elif m == 0xDA:
            sc = info.progressive[k]
            ns = data[a]
            assert [cids.index(data[a + 1 + 2 * i]) for i in range(ns)] == sc.comps
            for i in range(ns):
                td, ta = data[a + 2 + 2 * i] >> 4, data[a + 2 + 2 * i] & 15
                if sc.ss:
                    assert info.tables[sc.ac[i]].tobytes() == huff[(1, ta)][2].tobytes()
                elif not sc.ah:
                    assert info.tables[sc.dc[i]].tobytes() == huff[(0, td)][2].tobytes()
            assert sc.restart_interval == rst
            units = sc.units(info)
            assert len(sc.segments) == (-(-units // rst) if rst else 1)
            assert sc.segments[0, 0] == nxt[1] and sc.segments[-1, 1] == nxt[2]
            assert (sc.segments[:, 0] < sc.segments[:, 1]).all()
            k += 1
    assert k == len(want)


def _sos(data, k):
    """Byte offset of the k-th SOS marker."""
    pos = -1
    for _ in range(k + 1):
        pos = data.index(b"\xFF\xDA", pos + 1)
    return pos


def _host_files():
    data = penc(make_image(48, 64, "smooth_noise", 2), 80, "420")
    s4, s5 = _sos(data, 4), _sos(data, 5)          # scan 4: Y 6..63 Ah 0 Al 2; scan 5: Y 1..63 Ah 2 Al 1
    dht = data.rindex(b"\xFF\xC4", 0, s5)
    edit = lambda at, v: data[:at] + bytes([v]) + data[at + 1:]
    return {
        "cut_between_scans": (data[:s5], "ends between scans"),
        "cut_after_scan_data": (data[:dht], "incomplete"),
        "cut_in_table_between_scans": (data[:dht + 10], "ends between scans"),
        "al_above_13": (edit(s4 + 9, 0x0E), "illegal"),       # SOS: FF DA, length, Ns=1, Cs/Td:Ta, Ss, Se, Ah:Al
        "se_below_ss": (edit(s4 + 8, 5), "illegal"),
        "overlapping_first_scans": (edit(s4 + 7, 5), "inconsistent"),
        "refinement_of_unsent_bits": (edit(s5 + 9, 0x32), "inconsistent"),
        "dqt_between_scans": (data[:s5] + b"\xFF\xDB\x00\x43\x01" + bytes(range(1, 65)) + data[s5:], "0xDB"),
        "411": (penc(make_image(48, 64, "smooth", 3), 75, "411"), "sampling"),
    }


@pytest.mark.parametrize("kind", list(_host_files()))
def test_parser_sends_other_progressive_files_to_the_host(kind):
    data, why = _host_files()[kind]
    info = jpeg.parse(data, "h.jpg")
    assert not info.eligible and info.progressive is None
    assert why in info.reason, info.reason


def test_parser_caps_the_scan_count(monkeypatch):
    data = penc(make_image(24, 40, "noise", 4), 75, "420")
    assert len(jpeg.parse(data).progressive) == 10
    monkeypatch.setattr(jpeg, "MAX_SCANS", 9)
    info = jpeg.parse(data)
    assert info.progressive is None and "more than 9 scans" in info.reason


def test_truncated_last_scan_still_parses_and_the_model_flags_it():
    data = penc(make_image(64, 64, "noise", 5), 90, "420")
    cut = data[:(_sos(data, 9) + len(data)) // 2]
    info = jpeg.parse(cut)
    assert info.progressive and info.progressive[-1].segments[-1, 1] == len(cut)
    with pytest.raises(ValueError, match="data ends|run past Se"):    # zeros read past the cut may decode as a run
        model_progressive_coefficients(info, cut)


# ---- the model against cv2.imdecode ------------------------------------------------------------------------------------

@pytest.mark.parametrize("sampling", ["444", "422", "440", "420", "gray"])
@pytest.mark.parametrize("quality", QUALITIES)
def test_progressive_model_equals_cv2_imdecode(sampling, quality):
    n = 0
    for h, w in SIZES:
        for j, content in enumerate(CONTENTS):
            rst = RESTARTS[(j + h + quality) % len(RESTARTS)]     # every interval across the grid
            im = make_image(h, w, content, h * 1000 + w + quality, gray=sampling == "gray")
            data = penc(im, quality, sampling, rst)
            got, want = model_progressive_decode(data), cv2_decode(data)
            assert got.shape == want.shape, (h, w, content, rst)
            assert np.array_equal(got, want), (h, w, content, rst, int((got != want).sum()))
            n += 1
    assert n == len(SIZES) * len(CONTENTS)


def test_pack_lays_out_progressive_next_to_sequential_entries():
    """The launch buffer read back on the host: the scan records, their segments and tables sit at the offsets of
    each progressive entry, the sequential entries keep their layout, workspace ranges follow each other."""
    files = [penc(make_image(40, 56, "noise", 7), 75, "420", rst=3), encode(make_image(9, 11, "smooth", 8), 50, "444"),
             penc(make_image(33, 47, "smooth_noise", 9, True), 95, "gray"), penc(make_image(17, 23, "noise", 6), 60, "422")]
    infos = [jpeg.parse(d) for d in files]
    assert [i.progressive is not None for i in infos] == [True, False, True, True]
    dst = [0, 1000, 5000, 9000]
    buf, ws = jpeg.pack(infos, files, dst)
    table = buf[:len(files) * jpeg.JPEG_IMAGE.itemsize].view(jpeg.JPEG_IMAGE)
    end = 0
    for e, info, data, d in zip(table, infos, files, dst):
        assert e["dst_offset"] == d and (e["h"], e["w"], e["ncomp"], e["hs"], e["vs"]) == \
            (info.h, info.w, info.ncomp, info.hs, info.vs)
        assert e["coef_offset"] == end and e["plane_offset"] - e["coef_offset"] == info.workspace_bytes() * 2 // 3
        end = e["coef_offset"] + info.workspace_bytes()
        for c in range(info.ncomp):
            assert np.array_equal(e["qt"][c], info.qt[c])
        if info.progressive is None:
            assert e["nscan"] == 0 and e["nseg"] == len(info.segments)
            continue
        assert e["nscan"] == len(info.progressive) and e["scan_offset"] % 8 == 0 and e["huff_offset"] % 4 == 0
        scans = buf[e["scan_offset"]:e["scan_offset"] + e["nscan"] * jpeg.SCAN.itemsize].view(jpeg.SCAN)
        base = None
        for rec, sc in zip(scans, info.progressive):
            k = len(sc.comps)
            assert (rec["ncomp"], rec["ss"], rec["se"], rec["ah"], rec["al"], rec["restart_interval"]) == \
                (k, sc.ss, sc.se, sc.ah, sc.al, sc.restart_interval)
            assert list(rec["comp"][:k]) == sc.comps and rec["seg_offset"] % 8 == 0
            segs = buf[rec["seg_offset"]:rec["seg_offset"] + 16 * rec["nseg"]].view("<i8").reshape(-1, 2)
            base = segs[0, 0] - sc.segments[0, 0] if base is None else base
            assert np.array_equal(segs - base, sc.segments)
            for tbl, want in zip(list(rec["dc_tbl"][:k]) + list(rec["ac_tbl"][:k]), sc.dc + sc.ac):
                assert tbl == want
        assert buf[base:base + len(data)].tobytes() == data
        huff = buf[e["huff_offset"]:e["huff_offset"] + len(info.tables) * jpeg.HUFF.itemsize].view(jpeg.HUFF)
        assert all(a.tobytes() == b.tobytes() for a, b in zip(huff, info.tables))
    assert ws == end
