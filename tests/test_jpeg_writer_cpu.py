"""CPU tests of the JPEG parser and the numpy models of the device stages on files from tests/jpeg_writer.py, which
cv2.imencode cannot write: 16-bit DQT, table ids 0-3, long-code, single-symbol and all-ones Huffman tables, arbitrary
component ids, tables after SOF, fill bytes, missing EOI, custom progressive scripts with refinement and long EOB runs,
and blocks around the IDCT's 16-bit range.  Every file's route (device, flagged on the device, host, refused) is pinned
against ``jpeg.parse``, and every file the device decodes is pinned against cv2.imdecode through the models."""
import numpy as np
import pytest

from centerpose_b200 import jpeg
from tests import jpeg_writer as jw
from tests.test_jpeg_cpu import cv2_decode, model_decode
from tests.test_jpeg_progressive_cpu import model_progressive_decode

CASES = {c.name: c for c in jw.corpus()}


def _verdict(data):
    try:
        info = jpeg.parse(data, "w.jpg")
    except ValueError as e:
        return "raise", str(e)
    if info.eligible or info.progressive:
        return "device", ""
    return "host", info.reason


def test_corpus_reaches_every_knob():
    routes = {c.route for c in CASES.values()}
    assert routes == {"device", "range", "corrupt", "no_eoi", "host", "raise"}
    assert len(CASES) >= 130
    infos = [jpeg.parse(c.data) for c in CASES.values() if c.route == "device"]
    assert {(i.hs, i.vs) for i in infos if i.ncomp == 3} == {(1, 1), (2, 1), (1, 2), (2, 2)}
    assert any(i.ncomp == 1 for i in infos) and any(i.progressive for i in infos)
    assert {i.restart_interval for i in infos if i.eligible} >= {0, 1, 3, 1000}
    tables = [t for i in infos for t in ([i.huff[k][2] for k in i.huff] if i.eligible else i.tables)]
    assert any((t["maxcode"][16] >= 0) for t in tables)                         # 16-bit codes
    assert any((t["lut"] == 0).sum() > 256 for t in tables)                      # mostly longer than LUT_BITS
    assert any((t["maxcode"][2:17] < 0).all() for t in tables)                   # one 1-bit code
    scans = [s for i in infos if i.progressive for s in i.progressive]
    assert any(s.ah and s.ss for s in scans) and any(s.ah and not s.ss for s in scans)
    assert any(len(s.comps) == 1 and not s.ss for s in scans)
    assert len({s.restart_interval for s in scans}) >= 4


@pytest.mark.parametrize("name", list(CASES))
def test_parser_routes_writer_files(name):
    """``jpeg.parse`` sends each file where the corpus says: the device (its kernels decide status), the host with the
    expected reason, or a ValueError naming the image."""
    case = CASES[name]
    route, why = _verdict(case.data)
    want = "device" if case.route in ("device", "range", "corrupt", "no_eoi") else case.route
    assert route == want, (route, why)
    assert case.why in why
    if route == "device":
        assert jpeg.parse(case.data).eoi == (case.route != "no_eoi")


@pytest.mark.parametrize("name", [n for n, c in CASES.items() if c.route in ("device", "range")])
def test_device_files_decode_in_cv2(name):
    """No file the device is expected to decode with status 0 is one cv2 refuses (an all-ones Huffman code was the
    first such file), and out-of-range files decode in cv2 too, so the host fall-back returns an image."""
    assert cv2_decode(CASES[name].data) is not None


@pytest.mark.parametrize("name", [n for n, c in CASES.items() if c.route == "raise"])
def test_refused_files_are_refused_by_cv2(name):
    assert cv2_decode(CASES[name].data) is None


@pytest.mark.parametrize("name", [n for n, c in CASES.items() if c.route == "device"])
def test_models_equal_cv2_on_device_files(name):
    """The sequential or progressive entropy model, then the IDCT and colour models, equal cv2.imdecode byte for byte
    on every file the device decodes: legitimate-regime files, sparse and extreme blocks inside the IDCT range (peak
    exactly +-IDCT_RANGE included), DC categories 0-11, 16-bit quantisers and EOB runs of 32767 blocks."""
    data = CASES[name].data
    info = jpeg.parse(data)
    got = (model_progressive_decode if info.progressive else model_decode)(data)
    want = cv2_decode(data)
    assert got.shape == want.shape and np.array_equal(got, want), int((got != want).sum())


def test_range_routes_follow_the_block_peaks():
    """The boundary files sit on both sides of IDCT_RANGE: peaks of exactly IDCT_RANGE - 1 and IDCT_RANGE are
    decoded, IDCT_RANGE + 1 is flagged; a DC-only block of 4095 (pass 1: 16380) is decoded, 4096 flagged."""
    for name, want in (("boundary_16382", "device"), ("boundary_16383", "device"), ("boundary_16384", "range"),
                       ("dc_only_4095", "device"), ("dc_only_4096", "range")):
        assert CASES[name].route == want, name
    assert sum(c.route == "range" for c in CASES.values()) >= 10


def test_build_huff_refuses_an_all_ones_code():
    """The Annex K DC luminance table plus one 9-bit code: that code is 111111111, which libjpeg refuses (the next code
    after each length must still fit in that many bits)."""
    bits, vals = jw._annex_k()[0][(0, 0)]
    jpeg.build_huff(bits, vals, "ok.jpg", True)
    bits = list(bits)
    bits[8] += 1
    with pytest.raises(ValueError, match="ones.jpg"):
        jpeg.build_huff(bits, vals + [12], "ones.jpg", True)
    # a full code space one level down is refused the same way: two 1-bit codes
    with pytest.raises(ValueError, match="all-ones"):
        jpeg.build_huff([2] + [0] * 15, [0, 1], "x.jpg", True)
    jpeg.build_huff([1] + [0] * 15, [0], "x.jpg", True)


@pytest.mark.parametrize("progressive", [False, True])
def test_files_without_eoi_are_flagged_in_the_table(progressive):
    """cv2.imencode's own files cut just before EOI, and cut inside their last scan: ``eoi`` is False and ``pack``
    sets the entry's ``missing_eoi``, so the kernels give status 1 and cv2.imread decides.  With EOI, and with bytes
    after it, the flag is clear; with EOI after a cut the kernels find the missing data themselves."""
    from tests.test_jpeg_cpu import encode, make_image
    data = encode(make_image(40, 56, "smooth_noise", 3), 90, "420", progressive=progressive)
    assert data.endswith(b"\xFF\xD9")
    sos = data.rindex(b"\xFF\xDA")
    files = [data[:-2], data[:(sos + len(data)) // 2], data, data + b"trailing bytes",
             data[:(sos + len(data)) // 2] + b"\xFF\xD9"]
    infos = [jpeg.parse(d) for d in files]
    assert all(i.eligible or i.progressive for i in infos)
    assert [i.eoi for i in infos] == [False, False, True, True, True]
    buf, _ = jpeg.pack(infos, files, [0] * len(files))
    assert buf[:len(files) * jpeg.JPEG_IMAGE.itemsize].view(jpeg.JPEG_IMAGE)["missing_eoi"].tolist() == [1, 1, 0, 0, 0]


@pytest.mark.parametrize("name", [n for n, c in CASES.items() if n.startswith("cut_")])
def test_models_flag_data_ending_before_the_last_unit(name):
    """Files cut inside their last scan with EOI after the cut reach the kernels; the entropy models (as the kernels)
    run out of data or read a symbol they refuse."""
    from tests.test_jpeg_cpu import model_coefficients
    from tests.test_jpeg_progressive_cpu import model_progressive_coefficients
    data = CASES[name].data
    info = jpeg.parse(data)
    assert info.eoi
    with pytest.raises(ValueError, match="data ends|run past|refinement size"):   # zeros past the cut may decode
        (model_progressive_coefficients if info.progressive else model_coefficients)(info, data)
