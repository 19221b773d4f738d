"""GPU tests of the device PNG decoder: cpb200_png_decode_batch against cv2.imread over the CPU test matrix in one
launch, its status on corrupt streams, and MultiPoseDetector.run_images on PNG paths against run_images on the
cv2.imread arrays."""
import struct
import zlib

import cv2
import numpy as np
import pytest
import torch

from centerpose_b200 import png
from tests.test_jpeg_cpu import encode, make_image
from tests.test_jpeg_gpu import _detector
from tests.test_png_cpu import (COMBOS, chunk, cv2_decode, exif, matrix, palette_for, samples, write_png)

pytestmark = pytest.mark.gpu
CPB200_ERR_ARG = 1


def _launch(src, table, B, ws, ws_bytes, dst, status):
    from centerpose_b200 import _lib
    return _lib.lib().cpb200_png_decode_batch(src, table, B, ws, ws_bytes, dst, status,
                                              torch.cuda.current_stream().cuda_stream)


def _decode(datas):
    """One launch over all files; returns (images, status) after checking the bytes behind the last image were left
    alone."""
    from centerpose_b200 import _lib
    infos = [png.parse(d) for d in datas]
    assert all(i.eligible for i in infos)
    sizes = [i.oh * i.ow * 3 for i in infos]
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    buf, ws_bytes = png.pack(infos, datas, offs[:-1])
    src = torch.from_numpy(buf).cuda()
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    dst = torch.full((int(offs[-1]) + 256,), 77, dtype=torch.uint8, device="cuda")
    status = torch.full((len(datas),), -1, dtype=torch.int32, device="cuda")
    _lib.check(_launch(src.data_ptr(), src.data_ptr(), len(datas), ws.data_ptr(), ws_bytes, dst.data_ptr(),
                       status.data_ptr()), "png_decode_batch")
    out = dst.cpu().numpy()
    assert (out[offs[-1]:] == 77).all()
    return [out[offs[n]:offs[n + 1]].reshape(i.oh, i.ow, 3) for n, i in enumerate(infos)], status.cpu().numpy()


def _extra_files():
    """COCO-sized files from cv2.imwrite at compression 1 and 9, interlaced ones, split IDAT, EXIF orientations."""
    files = []
    for k, (h, w) in enumerate([(480, 640), (427, 640)]):
        im = make_image(h, w, "smooth_noise", k)
        for level in (1, 9):
            files.append(cv2.imencode(".png", im, [cv2.IMWRITE_PNG_COMPRESSION, level])[1].tobytes())
        files.append(write_png(im[:97, :203, ::-1].astype(np.uint16), 2, 8, 1, filters=[4, 1, 3]))
    for o in range(1, 9):
        files.append(write_png(samples(11, 17, 6, 8, o), 6, 8, o % 2, before=chunk(b"eXIf", exif(o))))
    files.append(write_png(samples(31, 29, 3, 2, 3), 3, 2, 1, palette=palette_for(2, 3), idat_split=5))
    return files


def test_png_kernel_equals_cv2_imread():
    """The CPU matrix (every colour type x depth, interlaced or not, all five filters, stored / fixed / dynamic
    blocks, 1x1 to 70x9) plus COCO-sized and orientation files, mixed in one launch, byte for byte."""
    files = [d for _, d in matrix()] + _extra_files()
    got, status = _decode(files)
    assert (status == 0).all(), np.flatnonzero(status)
    bad = [n for n, (g, d) in enumerate(zip(got, files)) if not np.array_equal(g, cv2_decode(d))]
    assert not bad, (len(bad), bad[:10])


def test_png_batched_equals_single_image_calls():
    files = [d for _, d in matrix()][::11] + _extra_files()[:3]
    batched, _ = _decode(files)
    for d, b in zip(files, batched):
        single, status = _decode([d])
        assert status[0] == 0 and np.array_equal(single[0], b)


def _zfile(z, w=16, h=8):
    """An RGB file of w x h, or 8-bit gray for 1 x 1, around zlib stream z."""
    ct = 0 if (w, h) == (1, 1) else 2
    return png.SIGNATURE + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, ct, 0, 0, 0)) + chunk(b"IDAT", z) + \
        chunk(b"IEND", b"")


def _corrupt():
    """Streams the device must refuse, each with a status: bad Adler-32, a bad Huffman code, a distance before the
    start of the data, a bad zlib header, too little data, a bad filter type, an incomplete literal / length code."""
    raw = b"".join(b"\x01" + bytes(range(k, k + 48)) for k in range(8))
    z = zlib.compress(raw, 9)
    out = {"adler": _zfile(z[:-1] + bytes([z[-1] ^ 1])),
           "header": _zfile(bytes([0x78, 0x9D]) + z[2:])}
    # a dynamic block header whose code-length code lengths over-subscribe: HCLEN 4, all of length 1
    bits = [0, 0, 1] + [0] * 5 + [0] * 5 + [0] * 4 + [1, 0, 0] * 4
    out["huffman"] = _zfile(b"\x78\x01" + np.packbits(np.array(bits + [0] * (-len(bits) % 8), np.uint8),
                                                      bitorder="little").tobytes() + b"\x00" * 16)
    # fixed block: literal 0, then a match of length 3 at distance 2 (only 1 byte written so far)
    bits = [1, 1, 0] + [0, 0, 1, 1, 0, 0, 0, 0] + [0, 0, 0, 0, 0, 0, 1] + [0, 0, 0, 0, 1] + [0] * 7
    out["distance"] = _zfile(b"\x78\x01" + np.packbits(np.array(bits + [0] * (-len(bits) % 8), np.uint8),
                                                       bitorder="little").tobytes() + b"\x00" * 4)
    out["short"] = _zfile(zlib.compress(raw[:-10]))
    out["filter"] = _zfile(zlib.compress(b"\x07" + raw[1:]))
    out["incomplete code"] = _zfile(incomplete_literal_code(), 1, 1)
    return out


def incomplete_literal_code(eob_length=2):
    """The zlib stream of a 1x1 8-bit gray image's scanline (two zero bytes) in one dynamic block whose literal /
    length code is {0: 1 bit, 256: ``eob_length`` bits}: incomplete for 2, which zlib refuses ("invalid
    literal/lengths set"), complete for 1."""
    bits = []
    put = lambda v, n: bits.extend((v >> k) & 1 for k in range(n))           # an n-bit field, LSB first
    code = lambda c, n: bits.extend((c >> (n - 1 - k)) & 1 for k in range(n))  # a Huffman code, MSB first
    put(1, 1); put(2, 2)                                     # final dynamic block
    put(0, 5); put(0, 5); put(18 - 4, 4)                     # HLIT 257, HDIST 1, HCLEN 18
    order = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1]
    for sym in order:                                        # code-length code: 0, 1, 2 and 18, 2 bits each
        put(2 if sym in (0, 1, 2, 18) else 0, 3)
    clc = {0: 0, 1: 1, 2: 2, 18: 3}                          # canonical codes in symbol order
    code(clc[1], 2)                                          # literal 0: 1 bit
    code(clc[18], 2); put(138 - 11, 7)                       # literals 1..138: none
    code(clc[18], 2); put(117 - 11, 7)                       # literals 139..255: none
    code(clc[eob_length], 2)                                 # end of block
    code(clc[0], 2)                                          # distance 0: none
    code(0, 1); code(0, 1)                                   # two literal zeros
    code(1 if eob_length == 1 else 2, eob_length)            # end of block
    packed = np.packbits(np.array(bits + [0] * (-len(bits) % 8), np.uint8), bitorder="little").tobytes()
    return b"\x78\x01" + packed + struct.pack(">I", zlib.adler32(b"\x00\x00"))


def test_corrupt_streams_set_status_and_spare_neighbours():
    good = [write_png(samples(20, 30, ct, d, ct + d), ct, d, ct % 2, palette=palette_for(d, 1) if ct == 3 else None)
            for ct, d in COMBOS[::3]]
    good.append(_zfile(incomplete_literal_code(1), 1, 1))  # the same stream with a complete code decodes
    bad = _corrupt()
    for d in bad.values():
        assert cv2_decode(d) is None                  # cv2.imread refuses these too
    files = good[:2] + list(bad.values()) + good[2:]
    got, status = _decode(files)
    nbad = len(bad)
    assert (status[2:2 + nbad] == 1).all(), dict(zip(bad, status[2:2 + nbad]))
    assert (status[:2] == 0).all() and (status[2 + nbad:] == 0).all()
    for n, (d, g) in enumerate(zip(files, got)):
        if 2 <= n < 2 + nbad:
            assert (g == 77).all(), n                # a refused image's slot is left unwritten
        else:
            assert np.array_equal(g, cv2_decode(d)), n


def test_png_rejects_host_checkable_arguments():
    from centerpose_b200 import _lib
    data = write_png(samples(16, 16, 2, 8, 1), 2, 8)
    info = png.parse(data)
    buf, ws_bytes = png.pack([info], [data], [0])
    src = torch.from_numpy(buf).cuda()
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    dst = torch.full((16 * 16 * 3,), 77, dtype=torch.uint8, device="cuda")
    status = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    s, w, d, st = src.data_ptr(), ws.data_ptr(), dst.data_ptr(), status.data_ptr()
    for args in ((s, s, 0, w, ws_bytes, d, st), (s, s, 65536, w, ws_bytes, d, st), (None, s, 1, w, ws_bytes, d, st),
                 (s, None, 1, w, ws_bytes, d, st), (s, s, 1, None, ws_bytes, d, st), (s, s, 1, w, ws_bytes, None, st),
                 (s, s, 1, w, ws_bytes, d, None)):
        assert _launch(*args) == CPB200_ERR_ARG, args
        assert b"png_decode_batch" in _lib.lib().cpb200_last_error()
    torch.cuda.synchronize()
    assert (dst.cpu().numpy() == 77).all() and status.item() == -1
    assert _launch(s, s, 1, w, ws_bytes - 1, d, st) == 0
    assert status.item() == 2 and (dst.cpu().numpy() == 77).all()
    assert _launch(s, s, 1, w, ws_bytes, d, st) == 0
    assert status.item() == 0 and np.array_equal(dst.cpu().numpy().reshape(16, 16, 3), cv2_decode(data))


def _png_paths(tmp_path):
    files = [cv2.imencode(".png", make_image(120, 160, "smooth_noise", 1), [cv2.IMWRITE_PNG_COMPRESSION, 1])[1],
             cv2.imencode(".png", make_image(100, 150, "smooth", 2)[:, :, 0])[1],
             write_png(samples(90, 130, 6, 16, 3), 6, 16, 1),
             write_png(samples(70, 110, 3, 4, 4), 3, 4, palette=palette_for(4, 4),
                       before=chunk(b"eXIf", exif(6))),
             write_png(samples(64, 64, 2, 8, 5), 2, 8, before=chunk(b"acTL", struct.pack(">II", 1, 0)))]  # host
    paths = []
    for n, d in enumerate(files):
        p = str(tmp_path / ("p%d.png" % n))
        with open(p, "wb") as f:
            f.write(bytes(d))
        paths.append(p)
    return paths


@pytest.fixture
def png_on_device(monkeypatch):
    """run_images sends PNG files to the device from the first one, so that calls with a few files test that path."""
    from centerpose_b200 import detector
    monkeypatch.setattr(detector, "PNG_DEVICE_MIN_IMAGES", 1)


def _count_png_launches(monkeypatch):
    from centerpose_b200 import png as png_mod
    packed = []
    pack = png_mod.pack
    monkeypatch.setattr(png_mod, "pack", lambda infos, *a, **k: packed.append(len(infos)) or pack(infos, *a, **k))
    return packed


@pytest.mark.parametrize("precision", ["fp32", "fp16x2"])
def test_run_images_png_paths_equal_run_images_arrays(tmp_path, precision, png_on_device, monkeypatch):
    """The same float rows from PNG paths (decoded on the device, an APNG and a corrupt file through cv2.imread),
    mixed with JPEG paths and an array, as from the cv2.imread arrays."""
    packed = _count_png_launches(monkeypatch)
    det = _detector("dla_34", precision, None)
    paths = _png_paths(tmp_path)
    jp = str(tmp_path / "j.jpg")
    with open(jp, "wb") as f:
        f.write(encode(make_image(120, 160, "noise", 9), 90, "420"))
    bad = str(tmp_path / "bad.png")
    with open(bad, "wb") as f:
        f.write(_corrupt()["adler"])
    inputs = paths + [jp, make_image(80, 100, "smooth", 11)]
    got = det.run_images(inputs)
    want = det.run_images([cv2.imread(x) if isinstance(x, str) else x for x in inputs])
    det.device_preprocess = False
    host = det.run_images(inputs)
    det.device_preprocess = True
    for n in range(len(inputs)):
        assert got[n].dtype == np.float32 and np.array_equal(got[n], want[n]), n
        assert np.array_equal(host[n], want[n]), n
    assert packed == [4]                             # the four PNG files but the APNG went to the device
    with pytest.raises(Exception):
        det.run_images([paths[0], bad])              # cv2.imread refuses the corrupt file, as on the host path


def _too_much_data_png(h, w, seed):
    """An RGB PNG whose stream inflates to more bytes than its scanlines: the device refuses it, libpng warns and
    decodes it."""
    im = make_image(h, w, "smooth_noise", seed)[:, :, ::-1]
    raw = b"".join(b"\x00" + im[y].tobytes() for y in range(h)) + b"\x00" * 40
    return png.SIGNATURE + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 0)) + \
        chunk(b"IDAT", zlib.compress(raw)) + chunk(b"IEND", b"")


def test_run_images_png_after_jpeg_chunks_falls_back_per_file(tmp_path, png_on_device, monkeypatch):
    """JPEG files are decoded in the launches before the PNG ones, so the PNG statuses sit after the JPEG ones.  A PNG
    the device refuses but cv2.imread reads (more inflated data than scanlines) takes cv2.imread's pixels, and every
    file gives the rows of the cv2.imread arrays."""
    det = _detector("dla_34", "fp16x2", None)
    extra = _too_much_data_png(96, 128, 21)
    assert png.parse(extra).eligible and cv2_decode(extra) is not None
    _, status = _decode([write_png(samples(8, 8, 2, 8, 1), 2, 8), extra])
    assert status.tolist() == [0, 1]
    packed = _count_png_launches(monkeypatch)
    paths = _png_paths(tmp_path)[:2]
    names = ["j0.jpg", "x.png", "j1.jpg"]
    datas = [encode(make_image(120, 160, "noise", 30), 90, "420"), extra,
             encode(make_image(100, 140, "smooth", 31), 85, "444", progressive=True)]
    for name, d in zip(names, datas):
        with open(str(tmp_path / name), "wb") as f:
            f.write(d)
    inputs = [paths[0], str(tmp_path / "j0.jpg"), str(tmp_path / "x.png"), make_image(90, 110, "noise", 32),
              str(tmp_path / "j1.jpg"), paths[1]]
    got = det.run_images(inputs)
    want = det.run_images([cv2.imread(x) if isinstance(x, str) else x for x in inputs])
    for n in range(len(inputs)):
        assert np.array_equal(got[n], want[n]), n
    assert packed == [3]


def test_run_images_keeps_a_few_png_files_on_the_host(tmp_path, monkeypatch):
    """Below PNG_DEVICE_MIN_IMAGES PNG files per call, cv2.imread reads them (one device launch costs about as much
    as a dozen host decodes); from that count on, they go to the device.  The rows are the same either way."""
    from centerpose_b200 import detector
    packed = _count_png_launches(monkeypatch)
    det = _detector("dla_34", "fp16x2", None)
    paths = _png_paths(tmp_path)[:2]
    want = det.run_images([cv2.imread(p) for p in paths])
    got = det.run_images(paths)
    assert packed == [] and detector.PNG_DEVICE_MIN_IMAGES > len(paths)
    monkeypatch.setattr(detector, "PNG_DEVICE_MIN_IMAGES", len(paths))
    got_device = det.run_images(paths)
    assert packed == [len(paths)]
    for n in range(len(paths)):
        assert np.array_equal(got[n], want[n]) and np.array_equal(got_device[n], want[n]), n
