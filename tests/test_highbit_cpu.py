"""CPU side of the 16-bit pose calls: tests/highbit_ref.py (convertTo(CV_8U, 2^-(bits-8)), then the 8-bit conversion and rotation
restatements) against real cv2, the records the wrappers build, and the wrappers' refusals before the library is called.

  1. every pinned source (every 16-bit layout and format, bits 10, 12, 16, every HB_SIZES size, every rotation): the reference's
     frame (the copy regime), oracle.resize_linear_u8 of it to the network size, its letterbox and its exact-2x area reduction have the
     cv2 sha of tests/golden/cv_pin_highbit.npz;
  2. where cv2 is installed, the reduction against cv2.convertScaleAbs for every 16-bit value and every bits in 9..16;
  3. yuv420_16_record / interleaved16_record: byte offsets and pitches of the planes and rows, and the bits;
  4. submit_pose_yuv420_16 / submit_pose_interleaved16 and their _device twins refuse a wrong dtype, shape, layout, format, bits and
     rotation before the library is called; accepted batches reach the 16-bit entry points with a rotation table or NULL."""
import ctypes
import os

import numpy as np
import pytest

import oracle
from hyperpose_b200 import capi
from tests import highbit_ref
from tests.golden.make_golden import sha
from tests.golden.make_golden_highbit import HB_BITS, HB_SIZES, NET, highbit_frame, key
from tests.golden.make_golden_rotated import ROTATIONS


@pytest.fixture(scope="module")
def pin(golden_dir):
    return np.load(os.path.join(golden_dir, "cv_pin_highbit.npz"))


@pytest.mark.parametrize("fmt", list(highbit_ref.ALL16))
def test_reference_matches_cv2(pin, fmt):
    for i, (h, w) in enumerate(HB_SIZES):
        for bits in HB_BITS:
            src = highbit_frame(fmt, i, bits)
            for deg in ROTATIONS:
                k = key(fmt, i, bits, deg)
                bgr = highbit_ref.to_bgr(src, fmt, bits, deg)
                assert bgr.shape[:2] == ((w, h) if deg % 180 else (h, w))
                assert sha(bgr) == str(pin[f"{k}_cvt_sha"]), k
                assert sha(oracle.resize_linear_u8(bgr, *NET)) == str(pin[f"{k}_rz_sha"]), k
                assert sha(oracle.resize_linear_u8(bgr, *NET, letterbox=True)) == str(pin[f"{k}_lb_sha"]), k
                assert sha(oracle.resize_linear_u8(bgr, bgr.shape[0] // 2, bgr.shape[1] // 2)) == str(pin[f"{k}_a2_sha"]), k


def test_reduction_against_cv2_directly():
    cv2 = pytest.importorskip("cv2")
    v = np.arange(1 << 16, dtype=np.uint16).reshape(256, 256)
    for bits in range(9, 17):
        assert np.array_equal(highbit_ref.reduce(v, bits), cv2.convertScaleAbs(v, alpha=2.0 ** -(bits - 8))), bits
    assert highbit_ref.reduce(np.array([1023, 1022, 2, 6, 65535], np.uint16), 10).tolist() == [255, 255, 0, 2, 255]
    assert highbit_ref.reduce(np.array([0x8080, 0x8180, 0x807f], np.uint16), 16).tolist() == [0x80, 0x82, 0x80]   # half to even


def test_records():
    f = np.zeros((9, 8), np.uint16)   # H = 6, W = 8
    p = f.ctypes.data
    for layout, (u, v, pitch_uv, step) in (("p016", (48, 49, 8, 2)), ("p016_vu", (49, 48, 8, 2)), ("i420", (48, 60, 4, 1)),
                                           ("yv12", (60, 48, 4, 1))):
        r = capi.yuv420_16_record(f, layout, 10)
        assert (r.y, r.u, r.v) == (p, p + 2 * u, p + 2 * v), layout
        assert (r.height, r.width, r.pitch_y, r.pitch_uv, r.uv_step, r.bits) == (6, 8, 16, 2 * pitch_uv, step, 10), layout
    big = np.zeros((5, 11, 4), np.uint16)
    r = capi.interleaved16_record(big[1:4, 2:9], "rgba64", 12)
    assert (r.data, r.height, r.width, r.pitch, r.format, r.bits) == (big.ctypes.data + 88 + 16, 3, 7, 88, capi.PIXEL_FORMATS["rgba"], 12)


def _recording(monkeypatch):
    """an Engine whose _submit_frame_table records its arguments, and a library that must not be called"""
    def no_library():
        raise AssertionError("the library was called")
    monkeypatch.setattr(capi, "lib", no_library)
    eng, parser = object.__new__(capi.Engine), capi.PafParser.__new__(capi.PafParser)
    seen = []

    def table_of(parser_, table, keep_ratio, device, fmt="u8", rotation=None):
        seen.append((fmt, device, [tuple(getattr(r, "bits") for r in table)], rotation))
        return 0
    monkeypatch.setattr(eng, "_submit_frame_table", table_of, raising=False)
    return eng, parser, seen


def test_wrapper_refusals(monkeypatch):
    eng, parser, seen = _recording(monkeypatch)
    p016, rgb = np.zeros((9, 8), np.uint16), np.zeros((6, 8, 3), np.uint16)
    yuv, inter = eng.submit_pose_yuv420_16, eng.submit_pose_interleaved16
    bad = [
        (yuv, [p016.astype(np.uint8)], "p016", 16, {}),                  # dtype
        (yuv, [p016.astype(np.int16)], "p016", 16, {}),
        (yuv, [p016.astype(np.float32)], "p016", 16, {}),
        (yuv, [np.zeros((8, 8), np.uint16)], "p016", 16, {}),            # shape: not 3H/2 rows
        (yuv, [np.zeros((9, 8, 1), np.uint16)], "p016", 16, {}),
        (yuv, [p016.tolist()], "p016", 16, {}),
        (yuv, [p016], "nv12", 16, {}),                                   # layout: the 8-bit names are not 16-bit layouts
        (yuv, [p016], "p010", 16, {}),
        (yuv, [p016, p016], ["p016"], 16, {}),
        (inter, [rgb[..., 0]], "rgb48", 16, {}),                         # shape
        (inter, [np.zeros((6, 8, 4), np.uint16)], "bgr48", 16, {}),
        (inter, [rgb], "gray16", 16, {}),
        (inter, [rgb.astype(np.uint8)], "rgb48", 16, {}),               # dtype
        (inter, [rgb], "rgb", 16, {}),                                   # format
        (inter, [rgb], "yuyv", 16, {}),
        (inter, [np.zeros((6, 8, 2), np.uint16)], "yuyv32", 16, {}),
        (inter, [np.zeros((6, 16, 3), np.uint16)[:, ::2]], "rgb48", 16, {}),   # samples of a row not contiguous
        (inter, [np.zeros((6, 8, 3), np.uint16).transpose(1, 0, 2)], "rgb48", 16, {}),
    ]
    for bits in (8, 17, 0, -10, 9.0, "16", None, True, [16], [16, 16, 16], [16, 8], [np.float64(12), 12]):
        bad += [(yuv, [p016, p016], "p016", bits, {}), (inter, [rgb, rgb], "rgb48", bits, {})]
    for rot in ([90], 45, -90, 360, [0, 45], 90.0, "90", True):
        bad += [(yuv, [p016, p016], "p016", 16, {"rotation": rot}), (inter, [rgb, rgb], "rgb48", 16, {"rotation": rot})]
    for submit, frames, what, bits, kw in bad:
        with pytest.raises(capi.HyperposeError) as e:
            submit(parser, frames, what, bits, **kw)
        assert e.value.status == capi.HP_ERR_ARG, (what, bits, kw)
    for submit, frames in ((eng.submit_pose_yuv420_16_device, [capi.FrameYUV420()]), (eng.submit_pose_yuv420_16_device, [p016]),
                           (eng.submit_pose_interleaved16_device, [capi.FrameInterleaved()]),
                           (eng.submit_pose_interleaved16_device, [capi.FrameYUV420_16()])):
        with pytest.raises(capi.HyperposeError) as e:
            submit(parser, frames)
        assert e.value.status == capi.HP_ERR_ARG
    with pytest.raises(capi.HyperposeError):
        eng.submit_pose_yuv420_16_device(parser, [capi.FrameYUV420_16()] * 2, rotation=[90, 91])
    assert seen == []
    # the 8-bit calls keep refusing 16-bit arrays
    for submit, frames, fmt in ((eng.submit_pose_yuv420, [p016], "nv12"), (eng.submit_pose_interleaved, [rgb], "rgb")):
        with pytest.raises(capi.HyperposeError):
            submit(parser, frames, fmt)
    assert seen == []


def test_wrapper_passes_tables(monkeypatch):
    eng, parser, seen = _recording(monkeypatch)
    p016, gray = np.zeros((9, 8), np.uint16), np.zeros((6, 8), np.uint16)
    calls = [("yuv420_16", False, lambda b, r: eng.submit_pose_yuv420_16(parser, [p016, p016], ["p016", "yv12"], b, rotation=r)),
             ("interleaved16", False, lambda b, r: eng.submit_pose_interleaved16(parser, [gray, gray], "gray16", b, rotation=r)),
             ("yuv420_16", True, lambda b, r: eng.submit_pose_yuv420_16_device(
                 parser, [capi.FrameYUV420_16(bits=b[0]), capi.FrameYUV420_16(bits=b[1])], rotation=r)),
             ("interleaved16", True, lambda b, r: eng.submit_pose_interleaved16_device(
                 parser, [capi.FrameInterleaved16(bits=b[0]), capi.FrameInterleaved16(bits=b[1])], rotation=r))]
    for fmt, device, submit in calls:
        for bits, rot, want in (([16, 10], None, None), ([12, 12], 90, [90, 90]), ([9, 16], [0, 270], [0, 270])):
            seen.clear()
            submit(bits if device else (bits[0] if bits[0] == bits[1] else bits), rot)
            (f, d, (got_bits,), table), = seen
            assert (f, d, list(got_bits)) == (fmt, device, bits)
            if want is None:
                assert table is None, "an upright batch passes NULL"
            else:
                assert table._type_ is ctypes.c_int32 and list(table) == want
