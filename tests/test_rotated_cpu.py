"""CPU side of the rotated pose calls: tests/rotated_ref.py (cv::rotate(cv::cvtColor(src, code)) composed from the conversion
restatements and np.rot90) against real cv2, and the wrapper's rotation argument before the library is called.

  1. every ROT_CASES source in every interleaved format and YUV 4:2:0 layout, at every rotation: the reference's rotated BGR frame,
     oracle.resize_linear_u8 of it and its letterbox have the cv2 sha of tests/golden/cv_pin_rotated.npz;
  2. where cv2 is installed, the same against cv2 itself, byte for byte, on small frames;
  3. a YUV 4:2:0 frame rotated in its planes converts to the rotated BGR frame (what the GPU tests feed the upright call);
  4. submit_pose_interleaved / _device and submit_pose_yuv420 / _device refuse a rotation of the wrong length, a value outside
     0, 90, 180, 270 and a non-int; accepted rotations reach the _rotated_ entry points as int32 tables, None the upright ones."""
import ctypes
import os

import numpy as np
import pytest

import oracle
from hyperpose_b200 import capi
from tests import rotated_ref
from tests.golden.make_golden import sha
from tests.golden.make_golden_rotated import ALL_FORMATS, ROT_CASES, ROTATIONS, cases, rotated_frame
from tests.yuv_ref import LAYOUTS


@pytest.fixture(scope="module")
def pin(golden_dir):
    return np.load(os.path.join(golden_dir, "cv_pin_rotated.npz"))


@pytest.mark.parametrize("fmt", ALL_FORMATS)
def test_reference_matches_cv2(pin, fmt):
    for i in cases(fmt):
        sh, sw, dh, dw = ROT_CASES[i]
        src = rotated_frame(i, fmt)
        for deg in ROTATIONS:
            key = f"{fmt}{i}_r{deg}"
            bgr = rotated_ref.to_bgr(src, fmt, deg)
            assert bgr.shape[:2] == ((sw, sh) if deg % 180 else (sh, sw))
            assert sha(bgr) == str(pin[f"{key}_cvt_sha"]), f"{fmt} {sh}x{sw} rotated {deg}"
            assert sha(oracle.resize_linear_u8(bgr, dh, dw)) == str(pin[f"{key}_rz_sha"]), f"{key} -> {dh}x{dw}"
            assert sha(oracle.resize_linear_u8(bgr, dh, dw, letterbox=True)) == str(pin[f"{key}_lb_sha"]), f"{key} letterbox"
    n = len(cases(fmt))
    assert n == (7 if fmt in LAYOUTS else 8 if fmt in ("yuyv", "uyvy", "yvyu") else len(ROT_CASES)), n


def test_rotations_against_cv2_directly():
    cv2 = pytest.importorskip("cv2")
    codes = {90: cv2.ROTATE_90_CLOCKWISE, 180: cv2.ROTATE_180, 270: cv2.ROTATE_90_COUNTERCLOCKWISE}
    rng = np.random.default_rng(3)
    for h, w in ((5, 7), (6, 4), (1, 3)):
        a = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        for deg, code in codes.items():
            assert np.array_equal(rotated_ref.rotate(a, deg), cv2.rotate(a, code)), (h, w, deg)
    y = rotated_frame(6, "nv12")
    for deg, code in codes.items():
        assert np.array_equal(rotated_ref.to_bgr(y, "nv12", deg), cv2.rotate(cv2.cvtColor(y, cv2.COLOR_YUV2BGR_NV12), code))


@pytest.mark.parametrize("layout", LAYOUTS)
def test_yuv420_rotated_in_its_planes(layout):
    for i in cases(layout):
        src = rotated_frame(i, layout)
        for deg in ROTATIONS:
            assert np.array_equal(rotated_ref.to_bgr(rotated_ref.rotate_yuv420(src, layout, deg), layout, 0),
                                  rotated_ref.to_bgr(src, layout, deg)), (layout, ROT_CASES[i], deg)


def _recording(monkeypatch):
    """an Engine whose _submit_frame_table records its arguments, and a library that must not be called"""
    def no_library():
        raise AssertionError("the library was called")
    monkeypatch.setattr(capi, "lib", no_library)
    eng, parser = object.__new__(capi.Engine), capi.PafParser.__new__(capi.PafParser)
    seen = []

    def table_of(parser_, table, keep_ratio, device, fmt="u8", **kw):
        seen.append((fmt, device, kw))
        return 0
    monkeypatch.setattr(eng, "_submit_frame_table", table_of, raising=False)
    return eng, parser, seen


def _calls(eng, parser):
    """(name, submit(rotation)) of the four calls that take a rotation, each on a batch of two frames"""
    rgb, nv12 = np.zeros((6, 8, 3), np.uint8), np.zeros((9, 8), np.uint8)
    return [("interleaved", lambda r: eng.submit_pose_interleaved(parser, [rgb, rgb], "rgb", rotation=r)),
            ("interleaved_device", lambda r: eng.submit_pose_interleaved_device(parser, [capi.FrameInterleaved()] * 2, rotation=r)),
            ("yuv420", lambda r: eng.submit_pose_yuv420(parser, [nv12, nv12], "nv12", rotation=r)),
            ("yuv420_device", lambda r: eng.submit_pose_yuv420_device(parser, [capi.FrameYUV420()] * 2, rotation=r))]


def test_wrapper_refuses_bad_rotations(monkeypatch):
    eng, parser, seen = _recording(monkeypatch)
    bad = [[90], [0, 90, 180], [], 45, -90, 360, [0, 45], [90, -90], [0, 1], 90.0, [0, 90.0], "90", ["90", "0"], [0, None], True,
           [False, 90], np.array([0.0, 90.0]), {0: 90}]
    for name, submit in _calls(eng, parser):
        for r in bad:
            with pytest.raises(capi.HyperposeError) as e:
                submit(r)
            assert e.value.status == capi.HP_ERR_ARG, (name, r)
    assert seen == []


def test_wrapper_passes_rotation_tables(monkeypatch):
    eng, parser, seen = _recording(monkeypatch)
    for name, submit in _calls(eng, parser):
        for r, want in ((None, None), (0, [0, 0]), (270, [270, 270]), ([90, 180], [90, 180]), ((0, 270), [0, 270]),
                        (np.array([180, 90], np.int64), [180, 90])):
            seen.clear()
            submit(r)
            (fmt, device, kw), = seen
            assert fmt == name.split("_")[0] and device == name.endswith("_device")
            if want is None:
                assert kw == {}, "an upright batch goes to the upright entry points"
            else:
                t = kw["rotation"]
                assert t._type_ is ctypes.c_int32 and list(t) == want, (name, r)
