"""CPU side of the YUV 4:2:0 pose calls: tests/yuv_ref.py (the restatement of cv::cvtColor(COLOR_YUV2BGR_NV12 / _NV21 / _I420 /
_YV12)) against real cv2, and the wrapper's refusals before the library is called.

  1. every YUV_CASES source in all four layouts: the restatement's BGR frame, oracle.resize_linear_u8 of it and its letterbox have
     the cv2 sha of tests/golden/cv_pin_yuv.npz;
  2. the YUV_SMALL frames stored in full (random planes and a sweep of every Y and V value) byte for byte;
  3. submit_pose_yuv420 / submit_pose_yuv420_device refuse what is not a uint8 (3H/2, W) frame, an unknown layout and records that
     are not FrameYUV420."""
import os

import numpy as np
import pytest

import oracle
from hyperpose_b200 import capi
from tests import yuv_ref
from tests.golden.make_golden import sha
from tests.golden.make_golden_yuv import YUV_CASES, YUV_LAYOUTS, YUV_SMALL, yuv_pack, yuv_planes


@pytest.fixture(scope="module")
def pin(golden_dir):
    return np.load(os.path.join(golden_dir, "cv_pin_yuv.npz"))


@pytest.mark.parametrize("i", range(len(YUV_CASES)))
def test_oracle_matches_cv2(pin, i):
    sh, sw, dh, dw = YUV_CASES[i]
    planes = yuv_planes(800 + i, sh, sw)
    for lay in YUV_LAYOUTS:
        bgr = yuv_ref.yuv420_to_bgr(yuv_pack(*planes, lay), lay)
        assert sha(bgr) == str(pin[f"{lay}{i}_cvt_sha"]), f"{lay} {sh}x{sw}"
        assert sha(oracle.resize_linear_u8(bgr, dh, dw)) == str(pin[f"{lay}{i}_rz_sha"]), f"{lay} {sh}x{sw} -> {dh}x{dw}"
        assert sha(oracle.resize_linear_u8(bgr, dh, dw, letterbox=True)) == str(pin[f"{lay}{i}_lb_sha"]), f"{lay} letterbox"


def test_oracle_small_frames_in_full(pin):
    for i in range(len(YUV_SMALL)):
        for lay in YUV_LAYOUTS:
            got = yuv_ref.yuv420_to_bgr(pin[f"small{i}_{lay}_in"], lay)
            want = pin[f"small{i}_{lay}_bgr"]
            assert np.array_equal(got, want), f"small{i} {lay}: {int((got != want).sum())} bytes differ"
    sweep = pin[f"small{len(YUV_SMALL) - 1}_nv12_bgr"]
    assert sweep.min() == 0 and sweep.max() == 255, "the sweep reaches both saturation limits"


def test_layouts_unpack_to_the_same_planes():
    """the four packed layouts of the same planes convert to the planes' bytes: the layouts differ only in where U and V are"""
    Y, U, V = yuv_planes(5, 12, 20)
    want = yuv_ref.planes_to_bgr(Y, U, V)
    assert len(np.unique(want)) > 100
    for lay in YUV_LAYOUTS:
        assert np.array_equal(yuv_ref.yuv420_to_bgr(yuv_pack(Y, U, V, lay), lay), want), lay


def test_wrapper_rejects_what_is_not_yuv420(monkeypatch):
    def no_library():
        raise AssertionError("the library was called")
    monkeypatch.setattr(capi, "lib", no_library)
    eng = object.__new__(capi.Engine)
    parser = capi.PafParser.__new__(capi.PafParser)
    good = np.zeros((6, 8), np.uint8)
    for bad in (np.zeros((6, 8), np.float32), np.zeros((6, 8, 3), np.uint8), np.zeros((7, 8), np.uint8), np.zeros((0, 8), np.uint8),
                [[1, 2, 3]]):
        with pytest.raises(capi.HyperposeError) as e:
            eng.submit_pose_yuv420(parser, [good, bad], "nv12")
        assert e.value.status == capi.HP_ERR_ARG
    for layout in ("nv16", ["nv12"], ["nv12", "bgr"]):   # unknown, one short, one unknown in the list
        with pytest.raises(capi.HyperposeError) as e:
            eng.submit_pose_yuv420(parser, [good, good], layout)
        assert e.value.status == capi.HP_ERR_ARG
    with pytest.raises(capi.HyperposeError) as e:
        eng.submit_pose_yuv420_device(parser, [capi.FrameYUV420(), (0, 0, 0, 4, 4, 4, 4, 2)])
    assert e.value.status == capi.HP_ERR_ARG


def test_packed_layout_records():
    """yuv420_record points into cv2's packed layouts as the oracle reads them"""
    f = np.zeros((12, 8), np.uint8)
    p = f.ctypes.data
    r = capi.yuv420_record(f, "nv12")
    assert (r.y, r.u - p, r.v - p, r.height, r.width, r.pitch_y, r.pitch_uv, r.uv_step) == (p, 64, 65, 8, 8, 8, 8, 2)
    r = capi.yuv420_record(f, "nv21")
    assert (r.u - p, r.v - p, r.uv_step) == (65, 64, 2)
    r = capi.yuv420_record(f, "i420")
    assert (r.u - p, r.v - p, r.pitch_uv, r.uv_step) == (64, 80, 4, 1)
    r = capi.yuv420_record(f, "yv12")
    assert (r.u - p, r.v - p, r.pitch_uv, r.uv_step) == (80, 64, 4, 1)
