"""CPU side of the interleaved-frame pose calls: tests/interleaved_ref.py (the restatement of cv::cvtColor(COLOR_RGB2BGR, _BGRA2BGR,
_RGBA2BGR, _GRAY2BGR, _YUV2BGR_YUYV / _UYVY / _YVYU)) against real cv2, and the wrapper's refusals before the library is called.

  1. every RESIZE_CASES source in every format (even widths for 4:2:2): the restatement's BGR frame, oracle.resize_linear_u8 of it
     and its letterbox have the cv2 sha of tests/golden/cv_pin_interleaved.npz;
  2. the SMALL frames stored in full (random bytes, random alpha) and the 4:2:2 sweep of every U, V pair byte for byte;
  3. submit_pose_interleaved / submit_pose_interleaved_device refuse a shape, dtype or format that does not match, rows whose bytes
     are not contiguous, and records that are not FrameInterleaved; a crop view passes its row stride as the pitch."""
import os
import re

import numpy as np
import pytest

import oracle
from hyperpose_b200 import capi
from tests import interleaved_ref
from tests.golden.make_golden import RESIZE_CASES, sha
from tests.golden.make_golden_interleaved import SMALL, case_frame, cases, sweep422
from tests.interleaved_ref import FORMATS


@pytest.fixture(scope="module")
def pin(golden_dir):
    return np.load(os.path.join(golden_dir, "cv_pin_interleaved.npz"))


@pytest.mark.parametrize("fmt", FORMATS)
def test_oracle_matches_cv2(pin, fmt):
    for i in cases(fmt):
        sh, sw, dh, dw = RESIZE_CASES[i]
        bgr = interleaved_ref.to_bgr(case_frame(i, fmt), fmt)
        assert sha(bgr) == str(pin[f"{fmt}{i}_cvt_sha"]), f"{fmt} {sh}x{sw}"
        assert sha(oracle.resize_linear_u8(bgr, dh, dw)) == str(pin[f"{fmt}{i}_rz_sha"]), f"{fmt} {sh}x{sw} -> {dh}x{dw}"
        assert sha(oracle.resize_linear_u8(bgr, dh, dw, letterbox=True)) == str(pin[f"{fmt}{i}_lb_sha"]), f"{fmt} letterbox"
    assert len(cases(fmt)) == (len(RESIZE_CASES) - 1 if fmt in interleaved_ref.YUV422 else len(RESIZE_CASES))


def test_oracle_small_frames_in_full(pin):
    for i in range(len(SMALL)):
        for fmt in FORMATS:
            got = interleaved_ref.to_bgr(pin[f"small{i}_{fmt}_in"], fmt)
            want = pin[f"small{i}_{fmt}_bgr"]
            assert np.array_equal(got, want), f"small{i} {fmt}: {int((got != want).sum())} bytes differ"
    alpha = pin["small0_bgra_in"][..., 3]
    assert len(np.unique(alpha)) > 100, "the 4-channel frames carry random alpha"


def test_oracle_sweep_in_full(pin):
    want = pin["sweep_bgr"]
    assert want.min() == 0 and want.max() == 255, "the sweep reaches both saturation limits"
    for fmt in interleaved_ref.YUV422:
        got = interleaved_ref.to_bgr(sweep422(fmt), fmt)
        assert np.array_equal(got, want), f"{fmt}: {int((got != want).sum())} bytes differ"
        assert sha(got) == str(pin[f"sweep_{fmt}_sha"])


def test_422_formats_differ_only_in_byte_order():
    rng = np.random.default_rng(5)
    Y = rng.integers(0, 256, (6, 10), dtype=np.uint8)
    U, V = rng.integers(0, 256, (2, 6, 5), dtype=np.uint8)
    want = interleaved_ref.to_bgr(interleaved_ref.pack422(Y, U, V, "yuyv"), "yuyv")
    assert len(np.unique(want)) > 50
    for fmt in ("uyvy", "yvyu"):
        assert np.array_equal(interleaved_ref.to_bgr(interleaved_ref.pack422(Y, U, V, fmt), fmt), want), fmt


def _no_library(monkeypatch):
    def no_library():
        raise AssertionError("the library was called")
    monkeypatch.setattr(capi, "lib", no_library)
    return object.__new__(capi.Engine), capi.PafParser.__new__(capi.PafParser)


def test_wrapper_rejects_mismatched_frames(monkeypatch):
    eng, parser = _no_library(monkeypatch)
    good = {"bgr": np.zeros((6, 8, 3), np.uint8), "gray": np.zeros((6, 8), np.uint8), "yuyv": np.zeros((6, 8, 2), np.uint8),
            "rgba": np.zeros((6, 8, 4), np.uint8)}
    big = np.zeros((10, 20, 4), np.uint8)
    bad = [("bgr", np.zeros((6, 8, 4), np.uint8)), ("bgra", np.zeros((6, 8, 3), np.uint8)), ("gray", np.zeros((6, 8, 1), np.uint8)),
           ("yuyv", np.zeros((6, 8), np.uint8)), ("uyvy", np.zeros((6, 8, 3), np.uint8)), ("rgb", np.zeros((6, 8, 3), np.float32)),
           ("rgb", np.zeros((6, 8, 3), np.int8)), ("gray", [[1, 2, 3]]),
           ("rgba", big[:, ::2]),                         # pixels not adjacent
           ("bgr", big[:, :, 2::-1]),                     # channels reversed by a negative stride
           ("gray", big[..., 0]),                         # bytes of a row 4 apart
           ("rgba", big[::-1]),                           # rows upward: a negative pitch
           ("bgr", np.zeros((8, 6, 3), np.uint8).transpose(1, 0, 2)), ("yvyu", np.asfortranarray(np.zeros((6, 8, 2), np.uint8)))]
    for fmt, f in bad:
        with pytest.raises(capi.HyperposeError) as e:
            eng.submit_pose_interleaved(parser, [good["bgr"], f], ["bgr", fmt])
        assert e.value.status == capi.HP_ERR_ARG, (fmt, getattr(f, "shape", None))
    for fmt in ("nv12", "BGR", ["bgr"], ["bgr", "xrgb"]):   # unknown, wrong case, one short, one unknown in the list
        with pytest.raises(capi.HyperposeError) as e:
            eng.submit_pose_interleaved(parser, [good["bgr"], good["bgr"]], fmt)
        assert e.value.status == capi.HP_ERR_ARG
    with pytest.raises(capi.HyperposeError) as e:
        eng.submit_pose_interleaved_device(parser, [capi.FrameInterleaved(), (0, 4, 4, 12, 0)])
    assert e.value.status == capi.HP_ERR_ARG


def test_wrapper_passes_crop_views_with_their_pitch(monkeypatch):
    """a crop of a larger frame is submitted in place, its row stride as the pitch; packed frames with pitch = row bytes"""
    eng = object.__new__(capi.Engine)
    parser = capi.PafParser.__new__(capi.PafParser)
    seen = {}

    def table_of(parser_, table, keep_ratio, device, fmt):
        seen["table"], seen["device"], seen["fmt"] = [(r.data, r.height, r.width, r.pitch, r.format) for r in table], device, fmt
        return 0
    monkeypatch.setattr(eng, "_submit_frame_table", table_of, raising=False)
    big = np.zeros((720, 1280, 4), np.uint8)
    crop = big[100:300, 40:640]
    y = np.zeros((4, 6, 2), np.uint8)
    g = np.zeros((3, 5), np.uint8)
    eng.submit_pose_interleaved(parser, [crop, y, g], ["rgba", "uyvy", "gray"])
    assert seen["device"] is False and seen["fmt"] == "interleaved"
    assert seen["table"] == [(crop.ctypes.data, 200, 600, 1280 * 4, capi.PIXEL_FORMATS["rgba"]), (y.ctypes.data, 4, 6, 12, 6),
                             (g.ctypes.data, 3, 5, 5, 4)]
    assert crop.ctypes.data == big.ctypes.data + (100 * 1280 + 40) * 4


def test_pixel_format_values_match_the_header():
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "hyperpose_b200.h")).read()
    body = hdr[hdr.index("typedef enum hp_pixel_format"):hdr.index("} hp_pixel_format;")]
    names = [n.lower() for n in re.findall(r"HP_PIX_([A-Z]+)", body)]
    assert names == list(capi.PIXEL_FORMATS) == list(FORMATS)
    assert [capi.PIXEL_FORMATS[n] for n in names] == list(range(len(names)))
