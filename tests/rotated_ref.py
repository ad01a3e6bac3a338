"""Reference for the rotated pose calls: cv::rotate(cv::cvtColor(src, code), rotate_code), composed from the conversion restatements
(tests/interleaved_ref.py, tests/yuv_ref.py) and np.rot90.  The conversion happens in the stored grid, then the BGR frame is rotated:

    0    upright                              180  ROTATE_180
    90   ROTATE_90_CLOCKWISE                  270  ROTATE_90_COUNTERCLOCKWISE

np.rot90(a, k) turns counter-clockwise for k > 0, so `deg` clockwise degrees is k = -deg // 90.  The resize after it is
oracle.resize_linear_u8 of the rotated frame.  Pinned against real cv2 (tests/golden/cv_pin_rotated.npz, tests/test_rotated_cpu.py)."""
import numpy as np

from tests import interleaved_ref, yuv_ref
from tests.golden.make_golden_yuv import yuv_pack

ROTATIONS = (0, 90, 180, 270)


def rotate(a: np.ndarray, deg: int) -> np.ndarray:
    """cv::rotate of an image (H, W, ...) by `deg` clockwise degrees"""
    assert deg in ROTATIONS
    return np.ascontiguousarray(np.rot90(a, k=-deg // 90))


def to_bgr(frame: np.ndarray, fmt: str, deg: int) -> np.ndarray:
    """cv::rotate(cv::cvtColor(frame, COLOR_..2BGR)) of an interleaved frame (interleaved_ref.FORMATS) or a YUV 4:2:0 frame in cv2's
    packed (3H/2, W) layout (yuv_ref.LAYOUTS)"""
    bgr = yuv_ref.yuv420_to_bgr(frame, fmt) if fmt in yuv_ref.LAYOUTS else interleaved_ref.to_bgr(frame, fmt)
    return rotate(bgr, deg)


def rotate_yuv420(frame: np.ndarray, layout: str, deg: int) -> np.ndarray:
    """a YUV 4:2:0 frame rotated in its planes, in the same packed layout: each chroma sample's 2x2 block turns with it, so its BGR frame
    is to_bgr(frame, layout, deg) (what the upright call is fed to check the rotated one)"""
    Y, U, V = yuv_ref.unpack(np.ascontiguousarray(frame), layout)
    return yuv_pack(rotate(Y, deg), rotate(U, deg), rotate(V, deg), layout)
