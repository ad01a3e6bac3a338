"""Reference for the 16-bit pose calls (hp_pose_submit{,_pifpaf,_ppn}_frames_{yuv420_16,interleaved16}_*): each 16-bit sample v
holding `bits` significant bits becomes the byte of OpenCV's src.convertTo(dst, CV_8U, 1.0 / (1 << (bits - 8))),

    u8 = saturate(rint_half_even(v * 2^-(bits - 8)))

and the reduced frame goes through the 8-bit restatements unchanged (tests/rotated_ref.py: cvtColor in the stored grid, then
cv::rotate).  v / 2^(bits-8) is exact in float64 and np.rint rounds half to even.  Pinned against real cv2
(tests/golden/cv_pin_highbit.npz, tests/test_highbit_cpu.py)."""
import numpy as np

from tests import rotated_ref

# the 16-bit layouts and formats, and the 8-bit layout or format each one is once reduced
LAYOUTS16 = {"p016": "nv12", "p016_vu": "nv21", "i420": "i420", "yv12": "yv12"}
FORMATS16 = {"bgr48": "bgr", "rgb48": "rgb", "bgra64": "bgra", "rgba64": "rgba", "gray16": "gray"}
ALL16 = {**LAYOUTS16, **FORMATS16}


def reduce(v: np.ndarray, bits: int) -> np.ndarray:
    """uint16 samples with `bits` significant bits -> the uint8 of convertTo(CV_8U, 2^-(bits - 8)), same shape"""
    assert v.dtype == np.uint16 and 9 <= bits <= 16
    return np.minimum(np.rint(v.astype(np.float64) / (1 << (bits - 8))), 255).astype(np.uint8)


def to_bgr(frame: np.ndarray, fmt: str, bits: int, deg: int = 0) -> np.ndarray:
    """cv::rotate(cv::cvtColor(convertTo(frame, CV_8U, 2^-(bits - 8)), code), deg) of a uint16 frame: (3H/2, W) in a LAYOUTS16 layout,
    or (H, W, C) / (H, W) in a FORMATS16 format"""
    return rotated_ref.to_bgr(reduce(frame, bits), ALL16[fmt], deg)
