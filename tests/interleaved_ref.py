"""Reference for the interleaved-frame pose calls: cv::cvtColor(src, dst, COLOR_<format>2BGR), restated in numpy.

    bgr   identity                       rgb   channels reversed (COLOR_RGB2BGR)
    bgra  alpha dropped (COLOR_BGRA2BGR) rgba  alpha dropped, channels reversed (COLOR_RGBA2BGR)
    gray  replicated (COLOR_GRAY2BGR)
    yuyv, uyvy, yvyu (COLOR_YUV2BGR_YUYV / _UYVY / _YVYU): 4:2:2, the 4 bytes of each 2 x 1 pixel pair holding both luma bytes and
          one U, V pair (Y0 U Y1 V, U Y0 V Y1, Y0 V Y1 U).  OpenCV's YUV422toRGB8Invoker (modules/imgproc/src/color_yuv.simd.hpp)
          uses the BT.601 limited-range 20-bit fixed point of its 4:2:0 path, so the arithmetic is yuv_ref.planes_to_bgr's: a 4:2:2
          frame is a 4:2:0 frame of twice the rows, each row duplicated, whose even rows are kept.

Pinned against real cv2 for every format (tests/golden/cv_pin_interleaved.npz, tests/test_interleaved_cpu.py)."""
import numpy as np

from tests import yuv_ref

FORMATS = ("bgr", "rgb", "bgra", "rgba", "gray", "yuyv", "uyvy", "yvyu")
# byte offsets of Y0, Y1, U and V in a 4:2:2 pixel pair
YUV422 = {"yuyv": (0, 2, 1, 3), "uyvy": (1, 3, 0, 2), "yvyu": (0, 2, 3, 1)}


def to_bgr(frame: np.ndarray, fmt: str) -> np.ndarray:
    """cv::cvtColor(frame, COLOR_<fmt>2BGR) (COLOR_YUV2BGR_<fmt> for 4:2:2) of a uint8 frame: (H, W, 3) bgr / rgb, (H, W, 4) bgra /
    rgba, (H, W) gray, (H, W, 2) 4:2:2 with W even"""
    assert frame.dtype == np.uint8 and fmt in FORMATS
    if fmt in ("bgr", "rgb", "bgra", "rgba"):
        assert frame.ndim == 3 and frame.shape[2] == len(fmt)
        bgr = frame[..., :3]
        return np.ascontiguousarray(bgr if fmt.startswith("bgr") else bgr[..., ::-1])
    if fmt == "gray":
        assert frame.ndim == 2
        return np.ascontiguousarray(np.repeat(frame[..., None], 3, 2))
    H, W = frame.shape[:2]
    assert frame.shape == (H, W, 2) and W % 2 == 0
    q = np.ascontiguousarray(frame).reshape(H, W // 2, 4)
    y0, y1, u, v = YUV422[fmt]
    Y = np.stack([q[..., y0], q[..., y1]], -1).reshape(H, W)
    return yuv_ref.planes_to_bgr(np.repeat(Y, 2, 0), q[..., u], q[..., v])[::2].copy()


def pack422(Y: np.ndarray, U: np.ndarray, V: np.ndarray, fmt: str) -> np.ndarray:
    """Y [H, W], U and V [H, W/2] as one uint8 (H, W, 2) 4:2:2 frame in `fmt`"""
    H, W = Y.shape
    q = np.empty((H, W // 2, 4), np.uint8)
    y0, y1, u, v = YUV422[fmt]
    q[..., y0], q[..., y1], q[..., u], q[..., v] = Y[:, 0::2], Y[:, 1::2], U, V
    return q.reshape(H, W, 2)
