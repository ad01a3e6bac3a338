"""Reference for the YUV 4:2:0 pose calls: cv::cvtColor(src, dst, COLOR_YUV2BGR_NV12 / _NV21 / _I420 / _YV12), restated in numpy.

OpenCV's 8-bit YUV 4:2:0 -> BGR path (modules/imgproc/src/color_yuv.simd.hpp, YUV420sp2RGB8Invoker / YUV420p2RGB8Invoker) is BT.601
limited range in 20-bit fixed point, each chroma sample covering its 2x2 luma block:
    ITUR_BT_601_SHIFT = 20, ITUR_BT_601_CY = 1220542, ITUR_BT_601_CUB = 2116026, ITUR_BT_601_CUG = -409993,
    ITUR_BT_601_CVG = -852492, ITUR_BT_601_CVR = 1673527
    y' = max(Y - 16, 0) * CY;  u = U - 128;  v = V - 128;  h = 1 << 19
    B = sat((y' + h + CUB u) >> 20),  G = sat((y' + h + CVG v + CUG u) >> 20),  R = sat((y' + h + CVR v) >> 20)
The sums are evaluated in int64, so nothing can overflow; every one stays below 2^30 in magnitude, so int32 arithmetic (the kernel's)
gives the same bytes.  The four layouts differ only in where U and V are.  Pinned against real cv2 for all four codes
(tests/golden/cv_pin_yuv.npz, tests/test_yuv_cpu.py)."""
import numpy as np

SHIFT, CY, CUB, CUG, CVG, CVR = 20, 1220542, 2116026, -409993, -852492, 1673527
LAYOUTS = ("nv12", "nv21", "i420", "yv12")


def planes_to_bgr(Y: np.ndarray, U: np.ndarray, V: np.ndarray) -> np.ndarray:
    """Y u8 [H, W], U and V u8 [H/2, W/2] -> BGR u8 [H, W, 3]"""
    H, W = Y.shape
    assert H % 2 == 0 and W % 2 == 0 and U.shape == V.shape == (H // 2, W // 2)
    y = np.maximum(Y.astype(np.int64) - 16, 0) * CY + (1 << (SHIFT - 1))
    u = np.repeat(np.repeat(U.astype(np.int64) - 128, 2, 0), 2, 1)
    v = np.repeat(np.repeat(V.astype(np.int64) - 128, 2, 0), 2, 1)
    bgr = np.stack([y + CUB * u, y + CVG * v + CUG * u, y + CVR * v], -1) >> SHIFT
    return np.clip(bgr, 0, 255).astype(np.uint8)


def unpack(frame: np.ndarray, layout: str):
    """(Y, U, V) of a uint8 (3H/2, W) frame in cv2's packed layout for `layout`"""
    assert frame.dtype == np.uint8 and frame.ndim == 2 and frame.shape[0] % 3 == 0 and layout in LAYOUTS
    H, W = frame.shape[0] * 2 // 3, frame.shape[1]
    Y, rest = frame[:H], frame[H:]
    if layout in ("nv12", "nv21"):   # one interleaved plane: U V U V ... (NV12) or V U V U ... (NV21)
        uv = rest.reshape(H // 2, W // 2, 2)
        a, b = uv[..., 0], uv[..., 1]
        return (Y, a, b) if layout == "nv12" else (Y, b, a)
    flat = rest.reshape(-1)          # two planes of (H/2) x (W/2), packed: U then V (I420) or V then U (YV12)
    n = H * W // 4
    a, b = flat[:n].reshape(H // 2, W // 2), flat[n:].reshape(H // 2, W // 2)
    return (Y, a, b) if layout == "i420" else (Y, b, a)


def yuv420_to_bgr(frame: np.ndarray, layout: str) -> np.ndarray:
    """cv::cvtColor(frame, COLOR_YUV2BGR_<layout>) on a uint8 (3H/2, W) frame in cv2's packed layout"""
    return planes_to_bgr(*unpack(np.ascontiguousarray(frame), layout))
