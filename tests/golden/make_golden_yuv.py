"""Generates tests/golden/cv_pin_yuv.npz from real OpenCV (Python cv2; not required at test time):

    python tests/golden/make_golden_yuv.py

For every layout (NV12, NV21, I420, YV12) and every YUV_CASES source: sha256 of cv2.cvtColor(COLOR_YUV2BGR_<layout>), of cv2.resize
of that to the case's destination size, and of the letterbox (non_scaling_resize, src/data.cpp:53-69) of it.  The YUV_SMALL frames
are stored in full, input and output.  The planes are seeded (yuv_planes), so the tests rebuild every input."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests.golden.make_golden import RESIZE_CASES, sha  # noqa: E402

# (src_h, src_w, dst_h, dst_w): the even-sized frame-resize cases and a 1080p frame (NVDEC decodes it into a 1088-row surface with a
# 2048-byte pitch; the visible 1080 rows are what is converted).  OpenCV refuses odd sizes for these codes.
YUV_CASES = [c for c in RESIZE_CASES if c[0] % 2 == 0 and c[1] % 2 == 0] + [(1080, 1920, 368, 656)]
YUV_LAYOUTS = ("nv12", "nv21", "i420", "yv12")
# (h, w) of the frames stored in full; the last is a sweep: every luma value against every V and 16 U values
YUV_SMALL = [(36, 50), (2, 2), (32, 512)]


def yuv_planes(seed, h, w):
    """seeded Y [h,w], U and V [h/2,w/2] planes"""
    rng = np.random.default_rng(seed)
    return (rng.integers(0, 256, (h, w), dtype=np.uint8), rng.integers(0, 256, (h // 2, w // 2), dtype=np.uint8),
            rng.integers(0, 256, (h // 2, w // 2), dtype=np.uint8))


def yuv_sweep():
    """Y [32,512] = column % 256; U [16,256] = 17 * row, V = column"""
    Y = np.tile(np.arange(512) % 256, (32, 1)).astype(np.uint8)
    U = np.repeat((np.arange(16) * 17).astype(np.uint8)[:, None], 256, 1)
    V = np.tile(np.arange(256, dtype=np.uint8), (16, 1))
    return Y, U, V


def yuv_pack(Y, U, V, layout):
    """the planes in cv2's packed (3H/2, W) layout"""
    h, w = Y.shape
    if layout in ("nv12", "nv21"):
        uv = np.stack([U, V] if layout == "nv12" else [V, U], -1).reshape(h // 2, w)
        return np.concatenate([Y, uv])
    a, b = (U, V) if layout == "i420" else (V, U)
    return np.concatenate([Y.ravel(), a.ravel(), b.ravel()]).reshape(h * 3 // 2, w)


def make_yuv():
    """planes of seed 800 + i for YUV_CASES[i]; seed 900 + i for YUV_SMALL[i], the sweep last"""
    import cv2
    codes = {"nv12": cv2.COLOR_YUV2BGR_NV12, "nv21": cv2.COLOR_YUV2BGR_NV21, "i420": cv2.COLOR_YUV2BGR_I420, "yv12": cv2.COLOR_YUV2BGR_YV12}
    out = {"cv2_version": np.array(cv2.__version__)}
    for i, (sh, sw, dh, dw) in enumerate(YUV_CASES):
        planes = yuv_planes(800 + i, sh, sw)
        for lay in YUV_LAYOUTS:
            bgr = cv2.cvtColor(yuv_pack(*planes, lay), codes[lay])
            out[f"{lay}{i}_cvt_sha"] = np.array(sha(bgr))
            out[f"{lay}{i}_rz_sha"] = np.array(sha(cv2.resize(bgr, (dw, dh))))
            h1 = dw * (sh / float(sw)); w2 = dh * (sw / float(sh))
            rw, rh = (dw, int(h1)) if h1 <= dh else (int(w2), dh)
            lb = cv2.copyMakeBorder(cv2.resize(bgr, (rw, rh)), 0, dh - rh, 0, dw - rw, cv2.BORDER_CONSTANT, value=(0, 0, 0))
            out[f"{lay}{i}_lb_sha"] = np.array(sha(lb))
    for i, (h, w) in enumerate(YUV_SMALL):
        planes = yuv_sweep() if i == len(YUV_SMALL) - 1 else yuv_planes(900 + i, h, w)
        for lay in YUV_LAYOUTS:
            src = yuv_pack(*planes, lay)
            out[f"small{i}_{lay}_in"] = src
            out[f"small{i}_{lay}_bgr"] = cv2.cvtColor(src, codes[lay])
    np.savez_compressed(os.path.join(HERE, "cv_pin_yuv.npz"), **out)


if __name__ == "__main__":
    make_yuv()
