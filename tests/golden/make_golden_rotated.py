"""Generates tests/golden/cv_pin_rotated.npz from real OpenCV (Python cv2; not required at test time):

    python tests/golden/make_golden_rotated.py

For every interleaved format (bgr, rgb, bgra, rgba, gray, yuyv, uyvy, yvyu), every YUV 4:2:0 layout (nv12, nv21, i420, yv12), every
clockwise rotation (0, 90, 180, 270) and every ROT_CASES source the format accepts: sha256 of cv2.rotate(cv2.cvtColor(src)), of
cv2.resize of that to the case's destination size, and of the letterbox (non_scaling_resize, src/data.cpp:53-69) of it, whose size
comes from the rotated frame.  The sources are seeded (rotated_frame), so the tests rebuild every input."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests.golden.make_golden import sha  # noqa: E402
from tests.golden.make_golden_interleaved import CHANNELS, interleaved_frame  # noqa: E402
from tests.golden.make_golden_yuv import yuv_pack, yuv_planes  # noqa: E402
from tests.interleaved_ref import FORMATS  # noqa: E402
from tests.yuv_ref import LAYOUTS  # noqa: E402

ROTATIONS = (0, 90, 180, 270)
ALL_FORMATS = FORMATS + LAYOUTS
# (src_h, src_w, dst_h, dst_w) as stored: a camera frame; a portrait frame stored as such; a frame whose 90 / 270 rotation is the
# network size (copy) and one whose rotation is twice it (exact-2x area); odd sizes (an odd height for 4:2:2); a tiny upscale; a
# downscale to an odd-width network; 1080p (portrait phone video stored landscape)
ROT_CASES = [(360, 640, 368, 656), (640, 480, 368, 656), (656, 368, 368, 656), (1312, 736, 368, 656), (37, 53, 64, 48),
             (37, 54, 64, 48), (2, 4, 64, 48), (300, 500, 207, 344), (1080, 1920, 368, 656)]


def accepts(fmt, h, w):
    """OpenCV's (and the calls') size rule: 4:2:2 needs an even width, 4:2:0 an even height and width"""
    if fmt in LAYOUTS:
        return h % 2 == 0 and w % 2 == 0
    return CHANNELS[fmt] != 2 or w % 2 == 0


def cases(fmt):
    """the indices into ROT_CASES a format is pinned on"""
    return [i for i, c in enumerate(ROT_CASES) if accepts(fmt, c[0], c[1])]


def rotated_frame(i, fmt):
    """the seeded source of ROT_CASES[i] in `fmt`: interleaved as interleaved_frame, 4:2:0 in cv2's packed (3H/2, W) layout"""
    h, w = ROT_CASES[i][:2]
    seed = 5000 + 16 * i + ALL_FORMATS.index(fmt)
    return yuv_pack(*yuv_planes(seed, h, w), fmt) if fmt in LAYOUTS else interleaved_frame(seed, h, w, fmt)


def letterbox_size(sh, sw, dh, dw):
    """non_scaling_resize's (rh, rw) of an sh x sw frame into dh x dw"""
    h1 = dw * (sh / float(sw)); w2 = dh * (sw / float(sh))
    return (int(h1), dw) if h1 <= dh else (dh, int(w2))


def make_rotated():
    import cv2
    codes = {"rgb": cv2.COLOR_RGB2BGR, "bgra": cv2.COLOR_BGRA2BGR, "rgba": cv2.COLOR_RGBA2BGR, "gray": cv2.COLOR_GRAY2BGR,
             "yuyv": cv2.COLOR_YUV2BGR_YUYV, "uyvy": cv2.COLOR_YUV2BGR_UYVY, "yvyu": cv2.COLOR_YUV2BGR_YVYU,
             "nv12": cv2.COLOR_YUV2BGR_NV12, "nv21": cv2.COLOR_YUV2BGR_NV21, "i420": cv2.COLOR_YUV2BGR_I420, "yv12": cv2.COLOR_YUV2BGR_YV12}
    rotate = {90: cv2.ROTATE_90_CLOCKWISE, 180: cv2.ROTATE_180, 270: cv2.ROTATE_90_COUNTERCLOCKWISE}
    out = {"cv2_version": np.array(cv2.__version__)}
    for fmt in ALL_FORMATS:
        for i in cases(fmt):
            dh, dw = ROT_CASES[i][2:]
            src = rotated_frame(i, fmt)
            bgr = src.copy() if fmt == "bgr" else cv2.cvtColor(src, codes[fmt])
            for deg in ROTATIONS:
                r = bgr if deg == 0 else cv2.rotate(bgr, rotate[deg])
                key = f"{fmt}{i}_r{deg}"
                out[f"{key}_cvt_sha"] = np.array(sha(r))
                out[f"{key}_rz_sha"] = np.array(sha(cv2.resize(r, (dw, dh))))
                rh, rw = letterbox_size(r.shape[0], r.shape[1], dh, dw)
                lb = cv2.copyMakeBorder(cv2.resize(r, (rw, rh)), 0, dh - rh, 0, dw - rw, cv2.BORDER_CONSTANT, value=(0, 0, 0))
                out[f"{key}_lb_sha"] = np.array(sha(lb))
    np.savez_compressed(os.path.join(HERE, "cv_pin_rotated.npz"), **out)


if __name__ == "__main__":
    make_rotated()
