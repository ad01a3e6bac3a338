"""Generates tests/golden/cv_pin_highbit.npz from real OpenCV (Python cv2; not required at test time):

    python tests/golden/make_golden_highbit.py

First asserts that cv2.convertScaleAbs(v, alpha=2^-(bits-8)) -- convertTo(CV_8U) for non-negative data -- equals
tests/highbit_ref.reduce for every v in 0..65535 and every bits in 9..16.  Then, for every 16-bit layout and format, bits 10, 12 and
16, every HB_SIZES source and every clockwise rotation: sha256 of cv2.rotate(cv2.cvtColor(convertScaleAbs(src))) (which is also the
copy regime: a resize to its own size), of cv2.resize of that to the network size NET (stretch), of the letterbox
(non_scaling_resize, src/data.cpp:53-69) into NET, and of cv2.resize to half its size (the exact-2x area regime).  The sources are
seeded (highbit_frame); interleaved ones are crop views of a wider buffer, so their rows carry garbage between the row's end and the
pitch."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests.golden.make_golden import sha  # noqa: E402
from tests.golden.make_golden_rotated import ROTATIONS, letterbox_size  # noqa: E402
from tests.highbit_ref import ALL16, LAYOUTS16, reduce  # noqa: E402

HB_SIZES = [(360, 640), (720, 1280), (1080, 1920), (362, 642)]   # stored (h, w): camera, 720p, 1080p, and odd halves (181 x 321)
HB_BITS = (10, 12, 16)
NET = (368, 656)
PAD = 8   # samples of garbage after each row of an interleaved source
CH = {"bgr48": 3, "rgb48": 3, "bgra64": 4, "rgba64": 4, "gray16": None}


def highbit_frame(fmt, i, bits):
    """the seeded uint16 source of HB_SIZES[i] in `fmt`: (3H/2, W) packed for a 4:2:0 layout, else an (H, W[, C]) crop view of an
    (H, W + PAD[, C]) buffer.  Samples are drawn below 1.25 * 2^bits (capped at 2^16), so a fifth of them saturate to 255."""
    h, w = HB_SIZES[i]
    rng = np.random.default_rng(7000 + 64 * i + 4 * list(ALL16).index(fmt) + HB_BITS.index(bits))
    hi = min(1 << 16, 5 << (bits - 2))
    if fmt in LAYOUTS16:
        return rng.integers(0, hi, (h * 3 // 2, w), dtype=np.uint16)
    ch = CH[fmt]
    buf = rng.integers(0, 1 << 16, (h, w + PAD) if ch is None else (h, w + PAD, ch), dtype=np.uint16)
    buf[:, :w] = rng.integers(0, hi, buf[:, :w].shape, dtype=np.uint16)
    return buf[:, :w]


def key(fmt, i, bits, deg):
    return f"{fmt}{i}_b{bits}_r{deg}"


def check_reduction(cv2):
    v = np.arange(1 << 16, dtype=np.uint16).reshape(256, 256)
    for bits in range(9, 17):
        got = cv2.convertScaleAbs(v, alpha=2.0 ** -(bits - 8))
        assert np.array_equal(got, reduce(v, bits)), f"bits {bits}: {int((got != reduce(v, bits)).sum())} values differ"


def make_highbit():
    import cv2
    check_reduction(cv2)
    codes = {"rgb48": cv2.COLOR_RGB2BGR, "bgra64": cv2.COLOR_BGRA2BGR, "rgba64": cv2.COLOR_RGBA2BGR, "gray16": cv2.COLOR_GRAY2BGR,
             "p016": cv2.COLOR_YUV2BGR_NV12, "p016_vu": cv2.COLOR_YUV2BGR_NV21, "i420": cv2.COLOR_YUV2BGR_I420,
             "yv12": cv2.COLOR_YUV2BGR_YV12}
    rotate = {90: cv2.ROTATE_90_CLOCKWISE, 180: cv2.ROTATE_180, 270: cv2.ROTATE_90_COUNTERCLOCKWISE}
    out = {"cv2_version": np.array(cv2.__version__)}
    dh, dw = NET
    for fmt in ALL16:
        for i in range(len(HB_SIZES)):
            for bits in HB_BITS:
                u8 = cv2.convertScaleAbs(highbit_frame(fmt, i, bits), alpha=2.0 ** -(bits - 8))
                bgr = u8 if fmt == "bgr48" else cv2.cvtColor(u8, codes[fmt])
                for deg in ROTATIONS:
                    r = bgr if deg == 0 else cv2.rotate(bgr, rotate[deg])
                    k = key(fmt, i, bits, deg)
                    out[f"{k}_cvt_sha"] = np.array(sha(r))
                    out[f"{k}_rz_sha"] = np.array(sha(cv2.resize(r, (dw, dh))))
                    rh, rw = letterbox_size(r.shape[0], r.shape[1], dh, dw)
                    lb = cv2.copyMakeBorder(cv2.resize(r, (rw, rh)), 0, dh - rh, 0, dw - rw, cv2.BORDER_CONSTANT, value=(0, 0, 0))
                    out[f"{k}_lb_sha"] = np.array(sha(lb))
                    out[f"{k}_a2_sha"] = np.array(sha(cv2.resize(r, (r.shape[1] // 2, r.shape[0] // 2))))
    np.savez_compressed(os.path.join(HERE, "cv_pin_highbit.npz"), **out)


if __name__ == "__main__":
    make_highbit()
