"""Generates tests/golden/cv_pin_interleaved.npz from real OpenCV (Python cv2; not required at test time):

    python tests/golden/make_golden_interleaved.py

For every format (bgr, rgb, bgra, rgba, gray, yuyv, uyvy, yvyu) and every RESIZE_CASES source (even widths only for 4:2:2, which
OpenCV refuses otherwise): sha256 of cv2.cvtColor(COLOR_<format>2BGR), of cv2.resize of that to the case's destination size, and of
the letterbox (non_scaling_resize, src/data.cpp:53-69) of it.  The SMALL frames are stored in full, input and output; the 4:2:2
sweep (sweep422) is the same planes in all three 4:2:2 formats: its BGR frame is stored in full once, with each format's sha.  The
sources are seeded (interleaved_frame), so the tests rebuild every input."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests.golden.make_golden import RESIZE_CASES, sha  # noqa: E402
from tests.interleaved_ref import FORMATS, pack422  # noqa: E402

CHANNELS = {"bgr": 3, "rgb": 3, "bgra": 4, "rgba": 4, "gray": None, "yuyv": 2, "uyvy": 2, "yvyu": 2}
# (h, w) of the frames stored in full, every format (random bytes: the 4-channel frames carry random alpha)
SMALL = [(36, 50), (2, 2), (5, 6)]


def cases(fmt):
    """the indices into RESIZE_CASES a format is pinned on"""
    return [i for i, c in enumerate(RESIZE_CASES) if CHANNELS[fmt] != 2 or c[1] % 2 == 0]


def interleaved_frame(seed, h, w, fmt):
    """seeded uint8 frame of `fmt`: (h, w, C), or (h, w) for gray"""
    ch = CHANNELS[fmt]
    return np.random.default_rng(seed).integers(0, 256, (h, w) if ch is None else (h, w, ch), dtype=np.uint8)


def case_frame(i, fmt):
    """the source of RESIZE_CASES[i] in `fmt`"""
    return interleaved_frame(1000 + 16 * i + FORMATS.index(fmt), *RESIZE_CASES[i][:2], fmt)


def sweep422(fmt):
    """a (256, 512) 4:2:2 frame: pixel pair k of row r has U = k, V = r and luma (2k + r, 2k + 1 + r) mod 256, so every U, V pair
    occurs, and every luma value against every U value and against every V value"""
    r, x = np.arange(256)[:, None], np.arange(512)[None, :]
    Y = ((x + r) % 256).astype(np.uint8)
    U = np.tile(np.arange(256, dtype=np.uint8), (256, 1))
    V = np.repeat(np.arange(256, dtype=np.uint8)[:, None], 256, 1)
    return pack422(Y, U, V, fmt)


def make_interleaved():
    """RESIZE_CASES[i] in format f: seed 1000 + 16 i + FORMATS.index(f); SMALL[i]: seed 1900 + 16 i + FORMATS.index(f)"""
    import cv2
    codes = {"rgb": cv2.COLOR_RGB2BGR, "bgra": cv2.COLOR_BGRA2BGR, "rgba": cv2.COLOR_RGBA2BGR, "gray": cv2.COLOR_GRAY2BGR,
             "yuyv": cv2.COLOR_YUV2BGR_YUYV, "uyvy": cv2.COLOR_YUV2BGR_UYVY, "yvyu": cv2.COLOR_YUV2BGR_YVYU}

    def cvt(src, fmt):
        return src.copy() if fmt == "bgr" else cv2.cvtColor(src, codes[fmt])

    out = {"cv2_version": np.array(cv2.__version__)}
    for fmt in FORMATS:
        for i in cases(fmt):
            sh, sw, dh, dw = RESIZE_CASES[i]
            bgr = cvt(case_frame(i, fmt), fmt)
            out[f"{fmt}{i}_cvt_sha"] = np.array(sha(bgr))
            out[f"{fmt}{i}_rz_sha"] = np.array(sha(cv2.resize(bgr, (dw, dh))))
            h1 = dw * (sh / float(sw)); w2 = dh * (sw / float(sh))
            rw, rh = (dw, int(h1)) if h1 <= dh else (int(w2), dh)
            lb = cv2.copyMakeBorder(cv2.resize(bgr, (rw, rh)), 0, dh - rh, 0, dw - rw, cv2.BORDER_CONSTANT, value=(0, 0, 0))
            out[f"{fmt}{i}_lb_sha"] = np.array(sha(lb))
        for i, (h, w) in enumerate(SMALL):
            src = interleaved_frame(1900 + 16 * i + FORMATS.index(fmt), h, w, fmt)
            out[f"small{i}_{fmt}_in"] = src
            out[f"small{i}_{fmt}_bgr"] = cvt(src, fmt)
        if CHANNELS[fmt] == 2:   # the three sweeps are the same planes: one BGR frame in full, each format's sha
            bgr = cvt(sweep422(fmt), fmt)
            out[f"sweep_{fmt}_sha"] = np.array(sha(bgr))
            out["sweep_bgr"] = bgr
    np.savez_compressed(os.path.join(HERE, "cv_pin_interleaved.npz"), **out)


if __name__ == "__main__":
    make_interleaved()
