"""Generates tests/golden/*.npz.  Run in the BUILD container only (needs Python cv2 and
/root/reference; neither is required at test time):

    python tests/golden/make_golden.py

1. cv_pin.npz      -- outputs of the real OpenCV (Python cv2) for the two third-party
                      primitives on the reference's path: cv::resize(INTER_AREA) upscale
                      (src/post_process.hpp:50) and cv::GaussianBlur(17x17, sigma=3)
                      (post_process.hpp:66-67), on seeded inputs; small cases stored in full,
                      full-size cases as sha256 of the output bytes.
2. ref_humans.npz  -- human_t lists produced by the reference's OWN src/paf.cpp (compiled
                      verbatim into oracle/_ref by oracle/Makefile) on the seeded synthetic
                      frames of hyperpose_b200/synthetic.py (SURVEY 8d configs).
3. ref_pifpaf_large.npz (`python tests/golden/make_golden.py pifpaf_large`) -- the reference's own
                      PifPaf decoder on fields of real frame sizes (PIFPAF_LARGE_CASES).
4. ref_humans_large.npz + cv_pin_large.npz (`python tests/golden/make_golden.py paf_large`) -- the reference's
                      own src/paf.cpp on PAF_LARGE_CASES, and sha256 of real cv2 INTER_AREA / GaussianBlur at each of
                      their geometries (PAF_LARGE_PINS).
"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
HERE = os.path.dirname(os.path.abspath(__file__))

# (name, seed, persons, hf, wf, res_w, res_h, conf_thresh, paf_thresh)
FRAME_CASES = [
    ("cfg1_p1", 0, 1, 46, 54, -1, -1, 0.05, 0.05),
    ("cfg1_p3", 1, 3, 46, 54, -1, -1, 0.05, 0.05),
    ("cfg3_p5", 2, 5, 46, 82, -1, -1, 0.05, 0.05),
    ("cfg4_crowd", 3, (10, 20), 46, 54, -1, -1, 0.05, 0.05),
    ("cfg3_crowd", 5, 12, 46, 82, -1, -1, 0.05, 0.05),
    ("square", 6, 4, 46, 46, -1, -1, 0.05, 0.05),
    ("user_res", 7, 3, 46, 54, 216, 184, 0.05, 0.05),       # untransposed 4x resolution set by the user
    ("user_res_odd", 8, 3, 46, 54, 300, 200, 0.1, 0.08),
    ("empty", 9, 0, 46, 54, -1, -1, 0.05, 0.05),
    ("tiny", 10, 1, 12, 16, -1, -1, 0.05, 0.05),
]


# (src_h, src_w, dst_h, dst_w) of the frame-resize pin
RESIZE_CASES = [(360, 640, 368, 656), (480, 640, 368, 656), (720, 1280, 368, 656), (736, 1312, 368, 656), (100, 80, 368, 432),
                (1080, 1920, 368, 656), (368, 656, 368, 656), (300, 500, 207, 344), (37, 53, 64, 48)]


# (name, seed, persons, h, w, keypoint_thresh) of the PifPaf decode pin (BASELINE config 5: 385x385 -> 49x49 fields)
PIFPAF_CASES = [("pp_p2", 4, 2, 49, 49, 0.1), ("pp_p5", 5, 5, 49, 49, 0.1), ("pp_crowd", 6, (6, 12), 49, 49, 0.1), ("pp_empty", 7, 0, 49, 49, 0.1),
                ("pp_rect", 8, 3, 47, 55, 0.1), ("pp_thr", 9, 4, 49, 49, 0.3), ("pp_small", 10, 2, 25, 33, 0.1)]


# (name, seed, persons, h, w, scale range in cells) of the PifPaf decode pin at real frame sizes (keypoint threshold 0.1):
# 99 x 124 = 12,276 cells and 99 x 125 bracket the field size a whole field's cells once fitted in 48 KiB of shared memory;
# 89 x 159 is a 1280 x 720 input, 91 x 161 a 1281 x 721 one.  Scales of 4-8 cells give 33-65 px footprints on the
# high-resolution map; "pl_dense" has more than 8192 seeds, the decoder's initial seed capacity.
PIFPAF_LARGE_CASES = [("pl_99x124", 30, (6, 10), 99, 124, (4.0, 8.0)), ("pl_99x125", 31, (6, 10), 99, 125, (4.0, 8.0)),
                      ("pl_89x159", 32, (6, 12), 89, 159, (1.0, 8.0)), ("pl_91x161", 33, (6, 12), 91, 161, (4.0, 8.0)),
                      ("pl_161x161", 34, (8, 12), 161, 161, (4.0, 8.0)), ("pl_dense", 35, 40, 161, 161, (1.0, 1.5))]


# (name, seed, persons, net_w, net_h, gh, gw, nh, nw, point_thresh, limb_thresh, nms_thresh, distractors) of the Pose Proposal pin
PPN_CASES = [("ppn_p1", 20, 1, 384, 384, 12, 12, 9, 9, 0.10, 0.05, 0.3, 12), ("ppn_p4", 21, 4, 384, 384, 12, 12, 9, 9, 0.10, 0.05, 0.3, 12),
             ("ppn_crowd", 22, (6, 10), 384, 384, 12, 12, 9, 9, 0.10, 0.05, 0.3, 40), ("ppn_empty", 23, 0, 384, 384, 12, 12, 9, 9, 0.10, 0.05, 0.3, 0),
             ("ppn_rect", 24, 3, 512, 384, 12, 16, 7, 9, 0.10, 0.05, 0.3, 12), ("ppn_thr", 25, 4, 384, 384, 12, 12, 9, 9, 0.30, 0.20, 0.5, 12),
             ("ppn_dense", 26, 5, 384, 384, 12, 12, 9, 9, 0.05, 0.03, 0.3, 60)]


# (src_h, src_w, dst_h, dst_w) of the INTER_AREA pin for the regimes beyond pure up-scaling (A5): mixed (one axis shrinks: 2-tap
# area-mode lerp on both), integer factors (resizeAreaFast_, incl. the 2x2 SIMD kernel and its scalar tail), fractional (DecimateAlpha)
AREA_CASES = [(46, 82, 100, 60), (46, 82, 30, 200), (46, 200, 800, 184), (46, 82, 23, 41), (48, 84, 16, 28), (48, 84, 12, 21), (46, 82, 46, 41),
              (46, 82, 23, 82), (40, 84, 20, 41), (46, 82, 30, 50), (46, 82, 45, 81), (46, 82, 20, 82), (54, 46, 13, 17), (46, 82, 46, 50), (46, 82, 11, 19)]

# parser cases whose up-map shrinks an axis: (name, seed, persons, hf, wf, res_w, res_h, conf_thresh, paf_thresh)
AREA_FRAME_CASES = [
    # default resolution (width 4*Hf, height 4*Wf) = (120, 520): width 120 < Wf = 130 -> mixed regime.  (Much wider maps, e.g. 24x120,
    # stretch rows ~20x: the plateaus give limb candidates with EXACTLY equal scores and the reference's unstable std::sort
    # (paf.cpp:246) then picks among them arbitrarily -- the region test_oracle_matches_live_reference_sweep documents.)
    ("wide_default", 11, 3, 30, 130, -1, -1, 0.05, 0.05),
    ("user_mixed", 12, 3, 46, 54, 40, 300, 0.05, 0.05),      # x shrinks, y grows
    ("user_half", 13, 3, 46, 54, 27, 23, 0.05, 0.05),        # exact 2x2 reduction (SIMD kernel + tail)
    ("user_third", 14, 2, 48, 54, 18, 16, 0.05, 0.05),       # 3x3 integer reduction
    ("user_frac", 15, 3, 46, 54, 41, 33, 0.05, 0.05),        # fractional reduction on both axes
    ("user_keep_x", 16, 3, 46, 54, 54, 30, 0.05, 0.05),      # one axis kept (scale 1), the other shrinks: area regime
]


# parser cases at real frame sizes: (name, seed, persons, hf, wf, res_w, res_h, conf_thresh, paf_thresh, person_height).  The map
# sizes straddle the size-dependent paths of paf_parser.cu (tests/test_paf_large.py asserts which ones each case takes, with the
# H100's 200 KiB of dynamic shared memory for the limb kernel): up-sampling tables in shared memory while UW + UH <= 1024
# (92 x 164 is the last, 92 x 165 / 93 x 164 the first beyond), both PAF planes of a limb while 8 H W + 12288 <= 200 KiB
# (128 x 188 is the last, 128 x 189 the first beyond), TMA or scalar plane copies (H W divisible by 4 or odd), the peak kernel's
# direct up-sampling (portrait maps: fewer than ~3.4 up-map rows per source row) and its generic source staging (a resolution
# within ~1.27x of the map width).  "noise" is a structureless field (uniform PAF noise, uniform conf noise on the parts of
# NOISY_PARTS, halved elsewhere so that those stay below the threshold): > 1000 peaks per noisy part, > 500 connections per
# limb between them, the unstaged assembly and capacity growth, while the partial humans of the assembly stay in shared memory.
PAF_LARGE_CASES = [
    ("l_90x160", 60, (6, 10), 90, 160, -1, -1, 0.05, 0.05, (0.25, 0.7)),        # 1280 x 720 input
    ("l_91x161", 61, (6, 10), 91, 161, -1, -1, 0.05, 0.05, (0.25, 0.7)),        # odd H W; UW = 364 = 4 mod 8
    ("l_92x164", 62, (6, 10), 92, 164, -1, -1, 0.05, 0.05, (0.25, 0.7)),        # 1312 x 736 input; UW + UH = 1024
    ("l_92x165", 63, (6, 10), 92, 165, -1, -1, 0.05, 0.05, (0.25, 0.7)),
    ("l_93x164", 64, (6, 10), 93, 164, -1, -1, 0.05, 0.05, (0.25, 0.7)),
    ("l_128x188", 65, (6, 10), 128, 188, -1, -1, 0.05, 0.05, (0.25, 0.7)),      # H W = 24064
    ("l_128x189", 66, (6, 10), 128, 189, -1, -1, 0.05, 0.05, (0.25, 0.7)),      # H W = 24192
    ("l_135x240", 67, (6, 10), 135, 240, -1, -1, 0.05, 0.05, (0.25, 0.7)),      # 1920 x 1080 input; UW = 540
    ("l_240x135", 68, (4, 8), 240, 135, -1, -1, 0.05, 0.05, (0.25, 0.7)),       # portrait 1080p
    ("l_160x90", 69, (4, 8), 160, 90, -1, -1, 0.05, 0.05, (0.25, 0.7)),         # portrait 720p
    ("l_100x110_res", 70, (4, 8), 100, 110, 110, 400, 0.05, 0.05, (0.3, 0.8)),  # up-map width = map width
    ("l_120x300_res", 71, (4, 8), 120, 300, 330, 1200, 0.05, 0.05, (0.3, 0.8)),  # UW = 330 = 2 mod 8
    ("l_crowd", 72, (30, 40), 135, 240, -1, -1, 0.05, 0.05, (0.1, 0.3)),
    ("l_noise", 73, "noise", 135, 240, -1, -1, 0.6, 0.05, None),
]
NOISY_PARTS = (1, 2, 3, 5)

# one parser handle fed several map sizes in turn: the resolution and the length penalty's feature height are fixed at its
# first call (paf.cpp:314-315, 321-332).  The second handle's small map is stretched 8x: much more (46 x 54 at 540 x 960 stretches
# rows 21x) gives plateaus with exactly equal limb scores, where the reference's unstable std::sort decides (see AREA_FRAME_CASES).
PAF_HANDLE_SEQUENCES = [((46, 82), (135, 240), (90, 160), (135, 240)), ((135, 240), (68, 120))]


def paf_handle_tensors(k, h, w):
    """(conf, paf) of call k of a PAF_HANDLE_SEQUENCES entry, on h x w maps"""
    from hyperpose_b200 import synthetic as syn
    return syn.make_frame_tensors(500 + k, (4, 8), h, w, person_height=(0.3, 0.8))


def paf_large_tensors(case):
    """(conf[19,hf,wf], paf[38,hf,wf]) of a PAF_LARGE_CASES entry"""
    name, seed, P, hf, wf = case[:5]
    if P == "noise":
        rng = np.random.default_rng(seed)
        conf, paf = rng.random((19, hf, wf), dtype=np.float32), rng.random((38, hf, wf), dtype=np.float32) - 0.5
        conf[[k for k in range(19) if k not in NOISY_PARTS]] *= np.float32(0.5)
        return conf, paf
    from hyperpose_b200 import synthetic as syn
    return syn.make_frame_tensors(seed, P, hf, wf, person_height=case[9])


def _handle_geometries():
    """(H, W, UH, UW) of every call of PAF_HANDLE_SEQUENCES"""
    out = []
    for seq in PAF_HANDLE_SEQUENCES:
        uw, uh = 4 * seq[0][0], 4 * seq[0][1]
        out += [(h, w, uh, uw) for (h, w) in seq]
    return out


# (H, W, UH, UW) of the INTER_AREA / GaussianBlur pin at the large geometries
PAF_LARGE_PINS = sorted({(c[3], c[4], c[6] if c[6] > 0 else 4 * c[4], c[5] if c[5] > 0 else 4 * c[3]) for c in PAF_LARGE_CASES}
                        | set(_handle_geometries()))


def make_paf_large():
    """tests/golden/ref_humans_large.npz (the reference's own paf.cpp) + cv_pin_large.npz (real cv2)"""
    import cv2
    import oracle
    oracle.build()
    pin = {"cv2_version": np.array(cv2.__version__)}
    for i, (h, w, uh, uw) in enumerate(PAF_LARGE_PINS):
        img = np.random.default_rng(400 + i).random((h, w), dtype=np.float32)
        up = cv2.resize(img, (uw, uh), interpolation=cv2.INTER_AREA)
        pin[f"pin{i}_dims"] = np.array([h, w, uh, uw])
        pin[f"pin{i}_up_sha"] = np.array(sha(up))
        pin[f"pin{i}_blur_sha"] = np.array(sha(cv2.GaussianBlur(up, (17, 17), 3.0)))
    np.savez_compressed(os.path.join(HERE, "cv_pin_large.npz"), **pin)
    ref = {}
    for case in PAF_LARGE_CASES:
        name, rw, rh, ct, pt = case[0], case[5], case[6], case[7], case[8]
        conf, paf = paf_large_tensors(case)
        rp = oracle.RefParser(ct, pt, rw, rh)
        ref[name + "_humans"] = rp.process(conf, paf, cap=4096)
        ref[name + "_in_sha"] = np.array(sha(conf) + sha(paf))
        rp.close()
    for s, seq in enumerate(PAF_HANDLE_SEQUENCES):   # one reference handle per sequence, every call through it
        rp = oracle.RefParser()
        for k, (h, w) in enumerate(seq):
            conf, paf = paf_handle_tensors(k, h, w)
            ref[f"handle{s}_{k}_humans"] = rp.process(conf, paf, cap=4096)
            ref[f"handle{s}_{k}_in_sha"] = np.array(sha(conf) + sha(paf))
        rp.close()
    np.savez_compressed(os.path.join(HERE, "ref_humans_large.npz"), **ref)
    print({k: len(v) for k, v in ref.items() if k.endswith("_humans")})


def make_area():
    """tests/golden/cv_pin_area.npz (real cv2) + ref_humans_area.npz (the reference's own paf.cpp over the pinned resize)"""
    import cv2
    import oracle
    from hyperpose_b200 import synthetic as syn
    oracle.build()
    out = {"cv2_version": np.array(cv2.__version__)}
    for i, (sh, sw, dh, dw) in enumerate(AREA_CASES):
        img = np.random.default_rng(300 + i).random((sh, sw), dtype=np.float32)
        ref = cv2.resize(img, (dw, dh), interpolation=cv2.INTER_AREA)
        out[f"area{i}_sha"] = np.array(sha(ref))
        if ref.size <= 4096:
            out[f"area{i}_out"] = ref
    np.savez_compressed(os.path.join(HERE, "cv_pin_area.npz"), **out)
    ref = {}
    for (name, seed, P, hf, wf, rw, rh, ct, pt) in AREA_FRAME_CASES:
        conf, paf = syn.make_frame_tensors(seed, P, hf, wf)
        rp = oracle.RefParser(ct, pt, rw, rh)
        ref[name + "_humans"] = rp.process(conf, paf)
        ref[name + "_in_sha"] = np.array(sha(conf) + sha(paf))
        rp.close()
    np.savez_compressed(os.path.join(HERE, "ref_humans_area.npz"), **ref)
    print({k: len(v) for k, v in ref.items() if k.endswith("_humans")})


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def main():
    import cv2
    from hyperpose_b200 import synthetic as syn
    import oracle

    out = {"cv2_version": np.array(cv2.__version__)}
    out["gauss_kernel"] = cv2.getGaussianKernel(17, 3.0, cv2.CV_32F).ravel()
    rng = np.random.default_rng(1234)
    small = [(23, 27, 108, 92), (12, 16, 64, 48), (9, 9, 36, 36), (10, 7, 31, 40), (5, 20, 80, 20)]
    for i, (sh, sw, dh, dw) in enumerate(small):
        img = rng.random((sh, sw), dtype=np.float32) * 2 - 0.5
        up = cv2.resize(img, (dw, dh), interpolation=cv2.INTER_AREA)
        out[f"small{i}_in"] = img
        out[f"small{i}_shape"] = np.array([dh, dw])
        out[f"small{i}_up"] = up
        out[f"small{i}_blur"] = cv2.GaussianBlur(up, (17, 17), 3.0)
    big = [(46, 54, 216, 184), (46, 82, 328, 184), (46, 46, 184, 184), (46, 54, 184, 216)]
    for i, (sh, sw, dh, dw) in enumerate(big):
        img = np.random.default_rng(100 + i).random((sh, sw), dtype=np.float32)
        up = cv2.resize(img, (dw, dh), interpolation=cv2.INTER_AREA)
        out[f"big{i}_dims"] = np.array([sh, sw, dh, dw])
        out[f"big{i}_up_sha"] = np.array(sha(up))
        out[f"big{i}_blur_sha"] = np.array(sha(cv2.GaussianBlur(up, (17, 17), 3.0)))
    # cv::resize(INTER_LINEAR) on u8 frames (src/tensorrt.cpp:451) and the letterbox path (src/data.cpp:53-69)
    for i, (sh, sw, dh, dw) in enumerate(RESIZE_CASES):
        img = np.random.default_rng(200 + i).integers(0, 256, (sh, sw, 3), dtype=np.uint8)
        out[f"rz{i}_sha"] = np.array(sha(cv2.resize(img, (dw, dh))))
        h1 = dw * (sh / float(sw)); w2 = dh * (sw / float(sh))
        rw, rh = (dw, int(h1)) if h1 <= dh else (int(w2), dh)
        lb = cv2.copyMakeBorder(cv2.resize(img, (rw, rh)), 0, dh - rh, 0, dw - rw, cv2.BORDER_CONSTANT, value=(0, 0, 0))
        out[f"lb{i}_sha"] = np.array(sha(lb))
    np.savez_compressed(os.path.join(HERE, "cv_pin.npz"), **out)

    ref = {}
    for (name, seed, P, hf, wf, rw, rh, ct, pt) in FRAME_CASES:
        conf, paf = syn.make_frame_tensors(seed, P, hf, wf)
        rp = oracle.RefParser(ct, pt, rw, rh)
        ref[name + "_humans"] = rp.process(conf, paf)
        ref[name + "_in_sha"] = np.array(sha(conf) + sha(paf))
        rp.close()
    np.savez_compressed(os.path.join(HERE, "ref_humans.npz"), **ref)
    pp = {}
    for (name, seed, P, h, w, thr) in PIFPAF_CASES:
        pif, paf = syn.make_pifpaf_fields(seed, P, h, w)
        pp[name + "_humans"] = oracle.ref_pifpaf_process(pif, paf, (h - 1) * 8 + 1, (w - 1) * 8 + 1, thr)
        pp[name + "_in_sha"] = np.array(sha(pif) + sha(paf))
    np.savez_compressed(os.path.join(HERE, "ref_pifpaf.npz"), **pp)
    make_pifpaf_live()
    make_ppn()


def make_pifpaf_live():
    """the reference decoder on the inputs of test_gpu_decoder_batched_vs_live_reference (batched_i) and test_pifpaf_fields_hand_off
    (handoff_i): those tests compare with these records where oracle/_ref is not built, and check them against it where it is"""
    from hyperpose_b200 import synthetic as syn
    import oracle
    out = {}
    for i in range(8):
        pif, paf = syn.make_pifpaf_fields(100 + i, (1, 9), 49, 49)
        out[f"batched_{i}"] = oracle.ref_pifpaf_process(pif, paf, 385, 385, 0.1)
    for i in range(2):
        pif, paf = syn.make_pifpaf_fields(20 + i, (2, 3), 49, 49)
        out[f"handoff_{i}"] = oracle.ref_pifpaf_process(pif.astype(np.float32), paf.astype(np.float32), 385, 385, 0.1)
    np.savez_compressed(os.path.join(HERE, "ref_pifpaf_live.npz"), **out)


def make_pifpaf_large():
    """the reference decoder on PIFPAF_LARGE_CASES (tests/test_pifpaf_stages.py)"""
    from hyperpose_b200 import synthetic as syn
    import oracle
    out = {}
    for (name, seed, P, h, w, scale) in PIFPAF_LARGE_CASES:
        pif, paf = syn.make_pifpaf_fields(seed, P, h, w, scale=scale)
        out[name + "_humans"] = oracle.ref_pifpaf_process(pif, paf, (h - 1) * 8 + 1, (w - 1) * 8 + 1, 0.1)
        out[name + "_in_sha"] = np.array(sha(pif) + sha(paf))
    np.savez_compressed(os.path.join(HERE, "ref_pifpaf_large.npz"), **out)
    print({k: len(v) for k, v in out.items() if k.endswith("_humans")})


def make_ppn():
    """goldens of the reference's own src/pose_proposal.cpp (oracle/_ref/libref_ppn.so) on seeded synthetic tensors"""
    from hyperpose_b200 import synthetic as syn
    import oracle
    pn = {}
    for (name, seed, P, net_w, net_h, gh, gw, nh, nw, pt, lt, nt, nd) in PPN_CASES:
        t = syn.make_ppn_tensors(seed, P, net_h, net_w, gh, gw, nh, nw, nd)
        pn[name + "_humans"] = oracle.ref_ppn_process(*t, net_w, net_h, pt, lt, nt)
        pn[name + "_in_sha"] = np.array("".join(sha(a) for a in t))
    np.savez_compressed(os.path.join(HERE, "ref_ppn.npz"), **pn)
    print("wrote", os.listdir(HERE))


if __name__ == "__main__" and "area" in sys.argv[1:]:
    make_area()
    sys.exit(0)

if __name__ == "__main__":
    if "ppn" in sys.argv[1:]:
        make_ppn()
    elif "pifpaf_large" in sys.argv[1:]:
        make_pifpaf_large()
    elif "paf_large" in sys.argv[1:]:
        make_paf_large()
    else:
        main()
