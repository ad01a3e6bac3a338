"""Seeded synthetic conf / PAF tensors and frames for tests and bench (SURVEY.md 8d).

There are no weights, media or fixtures in the reference tree (scripts/downloader.py
needs the network), so every measurement uses tensors synthesised the way the
reference synthesises its *training targets*:

* conf: per joint ``max_persons exp(-d^2 / (2*7^2))`` sampled at cell centres
  ``8*i + 3.5`` and cut at 4.6052  (hyperpose/Model/openpose/utils.py:55-86),
  background channel ``clip(1 - max, 0, 1)`` (utils.py:48);
* PAF: unit limb vector within 1 cell of the segment, averaged over overlaps
  (utils.py:174-216), channel pairs in ``CocoLimb`` order (openpose/define.py:24-25),
  which is the order ``COCOPAIRS_NET`` (src/coco.hpp:10-30) indexes.

numpy only; nothing here is on the product path.
"""
from __future__ import annotations

import numpy as np

STRIDE = 8
N_PARTS = 18
N_LIMBS = 19

# hyperpose/Model/openpose/define.py:24-25
COCO_LIMB = list(zip([1, 8, 9, 1, 11, 12, 1, 2, 3, 2, 1, 5, 6, 5, 1, 0, 0, 14, 15],
                     [8, 9, 10, 11, 12, 13, 2, 3, 4, 16, 5, 6, 7, 17, 0, 14, 15, 16, 17]))

# (x, y) of the 18 COCO parts in a unit person box (y down)
_TEMPLATE = np.array([
    (0.50, 0.08), (0.50, 0.20), (0.36, 0.20), (0.30, 0.37), (0.27, 0.52), (0.64, 0.20),
    (0.70, 0.37), (0.73, 0.52), (0.42, 0.53), (0.41, 0.73), (0.40, 0.93), (0.58, 0.53),
    (0.59, 0.73), (0.60, 0.93), (0.46, 0.05), (0.54, 0.05), (0.41, 0.08), (0.59, 0.08)],
    dtype=np.float64)


def random_skeletons(rng: np.random.Generator, n_persons: int, height: int, width: int,
                     person_height=(0.55, 0.9)) -> np.ndarray:
    """[P,18,2] joint (x, y) positions in network-input pixels; each person's height is drawn uniformly from
    `person_height` (fractions of the frame height)."""
    out = np.zeros((n_persons, N_PARTS, 2))
    for p in range(n_persons):
        ph = rng.uniform(person_height[0], person_height[1]) * height            # person height in pixels
        pw = ph * rng.uniform(0.75, 0.95)
        x0 = rng.uniform(-0.1 * pw, max(-0.1 * pw + 1.0, width - 0.9 * pw))
        y0 = rng.uniform(0.0, max(1.0, height - ph))
        jit = rng.normal(0.0, 0.012, size=(N_PARTS, 2))
        pts = (_TEMPLATE + jit) * np.array([pw, ph]) + np.array([x0, y0])
        out[p] = pts
    return out


def conf_paf_from_skeletons(skel: np.ndarray, hf: int, wf: int, rng: np.random.Generator | None = None,
                            noise: float = 0.02):
    """conf f32[19,hf,wf], paf f32[38,hf,wf] for joints given in input pixels."""
    conf = np.zeros((N_PARTS + 1, hf, wf), dtype=np.float64)
    ys = np.arange(hf) * STRIDE + (STRIDE / 2 - 0.5)
    xs = np.arange(wf) * STRIDE + (STRIDE / 2 - 0.5)
    for person in skel:
        for k, (cx, cy) in enumerate(person):
            if cx < 0 or cy < 0 or cx >= wf * STRIDE or cy >= hf * STRIDE:
                continue
            d2 = ((ys - cy) ** 2)[:, None] + ((xs - cx) ** 2)[None, :]
            e = d2 / (2 * 7.0 * 7.0)
            g = np.exp(-e)
            g[e > 4.6052] = 0
            conf[k] = np.maximum(conf[k], g)
    conf[-1] = np.clip(1 - conf[:-1].max(axis=0), 0.0, 1.0)

    vec = np.zeros((2 * N_LIMBS, hf, wf), dtype=np.float64)
    cnt = np.zeros((N_LIMBS, hf, wf), dtype=np.float64)
    yy, xx = np.mgrid[0:hf, 0:wf]
    for person in skel / STRIDE:
        for i, (a, b) in enumerate(COCO_LIMB):
            (x1, y1), (x2, y2) = person[a], person[b]
            vx, vy = x2 - x1, y2 - y1
            ln = np.hypot(vx, vy)
            if ln == 0:
                continue
            nx, ny = vx / ln, vy / ln
            x_lo, x_hi = max(0, int(round(min(x1, x2) - 1))), min(wf, int(round(max(x1, x2) + 1)))
            y_lo, y_hi = max(0, int(round(min(y1, y2) - 1))), min(hf, int(round(max(y1, y2) + 1)))
            if x_lo >= x_hi or y_lo >= y_hi:
                continue
            sub_x, sub_y = xx[y_lo:y_hi, x_lo:x_hi], yy[y_lo:y_hi, x_lo:x_hi]
            dist = np.abs((sub_x - x1) * ny - (sub_y - y1) * nx)
            m = (dist <= 1).astype(np.float64)
            cnt[i, y_lo:y_hi, x_lo:x_hi] += m
            vec[2 * i, y_lo:y_hi, x_lo:x_hi] += nx * m
            vec[2 * i + 1, y_lo:y_hi, x_lo:x_hi] += ny * m
    nz = cnt > 0
    for i in range(N_LIMBS):
        vec[2 * i][nz[i]] /= cnt[i][nz[i]]
        vec[2 * i + 1][nz[i]] /= cnt[i][nz[i]]
    if rng is not None and noise > 0:
        conf = conf + rng.uniform(0, noise, size=conf.shape)
        vec = vec + rng.uniform(-noise, noise, size=vec.shape)
    return conf.astype(np.float32), vec.astype(np.float32)


def make_frame_tensors(seed: int, n_persons, hf: int = 46, wf: int = 54, noise: float = 0.02, person_height=(0.55, 0.9)):
    """One frame: (conf[19,hf,wf], paf[38,hf,wf]).  n_persons: int or (lo, hi) inclusive; person_height: see random_skeletons."""
    rng = np.random.default_rng(seed)
    if isinstance(n_persons, tuple):
        n_persons = int(rng.integers(n_persons[0], n_persons[1] + 1))
    skel = random_skeletons(rng, n_persons, hf * STRIDE, wf * STRIDE, person_height)
    return conf_paf_from_skeletons(skel, hf, wf, rng, noise)


def make_batch_tensors(seed: int, n_frames: int, n_persons, hf: int = 46, wf: int = 54, noise: float = 0.02,
                       person_height=(0.55, 0.9)):
    """(conf[N,19,hf,wf], paf[N,38,hf,wf]); frame i uses seed ``seed*100003 + i``."""
    cs, ps = [], []
    for i in range(n_frames):
        c, p = make_frame_tensors(seed * 100003 + i, n_persons, hf, wf, noise, person_height)
        cs.append(c)
        ps.append(p)
    return np.stack(cs), np.stack(ps)


def make_frames_u8(seed: int, n_frames: int, height: int, width: int) -> np.ndarray:
    """u8[N,height,width,3] BGR frames (SURVEY 8d: cfg2 default_rng(1), cfg3 default_rng(2))."""
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, size=(n_frames, height, width, 3), dtype=np.uint8)


# ---------------------------------------------------------------------------------------------
# OpenPifPaf fields (BASELINE config 5; SURVEY 8d cfg5 recipe)
# ---------------------------------------------------------------------------------------------
# 17 COCO keypoints in OpenPifPaf order; 19 bones, 1-based (src/pifpaf_decoder/openpifpaf_postprocessor.cpp:64-84)
PIFPAF_BONES = [(16, 14), (14, 12), (17, 15), (15, 13), (12, 13), (6, 12), (7, 13), (6, 7), (6, 8), (7, 9), (8, 10), (9, 11),
                (2, 3), (1, 2), (1, 3), (2, 4), (3, 5), (4, 6), (5, 7)]
# (x, y) of the 17 keypoints in a unit person box: nose, l/r eye, l/r ear, l/r shoulder, l/r elbow, l/r wrist, l/r hip, l/r knee, l/r ankle
_PIF_TEMPLATE = np.array([
    (0.50, 0.08), (0.54, 0.05), (0.46, 0.05), (0.59, 0.08), (0.41, 0.08), (0.64, 0.20), (0.36, 0.20), (0.70, 0.37),
    (0.30, 0.37), (0.73, 0.52), (0.27, 0.52), (0.58, 0.53), (0.42, 0.53), (0.59, 0.73), (0.41, 0.73), (0.60, 0.93), (0.40, 0.93)])


def make_pifpaf_fields(seed: int, n_persons, h: int = 49, w: int = 49, scale=(1.0, 1.5)):
    """(pif f32[17,5,h,w] = {conf, x, y, b, scale}, paf f32[19,9,h,w] = {conf, x1, y1, x2, y2, b1, b2, s1, s2}); all
    coordinates / scales absolute, in feature-cell units (the decoder multiplies by its stride 8,
    openpifpaf_postprocessor.cpp:326-328,726-730).  Each person's scale is drawn uniformly from `scale` (cells)."""
    rng = np.random.default_rng(seed)
    if isinstance(n_persons, tuple):
        n_persons = int(rng.integers(n_persons[0], n_persons[1] + 1))
    pif = np.zeros((17, 5, h, w), np.float32)
    paf = np.zeros((19, 9, h, w), np.float32)
    pif[:, 0] = rng.uniform(0.0, 0.05, (17, h, w))          # background confidences stay below every threshold
    paf[:, 0] = rng.uniform(0.0, 0.05, (19, h, w))
    pif[:, 4] = 1.0
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    for _ in range(n_persons):
        ph = rng.uniform(0.45, 0.9) * h
        pw = ph * rng.uniform(0.6, 0.8)
        x0 = rng.uniform(0.0, max(1.0, w - pw)); y0 = rng.uniform(0.0, max(1.0, h - ph))
        pts = (_PIF_TEMPLATE + rng.normal(0, 0.01, (17, 2))) * np.array([pw, ph]) + np.array([x0, y0])
        s_p = float(rng.uniform(scale[0], scale[1]))
        for k, (cx, cy) in enumerate(pts):
            m = ((xx - cx) ** 2 + (yy - cy) ** 2) <= 2.3 ** 2
            n = int(m.sum())
            if n == 0:
                continue
            pif[k, 0][m] = rng.uniform(0.85, 0.95, n)
            pif[k, 1][m] = cx + rng.normal(0, 0.02, n)
            pif[k, 2][m] = cy + rng.normal(0, 0.02, n)
            pif[k, 3][m] = rng.uniform(0.2, 0.4, n)
            pif[k, 4][m] = s_p + rng.normal(0, 0.02, n)
        for b, (j1, j2) in enumerate(PIFPAF_BONES):
            (x1, y1), (x2, y2) = pts[j1 - 1], pts[j2 - 1]
            for t in np.linspace(0.0, 1.0, 9):
                cx, cy = int(round(x1 + t * (x2 - x1))), int(round(y1 + t * (y2 - y1)))
                if 0 <= cx < w and 0 <= cy < h:
                    paf[b, :, cy, cx] = (rng.uniform(0.85, 0.95), x1 + rng.normal(0, 0.02), y1 + rng.normal(0, 0.02),
                                         x2 + rng.normal(0, 0.02), y2 + rng.normal(0, 0.02), 0.3, 0.3, s_p, s_p)
    return pif, paf


# ---------------------------------------------------------------------------------------------
# Pose Proposal Network tensors (src/pose_proposal.cpp:14-20): conf_point / conf_iou / x / y / w / h [18,gh,gw] and
# edge [17,nh,nw,gh,gw]; boxes in network-input pixels
# ---------------------------------------------------------------------------------------------
# src/pose_proposal.cpp:24-42
PPN_PAIRS = [(1, 8), (8, 9), (9, 10), (1, 11), (11, 12), (12, 13), (1, 2), (2, 3), (3, 4), (1, 5), (5, 6), (6, 7),
             (1, 0), (0, 14), (0, 15), (14, 16), (15, 17)]


def make_ppn_tensors(seed: int, n_persons, net_h: int = 384, net_w: int = 384, gh: int = 12, gw: int = 12, nh: int = 9, nw: int = 9,
                     distractors: int = 12):
    """(conf_point, conf_iou, x, y, w, h) f32[18,gh,gw] + edge f32[17,nh,nw,gh,gw] for P random skeletons: the joint's cell
    proposes a box centred on the joint, its 4-neighbours propose weaker overlapping boxes (NMS food), the edge tensor
    points from the limb's first joint cell to the cell of the second one; `distractors` spurious edges/boxes above threshold."""
    rng = np.random.default_rng(seed)
    if isinstance(n_persons, tuple):
        n_persons = int(rng.integers(n_persons[0], n_persons[1] + 1))
    K, E = N_PARTS, len(PPN_PAIRS)
    conf = rng.uniform(0.0, 0.08, (K, gh, gw))
    xs = rng.uniform(0, net_w, (K, gh, gw)); ys = rng.uniform(0, net_h, (K, gh, gw))
    ws = rng.uniform(10, 60, (K, gh, gw)); hs = rng.uniform(10, 60, (K, gh, gw))
    edge = rng.uniform(0.0, 0.04, (E, nh, nw, gh, gw))
    ch, cw = net_h / gh, net_w / gw
    skel = random_skeletons(rng, n_persons, net_h, net_w)
    for person in skel:
        cells = {}
        bw = rng.uniform(24, 56)
        for k, (px, py) in enumerate(person):
            gx, gy = int(px // cw), int(py // ch)
            if not (0 <= gx < gw and 0 <= gy < gh):
                continue
            cells[k] = (gy, gx)
            conf[k, gy, gx] = rng.uniform(0.7, 0.95)
            xs[k, gy, gx], ys[k, gy, gx] = px, py
            ws[k, gy, gx], hs[k, gy, gx] = bw + rng.normal(0, 1), bw + rng.normal(0, 1)
            for dy, dx in ((0, 1), (1, 0), (0, -1), (-1, 0)):
                y2, x2 = gy + dy, gx + dx
                if 0 <= y2 < gh and 0 <= x2 < gw and conf[k, y2, x2] < 0.1 and rng.random() < 0.7:
                    conf[k, y2, x2] = rng.uniform(0.15, 0.5)
                    xs[k, y2, x2], ys[k, y2, x2] = px + rng.normal(0, 3), py + rng.normal(0, 3)
                    ws[k, y2, x2], hs[k, y2, x2] = bw + rng.normal(0, 2), bw + rng.normal(0, 2)
        for i, (a, b) in enumerate(PPN_PAIRS):
            if a in cells and b in cells:
                dy, dx = cells[b][0] - cells[a][0] + nh // 2, cells[b][1] - cells[a][1] + nw // 2
                if 0 <= dy < nh and 0 <= dx < nw:
                    edge[i, dy, dx, cells[a][0], cells[a][1]] = rng.uniform(0.5, 0.9)
    for _ in range(distractors):
        edge[rng.integers(E), rng.integers(nh), rng.integers(nw), rng.integers(gh), rng.integers(gw)] = rng.uniform(0.06, 0.4)
        conf[rng.integers(K), rng.integers(gh), rng.integers(gw)] = rng.uniform(0.11, 0.3)
    f = lambda a: a.astype(np.float32)
    return f(conf), f(rng.uniform(0, 1, (K, gh, gw))), f(xs), f(ys), f(ws), f(hs), f(edge)
