"""OpenPifPaf path (BASELINE config 5) stage by stage, at real frame sizes.

  a. pifpaf_head_kernel alone (pixel shuffle, crop to 2*hc-1, sigmoid, softplus, index grid) against a float64 evaluation,
     f16 and TF32 engines: every element within 2^-20 |ref| + 2^-40;
  b. the decoder's high-resolution core map (targetIntensities, openpifpaf_postprocessor.cpp:284-380) bit for bit against a
     NumPy float32 restatement, and the seed count (:679-706) against a NumPy restatement of the seed test;
  c. the whole decoder against the reference decoder at field sizes of real frames (tests/golden/ref_pifpaf_large.npz, and
     the live reference where oracle/_ref is built), including fields with more than 8192 seeds and one parser fed a
     sequence of batches of different sizes;
  d. the engine's pipelined pose calls at 721 x 1281 against process_batch on the engine's read-back fields."""
import os

import numpy as np
import pytest

import oracle
from hyperpose_b200 import capi, models, synthetic as syn
from tests.golden.make_golden import PIFPAF_LARGE_CASES, sha

F32, F64 = np.float32, np.float64
NKP = 17
LARGE = {c[0]: c for c in PIFPAF_LARGE_CASES}


def _large_fields(name):
    _, seed, P, h, w, scale = LARGE[name]
    return syn.make_pifpaf_fields(seed, P, h, w, scale=scale)


def _diff(a, b):
    if len(a) != len(b):
        return f"{len(a)} humans vs {len(b)}"
    for i, (x, y) in enumerate(zip(a, b)):
        if x.tobytes() != y.tobytes():
            return f"human {i}:\n gpu={x}\n ref={y}"
    return None


@pytest.fixture(scope="module")
def gold_large(golden_dir):
    return np.load(os.path.join(golden_dir, "ref_pifpaf_large.npz"))


# ---------------------------------------------------------------------------------------------
# a. head kernel alone
# ---------------------------------------------------------------------------------------------
PIF_COMPS, PAF_COMPS = 5, 9
SENTINEL = 30000.0        # written to the pad channels past 340 / 684; must never reach an output
# both sigmoid tails (expf(-v) overflows for v < -88), and both sides of softplus' v > 20 branch
SPECIAL = [-100.0, -90.5, -88.5, -87.5, -20.0, 19.90625, 20.0, 20.125, 21.0, 24.5, 60.0, 88.5, 95.0]


def _head_raw(N, hc, wc, C, used, f16):
    """raw head input [N,hc,wc,C]: a value that differs along every axis, with every SPECIAL value on every channel, and
    SENTINEL in the pad channels"""
    n, y, x, c = np.meshgrid(np.arange(N), np.arange(hc), np.arange(wc), np.arange(C), indexing="ij")
    v = np.sin(0.37 * c + 1.3 * x + 2.1 * y + 0.9 * n + 0.05 * c * (x + 1)) * 14.0 + 0.01 * (c % 7)
    k = (7 * n + 3 * y + x + c) % (2 * len(SPECIAL))
    sel = k < len(SPECIAL)
    v[sel] = np.asarray(SPECIAL)[k[sel]]
    v[..., used:] = SENTINEL
    return v.astype(np.float16 if f16 else np.float32)


def _head_ref(raw, fields, comps, is_paf, swap_shuffle=False, no_grid_comp=None):
    """float64 head: raw [N,hc,wc,C] -> [N,fields,comps,2hc-1,2wc-1].  `swap_shuffle` / `no_grid_comp` are deliberate faults
    (dx and dy swapped in the pixel shuffle; no index grid on one component) that the bound must catch."""
    N, hc, wc, _ = raw.shape
    ho, wo = 2 * hc - 1, 2 * wc - 1
    r = raw.astype(F64)
    y, x = np.arange(ho), np.arange(wo)
    nc = np.arange(fields * comps)
    dy, dx = (y & 1)[:, None], (x & 1)[None, :]
    if swap_shuffle:
        dy, dx = dx, dy
    ch = (nc[:, None, None] * 2 + dy[None]) * 2 + dx[None]                          # [fields*comps, ho, wo]
    g = r[:, (y >> 1)[None, :, None], (x >> 1)[None, None, :], ch]                   # [N, fields*comps, ho, wo]
    g = g.reshape(N, fields, comps, ho, wo)
    out = g.copy()
    out[:, :, 0] = 1.0 / (1.0 + np.exp(-g[:, :, 0]))
    xs, ys, ss = ((1, 3), (2, 4), (7, 8)) if is_paf else ((1,), (2,), (4,))
    for c in ss:
        out[:, :, c] = np.logaddexp(0.0, g[:, :, c])
    for c in xs:
        if c != no_grid_comp:
            out[:, :, c] += x[None, None, None, :]
    for c in ys:
        out[:, :, c] += y[None, None, :, None]
    return out, g


def _out_of_bound(got, ref):
    return np.abs(got.astype(F64) - ref) > 2.0 ** -20 * np.abs(ref) + 2.0 ** -40


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["f16", "tf32"])
@pytest.mark.parametrize("hw", [(129, 129), (129, 193), (721, 1281), (100, 150)], ids=lambda t: f"{t[0]}x{t[1]}")
def test_head_kernel_alone_against_float64(dtype, hw):
    H, W = hw
    N = 3
    g = models.resnet50_pifpaf(0)
    hi = next(i for i, op in enumerate(g.ops) if op.type == models.OP_PIFPAF_HEAD)
    pif_buf, paf_buf = g.ops[hi].in_buf, g.ops[hi].res_buf
    eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=N, dtype=dtype)
    assert eng.head_type == 1
    shape_a, shape_b = eng.debug_read_buffer(pif_buf, N).shape, eng.debug_read_buffer(paf_buf, N).shape
    hc, wc = shape_a[1], shape_a[2]
    assert shape_b[1:3] == (hc, wc) and shape_a[3] > 340 and shape_b[3] > 684
    ho, wo = 2 * hc - 1, 2 * wc - 1
    assert (eng.out_h, eng.out_w) == (ho, wo)
    f16 = dtype == "f16"
    raw_a, raw_b = _head_raw(N, hc, wc, shape_a[3], 340, f16), _head_raw(N, hc, wc, shape_b[3], 684, f16)
    eng.debug_write_buffer(pif_buf, raw_a)
    eng.debug_write_buffer(paf_buf, raw_b)
    eng.debug_run_ops(hi, hi, N)
    pif, paf = eng.read_outputs(N)
    eng.close()
    pif, paf = pif.reshape(N, 17, PIF_COMPS, ho, wo), paf.reshape(N, 19, PAF_COMPS, ho, wo)
    assert np.isfinite(pif).all() and np.isfinite(paf).all()
    assert np.abs(pif).max() < 0.5 * SENTINEL and np.abs(paf).max() < 0.5 * SENTINEL, "a pad channel reached an output"
    for got, raw, fields, comps, is_paf, what in ((pif, raw_a, 17, PIF_COMPS, False, "pif"), (paf, raw_b, 19, PAF_COMPS, True, "paf")):
        ref, pre = _head_ref(raw, fields, comps, is_paf)
        bad = np.argwhere(_out_of_bound(got, ref))
        assert len(bad) == 0, f"{what}: {len(bad)} elements out of bound, first at {tuple(bad[0])}: {got[tuple(bad[0])]!r} vs {ref[tuple(bad[0])]!r}"
        # not vacuous: both sigmoid tails (v < -88 included), both softplus branches, the grid on the last row and column
        conf_in = pre[:, :, 0]
        assert (conf_in < -88).any() and (conf_in > 88).any()
        assert got[:, :, 0][conf_in < -88].max() < 1e-30 and got[:, :, 0][conf_in > 20].min() == 1.0
        scale_in = pre[:, :, (7, 8) if is_paf else (4,)]
        assert (scale_in > 20).any() and (scale_in <= 20).any() and (scale_in == 20).any() and (scale_in == 19.90625).any()
        for cx in ((1, 3) if is_paf else (1,)):
            assert np.allclose(got[:, :, cx, :, -1] - pre[:, :, cx, :, -1], wo - 1, rtol=0, atol=1e-4 * max(1.0, np.abs(pre).max()))
        for cy in ((2, 4) if is_paf else (2,)):
            assert np.allclose(got[:, :, cy, -1, :] - pre[:, :, cy, -1, :], ho - 1, rtol=0, atol=1e-4 * max(1.0, np.abs(pre).max()))
    # the bound is tight enough to catch a swapped shuffle and a missing grid offset on one PAF component
    for mut in (dict(swap_shuffle=True), dict(no_grid_comp=3)):
        ref_m, _ = _head_ref(raw_b, 19, PAF_COMPS, True, **mut)
        ref, _ = _head_ref(raw_b, 19, PAF_COMPS, True)
        changed = ref_m != ref
        assert changed.sum() > 1000, mut
        caught = _out_of_bound(paf, ref_m)[changed].mean()
        assert caught > 0.9, f"{mut}: only {caught:.1%} of the changed elements break the bound"


# ---------------------------------------------------------------------------------------------
# b. high-resolution core map and seeds, NumPy restatements
# ---------------------------------------------------------------------------------------------
def _approx_exp(x):
    """openpifpaf_postprocessor.cpp:224-232 on a float32 array"""
    out = np.zeros_like(x)
    m = (x <= 2) & (x >= -2)
    y = F32(1) + x[m] / F32(8)
    y = y * y
    y = y * y
    y = y * y
    out[m] = y
    return out


def hr_core_map(p, stats=None):
    """targetsCoreOnly of one field (targetIntensities, :284-380 with scalarSquareAddGaussWitMax :192-241): p = pif[field]
    f32[5,H,W].  Cells with conf > 0.1 are applied in ascending order, each footprint vectorised; float32 arithmetic except
    where the reference promotes to double (the scale, :329, and the approx_exp argument, :233)."""
    _, H, W = p.shape
    HR, WR = (H - 1) * 8 + 1, (W - 1) * 8 + 1
    m = np.zeros((HR, WR), F32)
    conf, px, py, ps = (p[i].ravel() for i in (0, 1, 2, 4))
    clip = lambda v, lo, hi: max(lo, min(hi, v))
    for j in np.flatnonzero(conf > F32(0.1)):
        cx, cy = px[j] * F32(8), py[j] * F32(8)
        cs = F32(max(1.0, 0.5 * float(ps[j]) * 8.0))
        cv = conf[j] * F32(1.0 / 16.0)
        tc = cs * F32(1)
        minx = int(clip(cx - tc, F32(0), F32(WR - 1)))
        maxx = int(clip(cx + tc + F32(1), F32(minx + 1), F32(WR)))
        miny = int(clip(cy - tc, F32(0), F32(HR - 1)))
        maxy = int(clip(cy + tc + F32(1), F32(miny + 1), F32(HR)))
        dx2 = np.square(np.arange(minx, maxx).astype(F32) - cx)
        dy2 = np.square(np.arange(miny, maxy).astype(F32) - cy)
        d2 = dx2[None, :] + dy2[:, None]
        inside = ~(d2 > tc * tc)
        core = (dx2[None, :] < 0.25) & (dy2[:, None] < 0.25)
        arg = (-0.5 * d2.astype(F64) / F64(cs * cs)).astype(F32)
        vv = np.where(core, cv, cv * _approx_exp(arg))
        sub = m[miny:maxy, minx:maxx]
        sub[inside] = np.minimum(F32(1), sub[inside] + vv[inside])
        if stats is not None:
            stats["cells"] += 1
            stats["floor"] += bool(0.5 * float(ps[j]) * 8.0 < 1.0)
            stats["big"] += bool(cs >= 16)
            stats["clip"] |= {("x0" if cx - tc < 0 else None), ("x1" if cx + tc + 1 > WR else None),
                              ("y0" if cy - tc < 0 else None), ("y1" if cy + tc + 1 > HR else None)}
    return m


def seed_count(pif, hr):
    """number of seeds (:679-706): conf > 0.3, coordinates in range, 0.9 * core map at (y*8+0.5, x*8+0.5) + 0.1 * conf > 0.3"""
    _, _, H, W = pif.shape
    HR, WR = (H - 1) * 8 + 1, (W - 1) * 8 + 1
    maxx, maxy = F32(WR - 0.51), F32(HR - 0.51)
    n = 0
    for f in range(NKP):
        c, x, y = (pif[f, i].ravel() for i in (0, 1, 2))
        q = (c > F32(0.3)) & ~((x.astype(F64) < -0.49) | (y.astype(F64) < -0.49) | (x > maxx) | (y > maxy))
        iy = ((y[q] * F32(8)).astype(F64) + 0.5).astype(np.int64)
        ix = ((x[q] * F32(8)).astype(F64) + 0.5).astype(np.int64)
        v = (0.9 * hr[f][iy, ix].astype(F64) + 0.1 * c[q].astype(F64)).astype(F32)
        n += int((v > F32(0.3)).sum())
    return n


def make_hr_fields(seed, H, W, dense_fields=4, dense=0.2, sparse=0.03):
    """pif f32[17,5,H,W] for the core-map test: cells at exactly the 0.1 threshold and just above it, scales of 4-8 cells
    (33-65 px footprints) mixed with scales under the max(1, .) floor, coordinates spread over the whole map so footprints are
    clipped at all four borders, and per field two 6 x 6 blocks of cells aimed at one point (a corner, and a random point)
    whose Gaussians overlap far past the 1.0 clamp.  The first `dense_fields` fields have more than 2048 qualifying cells."""
    rng = np.random.default_rng(seed)
    pif = np.zeros((NKP, 5, H, W), F32)
    yy, xx = np.mgrid[0:H, 0:W].astype(F64)
    at_thr, above_thr = F32(0.1), np.nextafter(F32(0.1), F32(1))
    for f in range(NKP):
        frac = dense if f < dense_fields else sparse
        u = rng.random((H, W))
        conf = rng.uniform(0.0, 0.09, (H, W))
        conf[u < frac] = rng.uniform(0.1, 1.0, int((u < frac).sum()))
        conf[(u >= frac) & (u < frac + 0.01)] = at_thr
        conf[(u >= frac + 0.01) & (u < frac + 0.015)] = above_thr
        pif[f, 0] = conf
        pif[f, 1] = np.clip(xx + rng.normal(0, 3, (H, W)), 0, W - 1)
        pif[f, 2] = np.clip(yy + rng.normal(0, 3, (H, W)), 0, H - 1)
        pif[f, 3] = rng.uniform(0.2, 0.4, (H, W))
        r = rng.random((H, W))
        pif[f, 4] = np.where(r < 0.6, rng.uniform(4.0, 8.0, (H, W)), np.where(r < 0.8, rng.uniform(0.0, 0.24, (H, W)), rng.uniform(1.0, 4.0, (H, W))))
        for (by, bx), (ty, tx) in (((0, 0), (0.0, 0.0)), ((int(rng.integers(0, H - 6)), int(rng.integers(0, W - 6))), (rng.uniform(0, H - 1), rng.uniform(0, W - 1)))):
            pif[f, 0, by:by + 6, bx:bx + 6] = rng.uniform(0.9, 1.0, (6, 6))
            pif[f, 1, by:by + 6, bx:bx + 6] = tx
            pif[f, 2, by:by + 6, bx:bx + 6] = ty
            pif[f, 4, by:by + 6, bx:bx + 6] = rng.uniform(4.0, 8.0, (6, 6))
    return pif


def test_hr_fields_are_not_vacuous():
    """the core-map test's inputs reach what they are meant to: several chunks of 2048 cells in one field, the strict
    threshold, the scale floor, large footprints, clipping at all four borders, the clamp, and seeds"""
    pif = make_hr_fields(50, 99, 125)
    assert ((pif[0, 0] > F32(0.1)).sum()) > 2048 and (pif[:, 0] == F32(0.1)).sum() > 100
    st = {"cells": 0, "floor": 0, "big": 0, "clip": set()}
    maps = [hr_core_map(pif[f], st) for f in range(2)]
    assert st["floor"] > 50 and st["big"] > 1000 and {"x0", "x1", "y0", "y1"} <= st["clip"], st
    assert all((m == 1.0).any() for m in maps) and all(((m > 0) & (m < 1)).any() for m in maps)
    pif_s = make_hr_fields(51, 25, 33, dense_fields=0)
    assert seed_count(pif_s, [hr_core_map(pif_s[f]) for f in range(NKP)]) > 50


@pytest.mark.gpu
@pytest.mark.parametrize("hw", [(49, 49), (99, 125), (91, 161)], ids=lambda t: f"{t[0]}x{t[1]}")
def test_hr_core_map_bit_exact(hw):
    """debug_hr of every field of a two-frame batch == the NumPy restatement, bit for bit; debug_counts' seed count == the
    restated seed test.  The decode is only launched (process_device): these fields are not meant to be decoded into people."""
    import torch
    H, W = hw
    frames = [make_hr_fields(60 + H, H, W), make_hr_fields(61 + H, H, W, dense_fields=0)]
    pif = np.stack(frames)
    paf = np.zeros((2, 19, 9, H, W), F32)
    d_pif, d_paf = torch.from_numpy(pif).cuda(), torch.from_numpy(paf).cuda()
    dec = capi.PifPafParser((H - 1) * 8 + 1, (W - 1) * 8 + 1, 0.1)
    dec.process_device(d_pif.data_ptr(), d_paf.data_ptr(), 2, H, W)
    for i in range(2):
        maps = []
        for f in range(NKP):
            got = dec.debug_hr(i, f, H, W)
            want = hr_core_map(pif[i, f])
            bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
            assert len(bad) == 0, f"frame {i} field {f}: {len(bad)} pixels differ, first {tuple(bad[0])}: {got[tuple(bad[0])]!r} vs {want[tuple(bad[0])]!r}"
            maps.append(want)
        counts = dec.debug_counts(i)
        assert counts["flags"] & 1 == 0 and counts["seeds"] == seed_count(pif[i], maps), (counts, i)
        assert counts["seeds"] > 0
    dec.close()


# ---------------------------------------------------------------------------------------------
# c. decoder vs the reference decoder at real field sizes
# ---------------------------------------------------------------------------------------------
def test_large_goldens_not_vacuous(gold_large):
    for name, *_ in PIFPAF_LARGE_CASES:
        assert len(gold_large[name + "_humans"]) >= 4, name
    h = gold_large["pl_dense_humans"]
    assert len(h) >= 30 and int(h["parts"]["has_value"].sum()) > 30 * 12


@pytest.mark.parametrize("name", list(LARGE))
def test_large_generator_matches_golden_inputs(gold_large, name):
    pif, paf = _large_fields(name)
    assert sha(pif) + sha(paf) == str(gold_large[name + "_in_sha"])


@pytest.mark.skipif(not oracle.pifpaf_ref_available(), reason="oracle/_ref/libref_pifpaf.so not built")
@pytest.mark.parametrize("name", list(LARGE))
def test_live_reference_matches_large_golden(gold_large, name):
    pif, paf = _large_fields(name)
    h, w = pif.shape[2:]
    got = oracle.ref_pifpaf_process(pif, paf, (h - 1) * 8 + 1, (w - 1) * 8 + 1, 0.1)
    assert got.tobytes() == gold_large[name + "_humans"].tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(LARGE))
def test_decoder_equals_reference_at_real_sizes(gold_large, name):
    pif, paf = _large_fields(name)
    h, w = pif.shape[2:]
    dec = capi.PifPafParser((h - 1) * 8 + 1, (w - 1) * 8 + 1, 0.1)
    got = dec.process(pif, paf)
    d = _diff(got, gold_large[name + "_humans"])
    assert d is None, f"{name}: {d}"
    if name == "pl_dense":      # more seeds than the initial capacity: the decoder grew it and decoded again
        assert dec.debug_counts(0)["seeds"] > 8192
    dec.close()


def _renormalised(humans, h, w, net_h, net_w):
    """records decoded from [h,w] fields by a parser created for (h-1)*8+1 x (w-1)*8+1, as a parser created for net_h x net_w
    returns them: the keypoint pixels are integers divided by the network size (src/pifpaf.cpp:52-92), the neck is the mean
    of the shoulders"""
    out = humans.copy()
    parts = out["parts"]
    for c, full, net in (("x", (w - 1) * 8 + 1, net_w), ("y", (h - 1) * 8 + 1, net_h)):
        has = parts["has_value"] == 1
        px = np.round(parts[c].astype(F64) * full)
        parts[c][has] = px[has].astype(F32) / F32(net)
        parts[c][:, 1] = 0
        neck = (parts["has_value"][:, 2] == 1) & (parts["has_value"][:, 5] == 1)
        parts[c][neck, 1] = (parts[c][neck, 2] + parts[c][neck, 5]) / F32(2)
    return out


@pytest.mark.gpu
def test_one_parser_over_batches_of_different_sizes(gold_large):
    """one parser (network size 721 x 1281), batches whose field size goes up, down and up again, so its buffers are
    reallocated between calls; against the goldens rescaled to that network size, and the live reference where it is built"""
    live = oracle.pifpaf_ref_available()
    dec = capi.PifPafParser(721, 1281, 0.1)
    for names in (["pl_99x124"], ["pl_161x161", "pl_dense"], ["pl_89x159"], ["pl_99x125", "pl_99x125"], ["pl_91x161"]):
        fields = [_large_fields(n) for n in names]
        got = dec.process_batch(np.stack([f[0] for f in fields]), np.stack([f[1] for f in fields]))
        for n, (pif, paf), g in zip(names, fields, got):
            h, w = pif.shape[2:]
            want = _renormalised(gold_large[n + "_humans"], h, w, 721, 1281)
            if live:
                assert oracle.ref_pifpaf_process(pif, paf, 721, 1281, 0.1).tobytes() == want.tobytes(), n
            d = _diff(g, want)
            assert d is None, f"{names} / {n}: {d}"
    dec.close()


# ---------------------------------------------------------------------------------------------
# d. engine -> decoder at 721 x 1281
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_engine_pose_calls_at_721x1281(gold_large):
    """ResNet-50 PifPaf at a 1281 x 721 input (91 x 161 fields): the pipelined host-frame call (submit_pose / collect_pose) and
    the device-frame call (submit_pose_device / collect_pose) == process_batch on the engine's read-back fields, byte for byte.
    Random weights give fields without people, so crowd fields are copied over the network's outputs after its last op
    (hp_engine_set_output_override); the conv stack still runs at full size."""
    import torch
    N, H, W = 2, 721, 1281
    eng = capi.Engine(models.resnet50_pifpaf(0).to_pack(), (W, H), max_batch_size=N)
    assert (eng.out_h, eng.out_w) == (91, 161)
    fields = [_large_fields("pl_91x161"), syn.make_pifpaf_fields(36, (10, 14), 91, 161, scale=(1.0, 8.0))]
    pif = np.stack([f[0] for f in fields]); paf = np.stack([f[1] for f in fields])
    d_pif, d_paf = torch.from_numpy(pif).cuda(), torch.from_numpy(paf).cuda()
    eng.set_output_override(d_pif.data_ptr(), d_paf.data_ptr())
    frames = syn.make_frames_u8(44, N, H, W)
    eng.infer_u8(frames)
    rpif, rpaf = eng.read_outputs(N)
    assert rpif.tobytes() == pif.tobytes() and rpaf.tobytes() == paf.tobytes()
    ref_dec = capi.PifPafParser(H, W, 0.1)
    want = ref_dec.process_batch(rpif.reshape(pif.shape), rpaf.reshape(paf.shape))
    ref_dec.close()
    assert _diff(want[0], _renormalised(gold_large["pl_91x161_humans"], 91, 161, H, W)) is None
    assert len(want[1]) >= 5
    dec = capi.PifPafParser(H, W, 0.1)
    got_host = eng.collect_pose(eng.submit_pose(dec, frames), cap=128)
    d_frames = torch.from_numpy(frames).cuda()
    got_dev = eng.collect_pose(eng.submit_pose_device(dec, d_frames.data_ptr(), N), cap=128)
    for i in range(N):
        for what, g in (("host frames", got_host), ("device frames", got_dev)):
            d = _diff(g[i], want[i])
            assert d is None, f"{what}, frame {i}: {d}"
    eng.close(); dec.close()
