"""OpenPose PAF parser at real frame sizes (90 x 160 maps for a 1280 x 720 input, 135 x 240 for 1920 x 1080).

Both kernels of csrc/paf_parser.cu choose code paths from the map geometry: the limb kernel stages the up-sampling tables and
the two PAF planes of a limb in shared memory only up to a size, and the peak kernel has a direct up-sampling path and a
generic source-staging loop for tiles that read many source rows or columns.  Every case of PAF_LARGE_CASES states which
paths it takes (PafParser.debug_plan), so that a later change of a threshold cannot make a case quietly stop testing what it
was written for, and the cases together reach all of them.  Then, stage by stage against the oracle (oracle/paf_oracle.c):
peaks, connections and humans bit for bit; the connection scores also against a NumPy line integral in float64 that does not
go through the oracle; the humans against the reference's own src/paf.cpp (tests/golden/ref_humans_large.npz)."""
import os

import numpy as np
import pytest

import oracle
from hyperpose_b200 import capi, models, synthetic as syn
from tests.golden.make_golden import PAF_HANDLE_SEQUENCES, PAF_LARGE_CASES, PAF_LARGE_PINS, paf_handle_tensors, paf_large_tensors, sha

CASES = {c[0]: c for c in PAF_LARGE_CASES}
IDS = [c[0] for c in PAF_LARGE_CASES]
HANDLE_IDS = ["grow_then_shrink", "large_then_small"]

# paf_parser.cu: the peak kernel's tile (TH x TW interior, HALO each side) and the limits of its fast paths; the limb kernel's
# up-sampling table entries in shared memory and the bytes it keeps behind the staged PAF planes
TH, TW, HALO = 30, 62, 9
HL_ROWS, SRC_COLS, SM_TAB = 16, 64, 1024
LIMB_PHASE_B_EXTRA = SM_TAB * 8 + 2 * 512 * 4
H100_LIMB_DYN_BYTES = 200 * 1024
# channel pairs of the 19 limbs in the network's PAF tensor (src/coco.hpp COCOPAIRS_NET)
PAIRS_NET = [(12, 13), (20, 21), (14, 15), (16, 17), (22, 23), (24, 25), (0, 1), (2, 3), (4, 5), (6, 7), (8, 9), (10, 11), (28, 29),
             (30, 31), (34, 35), (32, 33), (36, 37), (18, 19), (26, 27)]
PAIRS = [(1, 2), (1, 5), (2, 3), (3, 4), (5, 6), (6, 7), (1, 8), (8, 9), (9, 10), (1, 11), (11, 12), (12, 13), (1, 0), (0, 14),
         (14, 16), (0, 15), (15, 17), (2, 16), (5, 17)]


def _geometry(case):
    """(H, W, UW, UH) of a case: the default resolution is (4 H, 4 W) transposed, as in the reference"""
    H, W, rw, rh = case[3], case[4], case[5], case[6]
    return H, W, rw if rw > 0 else 4 * H, rh if rh > 0 else 4 * W


def _area_up_table(src, dst):
    """cv::resize(INTER_AREA) up-scaling table (source index, fraction), restated in NumPy"""
    inv = dst / src
    d = np.arange(dst)
    s = np.floor(d * (1.0 / inv)).astype(np.int64)
    f = ((d + 1) - (s + 1) * inv).astype(np.float32)
    f = np.where(f <= 0, np.float32(0), f - np.floor(f)).astype(np.float32)
    last = s >= src - 1
    return np.where(last, src - 1, s), np.where(last, np.float32(0), f)


def _reflect101(p, n):
    p = np.abs(p)
    return np.where(p >= n, 2 * n - 2 - p, p) if n > 1 else np.zeros_like(p)


def _tile_source_extents(src, up, tile, window):
    """source rows (columns) each tile row (column) of the peak kernel reads, its halo window included"""
    idx, _ = _area_up_table(src, up)
    out = []
    for t in range((up + tile - 1) // tile):
        s = idx[_reflect101(np.arange(t * tile - HALO, t * tile - HALO + window), up)]
        out.append(int(np.minimum(s + 1, src - 1).max() - s.min() + 1))
    return np.array(out)


def expected_plan(case, limb_dyn_bytes, seq_assembly=False):
    """the debug_plan() a case must report (default: an up-scaling resolution, so nothing is materialised)"""
    H, W, UW, UH = _geometry(case)
    assert UW >= W and UH >= H
    want = 8 * H * W
    return {"generic": 0, "rz_mode": -1, "tab_staged": int(UW + UH <= SM_TAB),
            "stage_bytes": want if want + LIMB_PHASE_B_EXTRA <= limb_dyn_bytes else 0, "limb_dyn_bytes": limb_dyn_bytes,
            "fast_asm": 0 if seq_assembly else 1,
            "wide_tile_rows": int((_tile_source_extents(H, UH, TH, TH + 2 * HALO) > HL_ROWS).sum()),
            "wide_tile_cols": int((_tile_source_extents(W, UW, TW, TW + 2 * HALO) > SRC_COLS).sum())}


def _paths(plan, case):
    """the rows of the path table a plan reaches"""
    H, W, UW, UH = _geometry(case)
    out = set()
    out.add("tables staged" if plan["tab_staged"] else "tables from global memory")
    if plan["stage_bytes"]:
        out.add("PAF planes by TMA" if (H * W) % 4 == 0 else "PAF planes by scalar copy")
    else:
        out.add("PAF planes from global memory")
    if not plan["tab_staged"]:
        out.add("tables from global memory, PAF " + ("staged" if plan["stage_bytes"] else "from global memory"))
    if plan["wide_tile_rows"]:
        out.add("K1 direct up-sampling, PAF " + ("staged" if plan["stage_bytes"] else "from global memory"))
    if plan["wide_tile_rows"] < -(-UH // TH):
        out.add("K1 cached horizontal lerp")
    if plan["wide_tile_cols"]:
        out.add("K1 generic source loop, PAF " + ("staged" if plan["stage_bytes"] else "from global memory"))
    if plan["wide_tile_cols"] < -(-UW // TW):
        out.add("K1 source staging by (row mod 3, column)")
    return out


ALL_PATHS = {"tables staged", "tables from global memory", "PAF planes by TMA", "PAF planes by scalar copy", "PAF planes from global memory",
             "tables from global memory, PAF staged", "tables from global memory, PAF from global memory",
             "K1 direct up-sampling, PAF staged", "K1 direct up-sampling, PAF from global memory", "K1 cached horizontal lerp",
             "K1 generic source loop, PAF staged", "K1 generic source loop, PAF from global memory", "K1 source staging by (row mod 3, column)"}


def _line_integrals(paf, H, W, UW, UH, ax, ay, bx, by, ch1, ch2, swap_fractions=False, penalty_from_h=False):
    """scores (float64) of peak pairs (a -> b) on up-map coordinates, and their 10 sample products: the sample
    positions in float32 exactly as paf.cpp:74-78 computes them, the up-sampled PAF values and the sums in float64 (the
    resize's 2-tap area-mode interpolation, tables restated above).  swap_fractions / penalty_from_h: deliberately wrong
    restatements (the horizontal and vertical fractions exchanged; the length penalty from H instead of W) that the check
    must reject."""
    xi, xf = _area_up_table(W, UW)
    yi, yf = _area_up_table(H, UH)
    ax, ay, bx, by = (np.asarray(v, np.int64) for v in (ax, ay, bx, by))
    dx, dy = bx - ax, by - ay
    norm = np.sqrt((dx * dx + dy * dy).astype(np.float64))
    i = np.arange(10, dtype=np.float32)[None, :]
    stepx = dx.astype(np.float32)[:, None] / np.float32(10)
    stepy = dy.astype(np.float32)[:, None] / np.float32(10)
    fx = ax.astype(np.float32)[:, None] + i * stepx
    fy = ay.astype(np.float32)[:, None] + i * stepy
    assert fx.dtype == np.float32 and fy.dtype == np.float32
    lx = (fx.astype(np.float64) + 0.5).astype(np.int64)
    ly = (fy.astype(np.float64) + 0.5).astype(np.int64)
    a1 = (yf[ly] if swap_fractions else xf[lx]).astype(np.float64)
    b1 = (xf[lx] if swap_fractions else yf[ly]).astype(np.float64)
    sx0, sy0 = xi[lx], yi[ly]
    sx1, sy1 = np.minimum(sx0 + 1, W - 1), np.minimum(sy0 + 1, H - 1)

    def up(P):
        P = P.astype(np.float64)
        h0 = P[sy0, sx0] * (1 - a1) + P[sy0, sx1] * a1
        h1 = P[sy1, sx0] * (1 - a1) + P[sy1, sx1] * a1
        return h0 * (1 - b1) + h1 * b1

    s = (dx / norm)[:, None] * up(paf[ch1]) + (dy / norm)[:, None] * up(paf[ch2])
    feat_height = H if penalty_from_h else W
    score = s.sum(axis=1) / 10 + np.minimum(0.0, 0.5 * feat_height / norm - 1.0)
    return score, s


def _connection_scores(paf, case, peaks, pair, conns, **kw):
    H, W, UW, UH = _geometry(case)
    a, b = peaks[conns["cid1"]], peaks[conns["cid2"]]
    return _line_integrals(paf, H, W, UW, UH, a["x"], a["y"], b["x"], b["y"], *PAIRS_NET[pair], **kw)[0]


# ---------------------------------------------------------------------------------------------
# CPU: inputs, goldens, pins and the path inventory
# ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, "ref_humans_large.npz"))


@pytest.fixture(scope="module")
def oracle_runs():
    """oracle_process of every case, computed once per module"""
    out = {}
    for case in PAF_LARGE_CASES:
        conf, paf = paf_large_tensors(case)
        out[case[0]] = oracle.oracle_process(conf, paf, case[7], case[8], case[5], case[6], human_cap=4096, peak_cap=1 << 18,
                                             conn_cap=1 << 14)
    return out


def test_person_height_default_keeps_the_generator_byte_identical():
    for seed, P, hf, wf in ((0, 1, 46, 54), (3, (10, 20), 46, 54), (7, 3, 30, 40)):
        a = syn.make_frame_tensors(seed, P, hf, wf)
        b = syn.make_frame_tensors(seed, P, hf, wf, person_height=(0.55, 0.9))
        assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))
    small = syn.random_skeletons(np.random.default_rng(1), 50, 1080, 1920, person_height=(0.1, 0.2))
    tall = small[:, :, 1].max(axis=1) - small[:, :, 1].min(axis=1)
    assert tall.max() < 0.2 * 1080 and tall.min() > 0.08 * 1080


@pytest.mark.parametrize("name", IDS)
def test_generator_reproduces_golden_inputs(name, gold):
    conf, paf = paf_large_tensors(CASES[name])
    assert str(gold[name + "_in_sha"]) == sha(conf) + sha(paf)


@pytest.mark.parametrize("name", IDS)
def test_oracle_equals_reference_golden(name, gold, oracle_runs):
    assert oracle_runs[name]["humans"].tobytes() == gold[name + "_humans"].tobytes()


def test_oracle_resize_and_blur_equal_cv2_at_large_geometries(golden_dir):
    pin = np.load(os.path.join(golden_dir, "cv_pin_large.npz"))
    for i, (h, w, uh, uw) in enumerate(PAF_LARGE_PINS):
        assert pin[f"pin{i}_dims"].tolist() == [h, w, uh, uw]
        img = np.random.default_rng(400 + i).random((h, w), dtype=np.float32)
        up = oracle.resize_area_up(img, uh, uw) if (uh >= h and uw >= w) else oracle.resize_area(img, uh, uw)
        assert sha(up) == str(pin[f"pin{i}_up_sha"]), (h, w, uh, uw)
        assert sha(oracle.gaussian17(up)) == str(pin[f"pin{i}_blur_sha"]), (h, w, uh, uw)


def test_handle_sequences_oracle_equals_reference_golden(gold):
    """the handle sequences: inputs reproduce the golden's, and the oracle at the first call's resolution and feature height
    equals the reference handle's humans on every call; the fresh-handle answer (this frame's feature height) differs on some
    later call, so the sequences do test that the feature height is kept"""
    kept_matters = 0
    for s, seq in enumerate(PAF_HANDLE_SEQUENCES):
        res_w, res_h = 4 * seq[0][0], 4 * seq[0][1]
        for k, (h, w) in enumerate(seq):
            conf, paf = paf_handle_tensors(k, h, w)
            assert str(gold[f"handle{s}_{k}_in_sha"]) == sha(conf) + sha(paf)
            want = gold[f"handle{s}_{k}_humans"]
            assert len(want) > 0
            kept = oracle.oracle_process(conf, paf, 0.05, 0.05, res_w, res_h, feat_height=seq[0][1])["humans"]
            assert kept.tobytes() == want.tobytes(), (s, k)
            fresh = oracle.oracle_process(conf, paf, 0.05, 0.05, res_w, res_h)["humans"]
            kept_matters += fresh.tobytes() != want.tobytes()
    assert kept_matters > 0


@pytest.mark.skipif(not oracle.ref_available(), reason="oracle/_ref (the reference's own paf.cpp) is not built here")
@pytest.mark.parametrize("s", range(len(PAF_HANDLE_SEQUENCES)), ids=HANDLE_IDS)
def test_live_reference_handle_sequence_agrees(s, gold):
    rp = oracle.RefParser()
    for k, (h, w) in enumerate(PAF_HANDLE_SEQUENCES[s]):
        assert rp.process(*paf_handle_tensors(k, h, w), cap=4096).tobytes() == gold[f"handle{s}_{k}_humans"].tobytes(), k
    rp.close()


@pytest.mark.skipif(not oracle.ref_available(), reason="oracle/_ref (the reference's own paf.cpp) is not built here")
@pytest.mark.parametrize("name", IDS)
def test_live_reference_agrees(name, gold):
    case = CASES[name]
    conf, paf = paf_large_tensors(case)
    rp = oracle.RefParser(case[7], case[8], case[5], case[6])
    assert rp.process(conf, paf, cap=4096).tobytes() == gold[name + "_humans"].tobytes()
    rp.close()


def test_cases_reach_every_path_with_the_h100_limits():
    """with the H100's 200 KiB for the limb kernel, the cases reach every size-dependent path, and the boundary pairs
    straddle their limits (the GPU tests check that the device reports exactly this plan)"""
    plans = {c[0]: expected_plan(c, H100_LIMB_DYN_BYTES) for c in PAF_LARGE_CASES}
    reached = set().union(*(_paths(plans[c[0]], c) for c in PAF_LARGE_CASES))
    assert reached == ALL_PATHS, ALL_PATHS - reached
    assert plans["l_92x164"]["tab_staged"] == 1 and plans["l_92x165"]["tab_staged"] == plans["l_93x164"]["tab_staged"] == 0
    assert plans["l_92x165"]["stage_bytes"] > 0 and plans["l_93x164"]["stage_bytes"] > 0
    assert plans["l_128x188"]["stage_bytes"] > 0 and plans["l_128x189"]["stage_bytes"] == 0
    assert plans["l_135x240"]["tab_staged"] == 0 and plans["l_135x240"]["stage_bytes"] == 0
    assert _geometry(CASES["l_91x161"])[2] % 8 == 4 and _geometry(CASES["l_135x240"])[2] % 8 == 4
    assert _geometry(CASES["l_120x300_res"])[2] % 8 == 2


def test_noise_case_overflows_every_staging_limit(oracle_runs):
    """l_noise: > 2048 peaks and > 1024 connections in the frame, > 512 peaks of one part and > 512 candidates of one limb,
    more humans than the parser's initial capacity (64), every part <= 4096 peaks (the greedy pass' limit); the crowd stays
    within all of them"""
    case = CASES["l_noise"]
    o = oracle_runs["l_noise"]
    per_part = np.bincount(o["peaks"]["part_id"], minlength=18)
    n_conn = sum(len(c) for c in o["conns"])
    assert len(o["peaks"]) > 2048 and n_conn > 1024 and per_part.max() > 512 and per_part.max() <= 4096, (per_part, n_conn)
    assert len(o["humans"]) > 64
    # candidates of limb 0: every pair of its two parts through the float64 line integral (criterion 1: > 8 of the 10 samples
    # above the PAF threshold; criterion 2: score > 0), with a margin on both so that rounding cannot decide the count
    conf, paf = paf_large_tensors(case)
    H, W, UW, UH = _geometry(case)
    pk = o["peaks"]
    A, B = pk[pk["part_id"] == PAIRS[0][0]], pk[pk["part_id"] == PAIRS[0][1]]
    ia, ib = np.meshgrid(np.arange(len(A)), np.arange(len(B)), indexing="ij")
    a, b = A[ia.ravel()], B[ib.ravel()]
    keep = (a["x"] != b["x"]) | (a["y"] != b["y"])
    score, s = _line_integrals(paf, H, W, UW, UH, a["x"][keep], a["y"][keep], b["x"][keep], b["y"][keep], *PAIRS_NET[0])
    n_cand = int((((s > case[8] + 1e-4).sum(axis=1) > 8) & (score > 1e-4)).sum())
    assert n_cand > 512, n_cand
    c = oracle_runs["l_crowd"]
    assert 30 <= len(c["humans"]) and len(c["peaks"]) <= 2048 and sum(len(x) for x in c["conns"]) <= 1024


# ---------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------
def _cmp_humans(got, want, label):
    assert len(got) == len(want), f"{label}: {len(got)} humans vs {len(want)}"
    for i, (a, b) in enumerate(zip(got, want)):
        assert a.tobytes() == b.tobytes(), f"{label}: human {i} differs\n gpu={a}\n want={b}"


def _assembly_path(parser):
    """2: component-parallel get_humans, 1: sequential (needs HPB_PAF_TIMING=1)"""
    _, asm = parser.debug_timing(1)
    return int(asm[0, 1]) & 3


@pytest.mark.gpu
def test_plan_inventory():
    """every case reports the plan derived from the device's shared-memory limit; printed as the path inventory, which must
    reach every path"""
    reached = set()
    for case in PAF_LARGE_CASES:
        conf, paf = paf_large_tensors(case)
        parser = capi.PafParser(case[7], case[8], (case[5], case[6]))
        parser.process(conf, paf, cap=4096)
        plan = parser.debug_plan()
        parser.close()
        assert plan == expected_plan(case, plan["limb_dyn_bytes"]), case[0]
        paths = _paths(plan, case)
        reached |= paths
        print(f"{case[0]:>14}  {plan}  {sorted(paths)}")
    assert reached == ALL_PATHS, ALL_PATHS - reached


@pytest.mark.gpu
@pytest.mark.parametrize("name", IDS)
def test_stages_vs_oracle_and_reference(name, gold, oracle_runs, monkeypatch):
    """plan; peaks (part, x, y, id, score bits) and every limb's connections (ids, score bits) equal the oracle; the connection
    scores equal a float64 line integral within 1e-4 (the documented contract), which two wrong restatements break; humans equal
    the oracle and the reference's golden, on the component-parallel and on the sequential assembly"""
    monkeypatch.setenv("HPB_PAF_TIMING", "1")
    case = CASES[name]
    conf, paf = paf_large_tensors(case)
    orc = oracle_runs[name]
    parser = capi.PafParser(case[7], case[8], (case[5], case[6]))
    got = parser.process(conf, paf, cap=4096)
    plan = parser.debug_plan()
    assert plan == expected_plan(case, plan["limb_dyn_bytes"])

    pk = parser.debug_peaks(0, cap=1 << 18)
    op = orc["peaks"]
    assert len(pk) == len(op), f"{len(pk)} peaks vs oracle {len(op)}"
    for f in ("part_id", "x", "y", "id"):
        assert np.array_equal(pk[f], op[f]), f"peak field {f}"
    assert pk["score"].tobytes() == op["score"].tobytes(), "peak scores"

    n_conn = n_swap_bad = n_pen_changed = 0
    for pair in range(19):
        cn = parser.debug_connections(0, pair, cap=1 << 14)
        oc = orc["conns"][pair]
        assert len(cn) == len(oc), f"limb {pair}: {len(cn)} connections vs {len(oc)}"
        assert np.array_equal(cn["cid1"], oc["cid1"]) and np.array_equal(cn["cid2"], oc["cid2"]), f"limb {pair} ids"
        assert cn["score"].tobytes() == oc["score"].tobytes(), f"limb {pair} scores"
        if not len(cn):
            continue
        ref = _connection_scores(paf, case, pk, pair, cn)
        err = np.abs(ref - cn["score"].astype(np.float64))
        assert err.max() <= 1e-4, f"limb {pair}: line integral off by {err.max():.3g}"
        swapped = _connection_scores(paf, case, pk, pair, cn, swap_fractions=True)
        n_swap_bad += int((np.abs(swapped - cn["score"]) > 1e-4).sum())
        from_h = _connection_scores(paf, case, pk, pair, cn, penalty_from_h=True)
        changed = np.abs(from_h - ref) > 2e-4
        assert (np.abs(from_h - cn["score"])[changed] > 1e-4).all()
        n_pen_changed += int(changed.sum())
        n_conn += len(cn)
    H, W, UW, UH = _geometry(case)
    if n_conn and (_area_up_table(W, UW)[1].any() or _area_up_table(H, UH)[1].any()):   # integer factors: every fraction is 0
        assert n_swap_bad > n_conn // 2, f"exchanged fractions pass the check on {n_conn - n_swap_bad} of {n_conn} connections"
    if case[3] != case[4] and n_conn >= 20:
        assert n_pen_changed > 0, "no connection long enough for the H / W penalty to differ"

    _cmp_humans(got, orc["humans"], f"{name} vs oracle")
    _cmp_humans(got, gold[name + "_humans"], f"{name} vs reference golden")
    # the component-parallel assembly needs the frame's connections (<= 1024) and peak scores (<= 2048) in shared memory, so
    # the noise field's unstaged assembly always runs on the sequential path
    fast = _assembly_path(parser)
    assert fast == (1 if name == "l_noise" else 2)
    monkeypatch.setenv("HPB_PAF_SEQ_ASSEMBLY", "1")
    seq = parser.process(conf, paf, cap=4096)
    assert parser.debug_plan() == expected_plan(case, plan["limb_dyn_bytes"], seq_assembly=True)
    assert _assembly_path(parser) == 1
    _cmp_humans(seq, got, f"{name}: sequential assembly")
    parser.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", IDS)
def test_batched_equals_single_frames(name):
    """process_batch of [case, another frame of the same geometry, case]: every frame equals its single-frame result"""
    case = CASES[name]
    conf, paf = paf_large_tensors(case)
    other = paf_large_tensors((case[0], case[1] + 1000) + tuple(case[2:]))
    parser = capi.PafParser(case[7], case[8], (case[5], case[6]))
    want = [parser.process(conf, paf, cap=4096), parser.process(*other, cap=4096)]
    got = parser.process_batch(np.stack([conf, other[0], conf]), np.stack([paf, other[1], paf]), cap=4096)
    for i, w in enumerate((0, 1, 0)):
        _cmp_humans(got[i], want[w], f"{name} batch frame {i}")
    parser.close()


@pytest.mark.gpu
@pytest.mark.parametrize("s", range(len(PAF_HANDLE_SEQUENCES)), ids=HANDLE_IDS)
def test_one_handle_over_map_sizes(s, gold):
    """one handle fed maps of several sizes: the resolution and the length penalty's feature height stay those of its first call
    (paf.cpp:314-315, 321-332), later maps go through whichever path that resolution makes them take (135 x 240 at 184 x 328
    shrinks the width), and the buffers are reallocated as the size goes up and down.  Each call equals the reference's own
    handle fed the same sequence (golden) and the oracle at the first call's resolution and feature height."""
    seq = PAF_HANDLE_SEQUENCES[s]
    res_w, res_h = 4 * seq[0][0], 4 * seq[0][1]
    parser = capi.PafParser()
    plans = []
    for k, (h, w) in enumerate(seq):
        conf, paf = paf_handle_tensors(k, h, w)
        got = parser.process(conf, paf, cap=1024)
        plans.append(parser.debug_plan())
        label = f"call {k}: {h} x {w} at resolution {res_w} x {res_h}"
        _cmp_humans(got, gold[f"handle{s}_{k}_humans"], label + " vs reference golden")
        _cmp_humans(got, oracle.oracle_process(conf, paf, 0.05, 0.05, res_w, res_h, feat_height=seq[0][1])["humans"], label + " vs oracle")
    if seq[0] == (46, 82):
        assert [p["generic"] for p in plans] == [0, 1, 0, 1]
    parser.close()


@pytest.mark.gpu
def test_engine_pose_calls_with_1080p_maps():
    """the engine's pose calls on the 135 x 240 maps of a 1920 x 1080 frame: tiny_test_net (stride 2) at a 480 x 270 input, with
    crowd tensors copied over its outputs (hp_engine_set_output_override).  run_pose, submit_pose / collect_pose and
    submit_pose_device (CUDA graph, replayed twice) equal the oracle; a parser with tiny capacities makes hp_pose_collect grow
    them and rerun the batch"""
    import torch
    N, H, W = 2, 270, 480
    eng = capi.Engine(models.tiny_test_net(4).to_pack(), (W, H), max_batch_size=N)
    assert (eng.out_h, eng.out_w) == (135, 240)
    conf, paf = syn.make_batch_tensors(80, N, (30, 40), 135, 240, person_height=(0.1, 0.3))
    want = [oracle.oracle_process(conf[i], paf[i])["humans"] for i in range(N)]
    assert min(len(w) for w in want) >= 25
    dc, dp = torch.from_numpy(conf).cuda(), torch.from_numpy(paf).cuda()
    torch.cuda.synchronize()
    eng.set_output_override(dc.data_ptr(), dp.data_ptr())
    frames = syn.make_frames_u8(45, N, H, W)
    d_frames = torch.from_numpy(frames).cuda()
    parser = capi.PafParser()
    results = {"run_pose": eng.run_pose(parser, frames), "submit_pose": eng.collect_pose(eng.submit_pose(parser, frames))}
    launches0 = eng.pose_stats()["graph_launches"]
    for k in range(2):
        results[f"submit_pose_device #{k}"] = eng.collect_pose(eng.submit_pose_device(parser, d_frames.data_ptr(), N))
    assert eng.pose_stats()["graph_launches"] >= launches0 + 2
    small = capi.PafParser()
    small.set_capacity(peaks_per_part=8, candidates_per_limb=16, humans=4)
    results["collect with capacity growth"] = eng.collect_pose(eng.submit_pose_device(small, d_frames.data_ptr(), N))
    # the growth happened: more peaks per part and more humans than the initial capacities, and the peaks equal the oracle's
    orc0 = oracle.oracle_process(conf[0], paf[0])
    pk = small.debug_peaks(0)
    assert np.bincount(pk["part_id"], minlength=18).max() > 8 and len(want[0]) > 4
    assert pk.tobytes() == orc0["peaks"].tobytes()
    for what, got in results.items():
        for i in range(N):
            _cmp_humans(got[i], want[i], f"{what}, frame {i}")
    eng.close(); parser.close(); small.close()
