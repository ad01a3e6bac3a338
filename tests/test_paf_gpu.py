"""GPU parity tests (the parity tests proper): CUDA PAF parser, through the C ABI, against the
oracle on identical seeded tensors.  Bar (BASELINE.json north_star): peak indices bit-exact;
PAF line-integral scores and keypoint coordinates within 1e-4 -- this implementation is held to
BIT-EXACT on all of them (humans compared byte-for-byte), with 1e-4 documented as the contract."""
import os

import numpy as np
import pytest

import oracle
from hyperpose_b200 import capi, synthetic as syn
from tests.golden.make_golden import AREA_FRAME_CASES, FRAME_CASES

pytestmark = pytest.mark.gpu


def _cmp_frame(parser_out, orc, label=""):
    h, o = parser_out, orc["humans"]
    assert len(h) == len(o), f"{label}: {len(h)} humans vs oracle {len(o)}"
    if h.tobytes() != o.tobytes():
        for i, (a, b) in enumerate(zip(h, o)):
            if a.tobytes() != b.tobytes():
                raise AssertionError(f"{label}: human {i} differs\n gpu={a}\n orc={b}")


def _check_debug(parser, frame, orc, label=""):
    pk = parser.debug_peaks(frame)
    op = orc["peaks"]
    assert len(pk) == len(op), f"{label}: {len(pk)} peaks vs oracle {len(op)}"
    for f in ("part_id", "x", "y", "id"):
        assert np.array_equal(pk[f], op[f]), f"{label}: peak field {f} differs"
    assert pk["score"].tobytes() == op["score"].tobytes(), f"{label}: peak scores differ"
    for pair in range(19):
        cn = parser.debug_connections(frame, pair)
        oc = orc["conns"][pair]
        assert len(cn) == len(oc), f"{label}: limb {pair}: {len(cn)} conns vs {len(oc)}"
        assert np.array_equal(cn["cid1"], oc["cid1"]) and np.array_equal(cn["cid2"], oc["cid2"]), f"{label}: limb {pair} ids"
        assert np.allclose(cn["score"], oc["score"], rtol=0, atol=1e-4), f"{label}: limb {pair} scores (1e-4 contract)"
        assert cn["score"].tobytes() == oc["score"].tobytes(), f"{label}: limb {pair} scores not bit-exact"


@pytest.mark.parametrize("case", FRAME_CASES, ids=[c[0] for c in FRAME_CASES])
def test_frame_cases_vs_oracle_and_reference_golden(case, golden_dir):
    name, seed, P, hf, wf, rw, rh, ct, pt = case
    conf, paf = syn.make_frame_tensors(seed, P, hf, wf)
    orc = oracle.oracle_process(conf, paf, ct, pt, rw, rh)
    parser = capi.PafParser(ct, pt, (rw, rh))
    got = parser.process(conf, paf)
    _check_debug(parser, 0, orc, name)
    _cmp_frame(got, orc, name)
    # and against what the reference's own src/paf.cpp produced (committed golden)
    want = np.load(os.path.join(golden_dir, "ref_humans.npz"))[name + "_humans"]
    assert got.tobytes() == want.tobytes()
    parser.close()


@pytest.mark.parametrize("hf,wf,P,N", [(46, 54, (1, 3), 8), (46, 82, (2, 8), 16), (46, 54, (10, 20), 32)])
def test_batched_vs_oracle(hf, wf, P, N):
    conf, paf = syn.make_batch_tensors(11, N, P, hf, wf)
    parser = capi.PafParser()
    got = parser.process_batch(conf, paf)
    for i in range(N):
        orc = oracle.oracle_process(conf[i], paf[i])
        if i < 3:
            _check_debug(parser, i, orc, f"frame{i}")
        _cmp_frame(got[i], orc, f"frame{i}")
    parser.close()


@pytest.mark.parametrize("seed", range(40, 52))
def test_random_shapes_vs_oracle(seed):
    """ragged / odd geometries: every column class of the separable filter, reflect borders on tiny maps"""
    rng = np.random.default_rng(seed)
    hf = int(rng.integers(5, 60))
    wf = int(rng.integers(max(5, (hf + 3) // 4), min(90, 4 * hf) + 1))   # default resolution must up-scale both axes
    P = int(rng.integers(0, 6))
    conf, paf = syn.make_frame_tensors(seed, P, hf, wf)
    orc = oracle.oracle_process(conf, paf)
    parser = capi.PafParser()
    got = parser.process(conf, paf)
    _check_debug(parser, 0, orc, f"{hf}x{wf}")
    _cmp_frame(got, orc, f"{hf}x{wf}")
    parser.close()


def test_noise_field_many_peaks_capacity_growth():
    """structureless input: hundreds of spurious peaks per part -> internal capacities must grow, result still exact"""
    rng = np.random.default_rng(99)
    conf = rng.random((19, 24, 30), dtype=np.float32) * 0.3
    paf = rng.random((38, 24, 30), dtype=np.float32) - 0.5
    orc = oracle.oracle_process(conf, paf)
    parser = capi.PafParser()
    parser.set_capacity(peaks_per_part=8, candidates_per_limb=16, humans=2)
    got = parser.process(conf, paf)
    _check_debug(parser, 0, orc, "noise")
    _cmp_frame(got, orc, "noise")
    parser.close()


def _assembly_paths(parser, N):
    """which get_humans path assembled each frame of the last batch (needs HPB_PAF_TIMING=1): 2 component-parallel, 1 sequential"""
    _, asm = parser.debug_timing(N)
    return [int(v) & 3 for v in asm[:, 1]]


def test_component_parallel_assembly_is_the_path_taken_and_the_sequential_paths_agree(monkeypatch):
    """crowd frames: the component-parallel get_humans (one lane per connected component of the peak / connection graph) is what runs,
    and it equals the oracle; with HPB_PAF_SEQ_ASSEMBLY=1 the same frames go through the sequential path -- same bytes"""
    monkeypatch.setenv("HPB_PAF_TIMING", "1")
    N, hf, wf = 6, 46, 82
    conf, paf = syn.make_batch_tensors(1000, N, (10, 20), hf, wf)
    want = [oracle.oracle_process(conf[i], paf[i]) for i in range(N)]
    parser = capi.PafParser()
    parser.set_capacity(128, 2048, 64)
    got = parser.process_batch(conf, paf)
    assert _assembly_paths(parser, N) == [2] * N
    for i in range(N):
        _cmp_frame(got[i], want[i], f"fast frame{i}")
    monkeypatch.setenv("HPB_PAF_SEQ_ASSEMBLY", "1")
    got2 = parser.process_batch(conf, paf)
    assert _assembly_paths(parser, N) == [1] * N
    for i in range(N):
        assert got2[i].tobytes() == got[i].tobytes()
    parser.close()


def test_mixed_path_crowd_batch_vs_oracle(monkeypatch):
    """cfg4-sized crowd batch in which one frame (15) has a merge that invents a peak id: that frame alone is handed back to the
    sequential path, the other 31 stay on the component-parallel path, and every frame equals the oracle"""
    monkeypatch.setenv("HPB_PAF_TIMING", "1")
    N = 32
    conf, paf = syn.make_batch_tensors(1001, N, (10, 20), 46, 54)
    parser = capi.PafParser()
    got = parser.process_batch(conf, paf)
    assert _assembly_paths(parser, N) == [1 if i == 15 else 2 for i in range(N)]
    for i in range(N):
        _cmp_frame(got[i], oracle.oracle_process(conf[i], paf[i]), f"frame{i}")
    parser.close()


@pytest.mark.parametrize("seed", range(300, 312))
def test_noisy_crowds_vs_oracle(seed, monkeypatch):
    """skeletons + noise strong enough to add spurious peaks, connections, merges of partial humans and (some seeds) the
    reference's fabricated part ids: whichever assembly path a frame ends on, the humans equal the oracle's"""
    monkeypatch.setenv("HPB_PAF_TIMING", "1")
    rng = np.random.default_rng(seed)
    hf, wf = 30, 40
    conf, paf = syn.make_frame_tensors(seed, int(rng.integers(3, 9)), hf, wf)
    amp = float(rng.uniform(0.05, 0.25))
    conf = (conf + rng.random(conf.shape, dtype=np.float32) * amp).astype(np.float32)
    paf = (paf + (rng.random(paf.shape, dtype=np.float32) - 0.5) * 2 * amp).astype(np.float32)
    orc = oracle.oracle_process(conf, paf, peak_cap=1 << 18, conn_cap=1 << 14)
    parser = capi.PafParser()
    got = parser.process(conf, paf)
    _cmp_frame(got, orc, f"seed {seed} amp {amp:.2f} path {_assembly_paths(parser, 1)}")
    parser.close()


def test_thresholds_and_setters():
    conf, paf = syn.make_frame_tensors(3, (10, 20), 46, 54)
    parser = capi.PafParser(0.05, 0.05)
    for ct, pt in [(0.3, 0.05), (0.05, 0.3), (0.6, 0.6), (0.0, 0.0)]:
        parser.set_conf_thresh(ct)
        parser.set_paf_thresh(pt)
        orc = oracle.oracle_process(conf, paf, ct, pt)
        _cmp_frame(parser.process(conf, paf), orc, f"thr {ct},{pt}")
    parser.close()


def test_device_resident_hand_off():
    import torch
    conf, paf = syn.make_batch_tensors(5, 4, (2, 5), 46, 82)
    dc = torch.from_numpy(conf).cuda()
    dp = torch.from_numpy(paf).cuda()
    torch.cuda.synchronize()
    parser = capi.PafParser()
    parser.process_device(dc.data_ptr(), dp.data_ptr(), 4, 19, 38, 46, 82)
    got = parser.fetch(4)
    for i in range(4):
        _cmp_frame(got[i], oracle.oracle_process(conf[i], paf[i]), f"dev frame {i}")
    assert parser.launch_count >= 2
    parser.close()


def test_bad_rank_is_rejected():
    parser = capi.PafParser()
    with pytest.raises(capi.HyperposeError):
        parser.process(np.zeros((19, 46), np.float32), np.zeros((38, 46, 54), np.float32))
    with pytest.raises(capi.HyperposeError):
        parser.process(np.zeros((10, 46, 54), np.float32), np.zeros((38, 46, 54), np.float32))
    parser.close()


@pytest.mark.parametrize("case", AREA_FRAME_CASES, ids=[c[0] for c in AREA_FRAME_CASES])
def test_resolutions_that_shrink_an_axis(case, golden_dir):
    """A5 beyond pure up-scaling (src/post_process.hpp:27-52 works for ANY resolution): mixed regime (2-tap lerp), integer-factor and
    fractional area averaging -- peaks, connections and humans bit-exact against the oracle (pinned to cv2) and against what the
    reference's own src/paf.cpp produced (committed golden)"""
    name, seed, P, hf, wf, rw, rh, ct, pt = case
    conf, paf = syn.make_frame_tensors(seed, P, hf, wf)
    orc = oracle.oracle_process(conf, paf, ct, pt, rw, rh)
    parser = capi.PafParser(ct, pt, (rw, rh))
    got = parser.process(conf, paf)
    _check_debug(parser, 0, orc, name)
    _cmp_frame(got, orc, name)
    want = np.load(os.path.join(golden_dir, "ref_humans_area.npz"))[name + "_humans"]
    assert got.tobytes() == want.tobytes()
    # batched, mixed with itself: same answer per frame
    N = 3
    b = parser.process_batch(np.repeat(conf[None], N, 0), np.repeat(paf[None], N, 0))
    assert all(x.tobytes() == got.tobytes() for x in b)
    parser.close()


def test_shrinking_resolution_noise_field_vs_oracle():
    """structureless input through the down-scaling path: hundreds of peaks, no golden needed -- oracle parity on peaks and connections"""
    rng = np.random.default_rng(5)
    conf = rng.random((19, 40, 84), dtype=np.float32) * 0.3
    paf = (rng.random((38, 40, 84), dtype=np.float32) - 0.5)
    for res in ((42, 20), (41, 20), (50, 31), (30, 100)):       # 2x2 (SIMD + even width), 2x2 with a scalar tail, fractional, mixed
        parser = capi.PafParser(0.12, 0.05, res)
        parser.set_capacity(peaks_per_part=1024, candidates_per_limb=1 << 15, humans=256)
        got = parser.process(conf, paf, cap=256)
        orc = oracle.oracle_process(conf, paf, 0.12, 0.05, res[0], res[1], peak_cap=1 << 16, conn_cap=1 << 13)
        assert len(orc["peaks"]) > 30, res
        pk = parser.debug_peaks(0)
        assert np.array_equal(pk["x"], orc["peaks"]["x"]) and np.array_equal(pk["y"], orc["peaks"]["y"]) and pk["score"].tobytes() == orc["peaks"]["score"].tobytes(), res
        parser.close()


def test_full_size_property_permutation_invariance():
    """size-independent property at the full cfg3 batch: the parser is per-frame, so permuting the
    batch permutes the outputs; and the identical frame repeated gives identical humans."""
    conf, paf = syn.make_batch_tensors(21, 16, (3, 9), 46, 82)
    parser = capi.PafParser()
    a = parser.process_batch(conf, paf)
    perm = np.random.default_rng(0).permutation(16)
    b = parser.process_batch(conf[perm], paf[perm])
    for i, j in enumerate(perm):
        assert a[j].tobytes() == b[i].tobytes()
    c = parser.process_batch(np.repeat(conf[:1], 16, 0), np.repeat(paf[:1], 16, 0))
    assert all(x.tobytes() == c[0].tobytes() for x in c)
    parser.close()
