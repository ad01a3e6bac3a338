"""The benchmark networks in the precisions tests/test_network_ops.py does not build them in: TF32 (what data_type::kFLOAT, the
reference's default, maps to) and INT8, at the input sizes and batches bench.py and tools/bench_lw.py time their fp16 forms.  The
engine picks its plans from max_batch and the map sizes (items per persistent CTA, multi-round launches, n-tile splits), so these
launch sequences are only seen at these sizes.  The harness is test_network_ops's, imported; each INT8 pack is calibrated once, as
tools/bench_int8.py calibrates: one max_batch of seed-500 frames through a TF32 engine of the same max_batch.

  1. every launch group against float64 (TF32: |got - ref| <= 2^-11 |ref| + (K + 2) 2^-23 mag + 2^-24, K in 32-channel chunks) or
     byte for byte against tests/int8_sim.py (INT8), the channels outside each group's outputs kept, the tap mutation rejected, and
     the whole run byte-identical to the op-by-op replay: test_network_ops test 1, on the configs below;
  2. a short batch of B/2 + 1 frames at the benchmark plans: test_network_ops test 2;
  3. the pipelined pose call (submit_pose / collect_pose) computes every buffer and both outputs as infer_u8 does: PAF packs from a
     captured graph, OpenPifPaf with the decoder on its own stream and the conv grids narrowed by the SMs reserved for it (at least
     one TF32 conv launch of cfg5 has more work items than the SMs left, so the narrowed grid runs several rounds);
  4. the frame-format calls on a TF32 and an INT8 engine.  On these engines the slot's resized frames are read by im2col_c4_kernel
     inside the slot's captured graph (on f16 the fused u8 stem reads them).  Ten batches, two tickets in flight, the geometry,
     format and call changing from each batch to the next: camera-size BGR frames plain and letterboxed, host NV12 / I420 and pitched
     device NV12 surfaces, pitched host and device YUYV / BGRA, P016 and 16-bit gray, 4:2:0 rotated 90 / 270 and interleaved rotated
     180.  For every ticket the resized frames equal the restatements (tests/{yuv,interleaved,highbit,rotated}_ref.py) and the cv2 sha
     the source is pinned to, every buffer and both outputs equal infer_u8 on those frames, and the humans equal process_batch of
     those outputs (random weights give thousands of peaks but no people).  Then every batch goes once through the capacity-growth
     rerun in collect, over crowd tensors copied over the outputs, so the rerun's humans are compared with people in them.
The CPU tests check the harness on these precisions (the per-group references chained over their own buffers reproduce the whole
graph exactly) and that every network and precision the benchmarks build has a config here or in test_network_ops."""
import ast
import importlib.util
import os
import time

import numpy as np
import pytest
import torch

import oracle
from hyperpose_b200 import capi, models, synthetic as syn
from oracle import torch_backbone
from tests import highbit_ref, interleaved_ref, rotated_ref, test_network_ops as netops, yuv_ref
from tests.golden.make_golden import RESIZE_CASES, sha
from tests.golden.make_golden_highbit import HB_SIZES, highbit_frame, key as highbit_key
from tests.golden.make_golden_interleaved import case_frame
from tests.golden.make_golden_rotated import ROT_CASES, rotated_frame
from tests.golden.make_golden_yuv import YUV_CASES, yuv_pack, yuv_planes
from tests.test_engine_kernels import work_items
from tests.test_network_ops import (CAL_SEED, CPU_SIZES, FRAME_SEED, _buf_hw, _clean_env, _diff_state, _frame_hashes, _read, _ref_device,
                                    _replay, _state, launch_groups)

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (id, graph, H, W, max_batch, dtype): bench.py's cfg2, cfg4, cfg5 and tools/bench_lw.py's networks, in the other precisions
CONFIGS = [("cfg2-tf32", "mobilenet_thin_openpose", 368, 432, 8, "tf32"), ("cfg4-tf32", "resnet50_lw_openpose", 368, 432, 32, "tf32"),
           ("cfg5-tf32", "resnet50_pifpaf", 385, 385, 16, "tf32"),
           ("lw_vggtiny-256x384-tf32", "lw_openpose_vggtiny", 256, 384, 16, "tf32"),
           ("lw_vggtiny-342x368-tf32", "lw_openpose_vggtiny", 342, 368, 16, "tf32"),
           ("lw_resnet18-tf32", "lw_openpose_resnet18", 368, 432, 16, "tf32"),
           ("lw_mobilenet_dilated-tf32", "lw_openpose_mobilenet_dilated", 368, 432, 16, "tf32"),
           ("lw_vggtiny-256x384-int8", "lw_openpose_vggtiny", 256, 384, 16, "int8"),
           ("lw_vggtiny-342x368-int8", "lw_openpose_vggtiny", 342, 368, 16, "int8"),
           ("lw_resnet18-int8", "lw_openpose_resnet18", 368, 432, 16, "int8"),
           ("lw_mobilenet_dilated-int8", "lw_openpose_mobilenet_dilated", 368, 432, 16, "int8")]
CFG = {c[0]: c for c in CONFIGS}


def _calibrate(name, H, W, B):
    """tools/bench_int8.py's calibration: per-buffer max |x| of one max_batch of CAL_SEED frames through a TF32 engine"""
    cal = capi.Engine(getattr(models, name)(seed=0).to_pack(), (W, H), max_batch_size=B, dtype="tf32")
    absmax = cal.calibrate(syn.make_frames_u8(CAL_SEED, B, H, W))
    cal.close()
    return absmax


@pytest.fixture(scope="module")
def int8_absmax():
    """calibration of an INT8 config, computed on first use and kept for the module's other tests"""
    done = {}

    def get(cid):
        if cid not in done:
            _, name, H, W, B, _ = CFG[cid]
            done[cid] = _calibrate(name, H, W, B)
        return done[cid]
    return get


def _build(cid, monkeypatch, int8_absmax):
    """test_network_ops._build for this file's configs: seed-0 weights, FRAME_SEED frames, the INT8 scales from int8_absmax"""
    _, name, H, W, B, dtype = CFG[cid]
    _clean_env(monkeypatch)
    g = getattr(models, name)(seed=0)
    if dtype == "int8":
        g.set_int8_scales(int8_absmax(cid))
    eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=B, dtype=dtype)
    return g, eng, syn.make_frames_u8(FRAME_SEED, B, H, W)


@gpu
@pytest.mark.parametrize("cid", [c[0] for c in CONFIGS])
def test_network_ops_against_fp64_and_replay(cid, monkeypatch, int8_absmax):
    """test 1: every launch group against float64 (the INT8 model), and the op-by-op replay byte-identical to the whole run"""
    t0 = time.time()
    g, eng, frames = _build(cid, monkeypatch, int8_absmax)
    B = frames.shape[0]
    kernels = [eng.debug_op_kernel(i) for i in range(len(g.ops))]
    bufs = range(len(g.buffers))
    eng.infer_u8(frames)
    whole = _state(eng, bufs, B)
    groups = launch_groups(g, kernels, eng.dtype)
    worst, mutated = _replay(g, eng, frames, groups, B, _ref_device(), cid)
    replay = _state(eng, bufs, B)
    bad = _diff_state(whole, replay)
    assert not bad, f"{cid}: the op-by-op replay differs from the whole run at (buffer, frame) {bad[:8]} ({len(bad)} in all)"
    assert mutated, f"{cid}: no conv kernel"
    print(f"[network ops] {cid}: {len(groups)} launch groups, PDL {eng.debug_uses_pdl()}, conv kernels {sorted(mutated)}; " +
          ("every group byte-exact" if eng.dtype == "int8" else f"worst |got - ref| / bound {worst:.3f}") + f"; {time.time() - t0:.1f} s")
    eng.close()


@gpu
@pytest.mark.parametrize("cid", [c[0] for c in CONFIGS])
def test_short_batch_at_benchmark_plans(cid, monkeypatch, int8_absmax):
    """test 2: infer_u8 on N' = B/2 + 1 frames of the benchmark engine: frames < N' as in the full run, frames >= N' untouched"""
    g, eng, frames = _build(cid, monkeypatch, int8_absmax)
    B = frames.shape[0]
    n = B // 2 + 1
    bufs = range(len(g.buffers))
    eng.infer_u8(frames)
    full = _state(eng, bufs, B)
    sentinel = {}
    for bi in bufs:
        a = _read(eng, bi, B)
        a[n:] = -128 if eng.dtype == "int8" else np.nan
        eng.debug_write_buffer(bi, a)
        sentinel[bi] = _frame_hashes(a)
    eng.infer_u8(frames[:n])
    short = _state(eng, bufs, B)
    bad = _diff_state(full, short, range(n))
    assert not bad, f"{cid}: frames < {n} of the short batch differ from the full run at (buffer, frame) {bad[:8]}"
    past = [(bi, i) for bi in bufs for i in range(n, B) if short[bi][i] != sentinel[bi][i]]
    past += [(k, i) for k in ("conf", "paf") for i in range(n, B) if short[k][i] != full[k][i]]
    assert not past, f"{cid}: the {n}-frame batch wrote past frame {n} at (buffer, frame) {past[:8]}"
    eng.close()


@gpu
@pytest.mark.parametrize("cid", ["cfg2-tf32", "cfg4-tf32", "cfg5-tf32", "lw_resnet18-int8"])
def test_pipelined_pose_call_matches_infer(cid, monkeypatch, int8_absmax):
    """test 3: submit_pose / collect_pose compute every buffer and both outputs as infer_u8 does.  OpenPifPaf: the engine leaves
    min(max_batch, 16, SMs / 2) SMs (its default reserve; the HPB_ variables are cleared) to the decoder, and at least one TF32 conv
    launch has more work items than the SMs it keeps, so the narrowed grid is what computes it."""
    g, eng, frames = _build(cid, monkeypatch, int8_absmax)
    B, H, W = frames.shape[:3]
    bufs = range(len(g.buffers))
    if eng.head_type == 1:
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        kept = sms - min(B, 16, sms // 2)
        items = [work_items(k, g.ops[i], B, *_buf_hw(g, g.ops[i].in_buf, H, W))
                 for i, k in enumerate(eng.debug_op_kernel(i) for i in range(len(g.ops))) if k.startswith("conv<tf32")]
        assert max(items) > kept, f"{cid}: no TF32 conv launch has more than {kept} work items ({max(items)} at most)"
        print(f"[network ops] {cid}: {sum(n > kept for n in items)} of {len(items)} TF32 conv launches have more than {kept} work items")
    eng.infer_u8(frames)
    direct = _state(eng, bufs, B)
    conf, paf = eng.read_outputs(B)
    if eng.head_type == 1:
        parser = capi.PifPafParser(eng.in_h, eng.in_w, 0.1)
    else:
        parser = capi.PafParser(float(np.quantile(conf[:, :18], 0.97)), float(np.quantile(paf, 0.5)))
        parser.set_capacity(peaks_per_part=1024, candidates_per_limb=1 << 15, humans=128)
    humans = eng.collect_pose(eng.submit_pose(parser, frames), cap=128)
    piped = _state(eng, bufs, B)
    bad = _diff_state(direct, piped)
    assert not bad, f"{cid}: the pipelined call differs from infer_u8 at (buffer, frame) {bad[:8]}"
    assert len(humans) == B
    if eng.head_type != 1:   # (random weights give OpenPifPaf fields without people: its decode is tested in test_pifpaf_stages.py)
        want = parser.process_batch(conf, paf, cap=128)
        assert all(a.tobytes() == b.tobytes() for a, b in zip(humans, want)), f"{cid}: pipelined humans differ from a parse of the outputs"
        assert eng.pose_stats()["graph_captures"] >= 1
    parser.close()
    eng.close()


# ---- frame-format calls on TF32 and INT8 engines ----------------------------------------------------------------------------
NET_H, NET_W = 368, 656
FRAMES_PER_BATCH = 3   # one batch size throughout: each slot captures its graph once and replays it for every later batch


def _case(cases, h, w):
    """the index of the (h, w) -> NET_H x NET_W case of a pin table"""
    return next(i for i, c in enumerate(cases) if tuple(c) == (h, w, NET_H, NET_W))


def _pitched(frame, extra):
    """frame as a crop view of rows `extra` pixels longer, every other byte 255"""
    h, w = frame.shape[:2]
    buf = np.full((h, w + extra) + frame.shape[2:], 255, frame.dtype)
    buf[:, :w] = frame
    return buf[:, :w]


def _surface(frame, pitch):
    """an interleaved frame's rows in a u8 [rows, pitch] surface, every other byte 255"""
    h, row = frame.shape[0], frame[0].size
    s = np.full((h, pitch), 255, np.uint8)
    s[:, :row] = frame.reshape(h, row)
    return s


def _nv12_surface(Y, U, V, pitch, rows):
    """NV12 as a decoder leaves it: luma rows with `pitch`, padded to `rows` rows, the UV plane after them; every other byte 255"""
    h, w = Y.shape
    s = np.full((rows + rows // 2, pitch), 255, np.uint8)
    s[:h, :w] = Y
    s[rows:rows + h // 2, :w] = np.stack([U, V], -1).reshape(h // 2, w)
    return s


class FrameBatch:
    """one submitted batch: the call that submits it, its frames' reference conversion to BGR and the cv2 sha each resized frame
    is pinned to"""

    def __init__(self, label, keep, bgr, pins, submit):
        self.label, self.keep, self.pins, self.submit = label, keep, pins, submit
        self.want = np.stack([oracle.resize_linear_u8(b, NET_H, NET_W, letterbox=keep) for b in bgr])


def _frame_batches(golden_dir):
    """the ten batches of test 4, in submission order; device surfaces are allocated here and live as long as the list"""
    pin = {n: np.load(os.path.join(golden_dir, f"cv_pin{n}.npz")) for n in ("", "_yuv", "_interleaved", "_highbit", "_rotated")}
    rz = {False: "rz", True: "lb"}
    out = []
    dev = []

    def on_device(a):
        t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
        dev.append(t)
        return t.data_ptr()

    # camera-size BGR frames (test_network_ops' resize sources), plain and letterboxed
    for keep, sizes in ((False, [(720, 1280), (1080, 1920), (360, 640)]), (True, [(736, 1312), (368, 656), (480, 640)])):
        idx = [_case(RESIZE_CASES, h, w) for h, w in sizes]
        imgs = [netops._resize_src(i) for i in idx]
        out.append(FrameBatch(f"bgr keep_ratio={keep}", keep, imgs, [str(pin[""][f"{rz[keep]}{i}_sha"]) for i in idx],
                              lambda eng, p, imgs=imgs, keep=keep: eng.submit_pose_frames(p, imgs, keep_ratio=keep)))
    # host NV12 / I420, then pitched device NV12: a 1080p decoder surface (pitch 2048, 1088 rows) and two smaller ones
    spec = [("nv12", (720, 1280)), ("i420", (1080, 1920)), ("i420", (360, 640))]
    idx = [_case(YUV_CASES, h, w) for _, (h, w) in spec]
    frames = [yuv_pack(*yuv_planes(800 + i, *YUV_CASES[i][:2]), lay) for i, (lay, _) in zip(idx, spec)]
    lays = [lay for lay, _ in spec]
    out.append(FrameBatch("yuv420 host", False, [yuv_ref.yuv420_to_bgr(f, lay) for f, lay in zip(frames, lays)],
                          [str(pin["_yuv"][f"{lay}{i}_rz_sha"]) for i, lay in zip(idx, lays)],
                          lambda eng, p, frames=frames, lays=lays: eng.submit_pose_yuv420(p, frames, lays)))
    spec = [((1080, 1920), 2048, 1088), ((736, 1312), 1536, 744), ((480, 640), 768, 480)]
    idx = [_case(YUV_CASES, h, w) for (h, w), _, _ in spec]
    recs, bgr = [], []
    for i, (_, pitch, rows) in zip(idx, spec):
        Y, U, V = yuv_planes(800 + i, *YUV_CASES[i][:2])
        p = on_device(_nv12_surface(Y, U, V, pitch, rows))
        recs.append(capi.FrameYUV420(p, p + rows * pitch, p + rows * pitch + 1, Y.shape[0], Y.shape[1], pitch, pitch, 2))
        bgr.append(yuv_ref.yuv420_to_bgr(yuv_pack(Y, U, V, "nv12"), "nv12"))
    out.append(FrameBatch("nv12 device surfaces keep_ratio=True", True, bgr, [str(pin["_yuv"][f"nv12{i}_lb_sha"]) for i in idx],
                          lambda eng, p, recs=recs: eng.submit_pose_yuv420_device(p, recs, keep_ratio=True)))
    # pitched YUYV / BGRA: crop views of host frames, then device surfaces with 256-byte-aligned pitches
    spec = [("yuyv", (720, 1280)), ("bgra", (1080, 1920)), ("yuyv", (360, 640))]
    idx = [_case(RESIZE_CASES, h, w) for _, (h, w) in spec]
    fmts = [f for f, _ in spec]
    frames = [_pitched(case_frame(i, f), 6) for i, f in zip(idx, fmts)]
    out.append(FrameBatch("interleaved host pitched", False, [interleaved_ref.to_bgr(f, x) for f, x in zip(frames, fmts)],
                          [str(pin["_interleaved"][f"{x}{i}_rz_sha"]) for i, x in zip(idx, fmts)],
                          lambda eng, p, frames=frames, fmts=fmts: eng.submit_pose_interleaved(p, frames, fmts)))
    spec = [("bgra", (736, 1312)), ("yuyv", (480, 640)), ("bgra", (368, 656))]
    idx = [_case(RESIZE_CASES, h, w) for _, (h, w) in spec]
    fmts = [f for f, _ in spec]
    frames = [case_frame(i, f) for i, f in zip(idx, fmts)]
    recs = []
    for f, x in zip(frames, fmts):
        pitch = -(-f[0].size // 256) * 256 + 256
        recs.append(capi.FrameInterleaved(on_device(_surface(f, pitch)), f.shape[0], f.shape[1], pitch, capi.PIXEL_FORMATS[x]))
    out.append(FrameBatch("interleaved device surfaces keep_ratio=True", True, [interleaved_ref.to_bgr(f, x) for f, x in zip(frames, fmts)],
                          [str(pin["_interleaved"][f"{x}{i}_lb_sha"]) for i, x in zip(idx, fmts)],
                          lambda eng, p, recs=recs: eng.submit_pose_interleaved_device(p, recs, keep_ratio=True)))
    # P016, then 16-bit gray (crop views with garbage after each row), at 10, 12 and 16 significant bits
    for call, fmt, keep, spec in (("submit_pose_yuv420_16", "p016", False, [((1080, 1920), 16), ((360, 640), 10), ((720, 1280), 12)]),
                                  ("submit_pose_interleaved16", "gray16", True, [((720, 1280), 12), ((362, 642), 16), ((1080, 1920), 10)])):
        idx = [HB_SIZES.index(hw) for hw, _ in spec]
        bits = [b for _, b in spec]
        frames = [highbit_frame(fmt, i, b) for i, b in zip(idx, bits)]
        out.append(FrameBatch(f"{fmt} keep_ratio={keep}", keep, [highbit_ref.to_bgr(f, fmt, b) for f, b in zip(frames, bits)],
                              [str(pin["_highbit"][f"{highbit_key(fmt, i, b, 0)}_{rz[keep]}_sha"]) for i, b in zip(idx, bits)],
                              lambda eng, p, call=call, frames=frames, fmt=fmt, bits=bits, keep=keep:
                                  getattr(eng, call)(p, frames, fmt, bits, keep_ratio=keep)))
    # rotated: 4:2:0 frames at 90 and 270, interleaved frames at 180
    for call, keep, spec in (("submit_pose_yuv420", False, [("nv12", (1080, 1920), 90), ("i420", (360, 640), 270), ("nv12", (1312, 736), 90)]),
                             ("submit_pose_interleaved", True, [("yuyv", (640, 480), 180), ("bgra", (1080, 1920), 180), ("gray", (656, 368), 180)])):
        idx = [_case(ROT_CASES, h, w) for _, (h, w), _ in spec]
        fmts, rots = [f for f, _, _ in spec], [r for _, _, r in spec]
        frames = [rotated_frame(i, f) for i, f in zip(idx, fmts)]
        out.append(FrameBatch(f"{fmts} rotated {rots} keep_ratio={keep}", keep,
                              [rotated_ref.to_bgr(f, x, r) for f, x, r in zip(frames, fmts, rots)],
                              [str(pin["_rotated"][f"{x}{i}_r{r}_{rz[keep]}_sha"]) for i, x, r in zip(idx, fmts, rots)],
                              lambda eng, p, call=call, frames=frames, fmts=fmts, rots=rots, keep=keep:
                                  getattr(eng, call)(p, frames, fmts, keep_ratio=keep, rotation=rots)))
    torch.cuda.synchronize()
    assert all(len(b.pins) == FRAMES_PER_BATCH for b in out)
    return out, dev


def _same_humans(a, b):
    return len(a) == len(b) and all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


def _check_slot_frames(eng, t, b, what):
    got = eng.debug_read_slot_frames(t, FRAMES_PER_BATCH)
    for k in range(FRAMES_PER_BATCH):
        assert np.array_equal(got[k], b.want[k]), f"{what}: {b.label}: frame {k}: {int((got[k] != b.want[k]).sum())} bytes differ from the restatement"
        assert sha(got[k]) == b.pins[k], f"{what}: {b.label}: frame {k} differs from its cv2 pin"


@gpu
@pytest.mark.parametrize("dtype", ["tf32", "int8"])
def test_frame_calls_on_tf32_and_int8_engines(dtype, golden_dir, monkeypatch):
    """test 4: the ten batches of _frame_batches on tiny_test_net at 368 x 656.  Ticket pairs (batch k, batch k + 1), k = 0 .. 9 (the
    last pair wraps around): both are submitted before either is collected.  The activation buffers and outputs are the engine's, so
    they are compared after the second ticket of each pair: every batch is that ticket once."""
    N = FRAMES_PER_BATCH
    _clean_env(monkeypatch)
    g = models.tiny_test_net(0)
    if dtype == "int8":
        g.set_int8_scales(_calibrate("tiny_test_net", NET_H, NET_W, N))
    eng = capi.Engine(g.to_pack(), (NET_W, NET_H), max_batch_size=N, dtype=dtype)
    batches, dev = _frame_batches(golden_dir)
    bufs = range(len(g.buffers))
    eng.infer_u8(batches[0].want)
    conf, paf = eng.read_outputs(N)
    parser = capi.PafParser(float(np.quantile(conf[:, :18], 0.995)), float(np.quantile(paf, 0.5)))
    parser.set_capacity(peaks_per_part=4096, candidates_per_limb=1 << 15, humans=128)
    # per batch: infer_u8's buffers and outputs on the reference frames, and the parse of those outputs
    ref, n_peaks, n_humans = [], 0, 0
    for b in batches:
        eng.infer_u8(b.want)
        st = _state(eng, bufs, N)
        conf, paf = eng.read_outputs(N)
        humans = parser.process_batch(conf, paf, cap=128)
        n_peaks += sum(len(parser.debug_peaks(f)) for f in range(N))
        n_humans += sum(len(h) for h in humans)
        ref.append((st, humans))
    assert n_peaks > 50, "vacuous: no peaks at these thresholds"
    captures = None
    for k in range(len(batches)):
        pair = (k, (k + 1) % len(batches))
        tickets = [batches[j].submit(eng, parser) for j in pair]
        for j, t in zip(pair, tickets):
            _check_slot_frames(eng, t, batches[j], dtype)
            assert _same_humans(eng.collect_pose(t, cap=128), ref[j][1]), f"{dtype}: {batches[j].label}: humans differ from a parse of infer_u8's outputs"
        bad = _diff_state(ref[pair[1]][0], _state(eng, bufs, N))
        assert not bad, f"{dtype}: {batches[pair[1]].label} (after {batches[pair[0]].label}): differs from infer_u8 at (buffer, frame) {bad[:8]}"
        if k == 0:
            captures = eng.pose_stats()["graph_captures"]
            assert 1 <= captures <= 2
    stats = eng.pose_stats()
    assert stats["graph_captures"] == captures, "a new frame geometry, format or call recaptured the graph"
    assert stats["graph_launches"] >= 2 * len(batches)
    # the capacity-growth rerun: over crowd tensors every capacity of a small parser overflows, collect grows it and runs the slot
    # again from its resized frames
    cc, pp = syn.make_batch_tensors(13, N, (6, 10), eng.out_h, eng.out_w)
    d_conf, d_paf = torch.from_numpy(cc).cuda(), torch.from_numpy(pp).cuda()
    torch.cuda.synchronize()
    eng.set_output_override(d_conf.data_ptr(), d_paf.data_ptr())
    big = capi.PafParser()
    big.set_capacity(peaks_per_part=1024, candidates_per_limb=1 << 15, humans=128)
    want = big.process_batch(cc, pp, cap=128)
    assert max(len(h) for h in want) > 1
    for j, b in enumerate(batches):
        small = capi.PafParser()
        small.set_capacity(peaks_per_part=2, candidates_per_limb=2, humans=1)
        t = b.submit(eng, small)
        assert _same_humans(eng.collect_pose(t, cap=128), want), f"{dtype}: {b.label}: the growth rerun's humans differ"
        _check_slot_frames(eng, t, b, f"{dtype} growth rerun")
        st = _state(eng, bufs, N)
        bad = _diff_state({bi: ref[j][0][bi] for bi in bufs}, st)
        assert not bad, f"{dtype}: {b.label}: the growth rerun's buffers differ from infer_u8 at (buffer, frame) {bad[:8]}"
        conf, paf = eng.read_outputs(N)
        assert conf.tobytes() == cc.tobytes() and paf.tobytes() == pp.tobytes()
        small.close()
    print(f"[frame calls] {dtype}: {len(batches)} batches of {N} frames, {n_peaks} peaks, {n_humans} humans; "
          f"{stats['graph_captures']} captures, {stats['graph_launches']} graph launches")
    eng.set_output_override(0, 0)
    eng.close(); parser.close(); big.close()
    del dev


# ---- the harness on the CPU -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted({c[1] for c in CONFIGS + netops.CONFIGS if c[5] == "tf32"}))
def test_tf32_group_references_chain_to_the_whole_graph(name):
    """the per-group references of the TF32 engine's groups (one per op, the im2col op with the conv that reads its patches) under
    rounding="tf32", chained over their own buffers, reproduce run_graph of the whole graph bit for bit"""
    H, W = CPU_SIZES.get(name, (64, 96))
    g = getattr(models, name)(seed=0)
    frames = syn.make_frames_u8(3, 2, H, W)
    groups = launch_groups(g, ["op"] * len(g.ops), "tf32")
    stems = [grp for grp in groups if grp.stem]
    assert len(stems) == 1 and len(stems[0].ops) == 2 and len(groups) == len(g.ops) - 1
    conf, paf, whole = torch_backbone.run_graph(g, frames, device="cpu", dtype=torch.float64, rounding="tf32", round_stores=False)
    state = [torch.zeros_like(b) for b in whole]
    cc = pc = None
    for grp in groups:
        if grp.ops[-1].type == models.OP_PPN_HEAD:   # checked against ppn_head_ref on the GPU; run_graph has no PPN head
            continue
        bufs, c, p = grp.reference({b: state[b].numpy() for b in grp.used}, frames)
        for b, t in bufs.items():
            state[b] = t
        if c is not None:
            cc, pc = c, p
    for b, (x, y) in enumerate(zip(whole, state)):
        assert torch.equal(x, y), f"{name}: buffer {b} differs"
    if conf is not None:
        assert torch.equal(conf, cc) and torch.equal(paf, pc)


@pytest.mark.parametrize("name", sorted({c[1] for c in CONFIGS if c[5] == "int8"}))
def test_int8_group_references_chain_to_the_whole_graph(name):
    """test_network_ops' INT8 chain (one group per op, int8_sim byte for byte) on this file's INT8 graphs"""
    netops.test_int8_group_references_chain_to_the_whole_graph(name)


def _module(rel):
    spec = importlib.util.spec_from_file_location("_bench_" + os.path.splitext(os.path.basename(rel))[0], os.path.join(ROOT, rel))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def _option_default(rel, flag):
    """the default of a script's command-line option, read from its add_argument call"""
    with open(os.path.join(ROOT, rel)) as f:
        tree = ast.parse(f.read())
    for node in ast.walk(tree):
        if isinstance(node, ast.Call) and getattr(node.func, "attr", None) == "add_argument" and node.args and \
                isinstance(node.args[0], ast.Constant) and node.args[0].value == flag:
            return next(ast.literal_eval(k.value) for k in node.keywords if k.arg == "default")
    raise AssertionError(f"{rel}: no {flag} option")


def test_every_benchmark_network_and_precision_has_a_config():
    """every (graph, H, W, max_batch) that bench.py or tools/bench_{lw,ppn,int8}.py builds, in every precision the engine accepts
    for its head type (f16 and TF32 always; INT8 only for PAF heads, head_type 0: hp_engine_create refuses the others), has a
    config here or in test_network_ops.CONFIGS; and every config here is one of those builds"""
    bench, lw, ppn, i8 = (_module(p) for p in ("bench.py", "tools/bench_lw.py", "tools/bench_ppn.py", "tools/bench_int8.py"))
    built = {(w["graph"], w["in_h"], w["in_w"], w["batch"]) for w in bench.WORKLOADS.values()}
    built |= {(net, H, W, lw.B) for _, net, H, W in lw.WORKLOADS}
    built |= {(net, ppn.H, ppn.W, ppn.B) for net in _option_default("tools/bench_ppn.py", "--nets").split(",")}
    built |= {(net, H, W, B) for net, H, W, B, _ in i8.WORKLOADS.values()}
    have = {tuple(c[1:]) for c in CONFIGS + netops.CONFIGS}
    head = {net: getattr(models, net)(seed=0).head_type for net in {b[0] for b in built}}
    missing = [b + (dt,) for b in sorted(built) for dt in ("f16", "tf32", "int8")
               if (dt != "int8" or head[b[0]] == 0) and b + (dt,) not in have]
    assert not missing, f"benchmark builds without a config: {missing}"
    assert {tuple(c[1:5]) for c in CONFIGS} <= built, "a config here is not a benchmark build"
