"""The pipelined pose calls on YUV 4:2:0 frames (hp_pose_submit{,_pifpaf,_ppn}_frames_yuv420_host / _device): the BT.601 conversion
of cv::cvtColor fused into the batched resize's fetch, bit-exact with cv::resize(cv::cvtColor(src, code)).

  1. every YUV_CASES source in all four layouts, plain and letterboxed, through submit_pose_yuv420: the resized frames equal
     oracle.resize_linear_u8(yuv_ref.yuv420_to_bgr(...)) and the cv2 sha it is pinned to;
  2. a mixed batch (720p, 1080p, network size, the exact-2x path, an upscale, a portrait frame; NV12, I420, NV21 and YV12 frames in
     one batch): resized frames, engine outputs and humans equal submit_pose_frames on the reference-converted BGR frames, for a PAF, an
     OpenPifPaf and a Pose Proposal Network pack;
  3. device NV12 laid out as NVDEC writes 1080p: pitch 2048, a 1088-row luma surface, the UV plane after it, every padding byte 255;
  4. host frames pageable and page-locked, two tickets in flight with a different geometry and layout in every batch, no recapture;
  5. the refusals;
  6. a batch that overflows the PAF parser's capacities: the rerun in collect reuses the converted frames."""
import os

import numpy as np
import pytest

import oracle
from hyperpose_b200 import capi, models, synthetic as syn
from tests import yuv_ref
from tests.golden.make_golden import sha
from tests.golden.make_golden_yuv import YUV_CASES, YUV_LAYOUTS, yuv_pack, yuv_planes

gpu = pytest.mark.gpu
H, W = 368, 656
# the cameras' and the reference examples' frame sizes, the network size, the exact-2x area path, an upscale and a portrait frame
MIXED = [(720, 1280), (1080, 1920), (H, W), (736, 1312), (38, 54), (640, 360)]
MIXED_LAYOUTS = ["nv12", "i420", "nv21", "yv12", "nv12", "i420"]


def _yuv(seed, h, w, layout):
    return yuv_pack(*yuv_planes(seed, h, w), layout)


def _bgr(frames, layouts):
    return [yuv_ref.yuv420_to_bgr(f, lay) for f, lay in zip(frames, layouts)]


def _resized(frames, layouts, h, w, keep):
    return np.stack([oracle.resize_linear_u8(b, h, w, letterbox=keep) for b in _bgr(frames, layouts)])


def _tiny(max_batch, h=H, w=W):
    return capi.Engine(models.tiny_test_net(0).to_pack(), (w, h), max_batch_size=max_batch)


def _quiet():
    """a parser that finds no peak: random-weight maps at the default thresholds hold more than the parser's capacity limits"""
    return capi.PafParser(1e30, 1e30)


def _same_humans(a, b):
    return len(a) == len(b) and all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


def _status(fn, *a, **k):
    with pytest.raises(capi.HyperposeError) as e:
        fn(*a, **k)
    return e.value.status


@gpu
def test_every_pinned_case(golden_dir):
    pin = np.load(os.path.join(golden_dir, "cv_pin_yuv.npz"))
    by_dst = {}
    for i, (_, _, dh, dw) in enumerate(YUV_CASES):
        by_dst.setdefault((dh, dw), []).append(i)
    for (dh, dw), idx in by_dst.items():
        eng = _tiny(len(idx), dh, dw)
        parser = _quiet()
        for lay in YUV_LAYOUTS:
            frames = [_yuv(800 + i, *YUV_CASES[i][:2], lay) for i in idx]
            for keep in (False, True):
                t = eng.submit_pose_yuv420(parser, frames, lay, keep_ratio=keep)
                got = eng.debug_read_slot_frames(t, len(idx))
                eng.collect_pose(t)
                for k, i in enumerate(idx):
                    want = oracle.resize_linear_u8(yuv_ref.yuv420_to_bgr(frames[k], lay), dh, dw, letterbox=keep)
                    assert np.array_equal(got[k], want), f"case {i} {lay} {YUV_CASES[i][:2]} -> {dh}x{dw} keep_ratio={keep}: " \
                                                         f"{int((got[k] != want).sum())} bytes differ"
                    assert sha(got[k]) == str(pin[f"{lay}{i}_{'lb' if keep else 'rz'}_sha"])
        eng.close(); parser.close()


def _compare_heads(eng, quiet, parser, frames, keep, override, cap=128):
    """resized frames and engine outputs (quiet parser, no override), then humans over `override` (parser): the YUV call against
    submit_pose_frames on the reference-converted BGR frames"""
    N = len(frames)
    bgr = _bgr(frames, MIXED_LAYOUTS)
    want_frames = np.stack([oracle.resize_linear_u8(b, eng.in_h, eng.in_w, letterbox=keep) for b in bgr])
    t = eng.submit_pose_yuv420(quiet, frames, MIXED_LAYOUTS, keep_ratio=keep)
    eng.collect_pose(t, cap=cap)
    assert np.array_equal(eng.debug_read_slot_frames(t, N), want_frames)
    outs = eng.read_outputs(N)
    t = eng.submit_pose_frames(quiet, bgr, keep_ratio=keep)
    eng.collect_pose(t, cap=cap)
    assert np.array_equal(eng.debug_read_slot_frames(t, N), want_frames)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(outs, eng.read_outputs(N)))
    eng.set_output_override(override[0].data_ptr(), override[1].data_ptr())
    got = eng.collect_pose(eng.submit_pose_yuv420(parser, frames, MIXED_LAYOUTS, keep_ratio=keep), cap=cap)
    want = eng.collect_pose(eng.submit_pose_frames(parser, bgr, keep_ratio=keep), cap=cap)
    eng.set_output_override(0, 0)
    assert sum(len(h) for h in want) >= N, "vacuous: no humans over the override"
    assert _same_humans(got, want)


def _on_device(*arrays):
    import torch
    d = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]
    torch.cuda.synchronize()
    return d


@gpu
@pytest.mark.parametrize("keep", [False, True])
def test_mixed_batch_paf(keep):
    frames = [_yuv(300 + k, h, w, lay) for k, ((h, w), lay) in enumerate(zip(MIXED, MIXED_LAYOUTS))]
    N = len(frames)
    eng = _tiny(N)
    quiet, parser = _quiet(), capi.PafParser()
    override = _on_device(*syn.make_batch_tensors(11, N, (4, 8), eng.out_h, eng.out_w))
    _compare_heads(eng, quiet, parser, frames, keep, override)
    eng.close(); parser.close(); quiet.close()


@gpu
def test_mixed_batch_pifpaf():
    PH = PW = 385
    sizes = [(720, 1280), (1080, 1920), (386, 386), (770, 770), (38, 54), (640, 360)]
    frames = [_yuv(500 + k, h, w, lay) for k, ((h, w), lay) in enumerate(zip(sizes, MIXED_LAYOUTS))]
    N = len(frames)
    eng = capi.Engine(models.resnet50_pifpaf(0).to_pack(), (PW, PH), max_batch_size=N)
    dec = capi.PifPafParser(PH, PW, 0.1)
    fl = [syn.make_pifpaf_fields(600 + i, (2, 6), eng.out_h, eng.out_w) for i in range(N)]
    override = _on_device(np.stack([f[0] for f in fl]).reshape(N, 85, eng.out_h, eng.out_w),
                          np.stack([f[1] for f in fl]).reshape(N, 171, eng.out_h, eng.out_w))
    for keep in (False, True):
        _compare_heads(eng, dec, dec, frames, keep, override)
    eng.close(); dec.close()


@gpu
def test_mixed_batch_ppn():
    PH = PW = 384
    sizes = [(720, 1280), (1080, 1920), (PH, PW), (2 * PH, 2 * PW), (38, 54), (640, 360)]
    frames = [_yuv(700 + k, h, w, lay) for k, ((h, w), lay) in enumerate(zip(sizes, MIXED_LAYOUTS))]
    N = len(frames)
    K, GH, GW, E, NH, NW = 18, 12, 12, 17, 9, 9
    eng = capi.Engine(models.ppn_resnet18(0).to_pack(), (PW, PH), max_batch_size=8)
    parser = capi.PoseProposalParser((PW, PH))
    ts = [syn.make_ppn_tensors(3300 + i, (4, 8)) for i in range(N)]
    box = np.stack([np.stack(t[:6]) for t in ts]).reshape(N, 6 * K, GH, GW).astype(np.float32)
    edge = np.stack([t[6] for t in ts]).reshape(N, E * NH * NW, GH, GW).astype(np.float32)
    override = _on_device(box, edge)
    for keep in (False, True):
        _compare_heads(eng, parser, parser, frames, keep, override, cap=512)
    eng.close(); parser.close()


@gpu
@pytest.mark.parametrize("keep", [False, True])
def test_device_nv12_surface(keep):
    """NV12 as NVDEC leaves a 1080p frame: luma pitch 2048, 1088 luma rows, the UV plane right after them with the same pitch; the
    padding (columns 1920-2047, rows 1080-1087 and the UV rows past 540) holds 255, so any read outside the visible planes shows"""
    h, w, rows, pitch = 1080, 1920, 1088, 2048
    frames, want = [], []
    for k in range(3):
        Y, U, V = yuv_planes(820 + k, h, w)
        surf = np.full((rows + rows // 2, pitch), 255, np.uint8)
        surf[:h, :w] = Y
        surf[rows:rows + h // 2, :w] = np.stack([U, V], -1).reshape(h // 2, w)
        frames.append(surf)
        want.append(oracle.resize_linear_u8(yuv_ref.yuv420_to_bgr(yuv_pack(Y, U, V, "nv12"), "nv12"), H, W, letterbox=keep))
    d = _on_device(*frames)
    recs = [capi.FrameYUV420(t.data_ptr(), t.data_ptr() + rows * pitch, t.data_ptr() + rows * pitch + 1, h, w, pitch, pitch, 2) for t in d]
    eng = _tiny(3)
    parser = _quiet()
    t = eng.submit_pose_yuv420_device(parser, recs, keep_ratio=keep)
    eng.collect_pose(t)
    assert np.array_equal(eng.debug_read_slot_frames(t, 3), np.stack(want))
    # the same planes from host memory, read with the surface's pitches, land in the same frames
    t = eng._submit_frame_table(parser, (capi.FrameYUV420 * 3)(*[capi.FrameYUV420(f.ctypes.data, f.ctypes.data + rows * pitch,
                                                                                    f.ctypes.data + rows * pitch + 1, h, w, pitch, pitch, 2)
                                                                  for f in frames]), keep, device=False, fmt="yuv420")
    eng.collect_pose(t)
    assert np.array_equal(eng.debug_read_slot_frames(t, 3), np.stack(want))
    eng.close(); parser.close()


@gpu
def test_changing_geometry_and_layout_in_flight():
    import torch
    N = 3
    # (size, keep_ratio, page-locked, layouts) of consecutive batches; each slot's source buffer grows on its second batch
    plan = [((360, 640), False, False, ["nv12", "i420", "nv21"]), ((360, 640), True, True, ["yv12", "nv12", "i420"]),
            ((1080, 1920), False, False, ["i420", "nv21", "yv12"]), ((720, 1280), True, True, ["nv21", "yv12", "nv12"]),
            ((38, 54), False, True, ["nv12", "nv12", "i420"])]
    batches = []
    for b, ((h, w), keep, pinned, lays) in enumerate(plan):
        frames = [_yuv(400 + 10 * b + k, h + 2 * k, w - 2 * k, lays[k]) for k in range(N)]   # sizes differ inside a batch too
        if pinned:
            frames = [torch.from_numpy(f).pin_memory().numpy() for f in frames]
        batches.append((frames, lays, keep, _resized(frames, lays, H, W, keep)))
    eng = _tiny(N)
    eng.infer_u8(batches[0][3])
    conf, paf = eng.read_outputs(N)
    parser = capi.PafParser(float(np.quantile(conf[:, :18], 0.995)), float(np.quantile(paf, 0.5)))
    parser.set_capacity(peaks_per_part=1024, candidates_per_limb=1 << 15, humans=128)
    got, slot_frames = [None] * len(plan), [None] * len(plan)
    tickets, captures = [], None
    for b, (frames, lays, keep, _) in enumerate(batches):
        tickets.append(eng.submit_pose_yuv420(parser, frames, lays, keep_ratio=keep))
        if b == 1:
            captures = eng.pose_stats()["graph_captures"]
            assert 1 <= captures <= 2
        if len(tickets) == 2:
            slot_frames[b - 1] = eng.debug_read_slot_frames(tickets[0], N)
            got[b - 1] = eng.collect_pose(tickets.pop(0), cap=128)
    slot_frames[-1] = eng.debug_read_slot_frames(tickets[0], N)
    got[-1] = eng.collect_pose(tickets.pop(0), cap=128)
    assert eng.pose_stats()["graph_captures"] == captures, "a new frame geometry or layout recaptured the graph"
    n_peaks = 0
    for b, (_, _, _, want_frames) in enumerate(batches):
        assert np.array_equal(slot_frames[b], want_frames), f"batch {b}"
        assert _same_humans(got[b], eng.run_pose(parser, want_frames, cap=128)), f"batch {b}"
        n_peaks += sum(len(parser.debug_peaks(f)) for f in range(N))
    assert n_peaks > 50, "vacuous: no peaks at these thresholds"
    eng.close(); parser.close()


@gpu
def test_refusals():
    eng = _tiny(2, 64, 96)
    parser = _quiet()
    f = _yuv(1, 90, 150, "nv12")
    d = _on_device(f)[0]
    p = d.data_ptr()

    def rec(**kw):
        a = dict(y=p, u=p + 90 * 150, v=p + 90 * 150 + 1, height=90, width=150, pitch_y=150, pitch_uv=150, uv_step=2)
        a.update(kw)
        return capi.FrameYUV420(*a.values())

    assert _status(eng.submit_pose_yuv420, parser, [f] * 3, "nv12") == capi.HP_ERR_BATCH
    assert _status(eng.submit_pose_yuv420_device, parser, [rec()] * 3) == capi.HP_ERR_BATCH
    bad = [dict(y=0), dict(u=0), dict(v=0), dict(height=0), dict(width=-2), dict(height=89), dict(width=149), dict(pitch_y=148),
           dict(pitch_uv=148), dict(uv_step=0), dict(uv_step=3), dict(v=p + 90 * 150 + 2), dict(u=p + 90 * 150 + 1, v=p + 90 * 150 + 1),
           dict(uv_step=1, pitch_uv=74)]
    for kw in bad:
        assert _status(eng.submit_pose_yuv420_device, parser, [rec(), rec(**kw)]) == capi.HP_ERR_ARG, kw
    assert _status(eng.submit_pose_yuv420, parser, [np.zeros((135, 151), np.uint8)], "i420") == capi.HP_ERR_ARG   # odd width
    assert _status(eng.submit_pose_yuv420, capi.PifPafParser(64, 96), [f], "nv12") == capi.HP_ERR_UNSUPPORTED   # no OpenPifPaf heads
    # nothing was enqueued by the refusals: both tickets are free, the accepted forms run
    t0 = eng.submit_pose_yuv420(parser, [f], "nv12")
    t1 = eng.submit_pose_yuv420_device(parser, [rec(), rec(uv_step=1, pitch_uv=75)])
    assert _status(eng.submit_pose_yuv420, parser, [f], "nv12") == capi.HP_ERR_ARG      # a third batch in flight
    eng.collect_pose(t0); eng.collect_pose(t1)
    eng.close()
    ppn = capi.Engine(models.ppn_resnet18(0).to_pack(), (384, 384), max_batch_size=2)
    assert _status(ppn.submit_pose_yuv420, parser, [f], "nv12") == capi.HP_ERR_UNSUPPORTED
    ppn.close(); parser.close()


@gpu
def test_capacity_growth_rerun():
    frames = [_yuv(700 + k, h, w, lay) for k, ((h, w), lay) in enumerate(zip(MIXED, MIXED_LAYOUTS))]
    N = len(frames)
    want_frames = _resized(frames, MIXED_LAYOUTS, H, W, False)
    eng = _tiny(N)
    d_conf, d_paf = _on_device(*syn.make_batch_tensors(12, N, (6, 10), eng.out_h, eng.out_w))
    eng.set_output_override(d_conf.data_ptr(), d_paf.data_ptr())
    big = capi.PafParser()
    big.set_capacity(peaks_per_part=1024, candidates_per_limb=1 << 15, humans=128)
    want = eng.collect_pose(eng.submit_pose(big, want_frames), cap=128)
    assert max(len(h) for h in want) > 1
    small = capi.PafParser()
    small.set_capacity(peaks_per_part=2, candidates_per_limb=2, humans=1)     # everything overflows: collect grows and reruns
    t = eng.submit_pose_yuv420(small, frames, MIXED_LAYOUTS)
    got = eng.collect_pose(t, cap=128)
    assert _same_humans(got, want)
    assert np.array_equal(eng.debug_read_slot_frames(t, N), want_frames)
    eng.set_output_override(0, 0)
    eng.close(); big.close(); small.close()
