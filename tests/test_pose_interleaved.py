"""The pipelined pose calls on interleaved frames (hp_pose_submit{,_pifpaf,_ppn}_frames_interleaved_host / _device): cv::cvtColor's
conversion of RGB, BGRA, RGBA, gray and 4:2:2 (YUYV, UYVY, YVYU) fused into the batched resize's fetch, rows read with a pitch,
bit-exact with cv::resize(cv::cvtColor(src, code)).

  1. every pinned source in every format, plain and letterboxed, through submit_pose_interleaved: the resized frames equal
     oracle.resize_linear_u8(interleaved_ref.to_bgr(...)) and the cv2 sha it is pinned to;
  2. a mixed batch (a different size and format in every frame, one of them a crop view): resized frames, engine outputs and humans
     equal submit_pose_frames on the reference-converted BGR frames, for a PAF, an OpenPifPaf and a Pose Proposal Network pack;
  3. HP_PIX_BGR with pitch = 3 * width, host and device, against the hp_frame_u8 call on the same frames;
  4. pitched device surfaces (1080p BGRA, 720p YUYV, 720p BGR) with 255 in every padding byte, and a host crop view;
  5. host frames pageable and page-locked, two tickets in flight with a different geometry and format in every batch, no recapture;
  6. the refusals;
  7. a batch that overflows the PAF parser's capacities: the rerun in collect reuses the converted frames."""
import os

import numpy as np
import pytest

import oracle
from hyperpose_b200 import capi, models, synthetic as syn
from tests import interleaved_ref
from tests.golden.make_golden import RESIZE_CASES, sha
from tests.golden.make_golden_interleaved import case_frame, cases, interleaved_frame
from tests.interleaved_ref import FORMATS

gpu = pytest.mark.gpu
H, W = 368, 656
# the cameras' and the reference examples' frame sizes, the network size, the exact-2x area path, an upscale, a portrait frame and
# two more, one frame per format
MIXED = [(720, 1280), (1080, 1920), (H, W), (736, 1312), (38, 54), (640, 360), (480, 640), (100, 80)]
MIXED_FORMATS = ["yuyv", "bgra", "rgb", "uyvy", "gray", "rgba", "yvyu", "bgr"]


def _bgr(frames, formats):
    return [interleaved_ref.to_bgr(f, fmt) for f, fmt in zip(frames, formats)]


def _resized(frames, formats, h, w, keep):
    return np.stack([oracle.resize_linear_u8(b, h, w, letterbox=keep) for b in _bgr(frames, formats)])


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


def _on_device(*arrays):
    import torch
    d = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]
    torch.cuda.synchronize()
    return d


def _surface(frame, pitch, rows=None):
    """frame's rows in a u8 [rows, pitch] surface (rows >= the frame's), every other byte 255"""
    h = frame.shape[0]
    row = frame[0].size
    s = np.full((rows or h, pitch), 255, np.uint8)
    s[:h, :row] = frame.reshape(h, row)
    return s


def _mixed(seed, sizes):
    """one frame per MIXED_FORMATS entry; the rgb frame is a crop view of a larger frame"""
    frames = [interleaved_frame(seed + k, h, w, fmt) for k, ((h, w), fmt) in enumerate(zip(sizes, MIXED_FORMATS))]
    k = MIXED_FORMATS.index("rgb")
    h, w = sizes[k]
    frames[k] = interleaved_frame(seed + 50, h + 9, w + 14, "rgb")[5:5 + h, 3:3 + w]
    return frames


@gpu
@pytest.mark.parametrize("fmt", FORMATS)
def test_every_pinned_case(golden_dir, fmt):
    pin = np.load(os.path.join(golden_dir, "cv_pin_interleaved.npz"))
    by_dst = {}
    for i in cases(fmt):
        by_dst.setdefault(tuple(RESIZE_CASES[i][2:]), []).append(i)
    for (dh, dw), idx in by_dst.items():
        eng = _tiny(len(idx), dh, dw)
        parser = _quiet()
        frames = [case_frame(i, fmt) for i in idx]
        for keep in (False, True):
            t = eng.submit_pose_interleaved(parser, frames, fmt, keep_ratio=keep)
            got = eng.debug_read_slot_frames(t, len(idx))
            eng.collect_pose(t)
            for k, i in enumerate(idx):
                want = oracle.resize_linear_u8(interleaved_ref.to_bgr(frames[k], fmt), dh, dw, letterbox=keep)
                assert np.array_equal(got[k], want), f"case {i} {fmt} {RESIZE_CASES[i][:2]} -> {dh}x{dw} keep_ratio={keep}: " \
                                                     f"{int((got[k] != want).sum())} bytes differ"
                assert sha(got[k]) == str(pin[f"{fmt}{i}_{'lb' if keep else 'rz'}_sha"])
        eng.close(); parser.close()


def _compare_heads(eng, quiet, parser, frames, keep, override, cap=128):
    """resized frames and engine outputs (quiet parser, no override), then humans over `override` (parser): the interleaved call
    against submit_pose_frames on the reference-converted BGR frames"""
    N = len(frames)
    bgr = _bgr(frames, MIXED_FORMATS)
    want_frames = np.stack([oracle.resize_linear_u8(b, eng.in_h, eng.in_w, letterbox=keep) for b in bgr])
    t = eng.submit_pose_interleaved(quiet, frames, MIXED_FORMATS, keep_ratio=keep)
    eng.collect_pose(t, cap=cap)
    assert np.array_equal(eng.debug_read_slot_frames(t, N), want_frames)
    outs = eng.read_outputs(N)
    t = eng.submit_pose_frames(quiet, bgr, keep_ratio=keep)
    eng.collect_pose(t, cap=cap)
    assert np.array_equal(eng.debug_read_slot_frames(t, N), want_frames)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(outs, eng.read_outputs(N)))
    eng.set_output_override(override[0].data_ptr(), override[1].data_ptr())
    got = eng.collect_pose(eng.submit_pose_interleaved(parser, frames, MIXED_FORMATS, keep_ratio=keep), cap=cap)
    want = eng.collect_pose(eng.submit_pose_frames(parser, bgr, keep_ratio=keep), cap=cap)
    eng.set_output_override(0, 0)
    assert sum(len(h) for h in want) >= N, "vacuous: no humans over the override"
    assert _same_humans(got, want)


@gpu
@pytest.mark.parametrize("keep", [False, True])
def test_mixed_batch_paf(keep):
    frames = _mixed(300, MIXED)
    N = len(frames)
    eng = _tiny(N)
    quiet, parser = _quiet(), capi.PafParser()
    override = _on_device(*syn.make_batch_tensors(11, N, (4, 8), eng.out_h, eng.out_w))
    _compare_heads(eng, quiet, parser, frames, keep, override)
    eng.close(); parser.close(); quiet.close()


@gpu
def test_mixed_batch_pifpaf():
    PH = PW = 385
    sizes = [(720, 1280), (1080, 1920), (386, 386), (770, 770), (38, 54), (640, 360), (480, 640), (100, 80)]
    frames = _mixed(500, sizes)
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
    sizes = [(720, 1280), (1080, 1920), (PH, PW), (2 * PH, 2 * PW), (38, 54), (640, 360), (480, 640), (100, 80)]
    frames = _mixed(700, sizes)
    N = len(frames)
    K, GH, GW, E, NH, NW = 18, 12, 12, 17, 9, 9
    eng = capi.Engine(models.ppn_resnet18(0).to_pack(), (PW, PH), max_batch_size=N)
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
def test_bgr_is_the_frame_u8_call(keep):
    """HP_PIX_BGR with pitch = 3 * width, from host and from device memory, resizes exactly as hp_frame_u8 and gives the same outputs"""
    frames = [interleaved_frame(40 + k, h, w, "bgr") for k, (h, w) in enumerate(MIXED)]
    N = len(frames)
    eng = _tiny(N)
    parser = _quiet()
    d = _on_device(*frames)
    runs = [lambda: eng.submit_pose_frames(parser, frames, keep_ratio=keep),
            lambda: eng.submit_pose_interleaved(parser, frames, "bgr", keep_ratio=keep),
            lambda: eng.submit_pose_frames_device(parser, [(t.data_ptr(), *f.shape[:2]) for t, f in zip(d, frames)], keep_ratio=keep),
            lambda: eng.submit_pose_interleaved_device(parser, [capi.FrameInterleaved(t.data_ptr(), f.shape[0], f.shape[1], 3 * f.shape[1],
                                                                                      capi.PIXEL_FORMATS["bgr"]) for t, f in zip(d, frames)],
                                                       keep_ratio=keep)]
    got = []
    for run in runs:
        t = run()
        eng.collect_pose(t)
        got.append((eng.debug_read_slot_frames(t, N), eng.read_outputs(N)))
    assert np.array_equal(got[0][0], _resized(frames, ["bgr"] * N, H, W, keep))
    for fr, outs in got[1:]:
        assert np.array_equal(fr, got[0][0])
        assert all(a.tobytes() == b.tobytes() for a, b in zip(outs, got[0][1]))
    eng.close(); parser.close()


@gpu
@pytest.mark.parametrize("keep", [False, True])
def test_pitched_device_surfaces(keep):
    """1080p BGRA with a 8192-byte pitch, 720p YUYV with a 2816-byte pitch and 736 rows, 720p BGR with a 4096-byte pitch, each padding
    byte 255 (a read of the padding shows in the frame); then the same surfaces from host memory and a host crop view"""
    specs = [("bgra", 1080, 1920, 8192, 1080), ("yuyv", 720, 1280, 2816, 736), ("bgr", 720, 1280, 4096, 720)]
    frames = [interleaved_frame(60 + k, h, w, fmt) for k, (fmt, h, w, _, _) in enumerate(specs)]
    surfs = [_surface(f, pitch, rows) for f, (_, _, _, pitch, rows) in zip(frames, specs)]
    fmts = [s[0] for s in specs]
    want = _resized(frames, fmts, H, W, keep)
    d = _on_device(*surfs)
    recs = [capi.FrameInterleaved(t.data_ptr(), h, w, pitch, capi.PIXEL_FORMATS[fmt]) for t, (fmt, h, w, pitch, _) in zip(d, specs)]
    eng = _tiny(4)
    parser = _quiet()
    t = eng.submit_pose_interleaved_device(parser, recs, keep_ratio=keep)
    eng.collect_pose(t)
    assert np.array_equal(eng.debug_read_slot_frames(t, 3), want)
    # the same surfaces in host memory, read with their pitch, and a crop of the BGRA frame as a numpy view (pitch 1920 * 4)
    host = [capi.FrameInterleaved(s.ctypes.data, h, w, pitch, capi.PIXEL_FORMATS[fmt]) for s, (fmt, h, w, pitch, _) in zip(surfs, specs)]
    t = eng._submit_frame_table(parser, (capi.FrameInterleaved * 3)(*host), keep, device=False, fmt="interleaved")
    eng.collect_pose(t)
    assert np.array_equal(eng.debug_read_slot_frames(t, 3), want)
    crop = frames[0][100:820, 300:1580]
    assert crop.strides[0] == 1920 * 4 and not crop.flags.c_contiguous
    t = eng.submit_pose_interleaved(parser, [crop, frames[1]], ["bgra", "yuyv"], keep_ratio=keep)
    eng.collect_pose(t)
    assert np.array_equal(eng.debug_read_slot_frames(t, 2), _resized([crop, frames[1]], ["bgra", "yuyv"], H, W, keep))
    eng.close(); parser.close()


@gpu
def test_changing_geometry_and_format_in_flight():
    import torch
    N = 3
    # (size, keep_ratio, page-locked, formats) of consecutive batches; each slot's source buffer grows on its second batch
    plan = [((360, 640), False, False, ["yuyv", "rgb", "gray"]), ((360, 640), True, True, ["bgra", "uyvy", "rgba"]),
            ((1080, 1920), False, False, ["rgba", "yvyu", "bgr"]), ((720, 1280), True, True, ["gray", "bgra", "yuyv"]),
            ((38, 54), False, True, ["uyvy", "rgb", "bgr"])]
    batches = []
    for b, ((h, w), keep, pinned, fmts) in enumerate(plan):
        frames = [interleaved_frame(400 + 10 * b + k, h + 2 * k, w - 2 * k, fmts[k]) for k in range(N)]   # sizes differ in a batch too
        if pinned:
            frames = [torch.from_numpy(f).pin_memory().numpy() for f in frames]
        batches.append((frames, fmts, keep, _resized(frames, fmts, H, W, keep)))
    eng = _tiny(N)
    eng.infer_u8(batches[0][3])
    conf, paf = eng.read_outputs(N)
    parser = capi.PafParser(float(np.quantile(conf[:, :18], 0.995)), float(np.quantile(paf, 0.5)))
    # the largest peak capacity from the start: some of these frames give a part more than 1024 peaks at this threshold, and this test
    # is about the frames, not about capacity growth (test_capacity_growth_rerun)
    parser.set_capacity(peaks_per_part=4096, candidates_per_limb=1 << 15, humans=128)
    got, slot_frames = [None] * len(plan), [None] * len(plan)
    tickets, captures = [], None
    for b, (frames, fmts, keep, _) in enumerate(batches):
        tickets.append(eng.submit_pose_interleaved(parser, frames, fmts, keep_ratio=keep))
        if b == 1:
            captures = eng.pose_stats()["graph_captures"]
            assert 1 <= captures <= 2
        if len(tickets) == 2:
            slot_frames[b - 1] = eng.debug_read_slot_frames(tickets[0], N)
            got[b - 1] = eng.collect_pose(tickets.pop(0), cap=128)
    slot_frames[-1] = eng.debug_read_slot_frames(tickets[0], N)
    got[-1] = eng.collect_pose(tickets.pop(0), cap=128)
    assert eng.pose_stats()["graph_captures"] == captures, "a new frame geometry or format recaptured the graph"
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
    f = interleaved_frame(1, 90, 150, "yuyv")
    d = _on_device(f)[0]
    p = d.data_ptr()

    def rec(**kw):
        a = dict(data=p, height=90, width=150, pitch=300, format=capi.PIXEL_FORMATS["yuyv"])
        a.update(kw)
        return capi.FrameInterleaved(*a.values())

    assert _status(eng.submit_pose_interleaved, parser, [f] * 3, "yuyv") == capi.HP_ERR_BATCH
    assert _status(eng.submit_pose_interleaved_device, parser, [rec()] * 3) == capi.HP_ERR_BATCH
    bad = [dict(data=0), dict(height=0), dict(width=-2), dict(height=-1), dict(format=8), dict(format=-1), dict(width=149, pitch=300),
           dict(pitch=299), dict(pitch=0), dict(pitch=-300), dict(format=capi.PIXEL_FORMATS["bgra"], width=74, pitch=295),
           dict(format=capi.PIXEL_FORMATS["rgb"], width=100, pitch=299)]
    for kw in bad:
        assert _status(eng.submit_pose_interleaved_device, parser, [rec(), rec(**kw)]) == capi.HP_ERR_ARG, kw
    assert _status(eng.submit_pose_interleaved, parser, [np.zeros((20, 31, 2), np.uint8)], "uyvy") == capi.HP_ERR_ARG   # odd width
    assert _status(eng.submit_pose_interleaved, capi.PifPafParser(64, 96), [f], "yuyv") == capi.HP_ERR_UNSUPPORTED   # no OpenPifPaf heads
    # nothing was enqueued by the refusals: both tickets are free, the accepted forms run (gray and rgb of odd width are fine)
    t0 = eng.submit_pose_interleaved(parser, [f], "yuyv")
    t1 = eng.submit_pose_interleaved_device(parser, [rec(), rec(format=capi.PIXEL_FORMATS["gray"], width=299)])
    assert _status(eng.submit_pose_interleaved, parser, [f], "yuyv") == capi.HP_ERR_ARG      # a third batch in flight
    eng.collect_pose(t0); eng.collect_pose(t1)
    eng.close()
    ppn = capi.Engine(models.ppn_resnet18(0).to_pack(), (384, 384), max_batch_size=2)
    assert _status(ppn.submit_pose_interleaved, parser, [f], "yuyv") == capi.HP_ERR_UNSUPPORTED
    ppn.close(); parser.close()


@gpu
def test_capacity_growth_rerun():
    frames = _mixed(800, MIXED)
    N = len(frames)
    want_frames = _resized(frames, MIXED_FORMATS, H, W, False)
    eng = _tiny(N)
    d_conf, d_paf = _on_device(*syn.make_batch_tensors(12, N, (6, 10), eng.out_h, eng.out_w))
    eng.set_output_override(d_conf.data_ptr(), d_paf.data_ptr())
    big = capi.PafParser()
    big.set_capacity(peaks_per_part=1024, candidates_per_limb=1 << 15, humans=128)
    want = eng.collect_pose(eng.submit_pose(big, want_frames), cap=128)
    assert max(len(h) for h in want) > 1
    small = capi.PafParser()
    small.set_capacity(peaks_per_part=2, candidates_per_limb=2, humans=1)     # everything overflows: collect grows and reruns
    t = eng.submit_pose_interleaved(small, frames, MIXED_FORMATS)
    got = eng.collect_pose(t, cap=128)
    assert _same_humans(got, want)
    assert np.array_equal(eng.debug_read_slot_frames(t, N), want_frames)
    eng.set_output_override(0, 0)
    eng.close(); big.close(); small.close()
