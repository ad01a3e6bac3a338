"""The pipelined pose calls on rotated frames (hp_pose_submit{,_pifpaf,_ppn}_frames_{interleaved,yuv420}_rotated_host / _device):
cv::rotate fused into the batched resize's fetch after the conversion, bit-exact with cv::resize(cv::rotate(cv::cvtColor(src, code))).
The oracle is the upright call, already pinned, fed the frame rotated beforehand.

  1. every pinned source in every format and layout at every rotation, plain and letterboxed: the resized frames equal the upright call
     on the np.rot90'd frame (rotated in its planes for 4:2:0, converted to BGR for 4:2:2) and the cv2 sha they are pinned to;
  2. mixed batches (formats, sizes and rotations differ in every frame), from host and from device memory: resized frames, engine
     outputs and humans equal submit_pose_frames on the reference-rotated BGR frames, for a PAF, an OpenPifPaf and a PPN pack;
  3. pitched device surfaces rotated 90 and 270: an NVDEC-like NV12 surface (pitch 2048, 1088 rows) and a BGRA surface with its pitch
     rounded up to 256 bytes, each padding byte 255;
  4. two tickets in flight whose rotation, geometry and call change from batch to batch, with no recapture;
  5. a capacity-growth rerun in collect on a rotated batch;
  6. every bad rotation is HP_ERR_ARG and leaves the engine usable;
  7. a NULL or all-zero rotation gives the bytes of the upright entry points."""
import ctypes
import os

import numpy as np
import pytest

import oracle
from hyperpose_b200 import capi, models, synthetic as syn
from tests import rotated_ref
from tests.golden.make_golden import sha
from tests.golden.make_golden_interleaved import interleaved_frame
from tests.golden.make_golden_rotated import ALL_FORMATS, ROT_CASES, ROTATIONS, cases, rotated_frame
from tests.golden.make_golden_yuv import yuv_pack, yuv_planes
from tests.interleaved_ref import YUV422
from tests.test_pose_interleaved import _on_device, _quiet, _same_humans, _status, _surface, _tiny
from tests.yuv_ref import LAYOUTS

gpu = pytest.mark.gpu
H, W = 368, 656
# (format, stored size, rotation): every interleaved format once; rotated sizes that take the copy (656x368 at 90) and the exact-2x
# area path (1312x736 at 90) into 368x656, odd sizes, a portrait frame, 720p and 1080p
MIXED_INTERLEAVED = [("yuyv", (720, 1280), 90), ("bgra", (1080, 1920), 270), ("rgb", (H, W), 180), ("uyvy", (1312, 736), 90),
                     ("gray", (37, 53), 270), ("rgba", (656, 368), 90), ("yvyu", (480, 640), 0), ("bgr", (101, 80), 180)]
MIXED_YUV = [("nv12", (1080, 1920), 90), ("nv21", (720, 1280), 270), ("i420", (H, W), 180), ("yv12", (1312, 736), 90),
             ("nv12", (2, 4), 270), ("nv21", (480, 640), 0)]


def _source(seed, fmt, h, w):
    return yuv_pack(*yuv_planes(seed, h, w), fmt) if fmt in LAYOUTS else interleaved_frame(seed, h, w, fmt)


def _batch(seed, spec):
    """(frames, formats, rotations, reference-rotated BGR frames) of a mixed batch spec"""
    frames = [_source(seed + k, fmt, h, w) for k, (fmt, (h, w), _) in enumerate(spec)]
    fmts, rots = [s[0] for s in spec], [s[2] for s in spec]
    return frames, fmts, rots, [rotated_ref.to_bgr(f, fmt, r) for f, fmt, r in zip(frames, fmts, rots)]


def _submit(eng, parser, frames, fmts, keep, rotation=None):
    """the host call for the frames' kind (all YUV 4:2:0 or all interleaved)"""
    if fmts[0] in LAYOUTS:
        return eng.submit_pose_yuv420(parser, frames, fmts, keep_ratio=keep, rotation=rotation)
    return eng.submit_pose_interleaved(parser, frames, fmts, keep_ratio=keep, rotation=rotation)


def _device_records(frames, fmts):
    """(device tensors, records) of host frames copied to device memory with packed rows"""
    d = _on_device(*frames)
    recs = []
    for t, f, fmt in zip(d, frames, fmts):
        p = t.data_ptr()
        if fmt in LAYOUTS:
            h, w = f.shape[0] * 2 // 3, f.shape[1]
            u, v, pitch_uv, step = capi.YUV420_LAYOUTS[fmt](h, w)
            recs.append(capi.FrameYUV420(p, p + u, p + v, h, w, w, pitch_uv, step))
        else:
            recs.append(capi.FrameInterleaved(p, f.shape[0], f.shape[1], f.strides[0], capi.PIXEL_FORMATS[fmt]))
    return d, recs


def _submit_device(eng, parser, recs, keep, rotation):
    if isinstance(recs[0], capi.FrameYUV420):
        return eng.submit_pose_yuv420_device(parser, recs, keep_ratio=keep, rotation=rotation)
    return eng.submit_pose_interleaved_device(parser, recs, keep_ratio=keep, rotation=rotation)


def _upright(frame, fmt, deg):
    """(frame, format) for the upright call that equals `frame` in `fmt` rotated by `deg`: the same format rotated as an image, 4:2:0
    rotated in its planes, 4:2:2 (whose pixel pairs do not survive a quarter turn) as the reference-converted BGR frame"""
    if fmt in LAYOUTS:
        return rotated_ref.rotate_yuv420(frame, fmt, deg), fmt
    if fmt in YUV422:
        return rotated_ref.to_bgr(frame, fmt, deg), "bgr"
    return rotated_ref.rotate(frame, deg), fmt


def _run(eng, submit, n, cap=128):
    t = submit()
    humans = eng.collect_pose(t, cap=cap)
    return eng.debug_read_slot_frames(t, n), humans


@gpu
@pytest.mark.parametrize("fmt", ALL_FORMATS)
def test_every_pinned_case(golden_dir, fmt):
    pin = np.load(os.path.join(golden_dir, "cv_pin_rotated.npz"))
    by_dst = {}
    for i in cases(fmt):
        by_dst.setdefault(tuple(ROT_CASES[i][2:]), []).append(i)
    for (dh, dw), idx in by_dst.items():
        jobs = [(i, deg) for i in idx for deg in ROTATIONS]
        src = {i: rotated_frame(i, fmt) for i in idx}
        frames, rots = [src[i] for i, _ in jobs], [deg for _, deg in jobs]
        upright = [_upright(src[i], fmt, deg) for i, deg in jobs]
        eng = _tiny(len(jobs), dh, dw)
        parser = _quiet()
        for keep in (False, True):
            got, _ = _run(eng, lambda: _submit(eng, parser, frames, [fmt] * len(jobs), keep, rotation=rots), len(jobs))
            want, _ = _run(eng, lambda: _submit(eng, parser, [u[0] for u in upright], [u[1] for u in upright], keep), len(jobs))
            for k, (i, deg) in enumerate(jobs):
                what = f"case {i} {fmt} {ROT_CASES[i][:2]} rotated {deg} -> {dh}x{dw} keep_ratio={keep}"
                assert np.array_equal(got[k], want[k]), f"{what}: {int((got[k] != want[k]).sum())} bytes differ from the upright call"
                assert sha(got[k]) == str(pin[f"{fmt}{i}_r{deg}_{'lb' if keep else 'rz'}_sha"]), what
        eng.close(); parser.close()


def _compare_heads(eng, quiet, parser, seed, keep, override, cap=128):
    """for both mixed batches, from host and from device memory: resized frames and engine outputs (quiet parser, no override), then
    humans over `override` (parser), against submit_pose_frames on the reference-rotated BGR frames"""
    for spec in (MIXED_INTERLEAVED, MIXED_YUV):
        frames, fmts, rots, bgr = _batch(seed, spec)
        N = len(frames)
        want_frames, _ = _run(eng, lambda: eng.submit_pose_frames(quiet, bgr, keep_ratio=keep), N, cap)
        assert np.array_equal(want_frames, np.stack([oracle.resize_linear_u8(b, eng.in_h, eng.in_w, letterbox=keep) for b in bgr]))
        want_outs = eng.read_outputs(N)
        d, recs = _device_records(frames, fmts)
        runs = {"host": lambda p: _submit(eng, p, frames, fmts, keep, rotation=rots),
                "device": lambda p: _submit_device(eng, p, recs, keep, rots)}
        for where, submit in runs.items():
            got, _ = _run(eng, lambda: submit(quiet), N, cap)
            assert np.array_equal(got, want_frames), f"{fmts[0]} batch from {where} memory, keep_ratio={keep}"
            assert all(a.tobytes() == b.tobytes() for a, b in zip(eng.read_outputs(N), want_outs)), where
        eng.set_output_override(override[0].data_ptr(), override[1].data_ptr())
        want = eng.collect_pose(eng.submit_pose_frames(parser, bgr, keep_ratio=keep), cap=cap)
        assert sum(len(h) for h in want) >= N, "vacuous: no humans over the override"
        for where, submit in runs.items():
            assert _same_humans(eng.collect_pose(submit(parser), cap=cap), want), where
        eng.set_output_override(0, 0)
        del d


@gpu
@pytest.mark.parametrize("keep", [False, True])
def test_mixed_batch_paf(keep):
    N = len(MIXED_INTERLEAVED)
    eng = _tiny(N)
    quiet, parser = _quiet(), capi.PafParser()
    override = _on_device(*syn.make_batch_tensors(21, N, (4, 8), eng.out_h, eng.out_w))
    _compare_heads(eng, quiet, parser, 300, keep, override)
    eng.close(); parser.close(); quiet.close()


@gpu
def test_mixed_batch_pifpaf():
    PH = PW = 385
    N = len(MIXED_INTERLEAVED)
    eng = capi.Engine(models.resnet50_pifpaf(0).to_pack(), (PW, PH), max_batch_size=N)
    dec = capi.PifPafParser(PH, PW, 0.1)
    fl = [syn.make_pifpaf_fields(610 + i, (2, 6), eng.out_h, eng.out_w) for i in range(N)]
    override = _on_device(np.stack([f[0] for f in fl]).reshape(N, 85, eng.out_h, eng.out_w),
                          np.stack([f[1] for f in fl]).reshape(N, 171, eng.out_h, eng.out_w))
    for keep in (False, True):
        _compare_heads(eng, dec, dec, 500, keep, override)
    eng.close(); dec.close()


@gpu
def test_mixed_batch_ppn():
    PH = PW = 384
    N = len(MIXED_INTERLEAVED)
    K, GH, GW, E, NH, NW = 18, 12, 12, 17, 9, 9
    eng = capi.Engine(models.ppn_resnet18(0).to_pack(), (PW, PH), max_batch_size=N)
    parser = capi.PoseProposalParser((PW, PH))
    ts = [syn.make_ppn_tensors(3400 + i, (4, 8)) for i in range(N)]
    box = np.stack([np.stack(t[:6]) for t in ts]).reshape(N, 6 * K, GH, GW).astype(np.float32)
    edge = np.stack([t[6] for t in ts]).reshape(N, E * NH * NW, GH, GW).astype(np.float32)
    override = _on_device(box, edge)
    for keep in (False, True):
        _compare_heads(eng, parser, parser, 700, keep, override, cap=512)
    eng.close(); parser.close()


@gpu
@pytest.mark.parametrize("keep", [False, True])
def test_pitched_device_surfaces(keep):
    """a 1080p NV12 frame in an NVDEC-like surface (pitch 2048, 1088 luma rows, the UV plane after them) and a 720 x 1000 BGRA frame
    with a 4096-byte pitch, each padding byte 255 (a read of the padding shows in the frame), rotated 90 and 270"""
    eng = _tiny(2)
    parser = _quiet()
    Y, U, V = yuv_planes(71, 1080, 1920)
    surf = np.full((1088 + 544, 2048), 255, np.uint8)
    surf[:1080, :1920] = Y
    surf[1088:1088 + 540, :1920] = np.stack([U, V], -1).reshape(540, 1920)
    bgra = interleaved_frame(72, 720, 1000, "bgra")
    d_nv12, d_bgra = _on_device(surf, _surface(bgra, 4096))
    p = d_nv12.data_ptr()
    nv12 = capi.FrameYUV420(p, p + 1088 * 2048, p + 1088 * 2048 + 1, 1080, 1920, 2048, 2048, 2)
    bgra_rec = capi.FrameInterleaved(d_bgra.data_ptr(), 720, 1000, 4096, capi.PIXEL_FORMATS["bgra"])
    packed = yuv_pack(Y, U, V, "nv12")
    for rec, src, fmt in ((nv12, packed, "nv12"), (bgra_rec, bgra, "bgra")):
        want = np.stack([oracle.resize_linear_u8(rotated_ref.to_bgr(src, fmt, deg), H, W, letterbox=keep) for deg in (90, 270)])
        got, _ = _run(eng, lambda: _submit_device(eng, parser, [rec, rec], keep, [90, 270]), 2)
        assert np.array_equal(got, want), f"{fmt}: {int((got != want).sum())} bytes differ"
    eng.close(); parser.close()


@gpu
def test_changing_rotation_and_geometry_in_flight():
    import torch
    N = 3
    # (kind, stored size, keep_ratio, page-locked, rotations) of consecutive batches, two in flight; the formats differ in a batch
    plan = [("yuv", (360, 640), False, False, [90, 0, 270]), ("int", (360, 640), True, True, [180, 90, 90]),
            ("yuv", (1080, 1920), True, True, [270, 270, 180]), ("int", (720, 1280), False, False, [0, 270, 90]),
            ("int", (38, 54), True, False, [90, 180, 270])]
    batches = []
    for b, (kind, (h, w), keep, pinned, rots) in enumerate(plan):
        fmts = ["nv12", "i420", "nv21"] if kind == "yuv" else ["yuyv", "bgra", "gray"]
        frames = [_source(400 + 10 * b + k, fmts[k], h + 2 * k, w - 2 * k) for k in range(N)]   # sizes differ in a batch too
        if pinned:
            frames = [torch.from_numpy(f).pin_memory().numpy() for f in frames]
        bgr = [rotated_ref.to_bgr(f, fmt, r) for f, fmt, r in zip(frames, fmts, rots)]
        batches.append((frames, fmts, keep, rots, np.stack([oracle.resize_linear_u8(x, H, W, letterbox=keep) for x in bgr])))
    eng = _tiny(N)
    eng.infer_u8(batches[0][4])
    conf, paf = eng.read_outputs(N)
    parser = capi.PafParser(float(np.quantile(conf[:, :18], 0.995)), float(np.quantile(paf, 0.5)))
    parser.set_capacity(peaks_per_part=4096, candidates_per_limb=1 << 15, humans=128)
    got, slot_frames = [None] * len(plan), [None] * len(plan)
    tickets, captures = [], None
    for b, (frames, fmts, keep, rots, _) in enumerate(batches):
        tickets.append(_submit(eng, parser, frames, fmts, keep, rotation=rots))
        if b == 1:
            captures = eng.pose_stats()["graph_captures"]
            assert 1 <= captures <= 2
        if len(tickets) == 2:
            slot_frames[b - 1] = eng.debug_read_slot_frames(tickets[0], N)
            got[b - 1] = eng.collect_pose(tickets.pop(0), cap=128)
    slot_frames[-1] = eng.debug_read_slot_frames(tickets[0], N)
    got[-1] = eng.collect_pose(tickets.pop(0), cap=128)
    assert eng.pose_stats()["graph_captures"] == captures, "a new rotation or frame geometry recaptured the graph"
    n_peaks = 0
    for b, (*_, want_frames) in enumerate(batches):
        assert np.array_equal(slot_frames[b], want_frames), f"batch {b}"
        assert _same_humans(got[b], eng.run_pose(parser, want_frames, cap=128)), f"batch {b}"
        n_peaks += sum(len(parser.debug_peaks(f)) for f in range(N))
    assert n_peaks > 50, "vacuous: no peaks at these thresholds"
    eng.close(); parser.close()


@gpu
def test_capacity_growth_rerun():
    frames, fmts, rots, bgr = _batch(800, MIXED_INTERLEAVED)
    N = len(frames)
    want_frames = np.stack([oracle.resize_linear_u8(b, H, W) for b in bgr])
    eng = _tiny(N)
    d_conf, d_paf = _on_device(*syn.make_batch_tensors(13, N, (6, 10), eng.out_h, eng.out_w))
    eng.set_output_override(d_conf.data_ptr(), d_paf.data_ptr())
    big = capi.PafParser()
    big.set_capacity(peaks_per_part=1024, candidates_per_limb=1 << 15, humans=128)
    want = eng.collect_pose(eng.submit_pose(big, want_frames), cap=128)
    assert max(len(h) for h in want) > 1
    small = capi.PafParser()
    small.set_capacity(peaks_per_part=2, candidates_per_limb=2, humans=1)     # everything overflows: collect grows and reruns
    t = eng.submit_pose_interleaved(small, frames, fmts, rotation=rots)
    assert _same_humans(eng.collect_pose(t, cap=128), want)
    assert np.array_equal(eng.debug_read_slot_frames(t, N), want_frames)
    eng.set_output_override(0, 0)
    eng.close(); big.close(); small.close()


@gpu
def test_refusals():
    eng = _tiny(2, 64, 96)
    parser = _quiet()
    yuyv = interleaved_frame(1, 90, 150, "yuyv")
    nv12 = _source(2, "nv12", 90, 150)
    d, recs = _device_records([yuyv, nv12], ["yuyv", "nv12"])
    yuvs = [recs[1]] * 2
    # (table, fmt, device): host records of host frames, device records of device frames
    tables = [((capi.FrameInterleaved * 2)(*[capi.interleaved_record(yuyv, "yuyv")] * 2), "interleaved", False),
              ((capi.FrameYUV420 * 2)(*[capi.yuv420_record(nv12, "nv12")] * 2), "yuv420", False),
              ((capi.FrameInterleaved * 2)(*[recs[0]] * 2), "interleaved", True), ((capi.FrameYUV420 * 2)(*yuvs), "yuv420", True)]
    for bad in ([0, 45], [-90, 0], [90, 360], [1, 0], [0, 91], [-2 ** 31, 0], [0, 2 ** 31 - 1], [450, 90], [-270, 0]):
        for table, fmt, device in tables:
            rot = (ctypes.c_int32 * 2)(*bad)
            assert _status(eng._submit_frame_table, parser, table, False, device, fmt, rotation=rot) == capi.HP_ERR_ARG, (bad, fmt, device)
    # the existing refusals stand with a rotation: 4:2:2 of odd width, 4:2:0 of odd size
    assert _status(eng.submit_pose_interleaved, parser, [np.zeros((20, 31, 2), np.uint8)], "uyvy", rotation=90) == capi.HP_ERR_ARG
    assert _status(eng.submit_pose_yuv420, parser, [np.zeros((30, 31), np.uint8)], "nv12", rotation=270) == capi.HP_ERR_ARG
    assert _status(eng.submit_pose_interleaved, parser, [yuyv] * 3, "yuyv", rotation=90) == capi.HP_ERR_BATCH
    # nothing was enqueued by the refusals: both tickets are free and the accepted forms run
    t0 = eng.submit_pose_interleaved(parser, [yuyv], "yuyv", rotation=[270])
    t1 = eng.submit_pose_yuv420_device(parser, yuvs, rotation=[90, 180])
    assert _status(eng.submit_pose_interleaved, parser, [yuyv], "yuyv", rotation=90) == capi.HP_ERR_ARG   # a third batch in flight
    eng.collect_pose(t0); eng.collect_pose(t1)
    want = np.stack([oracle.resize_linear_u8(rotated_ref.to_bgr(nv12, "nv12", r), 64, 96) for r in (90, 180)])
    assert np.array_equal(eng.debug_read_slot_frames(t1, 2), want)
    eng.close(); parser.close()


@gpu
@pytest.mark.parametrize("spec", ["interleaved", "yuv"])
def test_upright_rotation_is_the_upright_call(spec):
    """rotation NULL (through the library), 0 for the batch and all zero per frame: the bytes and outputs of the upright entry point"""
    frames, fmts, _, _ = _batch(900, MIXED_INTERLEAVED if spec == "interleaved" else MIXED_YUV)
    N = len(frames)
    eng = _tiny(N)
    parser = _quiet()
    fmt = "yuv420" if fmts[0] in LAYOUTS else "interleaved"
    table = ((capi.FrameYUV420 if fmt == "yuv420" else capi.FrameInterleaved) * N)(
        *[capi.yuv420_record(f, x) if fmt == "yuv420" else capi.interleaved_record(f, x) for f, x in zip(frames, fmts)])

    def null_rotation():
        t = ctypes.c_int(-1)
        capi.check(getattr(capi.lib(), f"hp_pose_submit_frames_{fmt}_rotated_host")(eng._h, parser._h, table, None, N, 1, ctypes.byref(t)))
        eng._ticket_n[t.value] = N
        return t.value
    runs = [lambda: _submit(eng, parser, frames, fmts, True), null_rotation, lambda: _submit(eng, parser, frames, fmts, True, rotation=0),
            lambda: _submit(eng, parser, frames, fmts, True, rotation=[0] * N)]
    got = []
    for run in runs:
        fr, _ = _run(eng, run, N)
        got.append((fr, eng.read_outputs(N)))
    for fr, outs in got[1:]:
        assert np.array_equal(fr, got[0][0])
        assert all(a.tobytes() == b.tobytes() for a, b in zip(outs, got[0][1]))
    eng.close(); parser.close()
