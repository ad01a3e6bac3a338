"""The pipelined pose calls on frames of 16-bit samples (hp_pose_submit{,_pifpaf,_ppn}_frames_{yuv420_16,interleaved16}_host /
_device): each sample reduced as convertTo(CV_8U, 2^-(bits-8)) in the batched resize's fetch, then converted, rotated and resized as
the 8-bit calls do, bit-exact with cv::resize(cv::rotate(cv::cvtColor(convertTo(src16, CV_8U, 2^-(bits-8)), code))).

  1. every pinned source (every layout and format, bits 10, 12, 16, 640x360 to 1080p and 642x362, every rotation) from host and from
     device memory: the resized frames have the cv2 sha of the stretch and the letterbox into 368x656, and of the copy and exact-2x
     area regimes;
  2. mixed batches (layout or format, size, bits and rotation differ in every frame) from pageable, page-locked and device memory:
     resized frames, engine outputs and humans equal the 8-bit call (submit_pose_yuv420 / submit_pose_interleaved, same rotations) on
     the frames reduced on the host, for a PAF, an OpenPifPaf and a PPN pack; the frames equal the restatement;
  3. pitched device surfaces, every padding sample 0xffff: a 1080p P016 NVDEC-like surface, a BGRA64 surface and a torch slice of a
     larger RGB48 tensor, against the restatement;
  4. every argument the C ABI refuses is HP_ERR_ARG (N > max_batch HP_ERR_BATCH, the wrong head type HP_ERR_UNSUPPORTED) with
     nothing enqueued: the next two submits are accepted and give the right frames."""
import ctypes
import os

import numpy as np
import pytest

import oracle
from hyperpose_b200 import capi, models, synthetic as syn
from tests import highbit_ref
from tests.golden.make_golden import sha
from tests.golden.make_golden_highbit import HB_BITS, HB_SIZES, highbit_frame, key
from tests.golden.make_golden_rotated import ROTATIONS
from tests.highbit_ref import ALL16, FORMATS16, LAYOUTS16
from tests.test_pose_interleaved import _quiet, _same_humans, _status, _tiny

gpu = pytest.mark.gpu
H, W = 368, 656
# (layout or format, stored size, bits, rotation)
MIXED_INTERLEAVED16 = [("bgr48", (720, 1280), 10, 90), ("rgba64", (1080, 1920), 16, 270), ("gray16", (362, 642), 12, 0),
                       ("rgb48", (H, W), 16, 180), ("bgra64", (37, 53), 9, 90), ("gray16", (656, 368), 14, 90)]
MIXED_YUV16 = [("p016", (1080, 1920), 16, 90), ("p016_vu", (720, 1280), 10, 0), ("i420", (362, 642), 12, 270),
               ("yv12", (H, W), 16, 180), ("p016", (2, 4), 12, 90), ("i420", (480, 640), 10, 0)]


def _on_device(*arrays):
    """uint16 arrays as int16 CUDA tensors of the same bytes"""
    import torch
    d = [torch.from_numpy(np.ascontiguousarray(a).view(np.int16)).cuda() for a in arrays]
    torch.cuda.synchronize()
    return d


def _pinned(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int16)).pin_memory().numpy().view(np.uint16)


def _source(seed, fmt, h, w, bits):
    """a seeded uint16 source: (3H/2, W) packed 4:2:0, or an interleaved crop view with 0xffff after each row"""
    rng = np.random.default_rng(seed)
    hi = min(1 << 16, 5 << (bits - 2))
    if fmt in LAYOUTS16:
        return rng.integers(0, hi, (h * 3 // 2, w), dtype=np.uint16)
    ch = {"bgr48": 3, "rgb48": 3, "bgra64": 4, "rgba64": 4, "gray16": None}[fmt]
    buf = np.full((h, w + 5) if ch is None else (h, w + 5, ch), 0xffff, np.uint16)
    buf[:, :w] = rng.integers(0, hi, buf[:, :w].shape, dtype=np.uint16)
    return buf[:, :w]


def _submit(eng, parser, frames, fmts, bits, keep, rotation):
    if fmts[0] in LAYOUTS16:
        return eng.submit_pose_yuv420_16(parser, frames, fmts, bits, keep_ratio=keep, rotation=rotation)
    return eng.submit_pose_interleaved16(parser, frames, fmts, bits, keep_ratio=keep, rotation=rotation)


def _submit_device(eng, parser, recs, keep, rotation):
    if isinstance(recs[0], capi.FrameYUV420_16):
        return eng.submit_pose_yuv420_16_device(parser, recs, keep_ratio=keep, rotation=rotation)
    return eng.submit_pose_interleaved16_device(parser, recs, keep_ratio=keep, rotation=rotation)


def _submit8(eng, parser, frames, fmts, bits, keep, rotation):
    """the 8-bit call on the frames reduced on the host"""
    r8, f8 = [highbit_ref.reduce(f, b) for f, b in zip(frames, bits)], [ALL16[x] for x in fmts]
    if fmts[0] in LAYOUTS16:
        return eng.submit_pose_yuv420(parser, r8, f8, keep_ratio=keep, rotation=rotation)
    return eng.submit_pose_interleaved(parser, r8, f8, keep_ratio=keep, rotation=rotation)


def _records(frames, fmts, bits):
    """(device tensors, records) of host frames copied to device memory with packed rows"""
    d = _on_device(*frames)
    recs = []
    for t, f, fmt, b in zip(d, frames, fmts, bits):
        p = t.data_ptr()
        if fmt in LAYOUTS16:
            h, w = f.shape[0] * 2 // 3, f.shape[1]
            u, v, pitch_uv, step = capi.YUV420_LAYOUTS[LAYOUTS16[fmt]](h, w)
            recs.append(capi.FrameYUV420_16(p, p + 2 * u, p + 2 * v, h, w, 2 * w, 2 * pitch_uv, step, b))
        else:
            recs.append(capi.FrameInterleaved16(p, f.shape[0], f.shape[1], 2 * f[0].size, capi.PIXEL_FORMATS[FORMATS16[fmt]], b))
    return d, recs


def _run(eng, submit, n, cap=128):
    t = submit()
    humans = eng.collect_pose(t, cap=cap)
    return eng.debug_read_slot_frames(t, n), humans


def _want(frames, fmts, bits, rots, h, w, keep):
    return np.stack([oracle.resize_linear_u8(highbit_ref.to_bgr(f, x, b, r), h, w, letterbox=keep)
                     for f, x, b, r in zip(frames, fmts, bits, rots)])


@gpu
@pytest.mark.parametrize("fmt", list(ALL16))
def test_every_pinned_case(golden_dir, fmt):
    pin = np.load(os.path.join(golden_dir, "cv_pin_highbit.npz"))
    parser = _quiet()
    # stretch and letterbox into H x W: the four rotations of one source per batch, from host and from device memory
    eng = _tiny(len(ROTATIONS))
    for i in range(len(HB_SIZES)):
        for bits in HB_BITS:
            src = highbit_frame(fmt, i, bits)
            d, recs = _records([src], [fmt], [bits])
            n = len(ROTATIONS)
            runs = {"host": lambda keep: _submit(eng, parser, [src] * n, [fmt] * n, bits, keep, list(ROTATIONS)),
                    "device": lambda keep: _submit_device(eng, parser, recs * n, keep, list(ROTATIONS))}
            for where, submit in runs.items():
                for keep in (False, True):
                    got, _ = _run(eng, lambda: submit(keep), n)
                    for k, deg in enumerate(ROTATIONS):
                        what = f"{key(fmt, i, bits, deg)} {HB_SIZES[i]} from {where} keep_ratio={keep}"
                        assert sha(got[k]) == str(pin[f"{key(fmt, i, bits, deg)}_{'lb' if keep else 'rz'}_sha"]), what
            del d
    eng.close()
    # the copy regime (640x360 at its own rotated size) and the exact-2x area regime (1280x720 into it)
    for net, degs in (((360, 640), (0, 180)), ((640, 360), (90, 270))):
        jobs = [(i, bits, deg) for i in (0, 1) for bits in HB_BITS for deg in degs]
        eng = _tiny(len(jobs), *net)
        frames = [highbit_frame(fmt, i, bits) for i, bits, _ in jobs]
        bl, rots = [b for _, b, _ in jobs], [deg for *_, deg in jobs]
        d, recs = _records(frames, [fmt] * len(jobs), bl)
        for where, submit in (("host", lambda: _submit(eng, parser, frames, [fmt] * len(jobs), bl, False, rots)),
                              ("device", lambda: _submit_device(eng, parser, recs, False, rots))):
            got, _ = _run(eng, submit, len(jobs))
            for k, (i, bits, deg) in enumerate(jobs):
                regime = "cvt" if i == 0 else "a2"
                assert sha(got[k]) == str(pin[f"{key(fmt, i, bits, deg)}_{regime}_sha"]), f"{key(fmt, i, bits, deg)} {regime} {where}"
        del d
        eng.close()
    parser.close()


def _batch(seed, spec):
    frames = [_source(seed + k, fmt, h, w, b) for k, (fmt, (h, w), b, _) in enumerate(spec)]
    return frames, [s[0] for s in spec], [s[2] for s in spec], [s[3] for s in spec]


def _compare_heads(eng, quiet, parser, seed, keep, override, cap=128):
    """both mixed batches from pageable, page-locked and device memory: resized frames and engine outputs (quiet parser, no override),
    then humans over `override` (parser), against the 8-bit call on the frames reduced on the host"""
    for spec in (MIXED_INTERLEAVED16, MIXED_YUV16):
        frames, fmts, bits, rots = _batch(seed, spec)
        N = len(frames)
        want_frames, _ = _run(eng, lambda: _submit8(eng, quiet, frames, fmts, bits, keep, rots), N, cap)
        assert np.array_equal(want_frames, _want(frames, fmts, bits, rots, eng.in_h, eng.in_w, keep))
        want_outs = eng.read_outputs(N)
        d, recs = _records(frames, fmts, bits)
        pinned = [_pinned(f) for f in frames]
        runs = {"pageable": lambda p: _submit(eng, p, frames, fmts, bits, keep, rots),
                "page-locked": lambda p: _submit(eng, p, pinned, fmts, bits, keep, rots),
                "device": lambda p: _submit_device(eng, p, recs, keep, rots)}
        for where, submit in runs.items():
            got, _ = _run(eng, lambda: submit(quiet), N, cap)
            assert np.array_equal(got, want_frames), f"{fmts[0]} batch from {where} memory, keep_ratio={keep}: " \
                                                     f"{int((got != want_frames).sum())} bytes differ"
            assert all(a.tobytes() == b.tobytes() for a, b in zip(eng.read_outputs(N), want_outs)), where
        eng.set_output_override(override[0].data_ptr(), override[1].data_ptr())
        want = eng.collect_pose(_submit8(eng, parser, frames, fmts, bits, keep, rots), cap=cap)
        assert sum(len(h) for h in want) >= N, "vacuous: no humans over the override"
        for where, submit in runs.items():
            assert _same_humans(eng.collect_pose(submit(parser), cap=cap), want), where
        eng.set_output_override(0, 0)
        del d


def _float_on_device(*arrays):
    import torch
    d = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]
    torch.cuda.synchronize()
    return d


@gpu
@pytest.mark.parametrize("keep", [False, True])
def test_mixed_batch_paf(keep):
    N = len(MIXED_INTERLEAVED16)
    eng = _tiny(N)
    quiet, parser = _quiet(), capi.PafParser()
    override = _float_on_device(*syn.make_batch_tensors(23, N, (4, 8), eng.out_h, eng.out_w))
    _compare_heads(eng, quiet, parser, 300, keep, override)
    eng.close(); parser.close(); quiet.close()


@gpu
def test_mixed_batch_pifpaf():
    PH = PW = 385
    N = len(MIXED_INTERLEAVED16)
    eng = capi.Engine(models.resnet50_pifpaf(0).to_pack(), (PW, PH), max_batch_size=N)
    dec = capi.PifPafParser(PH, PW, 0.1)
    fl = [syn.make_pifpaf_fields(710 + i, (2, 6), eng.out_h, eng.out_w) for i in range(N)]
    override = _float_on_device(np.stack([f[0] for f in fl]).reshape(N, 85, eng.out_h, eng.out_w),
                                np.stack([f[1] for f in fl]).reshape(N, 171, eng.out_h, eng.out_w))
    for keep in (False, True):
        _compare_heads(eng, dec, dec, 500, keep, override)
    eng.close(); dec.close()


@gpu
def test_mixed_batch_ppn():
    PH = PW = 384
    N = len(MIXED_INTERLEAVED16)
    K, GH, GW, E, NH, NW = 18, 12, 12, 17, 9, 9
    eng = capi.Engine(models.ppn_resnet18(0).to_pack(), (PW, PH), max_batch_size=N)
    parser = capi.PoseProposalParser((PW, PH))
    ts = [syn.make_ppn_tensors(3500 + i, (4, 8)) for i in range(N)]
    box = np.stack([np.stack(t[:6]) for t in ts]).reshape(N, 6 * K, GH, GW).astype(np.float32)
    edge = np.stack([t[6] for t in ts]).reshape(N, E * NH * NW, GH, GW).astype(np.float32)
    override = _float_on_device(box, edge)
    for keep in (False, True):
        _compare_heads(eng, parser, parser, 700, keep, override, cap=512)
    eng.close(); parser.close()


@gpu
@pytest.mark.parametrize("keep", [False, True])
def test_pitched_device_surfaces(keep):
    """a 1080p P016 frame in an NVDEC-like surface (pitch 4096 bytes, 1088 luma rows, the UV plane after them), a 720 x 1000 BGRA64
    frame with an 8192-byte pitch, each padding sample 0xffff, and a crop of a larger RGB48 device tensor (a torch slice)"""
    import torch
    eng = _tiny(2)
    parser = _quiet()
    packed = _source(81, "p016", 1080, 1920, 16)
    surf = np.full((1088 + 544, 2048), 0xffff, np.uint16)
    surf[:1080, :1920] = packed[:1080]
    surf[1088:1088 + 540, :1920] = packed[1080:]
    bgra = _source(82, "bgra64", 720, 1000, 12)
    bgra_surf = np.full((720, 4096), 0xffff, np.uint16)
    bgra_surf[:, :4000] = bgra.reshape(720, 4000)
    big = _source(83, "rgb48", 500, 700, 10).copy()
    d_p016, d_bgra, d_big = _on_device(surf, bgra_surf, big)
    crop = d_big[40:40 + 400, 30:30 + 600]
    assert not crop.is_contiguous()
    p = d_p016.data_ptr()
    cases = [(capi.FrameYUV420_16(p, p + 1088 * 4096, p + 1088 * 4096 + 2, 1080, 1920, 4096, 4096, 2, 16), packed, "p016", 16),
             (capi.FrameInterleaved16(d_bgra.data_ptr(), 720, 1000, 4096 * 2, capi.PIXEL_FORMATS["bgra"], 12), bgra, "bgra64", 12),
             (capi.FrameInterleaved16(crop.data_ptr(), 400, 600, crop.stride(0) * 2, capi.PIXEL_FORMATS["rgb"], 10),
              big[40:440, 30:630], "rgb48", 10)]
    for rec, src, fmt, bits in cases:
        want = _want([src, src], [fmt] * 2, [bits] * 2, [90, 0], H, W, keep)
        got, _ = _run(eng, lambda: _submit_device(eng, parser, [rec, rec], keep, [90, 0]), 2)
        assert np.array_equal(got, want), f"{fmt}: {int((got != want).sum())} bytes differ"
    del d_p016, d_bgra, d_big, crop
    torch.cuda.synchronize()
    eng.close(); parser.close()


def _variant(rec, **kw):
    r = type(rec).from_buffer_copy(rec)
    for k, v in kw.items():
        setattr(r, k, v)
    return r


@gpu
def test_refusals():
    eng = _tiny(2, 64, 96)
    parser = _quiet()
    p016, rgb = _source(1, "p016", 90, 150, 10), np.ascontiguousarray(_source(2, "rgb48", 90, 150, 12))
    d, (drec_y, drec_i) = _records([p016, rgb], ["p016", "rgb48"], [10, 12])
    hrec_y, hrec_i = capi.yuv420_16_record(p016, "p016", 10), capi.interleaved16_record(rgb, "rgb48", 12)
    bad_yuv = [dict(bits=8), dict(bits=17), dict(bits=0), dict(bits=-16), dict(height=89), dict(width=149), dict(height=0),
               dict(pitch_y=298), dict(pitch_uv=298), dict(pitch_y=301), dict(pitch_uv=303), dict(uv_step=3), dict(uv_step=0)]
    bad_int = [dict(bits=8), dict(bits=17), dict(bits=1 << 20), dict(pitch=898), dict(pitch=901), dict(format=5), dict(format=6),
               dict(format=7), dict(format=8), dict(format=-1), dict(width=0), dict(data=None)]
    tables = []
    for rec, bads in ((hrec_y, bad_yuv), (drec_y, bad_yuv), (hrec_i, bad_int), (drec_i, bad_int)):
        device = rec is drec_y or rec is drec_i
        fmt = "yuv420_16" if isinstance(rec, capi.FrameYUV420_16) else "interleaved16"
        variants = [_variant(rec, **kw) for kw in bads]
        if fmt == "yuv420_16":
            variants += [_variant(rec, y=rec.y + 1), _variant(rec, u=rec.u + 1, v=rec.v + 1), _variant(rec, v=rec.u + 4),
                         _variant(rec, y=None)]   # misaligned, not one sample apart, null
        else:
            variants += [_variant(rec, data=rec.data + 1)]
        tables += [((type(rec) * 2)(rec, v), fmt, device, None) for v in variants]
        for rot in ([0, 45], [-90, 0], [90, 360], [0, 1]):
            tables.append(((type(rec) * 2)(rec, rec), fmt, device, (ctypes.c_int32 * 2)(*rot)))
    for table, fmt, device, rot in tables:
        assert _status(eng._submit_frame_table, parser, table, False, device, fmt, rotation=rot) == capi.HP_ERR_ARG, \
            (fmt, device, [getattr(r, f) for r in table for f, _ in r._fields_])
    for rec, fmt in ((hrec_y, "yuv420_16"), (drec_i, "interleaved16")):
        assert _status(eng._submit_frame_table, parser, (type(rec) * 3)(rec, rec, rec), False, rec is drec_i, fmt) == capi.HP_ERR_BATCH
    ppn, dec = capi.PoseProposalParser((384, 384)), capi.PifPafParser(385, 385, 0.1)
    for head in (ppn, dec):
        assert _status(eng.submit_pose_yuv420_16, head, [p016], "p016", 10) == capi.HP_ERR_UNSUPPORTED
        assert _status(eng.submit_pose_interleaved16_device, head, [drec_i]) == capi.HP_ERR_UNSUPPORTED
    # nothing was enqueued: both tickets are free and the accepted forms give the right frames
    t0 = eng.submit_pose_yuv420_16(parser, [p016], "p016", 10, rotation=90)
    t1 = eng.submit_pose_interleaved16_device(parser, [drec_i, drec_i], rotation=[270, 0])
    assert _status(eng.submit_pose_yuv420_16, parser, [p016], "p016", 10) == capi.HP_ERR_ARG   # a third batch in flight
    eng.collect_pose(t0); eng.collect_pose(t1)
    assert np.array_equal(eng.debug_read_slot_frames(t0, 1), _want([p016], ["p016"], [10], [90], 64, 96, False))
    assert np.array_equal(eng.debug_read_slot_frames(t1, 2), _want([rgb] * 2, ["rgb48"] * 2, [12] * 2, [270, 0], 64, 96, False))
    del d
    eng.close(); parser.close(); ppn.close(); dec.close()
