"""The pipelined pose calls on frames of any size (hp_pose_submit_frames_u8_host / _device and their OpenPifPaf forms): one batched
resize kernel on the engine stream ahead of the captured graph, bit-exact with cv::resize / non_scaling_resize.

  1. every make_golden.RESIZE_CASES source, plain and letterboxed, through submit_pose_frames: the resized frames equal the oracle
     and the cv2 sha it is pinned to;
  2. a mixed batch (720p, 1080p, network size, the exact-2x path, an upscale, a portrait frame): resized frames, engine outputs and
     humans equal the network-size calls on the oracle-resized frames;
  3. two tickets in flight with a different geometry and keep_ratio in every batch, the source buffers growing, host frames pageable
     and page-locked: every result is right and no batch recaptures the graph;
  4. the mixed batch from device memory;
  5. OpenPifPaf: fields and humans equal submit_pose on the oracle-resized frames;
  6. the refusals;
  7. a batch that overflows the PAF parser's capacities: the rerun in collect reuses the resized frames.
The CPU test checks that the wrapper refuses frames that are not uint8 HWC3 before the library is called."""
import os

import numpy as np
import pytest

import oracle
from hyperpose_b200 import capi, models, synthetic as syn
from tests.golden.make_golden import RESIZE_CASES, sha

gpu = pytest.mark.gpu
H, W = 368, 656
# the cameras' and the reference examples' frame sizes, the network size, the exact-2x area path, an upscale and a portrait frame
MIXED = [(720, 1280), (1080, 1920), (H, W), (736, 1312), (37, 53), (640, 360)]


def _src(seed, h, w):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def _resized(frames, h, w, keep):
    return np.stack([oracle.resize_linear_u8(f, h, w, letterbox=keep) for f in frames])


def _tiny(max_batch, h=H, w=W):
    return capi.Engine(models.tiny_test_net(0).to_pack(), (w, h), max_batch_size=max_batch)


def _thresholds(eng, frames):
    """thresholds that keep a parse of random-weight 46 x 82 maps a few peaks per part deep"""
    eng.infer_u8(frames)
    conf, paf = eng.read_outputs(frames.shape[0])
    return float(np.quantile(conf[:, :18], 0.995)), float(np.quantile(paf, 0.5))


def _quiet():
    """a parser that finds no peak: random-weight maps at the default thresholds hold more than the parser's capacity limits"""
    return capi.PafParser(1e30, 1e30)


def _same_humans(a, b):
    return len(a) == len(b) and all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


@gpu
def test_every_pinned_case(golden_dir):
    pin = np.load(os.path.join(golden_dir, "cv_pin.npz"))
    by_dst = {}
    for i, (_, _, dh, dw) in enumerate(RESIZE_CASES):
        by_dst.setdefault((dh, dw), []).append(i)
    for (dh, dw), idx in by_dst.items():
        eng = _tiny(len(idx), dh, dw)
        parser = _quiet()
        imgs = [_src(200 + i, *RESIZE_CASES[i][:2]) for i in idx]
        for keep in (False, True):
            t = eng.submit_pose_frames(parser, imgs, keep_ratio=keep)
            got = eng.debug_read_slot_frames(t, len(idx))
            eng.collect_pose(t)
            for k, i in enumerate(idx):
                want = oracle.resize_linear_u8(imgs[k], dh, dw, letterbox=keep)
                assert np.array_equal(got[k], want), f"case {i} {imgs[k].shape[:2]} -> {dh}x{dw} keep_ratio={keep}: max |diff| " \
                                                     f"{np.abs(got[k].astype(int) - want.astype(int)).max()}"
                assert sha(got[k]) == str(pin[f"{'lb' if keep else 'rz'}{i}_sha"])
        eng.close(); parser.close()


@gpu
@pytest.mark.parametrize("keep", [False, True])
def test_mixed_batch(keep):
    import torch
    imgs = [_src(300 + k, h, w) for k, (h, w) in enumerate(MIXED)]
    want_frames = _resized(imgs, H, W, keep)
    N = len(imgs)
    eng = _tiny(N)
    quiet = _quiet()
    # resized frames and engine outputs, one batch in flight
    t = eng.submit_pose_frames(quiet, imgs, keep_ratio=keep)
    eng.collect_pose(t)
    assert np.array_equal(eng.debug_read_slot_frames(t, N), want_frames)
    conf, paf = eng.read_outputs(N)
    eng.infer_u8(want_frames)
    conf2, paf2 = eng.read_outputs(N)
    assert conf.tobytes() == conf2.tobytes() and paf.tobytes() == paf2.tobytes()
    # humans over crowd maps
    cc, pp = syn.make_batch_tensors(11, N, (4, 8), eng.out_h, eng.out_w)
    d_conf, d_paf = torch.from_numpy(cc).cuda(), torch.from_numpy(pp).cuda()
    torch.cuda.synchronize()
    eng.set_output_override(d_conf.data_ptr(), d_paf.data_ptr())
    parser = capi.PafParser()
    got = eng.collect_pose(eng.submit_pose_frames(parser, imgs, keep_ratio=keep))
    want = eng.run_pose(parser, want_frames)
    assert sum(len(h) for h in want) >= N, "vacuous: no humans in the crowd maps"
    assert _same_humans(got, want)
    eng.set_output_override(0, 0)
    eng.close(); parser.close(); quiet.close()


@gpu
def test_changing_geometry_in_flight():
    import torch
    N = 3
    # (size, keep_ratio, page-locked) of consecutive batches; each slot's source buffer grows on its second batch
    plan = [((360, 640), False, False), ((360, 640), True, True), ((1080, 1920), False, False), ((720, 1280), True, True),
            ((37, 53), False, False)]
    batches = []
    for b, ((h, w), keep, pinned) in enumerate(plan):
        imgs = [_src(400 + 10 * b + k, h + k, w - 2 * k) for k in range(N)]   # sizes differ inside a batch too
        if pinned:
            imgs = [torch.from_numpy(f).pin_memory().numpy() for f in imgs]
        batches.append((imgs, keep, _resized(imgs, H, W, keep)))
    eng = _tiny(N)
    ct, pt = _thresholds(eng, batches[0][2])
    parser = capi.PafParser(ct, pt)
    parser.set_capacity(peaks_per_part=1024, candidates_per_limb=1 << 15, humans=128)
    got, frames = [None] * len(plan), [None] * len(plan)
    tickets = []
    captures = None
    for b, (imgs, keep, _) in enumerate(batches):
        tickets.append(eng.submit_pose_frames(parser, imgs, keep_ratio=keep))
        if b == 1:
            captures = eng.pose_stats()["graph_captures"]
            assert 1 <= captures <= 2
        if len(tickets) == 2:
            k = b - 1
            frames[k] = eng.debug_read_slot_frames(tickets[0], N)
            got[k] = eng.collect_pose(tickets.pop(0), cap=128)
    frames[-1] = eng.debug_read_slot_frames(tickets[0], N)
    got[-1] = eng.collect_pose(tickets.pop(0), cap=128)
    assert eng.pose_stats()["graph_captures"] == captures, "a new frame geometry recaptured the graph"
    n_humans = n_peaks = 0
    for b, (imgs, keep, want_frames) in enumerate(batches):
        assert np.array_equal(frames[b], want_frames), f"batch {b}"
        want = eng.run_pose(parser, want_frames, cap=128)
        assert _same_humans(got[b], want), f"batch {b}"
        n_humans += sum(len(h) for h in want)
        n_peaks += sum(len(parser.debug_peaks(f)) for f in range(N))
    print(f"[frames] over {len(plan)} batches: {n_peaks} peaks, {n_humans} humans")
    assert n_peaks > 50, "vacuous: no peaks at these thresholds"
    eng.close(); parser.close()


@gpu
@pytest.mark.parametrize("keep", [False, True])
def test_device_frames(keep):
    import torch
    imgs = [_src(300 + k, h, w) for k, (h, w) in enumerate(MIXED)]
    want_frames = _resized(imgs, H, W, keep)
    N = len(imgs)
    eng = _tiny(N)
    parser = _quiet()
    d_imgs = [torch.from_numpy(f).cuda() for f in imgs]
    torch.cuda.synchronize()
    t = eng.submit_pose_frames_device(parser, [(d.data_ptr(), d.shape[0], d.shape[1]) for d in d_imgs], keep_ratio=keep)
    eng.collect_pose(t)
    assert np.array_equal(eng.debug_read_slot_frames(t, N), want_frames)
    conf, paf = eng.read_outputs(N)
    eng.infer_u8(want_frames)
    conf2, paf2 = eng.read_outputs(N)
    assert conf.tobytes() == conf2.tobytes() and paf.tobytes() == paf2.tobytes()
    eng.close(); parser.close()


@gpu
def test_pifpaf():
    import torch
    PH = PW = 385
    sizes = [(720, 1280), (PH, PW), (1080, 1920), (640, 360)]
    imgs = [_src(500 + k, h, w) for k, (h, w) in enumerate(sizes)]
    N = len(imgs)
    eng = capi.Engine(models.resnet50_pifpaf(0).to_pack(), (PW, PH), max_batch_size=N)
    dec = capi.PifPafParser(PH, PW, 0.1)
    for keep in (False, True):
        want_frames = _resized(imgs, PH, PW, keep)
        t = eng.submit_pose_frames(dec, imgs, keep_ratio=keep)
        eng.collect_pose(t)
        assert np.array_equal(eng.debug_read_slot_frames(t, N), want_frames)
        fields = eng.read_outputs(N)
        eng.collect_pose(eng.submit_pose(dec, want_frames))
        want_fields = eng.read_outputs(N)
        assert all(a.tobytes() == b.tobytes() for a, b in zip(fields, want_fields)), f"keep_ratio={keep}"
    # humans over synthetic fields (random weights give fields without people)
    fl = [syn.make_pifpaf_fields(600 + i, (2, 6), eng.out_h, eng.out_w) for i in range(N)]
    pif = np.stack([f[0] for f in fl]).reshape(N, 85, eng.out_h, eng.out_w)
    paf = np.stack([f[1] for f in fl]).reshape(N, 171, eng.out_h, eng.out_w)
    d_pif, d_paf = torch.from_numpy(pif).cuda(), torch.from_numpy(paf).cuda()
    torch.cuda.synchronize()
    eng.set_output_override(d_pif.data_ptr(), d_paf.data_ptr())
    got = eng.collect_pose(eng.submit_pose_frames(dec, imgs, keep_ratio=True))
    want = eng.collect_pose(eng.submit_pose(dec, _resized(imgs, PH, PW, True)))
    assert sum(len(h) for h in want) >= N, "vacuous: no humans in the synthetic fields"
    assert _same_humans(got, want)
    eng.set_output_override(0, 0)
    eng.close(); dec.close()


@gpu
def test_refusals():
    eng = _tiny(2, 64, 96)
    parser = _quiet()
    img = _src(1, 90, 150)

    def status(fn, *a, **k):
        with pytest.raises(capi.HyperposeError) as e:
            fn(*a, **k)
        return e.value.status

    assert status(eng.submit_pose_frames, parser, [img] * 3) == capi.HP_ERR_BATCH
    assert status(eng.submit_pose_frames_device, parser, [(0, 90, 150)]) == capi.HP_ERR_ARG
    assert status(eng.submit_pose_frames, parser, [img, np.zeros((0, 150, 3), np.uint8)]) == capi.HP_ERR_ARG
    assert status(eng.submit_pose_frames, parser, [img, np.zeros((90, 0, 3), np.uint8)]) == capi.HP_ERR_ARG
    assert status(eng.submit_pose_frames, capi.PifPafParser(64, 96), [img]) == capi.HP_ERR_UNSUPPORTED   # no OpenPifPaf heads
    t0 = eng.submit_pose_frames(parser, [img])
    t1 = eng.submit_pose_frames(parser, [img, img])
    assert status(eng.submit_pose_frames, parser, [img]) == capi.HP_ERR_ARG      # a third batch in flight
    eng.collect_pose(t0); eng.collect_pose(t1)
    eng.close()
    ppn = capi.Engine(models.ppn_resnet18(0).to_pack(), (384, 384), max_batch_size=2)
    assert status(ppn.submit_pose_frames, parser, [img]) == capi.HP_ERR_UNSUPPORTED
    ppn.close(); parser.close()


@gpu
def test_capacity_growth_rerun():
    import torch
    imgs = [_src(700 + k, h, w) for k, (h, w) in enumerate(MIXED)]
    N = len(imgs)
    want_frames = _resized(imgs, H, W, False)
    eng = _tiny(N)
    cc, pp = syn.make_batch_tensors(12, N, (6, 10), eng.out_h, eng.out_w)
    d_conf, d_paf = torch.from_numpy(cc).cuda(), torch.from_numpy(pp).cuda()
    torch.cuda.synchronize()
    eng.set_output_override(d_conf.data_ptr(), d_paf.data_ptr())
    big = capi.PafParser()
    big.set_capacity(peaks_per_part=1024, candidates_per_limb=1 << 15, humans=128)
    want = eng.collect_pose(eng.submit_pose(big, want_frames), cap=128)
    assert max(len(h) for h in want) > 1
    small = capi.PafParser()
    small.set_capacity(peaks_per_part=2, candidates_per_limb=2, humans=1)     # everything overflows: collect grows and reruns
    got = eng.collect_pose(eng.submit_pose_frames(small, imgs), cap=128)
    assert _same_humans(got, want)
    eng.set_output_override(0, 0)
    eng.close(); big.close(); small.close()


def test_wrapper_rejects_frames_that_are_not_u8_hwc3(monkeypatch):
    def no_library():
        raise AssertionError("the library was called")
    monkeypatch.setattr(capi, "lib", no_library)
    eng = object.__new__(capi.Engine)
    good = np.zeros((4, 6, 3), np.uint8)
    for bad in (np.zeros((4, 6, 3), np.float32), np.zeros((4, 6), np.uint8), np.zeros((4, 6, 4), np.uint8),
                np.zeros((1, 4, 6, 3), np.uint8), [[1, 2, 3]]):
        with pytest.raises(capi.HyperposeError) as e:
            eng.submit_pose_frames(capi.PafParser.__new__(capi.PafParser), [good, bad])
        assert e.value.status == capi.HP_ERR_ARG
