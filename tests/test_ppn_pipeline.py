"""The pipelined pose calls for Pose Proposal Network packs (hp_pose_submit_ppn_u8_host / _device, hp_pose_submit_ppn_frames_u8_host /
_device, results by hp_pose_collect): the network, the PPN parse of its outputs in place and the record D2H replayed from one CUDA
graph per ticket, two batches in flight.

The yardstick everywhere is the two-call path on the same frames, parser thresholds and engine: hp_engine_infer_u8_* on the engine
stream, hp_ppn_process_device_strided on the engine's outputs on the same stream, hp_ppn_fetch, retried on HP_ERR_CAPACITY the way
hp_ppn_process_host retries.  Records are compared byte for byte.

  1. ppn_resnet18 / ppn_resnet50, f16 / TF32, at 384 x 384: a full batch of 16 and 5 frames in an engine built for 8, over synthetic
     crowd tensors (output override) and over the network's own outputs (quantile thresholds);
  2. two tickets in flight with different N, override tensors and thresholds: one capture per slot per key, a recapture exactly when
     a threshold or N changes, every other submit a replay;
  3. camera-size frames from pageable, page-locked and device memory, with and without keep_ratio;
  4. capacity growth in collect with the other ticket in flight: the spill variant (the ppn_dense golden case) and the record
     capacity (144 humans in one frame, more than the 128 records a frame starts with);
  5. the refusals;
  6. hp_engine_launch_count + the parser's count advance alike per replayed and per direct batch.
The CPU test checks that the Python wrapper dispatches a PoseProposalParser to the PPN entry points."""
import ctypes as C
import functools

import numpy as np
import pytest

import oracle
from hyperpose_b200 import capi, models, synthetic as syn
from tests.golden.make_golden import PPN_CASES

gpu = pytest.mark.gpu
H = W = 384
K, GH, GW, E, NH, NW = 18, 12, 12, 17, 9, 9
CAP = 512
DEFAULT_THR = (0.10, 0.05, 0.3)
# camera and video sizes, the network size, the exact-2x area path, an upscale and a portrait frame
MIXED = [(720, 1280), (1080, 1920), (H, W), (2 * H, 2 * W), (37, 53), (640, 360)]


@functools.lru_cache(maxsize=None)
def _pack(net):
    return getattr(models, net)(0).to_pack()


def _engine(net="ppn_resnet18", max_batch=8, dtype="f16"):
    return capi.Engine(_pack(net), (W, H), max_batch_size=max_batch, dtype=dtype)


def _crowd(seed, N, persons=(4, 8)):
    """N frames of synthetic crowd tensors in the engine's output layout: box [N,6K,gh,gw], edge [N,E*nh*nw,gh,gw]"""
    ts = [syn.make_ppn_tensors(seed + i, persons) for i in range(N)]
    return _stack(ts)


def _stack(ts):
    N = len(ts)
    box = np.ascontiguousarray(np.stack([np.stack(t[:6]) for t in ts]).reshape(N, 6 * K, GH, GW), np.float32)
    edge = np.ascontiguousarray(np.stack([t[6] for t in ts]).reshape(N, E * NH * NW, GH, GW), np.float32)
    return box, edge


def _on_device(box, edge):
    import torch
    d = torch.from_numpy(box).cuda(), torch.from_numpy(edge).cuda()
    torch.cuda.synchronize()
    return d


def _host_parse(box, edge, thr, cap=CAP):
    """hp_ppn_process_host on the tensors the override copies over the engine's outputs"""
    N = box.shape[0]
    b = box.reshape(N, 6, K, GH, GW)
    e = edge.reshape(N, E, NH, NW, GH, GW)
    p = capi.PoseProposalParser((W, H), *thr)
    out = p.process_batch(b[:, 0], b[:, 2], b[:, 3], b[:, 4], b[:, 5], e, cap=cap)
    p.close()
    return out


def _two_call(eng, thr, N, frames=None, d_frames=None, cap=CAP):
    """engine inference, then the strided parse of its outputs in place on the engine stream, then fetch; retried after a capacity
    the parser grew (what hp_ppn_process_host does)"""
    parser = capi.PoseProposalParser((eng.in_w, eng.in_h), *thr)
    st = eng.device_outputs()[2]
    p = capi.ppn_engine_pointers(eng)
    for _ in range(3):
        if d_frames is not None:
            eng.infer_u8_device(d_frames, N, st)
        else:
            eng.infer_u8(frames)
        parser.process_device(*p["ptrs"], N, p["K"], p["gh"], p["gw"], E, NH, NW, stream=st,
                              box_frame_stride=p["box_frame_stride"], edge_frame_stride=p["edge_frame_stride"])
        try:
            out = parser.fetch(N, cap)
            parser.close()
            return out
        except capi.HyperposeError as ex:
            assert ex.status == capi.HP_ERR_CAPACITY, ex
    raise AssertionError("capacity kept growing")


def _same(a, b):
    return len(a) == len(b) and all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


def _status(fn, *a, **k):
    with pytest.raises(capi.HyperposeError) as e:
        fn(*a, **k)
    return e.value.status, str(e.value)


def _src(seed, h, w):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def _many_humans(n_cells_used=GH * GW):
    """one frame with a whole 18-part person in each of the first n grid cells: every part's box in that cell, an 8 x 8 box at the
    cell's centre (no two boxes of a type overlap, so NMS keeps all), and every limb's edge to the same cell (the centre neighbour).
    At the default thresholds each limb opens or extends one human per cell and no two humans share a part position: n humans"""
    rng = np.random.default_rng(5)
    yy, xx = np.meshgrid(np.arange(GH), np.arange(GW), indexing="ij")
    used = (yy * GW + xx) < n_cells_used
    cw, ch = W / GW, H / GH
    conf = np.where(used, rng.uniform(0.5, 0.9, (K, GH, GW)), 0.0).astype(np.float32)
    x = np.broadcast_to(xx * cw + cw / 2, (K, GH, GW)).astype(np.float32)
    y = np.broadcast_to(yy * ch + ch / 2, (K, GH, GW)).astype(np.float32)
    wh = np.full((K, GH, GW), 8, np.float32)
    edge = np.zeros((E, NH, NW, GH, GW), np.float32)
    edge[:, NH // 2, NW // 2] = np.where(used, rng.uniform(0.5, 0.9, (E, GH, GW)), 0.0)
    return conf, np.zeros_like(conf), x, y, wh, wh.copy(), edge


# ---- 1. equality with the two-call path ----------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dtype", ["f16", "tf32"])
@pytest.mark.parametrize("net", ["ppn_resnet18", "ppn_resnet50"])
def test_equals_two_call_path(net, dtype):
    import torch
    for max_batch, N in ((16, 16), (8, 5)):
        eng = _engine(net, max_batch, dtype)
        frames = syn.make_frames_u8(60 + N, N, H, W)
        d_frames = torch.from_numpy(frames).cuda()
        torch.cuda.synchronize()
        # synthetic crowd tensors through the output override
        box, edge = _crowd(3000 + N, N)
        d_box, d_edge = _on_device(box, edge)
        eng.set_output_override(d_box.data_ptr(), d_edge.data_ptr())
        parser = capi.PoseProposalParser((W, H), *DEFAULT_THR)
        got = eng.collect_pose(eng.submit_pose_device(parser, d_frames.data_ptr(), N), cap=CAP)
        want = _two_call(eng, DEFAULT_THR, N, d_frames=d_frames.data_ptr())
        n_crowd = sum(len(h) for h in want)
        assert n_crowd >= N, "vacuous: no humans in the crowd tensors"
        assert _same(got, want), f"{net} {dtype} N={N}: crowd tensors"
        assert _same(got, _host_parse(box, edge, DEFAULT_THR))
        # the network's own outputs: random weights give structureless maps; thresholds at the median box confidence and the 70 %
        # quantile of the edges assemble a few humans per frame
        eng.set_output_override(0, 0)
        eng.infer_u8(frames)
        ob, oe = eng.read_outputs(N)
        thr = (float(np.quantile(ob.reshape(N, 6, K, -1)[:, 0], 0.5)), float(np.quantile(oe, 0.7)), 0.3)
        parser2 = capi.PoseProposalParser((W, H), *thr)
        got = eng.collect_pose(eng.submit_pose(parser2, frames), cap=CAP)
        want = _two_call(eng, thr, N, frames=frames)
        assert sum(len(h) for h in want) >= N, "vacuous: no humans in the network's outputs"
        assert _same(got, want), f"{net} {dtype} N={N}: network outputs"
        print(f"[ppn pipeline] {net} {dtype} N={N}: crowd {n_crowd} humans, network outputs {[len(h) for h in got]}")
        eng.close(); parser.close(); parser2.close()


# ---- 2. two tickets in flight ----------------------------------------------------------------------------------------------------
@gpu
def test_two_tickets_in_flight():
    eng = _engine("ppn_resnet18", 8)
    tensors = {"a": _crowd(3100, 8), "b": _crowd(3200, 8, (6, 10))}
    dev = {k: _on_device(*v) for k, v in tensors.items()}
    thr_a, thr_a2, thr_b = (0.10, 0.05, 0.3), (0.12, 0.06, 0.3), (0.08, 0.04, 0.4)
    pa, pb = capi.PoseProposalParser((W, H), *thr_a), capi.PoseProposalParser((W, H), *thr_b)
    frames = syn.make_frames_u8(70, 8, H, W)
    # (override, parser, N, thresholds of pa, expected captures after the submit): slot 0 always gets pa, slot 1 pb
    plan = [("a", pa, 8, thr_a, 1), ("b", pb, 5, None, 2), ("a", pa, 8, thr_a, 2), ("b", pb, 5, None, 2),
            ("a", pa, 8, thr_a2, 3), ("b", pb, 6, None, 4), ("a", pa, 8, thr_a2, 4), ("b", pb, 6, None, 4), ("a", pa, 7, thr_a2, 5)]
    pending, results = [], []
    for i, (ov, parser, N, thr, captures) in enumerate(plan):
        if thr is not None:
            parser.set_point_thresh(thr[0]); parser.set_limb_thresh(thr[1]); parser.set_nms_thresh(thr[2])
        eng.set_output_override(dev[ov][0].data_ptr(), dev[ov][1].data_ptr())
        pending.append((eng.submit_pose(parser, frames[:N]), ov, N, thr or thr_b))
        st = eng.pose_stats()
        assert st["graph_captures"] == captures, (i, st)
        assert st["graph_launches"] == i + 1, (i, st)
        if len(pending) == 2:
            t, ov_, N_, thr_ = pending.pop(0)
            results.append((eng.collect_pose(t, cap=CAP), ov_, N_, thr_))
    t, ov_, N_, thr_ = pending.pop(0)
    results.append((eng.collect_pose(t, cap=CAP), ov_, N_, thr_))
    n = 0
    for i, (got, ov, N, thr) in enumerate(results):
        box, edge = tensors[ov]
        eng.set_output_override(dev[ov][0].data_ptr(), dev[ov][1].data_ptr())
        want = _two_call(eng, thr, N, frames=frames[:N])
        assert _same(got, want), f"batch {i}"
        n += sum(len(h) for h in want)
    assert n >= len(plan) * 5, f"vacuous: {n} humans"
    eng.set_output_override(0, 0)
    eng.close(); pa.close(); pb.close()


# ---- 3. camera-size frames ----------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("keep", [False, True])
def test_camera_size_frames(keep):
    import torch
    imgs = [_src(800 + k, h, w) for k, (h, w) in enumerate(MIXED)]
    N = len(imgs)
    want_frames = np.stack([oracle.resize_linear_u8(f, H, W, letterbox=keep) for f in imgs])
    pinned = [torch.from_numpy(f).pin_memory().numpy() for f in imgs]
    d_imgs = [torch.from_numpy(f).cuda() for f in imgs]
    torch.cuda.synchronize()
    eng = _engine("ppn_resnet18", 8)
    parser = capi.PoseProposalParser((W, H))

    def submit(mode):
        if mode == "device":
            return eng.submit_pose_frames_device(parser, [(d.data_ptr(), d.shape[0], d.shape[1]) for d in d_imgs], keep_ratio=keep)
        return eng.submit_pose_frames(parser, pinned if mode == "pinned" else imgs, keep_ratio=keep)

    eng.infer_u8(want_frames)
    want_box, want_edge = eng.read_outputs(N)
    for mode in ("pageable", "pinned", "device"):
        t = submit(mode)
        eng.collect_pose(t, cap=CAP)
        assert np.array_equal(eng.debug_read_slot_frames(t, N), want_frames), f"{mode} keep_ratio={keep}"
        box, edge = eng.read_outputs(N)
        assert box.tobytes() == want_box.tobytes() and edge.tobytes() == want_edge.tobytes(), f"{mode} keep_ratio={keep}"
    # humans over crowd tensors equal the network-size pipelined call
    cb, ce = _crowd(3300, N)
    d_box, d_edge = _on_device(cb, ce)
    eng.set_output_override(d_box.data_ptr(), d_edge.data_ptr())
    want = eng.collect_pose(eng.submit_pose(parser, want_frames), cap=CAP)
    assert sum(len(h) for h in want) >= N, "vacuous: no humans in the crowd tensors"
    for mode in ("pageable", "pinned", "device"):
        assert _same(eng.collect_pose(submit(mode), cap=CAP), want), f"{mode} keep_ratio={keep}"
    eng.set_output_override(0, 0)
    eng.close(); parser.close()


# ---- 4. capacity growth in collect, the other ticket in flight -------------------------------------------------------------------
def _growth(first, second, thr):
    """ticket A over `first` (it overflows), ticket B over `second` submitted before A is collected: both collects return the host
    parse's records, and the next submit of each slot recaptures"""
    eng = _engine("ppn_resnet18", 4)
    parser = capi.PoseProposalParser((W, H), *thr)
    dev = [_on_device(*first), _on_device(*second)]
    frames = syn.make_frames_u8(71, 4, H, W)
    n1, n2 = first[0].shape[0], second[0].shape[0]
    eng.set_output_override(dev[0][0].data_ptr(), dev[0][1].data_ptr())
    ta = eng.submit_pose(parser, frames[:n1])
    eng.set_output_override(dev[1][0].data_ptr(), dev[1][1].data_ptr())
    tb = eng.submit_pose(parser, frames[:n2])
    assert eng.pose_stats()["graph_captures"] == 2
    got_a = eng.collect_pose(ta, cap=CAP)
    got_b = eng.collect_pose(tb, cap=CAP)
    want_a, want_b = _host_parse(*first, thr), _host_parse(*second, thr)
    assert _same(got_a, want_a), "ticket A (grown in collect)"
    assert _same(got_b, want_b), "ticket B (in flight while A grew)"
    # the next submits: both slots' keys changed (A's in its rerun, B's because the parser grew)
    eng.set_output_override(dev[0][0].data_ptr(), dev[0][1].data_ptr())
    t = eng.submit_pose(parser, frames[:n1])
    assert eng.pose_stats()["graph_captures"] == 3
    assert _same(eng.collect_pose(t, cap=CAP), want_a)
    eng.set_output_override(dev[1][0].data_ptr(), dev[1][1].data_ptr())
    t = eng.submit_pose(parser, frames[:n2])
    assert eng.pose_stats()["graph_captures"] == 4
    assert _same(eng.collect_pose(t, cap=CAP), want_b)
    eng.set_output_override(0, 0)
    eng.close(); parser.close()
    return want_a, want_b


@gpu
def test_growth_to_the_spill_variant():
    case = next(c for c in PPN_CASES if c[0] == "ppn_dense")
    name, seed, P, net_w, net_h, gh, gw, nh, nw, pt, lt, nt, nd = case
    assert (net_w, net_h, gh, gw, nh, nw) == (W, H, GH, GW, NH, NW)
    dense = syn.make_ppn_tensors(seed, P, net_h, net_w, gh, gw, nh, nw, nd)
    crowd = [syn.make_ppn_tensors(3400 + i, (4, 8)) for i in range(3)]
    want_a, _ = _growth(_stack([crowd[0], dense]), _stack(crowd[1:]), (pt, lt, nt))
    assert len(want_a[1]) == 87


@gpu
def test_growth_of_the_record_capacity():
    many = _many_humans()
    crowd = [syn.make_ppn_tensors(3500 + i, (4, 8)) for i in range(4)]
    want_a, _ = _growth(_stack([many, crowd[0]]), _stack(crowd[1:]), DEFAULT_THR)
    assert len(want_a[0]) == GH * GW > 128   # more than the records a frame starts with


def test_many_humans_frame_on_the_cpu():
    """the frame test_growth_of_the_record_capacity relies on: oracle.ppn_process finds 144 whole humans in it"""
    humans = oracle.ppn_process(*_many_humans(), W, H, *DEFAULT_THR)
    assert len(humans) == GH * GW and all(float(h["score"]) == 18.0 for h in humans)


# ---- 5. refusals --------------------------------------------------------------------------------------------------------------
@gpu
def test_refusals():
    import torch
    eng = _engine("ppn_resnet18", 2)
    parser = capi.PoseProposalParser((W, H))
    frames = syn.make_frames_u8(72, 3, H, W)
    d = torch.from_numpy(frames).cuda()
    torch.cuda.synchronize()
    img = _src(1, 90, 150)
    L = capi.lib()
    t = C.c_int(-1)
    # null arguments
    for rc in (L.hp_pose_submit_ppn_u8_host(eng._h, None, frames.ctypes.data, 1, C.byref(t)),
               L.hp_pose_submit_ppn_u8_device(eng._h, parser._h, None, 1, C.byref(t)),
               L.hp_pose_submit_ppn_u8_device(eng._h, parser._h, d.data_ptr(), 1, None),
               L.hp_pose_submit_ppn_u8_host(None, parser._h, frames.ctypes.data, 1, C.byref(t))):
        assert rc == capi.HP_ERR_ARG and "null argument" in L.hp_last_error().decode()
    assert _status(eng.submit_pose_frames_device, parser, [(0, 90, 150)])[0] == capi.HP_ERR_ARG
    # more frames than max_batch
    assert _status(eng.submit_pose, parser, frames)[0] == capi.HP_ERR_BATCH
    assert _status(eng.submit_pose_device, parser, d.data_ptr(), 3)[0] == capi.HP_ERR_BATCH
    assert _status(eng.submit_pose_frames, parser, [img] * 3)[0] == capi.HP_ERR_BATCH
    # a third batch in flight
    t0 = eng.submit_pose(parser, frames[:1])
    t1 = eng.submit_pose_frames(parser, [img, img])
    st, msg = _status(eng.submit_pose_device, parser, d.data_ptr(), 1)
    assert st == capi.HP_ERR_ARG and "in flight" in msg
    eng.collect_pose(t0); eng.collect_pose(t1)
    # the caller's capacity, at collect
    box, edge = _crowd(3600, 2, (4, 7))
    d_box, d_edge = _on_device(box, edge)
    eng.set_output_override(d_box.data_ptr(), d_edge.data_ptr())
    t = eng.submit_pose(parser, frames[:2])
    st, msg = _status(eng.collect_pose, t, cap=1)
    assert st == capi.HP_ERR_CAPACITY and "caller's capacity is 1" in msg
    eng.set_output_override(0, 0)
    # the PAF-parser calls keep refusing the PPN pack
    paf = capi.PafParser()
    st, msg = _status(eng.submit_pose, paf, frames[:1])
    assert st == capi.HP_ERR_UNSUPPORTED and "Pose Proposal Network" in msg and "hp_pose_submit_ppn" in msg
    paf.close(); eng.close()
    # a pack without PPN heads
    tiny = capi.Engine(models.tiny_test_net(0).to_pack(), (96, 64), max_batch_size=2)
    st, msg = _status(tiny.submit_pose, parser, syn.make_frames_u8(73, 1, 64, 96))
    assert st == capi.HP_ERR_UNSUPPORTED and "head_type 0" in msg
    assert _status(tiny.submit_pose_frames, parser, [img])[0] == capi.HP_ERR_UNSUPPORTED
    tiny.close(); parser.close()


@gpu
def test_refuses_a_parser_on_another_device():
    if capi.lib().hp_device_count() < 2:
        pytest.skip("needs two GPUs")
    eng = _engine("ppn_resnet18", 2)
    parser = capi.PoseProposalParser((W, H), device=1)
    st, msg = _status(eng.submit_pose, parser, syn.make_frames_u8(74, 1, H, W))
    assert st == capi.HP_ERR_ARG and "device 1" in msg
    eng.close(); parser.close()


# ---- 6. launch counts ---------------------------------------------------------------------------------------------------------
@gpu
def test_launch_count_per_replay_equals_direct():
    import torch
    eng = _engine("ppn_resnet18", 4)
    box, edge = _crowd(3700, 4)
    d_box, d_edge = _on_device(box, edge)
    eng.set_output_override(d_box.data_ptr(), d_edge.data_ptr())
    frames = syn.make_frames_u8(75, 4, H, W)
    d = torch.from_numpy(frames).cuda()
    torch.cuda.synchronize()
    parser = capi.PoseProposalParser((W, H))
    st = eng.device_outputs()[2]
    p = capi.ppn_engine_pointers(eng)

    def total():
        return eng.launch_count + parser.launch_count

    n0 = total()
    eng.infer_u8_device(d.data_ptr(), 4, st)
    parser.process_device(*p["ptrs"], 4, p["K"], p["gh"], p["gw"], E, NH, NW, stream=st,
                          box_frame_stride=p["box_frame_stride"], edge_frame_stride=p["edge_frame_stride"])
    parser.fetch(4, CAP)
    direct = total() - n0
    assert direct > 1
    for i in range(4):   # a capture, then replays of both slots
        n0 = total()
        eng.collect_pose(eng.submit_pose_device(parser, d.data_ptr(), 4), cap=CAP)
        assert total() - n0 == direct, (i, total() - n0, direct)
    assert eng.pose_stats() == {"graph_captures": 2, "graph_launches": 4}
    eng.set_output_override(0, 0)
    eng.close(); parser.close()


# ---- CPU: the wrapper's dispatch ------------------------------------------------------------------------------------------------
def test_wrapper_dispatches_ppn_parsers(monkeypatch):
    calls = []

    class FakeLib:
        def __getattr__(self, name):
            def fn(*a):
                calls.append(name)
                return capi.HP_OK
            return fn

    monkeypatch.setattr(capi, "lib", lambda: FakeLib())
    eng = object.__new__(capi.Engine)
    eng._h = None
    parser = capi.PoseProposalParser.__new__(capi.PoseProposalParser)
    parser._h = None
    frames = np.zeros((2, 4, 6, 3), np.uint8)
    eng.submit_pose(parser, frames)
    eng.submit_pose_device(parser, 1, 2)
    eng.submit_pose_frames(parser, [frames[0]])
    eng.submit_pose_frames_device(parser, [(1, 4, 6)])
    assert calls == ["hp_pose_submit_ppn_u8_host", "hp_pose_submit_ppn_u8_device", "hp_pose_submit_ppn_frames_u8_host",
                     "hp_pose_submit_ppn_frames_u8_device"]
