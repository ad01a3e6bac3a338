"""Pose Proposal Network packs on the engine (head_type 2, OP_PPN_HEAD / ppn_head_kernel) and the parse of its outputs in place
(hp_ppn_process_device_strided).

  * the head kernel alone, on chosen raw values, against a float64 evaluation of its formulas (tests/ppn_head_ref.py): every element
    within 2^-20 |ref| + 2^-40, f16 and TF32 engines, square and non-square inputs;
  * both networks at 384 x 384 against the torch oracle, every buffer and both outputs (the ResNet-50 rule of
    test_backbone_fullsize.py for f16, test_engine_tf32.py's for TF32);
  * engine -> strided device parse == host parse of the read-back tensors == oracle.ppn_process, byte for byte;
  * malformed packs and unsupported calls are refused with a message naming the op or head type;
  * the reference's own pose_proposal example and `cli --post=ppn` run unmodified on a PPN pack."""
import os
import subprocess

import numpy as np
import pytest
import torch

import oracle
from hyperpose_b200 import capi, models, synthetic as syn
from oracle import torch_backbone
from tests.ppn_head_ref import ppn_head_ref
from tests.test_ppn import _as_records
from tests.test_reference_examples import _exes, _read_p6_stream, _write_inputs

pytestmark = pytest.mark.gpu

K, E = 18, 17 * 9 * 9


def _head_index(g):
    return next(i for i, op in enumerate(g.ops) if op.type == models.OP_PPN_HEAD)


def _raw_values(n, gh, gw, C, f16):
    """a value per (frame, pixel, channel) that differs along every axis, in [-14, 14] (both tails of the sigmoid)"""
    n_, y, x, c = np.meshgrid(np.arange(n), np.arange(gh), np.arange(gw), np.arange(C), indexing="ij")
    v = np.sin(0.37 * c + 1.3 * x + 2.1 * y + 0.9 * n_ + 0.05 * c * (x + 1)) * 14.0 + 0.01 * (c % 7)
    return v.astype(np.float16) if f16 else v.astype(np.float32)


@pytest.mark.parametrize("dtype", ["f16", "tf32"])
@pytest.mark.parametrize("hw", [(320, 448), (384, 384)])
def test_head_kernel_alone_against_float64(dtype, hw):
    H, W = hw
    g = models.ppn_resnet18(0)
    hi = _head_index(g)
    raw_buf = g.ops[hi].in_buf
    N = 2
    eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=N, dtype=dtype)
    assert eng.debug_op_kernel(hi) == "ppn_head" and eng.head_type == 2
    gh, gw = eng.out_h, eng.out_w
    assert (gh, gw) == ((H + 31) // 32, (W + 31) // 32) and (eng.c_conf, eng.c_paf) == (6 * K, E)
    raw = _raw_values(N, gh, gw, 1488, dtype == "f16")
    eng.debug_write_buffer(raw_buf, raw)
    eng.debug_run_ops(hi, hi, N)
    box, edge = eng.read_outputs(N)
    rbox, redge = ppn_head_ref(raw.astype(np.float64).transpose(0, 3, 1, 2), K, E, H, W)
    for got, ref, what in ((box, rbox, "boxes"), (edge, redge, "edges")):
        err = np.abs(got.astype(np.float64) - ref)
        bound = 2.0 ** -20 * np.abs(ref) + 2.0 ** -40
        bad = np.argwhere(err > bound)
        assert len(bad) == 0, f"{what}: {len(bad)} elements out of bound, first at {tuple(bad[0])}: {got[tuple(bad[0])]!r} vs {ref[tuple(bad[0])]!r}"
    # not vacuous: both sigmoid tails, every slot, the grid offsets along both axes
    assert redge.min() < 1e-5 and redge.max() > 1 - 1e-5
    b = box.reshape(N, 6, K, gh, gw)
    assert b[:, 2].max() > (gw - 1) * W / gw and b[:, 3].max() > (gh - 1) * H / gh and b[:, 4].max() > 0.99 * W and b[:, 5].max() > 0.99 * H
    eng.close()


@pytest.mark.parametrize("dtype", ["f16", "tf32"])
@pytest.mark.parametrize("net", ["ppn_resnet18", "ppn_resnet50"])
def test_whole_network_against_oracle(net, dtype):
    """every buffer and both outputs at 384 x 384, batch 4.  f16: the fp16-emulated oracle, max|diff| <= 8e-3 max|ref| + 8e-3 (the
    ResNet-50 PifPaf constants of test_backbone_fullsize.py); TF32: plain fp32, 6e-3 max|ref| + 1e-3 (test_engine_tf32.py).  The outputs
    are the head's formulas on the raw buffer: the sigmoid's slope is at most 1/4, so each slot's bound is 1/4 of the raw buffer's, times
    the slot's scale (1, or the grid size / input size the coordinates are multiplied by)."""
    H = W = 384
    N = 4
    g = getattr(models, net)(0)
    rel, abs_ = (8e-3, 8e-3) if dtype == "f16" else (6e-3, 1e-3)
    frames = syn.make_frames_u8(41, N, H, W)
    eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=N, dtype=dtype)
    eng.infer_u8(frames)
    box, edge = eng.read_outputs(N)
    _, _, rbufs = torch_backbone.run_graph(g, frames, emulate_fp16=dtype == "f16")
    worst = 0.0
    for bi in range(1, len(g.buffers)):             # buffer 0: the stem's patch buffer, which the fused u8 stem never writes
        try:
            got = eng.debug_read_buffer(bi, N).astype(np.float32).transpose(0, 3, 1, 2)
        except capi.HyperposeError as ex:           # an un-pooled conv output whose max-pool runs in the conv's epilogue
            assert ex.status == capi.HP_ERR_UNSUPPORTED, ex
            continue
        ref = rbufs[bi].cpu().numpy()
        d, m = float(np.abs(got[:, :ref.shape[1]] - ref).max()), float(np.abs(ref).max())
        assert np.isfinite(got).all() and d <= rel * m + abs_, f"{net} {dtype} buffer {bi} {ref.shape}: max|diff| {d:.3e} vs max|ref| {m:.3e}"
        worst = max(worst, d / max(m, 1e-30))
    raw = rbufs[g.ops[-1].in_buf].cpu().numpy()[:, :6 * K + E]
    raw_budget = rel * float(np.abs(raw).max()) + abs_
    rbox, redge = ppn_head_ref(raw, K, E, H, W)
    gh, gw = eng.out_h, eng.out_w
    scale = [1.0, 1.0, W / gw, H / gh, W, H]
    b, rb = box.reshape(N, 6, K, gh, gw), rbox.reshape(N, 6, K, gh, gw)
    for t in range(6):
        d = float(np.abs(b[:, t] - rb[:, t]).max())
        assert d <= 0.25 * raw_budget * scale[t] + 1e-6 * scale[t], f"{net} {dtype} box slot {t}: {d:.3e} (raw budget {raw_budget:.3e})"
    d = float(np.abs(edge - redge).max())
    assert d <= 0.25 * raw_budget + 1e-6, f"{net} {dtype} edges: {d:.3e}"
    print(f"[ppn] {net} {dtype} 384x384 batch {N}: worst buffer rel err {worst:.2e}; raw max {np.abs(raw).max():.3g}, edges max|diff| {d:.2e}")
    eng.close()


def _parse_device(parser, eng, N, cap=512):
    p = capi.ppn_engine_pointers(eng)
    for _ in range(3):          # a capacity the parser raised on the way: run again (as hp_ppn_process_host does)
        parser.process_device(*p["ptrs"], N, p["K"], p["gh"], p["gw"], 17, 9, 9, box_frame_stride=p["box_frame_stride"],
                              edge_frame_stride=p["edge_frame_stride"])
        try:
            return parser.fetch(N, cap)
        except capi.HyperposeError as ex:
            assert ex.status == capi.HP_ERR_CAPACITY, ex
    raise AssertionError("capacity kept growing")


def _check_parse(eng, N, thr, min_humans):
    """device parse of the engine's outputs in place == host parse of the read-back == the restatement, frame by frame"""
    box, edge = eng.read_outputs(N)
    gh, gw = eng.out_h, eng.out_w
    b = box.reshape(N, 6, K, gh, gw)
    e = edge.reshape(N, 17, 9, 9, gh, gw)
    parser = capi.PoseProposalParser((eng.in_w, eng.in_h), *thr)
    got = _parse_device(parser, eng, N)
    host = parser.process_batch(b[:, 0], b[:, 2], b[:, 3], b[:, 4], b[:, 5], e, cap=512)
    for i in range(N):
        assert got[i].tobytes() == host[i].tobytes(), f"frame {i}: device-strided parse differs from the host parse"
        want = _as_records(oracle.ppn_process(b[i, 0], b[i, 1], b[i, 2], b[i, 3], b[i, 4], b[i, 5], e[i], eng.in_w, eng.in_h, *thr))
        assert got[i].tobytes() == want.tobytes(), f"frame {i}: differs from oracle.ppn_process"
        assert len(got[i]) >= min_humans, (i, len(got[i]))
    parser.close()
    return [len(h) for h in got]


def test_engine_outputs_parse_in_place_network_outputs():
    """N = 3 frames in an engine built for 8: the strides are the per-frame distances of the engine's slots, not max_batch's"""
    g = models.ppn_resnet18(0)
    N = 3
    eng = capi.Engine(g.to_pack(), (384, 384), max_batch_size=8)
    frames = syn.make_frames_u8(43, N, 384, 384)
    d_frames = torch.from_numpy(frames).cuda()
    eng.infer_u8_device(d_frames.data_ptr(), N)
    eng.sync()
    box, edge = eng.read_outputs(N)
    # random weights give structureless maps: thresholds at high quantiles keep the parse a few hundred candidates deep
    pt = float(np.quantile(box.reshape(N, 6, K, -1)[:, 0], 0.97))
    lt = float(np.quantile(edge, 0.999))
    n = _check_parse(eng, N, (pt, lt, 0.3), 0)
    print(f"[ppn] network outputs: humans per frame {n} (point_thresh {pt:.4g}, limb_thresh {lt:.4g})")
    eng.close()


def test_engine_outputs_parse_in_place_crowd_override():
    N = 3
    eng = capi.Engine(models.ppn_resnet18(0).to_pack(), (384, 384), max_batch_size=8)
    ts = [syn.make_ppn_tensors(900 + i, (4, 7)) for i in range(N)]
    box = np.stack([np.stack(t[:6]) for t in ts]).reshape(N, 6 * K, 12, 12)
    edge = np.stack([t[6] for t in ts]).reshape(N, E, 12, 12)
    d_box, d_edge = torch.from_numpy(np.ascontiguousarray(box)).cuda(), torch.from_numpy(np.ascontiguousarray(edge)).cuda()
    eng.set_output_override(d_box.data_ptr(), d_edge.data_ptr())
    eng.infer_u8(syn.make_frames_u8(44, N, 384, 384))
    eng.sync()
    rb, re_ = eng.read_outputs(N)
    assert np.array_equal(rb, box) and np.array_equal(re_, edge)
    n = _check_parse(eng, N, (0.10, 0.05, 0.3), 3)
    print(f"[ppn] crowd tensors: humans per frame {n}")
    eng.close()


def _head_only(down=5, channels=1488, Kp=18, conf=108, paf=1377, head_type=2):
    g = models.Graph("ppn_head_only", conf, paf, 5, head_type=head_type)
    b = g.add_buffer(channels, down)
    g.ops.append(models.Op(models.OP_PPN_HEAD, in_buf=b, cout_g=Kp, groups=17, R=9, S=9, name="ppn_head"))
    return g.to_pack()


@pytest.mark.parametrize("case,pack,words", [
    ("wrong head_type", lambda: _head_only(head_type=0), ["PPN head op 0", "head_type 0"]),
    ("wrong resolution", lambda: _head_only(down=4), ["PPN head op 0", "down-shift 4"]),
    ("too few channels", lambda: _head_only(channels=1480), ["PPN head op 0", "1485 channels"]),
    ("header channel counts", lambda: _head_only(paf=1376), ["PPN head op 0", "paf 1376"]),
    ("K < 18", lambda: _head_only(Kp=17, conf=102), ["PPN head op 0", "K=17"]),
])
def test_malformed_packs_are_refused(case, pack, words):
    with pytest.raises(capi.HyperposeError) as ex:
        capi.Engine(pack(), (384, 384), max_batch_size=2)
    assert ex.value.status == capi.HP_ERR_ARG
    for w in words:
        assert w in str(ex.value), (case, str(ex.value))


def test_head_only_pack_is_accepted():
    """the rejection cases above differ from this pack in one field each"""
    eng = capi.Engine(_head_only(), (384, 384), max_batch_size=2)
    assert eng.debug_op_kernel(0) == "ppn_head"
    eng.close()


def test_int8_engine_and_pose_calls_refuse_ppn_packs():
    g = models.ppn_resnet18(0)
    g.set_int8_scales(np.ones(len(g.buffers), np.float32))
    with pytest.raises(capi.HyperposeError) as ex:
        capi.Engine(g.to_pack(), (384, 384), max_batch_size=2, dtype="int8")
    assert ex.value.status == capi.HP_ERR_ARG and "head_type 2" in str(ex.value)
    eng = capi.Engine(models.ppn_resnet18(0).to_pack(), (384, 384), max_batch_size=2)
    frames = syn.make_frames_u8(45, 2, 384, 384)
    parser = capi.PafParser()
    for call in (lambda: eng.submit_pose(parser, frames), lambda: eng.run_pose(parser, frames)):
        with pytest.raises(capi.HyperposeError) as ex:
            call()
        assert ex.value.status == capi.HP_ERR_UNSUPPORTED and "Pose Proposal Network" in str(ex.value)
    eng.close(); parser.close()


def test_reference_pose_proposal_example_runs(tmp_path):
    """examples/operator_api_batched_images_pose_proposal.example.cpp, unmodified: seven maps per image, parser.process(packet)"""
    exes = _exes()
    folder, _, _ = _write_inputs(tmp_path, 3, 300, 420)
    pack = tmp_path / "ppn.onnx"
    pack.write_bytes(models.ppn_resnet18(0).to_pack())
    r = subprocess.run([exes["operator_api_batched_images_pose_proposal.example"], f"--model_file={pack}", f"--input_folder={folder}"],
                       capture_output=True, text=True, timeout=300, cwd=tmp_path)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "3 images got processed" in r.stdout
    assert r.stdout.count("[18, 12, 12, ]") == 18 and r.stdout.count("[17, 9, 9, 12, 12, ]") == 3, r.stdout
    outs = sorted(p for p in os.listdir(tmp_path) if p.startswith("output_"))
    assert outs == ["output_0.png", "output_1.png", "output_2.png"]
    assert _read_p6_stream(tmp_path / "output_0.png")[0].shape == (384, 384, 3)


@pytest.mark.parametrize("runtime,source", [("operator", "folder"), ("stream", "video")])
def test_cli_post_ppn_runs(tmp_path, runtime, source):
    exes = _exes()
    folder, video, _ = _write_inputs(tmp_path, 5, 96, 128)
    pack = tmp_path / "ppn.pack"
    pack.write_bytes(models.ppn_resnet18(0).to_pack())
    src = folder if source == "folder" else video
    r = subprocess.run([exes["cli"], f"--model={pack}", "--w=128", "--h=96", "--max_batch_size=2", f"--source={src}", f"--runtime={runtime}", "--post=ppn",
                        "--imshow=false", f"--saving_prefix={tmp_path / 'out'}"], capture_output=True, text=True, timeout=300, cwd=tmp_path)
    assert r.returncode == 0, r.stdout + r.stderr
    assert ("6 images got processed" if runtime == "stream" else "5 images got processed") in r.stdout, r.stdout
    if source == "folder":
        assert len([p for p in os.listdir(tmp_path) if p.startswith("out_") and p.endswith(".png")]) == 5
    else:
        assert len(_read_p6_stream(tmp_path / "out.avi")) == 5
