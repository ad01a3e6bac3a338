"""Lightweight-OpenPose on TinyVGG and on ResNet-18 (lw_openpose.py:13-45 with vggtiny_backbone / Resnet18_backbone at scale_size 8,
backbones.py:343-391 / :512-585).

CPU: the ResNet-50 graph (BASELINE cfg4) keeps its exact pack after the LW head moved into a shared builder; both new graphs, on
weights written in TensorLayer's all_weights order and imported, equal a plain fp32 PyTorch model written from the reference
definitions (BatchNorm unfolded, explicit TF 'SAME' padding, ceil max-pools), at 64 x 96 and at an odd 86 x 92 (11 x 12 maps); the
seeded random-init graphs have the imported graphs' layout; the exporter round-trips both.

GPU: every buffer and both outputs at the published / model-zoo sizes against oracle/torch_backbone.py (fp16 and TF32 engines,
batch 16 and a ragged 5 on a batch-16 engine), a calibrated INT8 pack of each byte for byte against tests/int8_sim.py, the kernel
instantiations these graphs introduce against float64 at their real shapes (tests/test_engine_kernels.py), the kernel every layer
lands on, and the pose-level paths: the pipelined hp_pose_submit / hp_pose_collect call and hp_pool on synthetic crowd maps, and
the reference's unmodified cli on a TinyVGG pack."""
import hashlib
import os
import subprocess
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from hyperpose_b200 import export, models, synthetic as syn, weights as W
from oracle import torch_backbone as torch_ref
from tests.test_weights_import import _tl_arrays, _TlReader

NETS = {"lw_openpose_vggtiny": (models.lw_openpose_vggtiny, W.LwVggtinyWeights, W.lw_vggtiny_layer_order),
        "lw_openpose_resnet18": (models.lw_openpose_resnet18, W.LwResnet18Weights, W.lw_resnet18_layer_order)}

# sha256 of resnet50_lw_openpose(seed=0).to_pack() before the LW head became a shared builder
CFG4_PACK_SHA256 = "44e23dbdbf5e47a770bd1009ee80d3ca55e74ef832eddbc43d95933f4f9ba5a9"


def test_cfg4_pack_is_unchanged():
    assert hashlib.sha256(models.resnet50_lw_openpose(seed=0).to_pack()).hexdigest() == CFG4_PACK_SHA256


# ---- plain PyTorch models written from the reference definitions --------------------------------------------------------------
def _pool_same(x, k):
    """MaxPool2d(k, 2, 'SAME'): out = ceil(in / 2), TF's padding (the odd pixel after) filled with -inf"""
    pads = []
    for n in (x.shape[3], x.shape[2]):
        total = max((-(-n // 2) - 1) * 2 + k - n, 0)
        pads += [total // 2, total - total // 2]
    return F.max_pool2d(F.pad(x, pads, value=float("-inf")), k, 2)


def _vggtiny_reference(r, x):
    """vggtiny_backbone(scale_size=8), backbones.py:350-365: conv_block = Conv2d(+bias) + BatchNorm2d(relu)"""
    for c in (32, 64, "P", 128, 128, "P", 200, 200, 200, "P", 384, 384):
        x = _pool_same(x, 2) if c == "P" else F.relu(r.bn(r.conv(x)))
        assert c == "P" or x.shape[1] == c
    return x


def _resnet18_reference(r, x):
    """Resnet18_backbone(scale_size=8), backbones.py:513-585: the blocks 4_1 and 5_1 keep stride 1"""
    bn = r.bn
    x = F.relu(bn(r.conv(x, stride=2, bias=False)))
    x = _pool_same(x, 3)
    for st, ds in ((1, False), (1, False), (2, True), (1, False), (1, True), (1, False), (1, True)):
        y = F.relu(bn(r.conv(x, stride=st, bias=False)))                   # main_block, then down_sample (created in that order)
        y = bn(r.conv(y, bias=False))
        res = bn(r.conv(x, stride=st, bias=False)) if ds else x
        x = F.relu(y + res)
    return x


def _lw_head_reference(r, feat):
    """Cpm_stage, Init_stage, Refinement_stage of lw_openpose.py:106-191"""
    cb = lambda t: F.relu(r.bn(r.conv(t)))                                  # conv_block: Conv2d(+bias), BatchNorm(relu)
    t = F.relu(r.conv(feat))
    t = t + cb(cb(cb(t)))
    cpm = F.relu(r.conv(t))
    t = F.relu(r.conv(F.relu(r.conv(F.relu(r.conv(cpm))))))
    conf = r.conv(F.relu(r.conv(t)))
    paf = r.conv(F.relu(r.conv(t)))
    t = torch.cat([cpm, conf, paf], 1)
    for _ in range(5):
        t = F.relu(r.conv(t))
        t = t + cb(cb(t))
    conf = r.conv(F.relu(r.conv(t)))
    paf = r.conv(F.relu(r.conv(t)))
    r.done()
    return conf, paf


def _reference(net, arrays, frames):
    x = torch.from_numpy(np.ascontiguousarray((frames.astype(np.float64) / 255).astype(np.float32)[..., ::-1].transpose(0, 3, 1, 2)))
    r = _TlReader(arrays)
    feat = _vggtiny_reference(r, x) if net == "lw_openpose_vggtiny" else _resnet18_reference(r, x)
    return _lw_head_reference(r, feat)


def _params_npz(path, arrays):
    """tl.files.save_npz / Model.save_weights(format="npz"): one object array 'params' in all_weights order"""
    params = np.empty(len(arrays), object)
    params[:] = arrays
    np.savez(path, params=params)


@pytest.mark.parametrize("net", sorted(NETS))
@pytest.mark.parametrize("hw", [(64, 96), (86, 92)])
def test_imported_graph_equals_reference_definition(net, hw, tmp_path):
    build, cls, order = NETS[net]
    arrays = _tl_arrays(order(), 61)
    _params_npz(tmp_path / "w.npz", arrays)
    g = build(weights=cls.from_npz(str(tmp_path / "w.npz")))
    assert g.to_pack() == build(weights=cls(arrays)).to_pack()
    H, Wd = hw
    frames = np.random.default_rng(8).integers(0, 256, (2, H, Wd, 3), dtype=np.uint8)
    conf, paf, _ = torch_ref.run_graph(g, frames, flip_rgb=True, device="cpu")
    rc, rp = _reference(net, arrays, frames)
    h8, w8 = -(-H // 8), -(-Wd // 8)
    assert conf.shape == rc.shape == (2, 19, h8, w8) and paf.shape == rp.shape == (2, 38, h8, w8)
    tol = 2e-4 * max(1.0, float(rc.abs().max()), float(rp.abs().max()))
    assert float((conf.cpu() - rc).abs().max()) < tol and float((paf.cpu() - rp).abs().max()) < tol


def _layout(g):
    return ([(op.type, op.in_buf, op.out_buf, op.in_ch_off, op.out_ch_off, op.R, op.S, op.groups, op.cin_g, op.cout_g, op.out_mode,
              op.split, op.im2col_input, op.stride, op.res_buf, op.res_mode, op.name, None if op.weight is None else op.weight.shape)
             for op in g.ops], g.buffers, (g.conf_channels, g.paf_channels, g.out_down_shift, g.mean, g.head_type))


@pytest.mark.parametrize("net", sorted(NETS))
def test_seeded_graph_has_the_imported_layout(net):
    """the random-init graph (what the benchmark and the GPU tests run) is the network the imported one is"""
    build, cls, order = NETS[net]
    g = build(0)
    assert _layout(g) == _layout(build(weights=cls(_tl_arrays(order(), 3))))
    assert g.to_pack() == build(0).to_pack() != build(1).to_pack()


def test_graph_shapes():
    vt, r18 = models.lw_openpose_vggtiny(0), models.lw_openpose_resnet18(0)
    for g in (vt, r18):
        assert (g.head_type, g.out_down_shift, g.conf_channels, g.paf_channels, g.mean) == (0, 3, 19, 38, (0.0, 0.0, 0.0))
        assert g.ops[-1].out_mode == models.OUT_F32_NCHW_SPLIT and g.ops[-1].split == 19
        cpm = next(op for op in g.ops if op.name == "cpm_init")
        assert cpm.weight.shape == (1, 128, 384 if g is vt else 512, 1, 1) and g.buffers[cpm.in_buf][1] == 3
    pools = [op for op in vt.ops if op.type == models.OP_MAXPOOL2]
    assert [(op.R, op.cout_g) for op in pools] == [(2, 64), (2, 128), (2, 200)]
    assert [vt.buffers[op.out_buf] for op in pools] == [(64, 1), (128, 2), (256, 3)]            # 200 channels in a 256-channel buffer
    trunk = [op for op in vt.ops[:13] if op.type == models.OP_CONV]
    assert len(trunk) == 9 and all(np.all(op.alpha == 0) for op in trunk)                   # BatchNorm(relu) after every conv
    names = [op.name for op in r18.ops]
    assert not any(n.startswith("block_5_2") for n in names)
    assert sorted(n for n in names if n.endswith("_ds")) == ["block_3_1_ds", "block_4_1_ds", "block_5_1_ds"]
    assert [op.name for op in r18.ops if op.type == models.OP_DWCONV] == ["block_3_1_1_sub", "block_3_1_ds_sub"]   # only 3_1 strides
    assert sum(op.res_mode == 1 for op in r18.ops) == 7 and sum(op.res_mode == 2 for op in r18.ops) == 6


def test_head_order_is_shared():
    """the backbone's arrays first, then the ResNet-50 network's head with the CPM init_layer on the backbone width"""
    head = lambda order: [e for e in order if e[1].split(".")[0] in ("cpm", "init", "ref")]
    r50 = head(W.resnet50_lw_layer_order())
    for order, cin in ((W.lw_vggtiny_layer_order(), 384), (W.lw_resnet18_layer_order(), 512)):
        assert order[-len(r50):] == head(order)
        assert head(order)[0] == ("conv", "cpm.init", 128, cin, 1) and head(order)[1:] == r50[1:]
    assert W.lw_resnet18_layer_order()[:-len(r50)] == W.ppn_resnet18_layer_order()[:-5]


@pytest.mark.parametrize("net", sorted(NETS))
def test_importers_reject_wrong_lists(net):
    _, cls, order = NETS[net]
    arrays = _tl_arrays(order(), 4)
    with pytest.raises(ValueError):
        cls(arrays[:-1])
    with pytest.raises(ValueError):
        cls(arrays + [np.zeros(3, np.float32)])
    other = W.LwResnet18Weights if cls is W.LwVggtinyWeights else W.LwVggtinyWeights
    with pytest.raises(ValueError):
        other(arrays)


@pytest.mark.parametrize("net", sorted(NETS))
def test_export_round_trips(tmp_path, net):
    build, cls, order = NETS[net]
    out = tmp_path / f"{net}.pack"
    assert export.main(["--model", net, "--out", str(out), "--seed", "3"]) == 0
    assert out.read_bytes() == build(3).to_pack()
    arrays = _tl_arrays(order(), 12)
    _params_npz(tmp_path / "w.npz", arrays)
    out2 = tmp_path / f"{net}_trained.pack"
    assert export.main(["--model", net, "--out", str(out2), "--weights", str(tmp_path / "w.npz")]) == 0
    assert out2.read_bytes() == build(weights=cls(arrays)).to_pack()


# ================================================ GPU ===========================================================================
gpu = pytest.mark.gpu
WORKLOADS = {"vggtiny_256x384": ("lw_openpose_vggtiny", 256, 384), "vggtiny_342x368": ("lw_openpose_vggtiny", 342, 368),
             "resnet18_368x432": ("lw_openpose_resnet18", 368, 432)}
B = 16


def _cmp(got, ref, rel, abs_, what):
    d = float(np.abs(got - ref).max())
    m = float(np.abs(ref).max())
    assert np.isfinite(got).all(), f"{what}: non-finite values"
    assert d <= rel * m + abs_, f"{what}: max|diff| {d:.3e} vs max|ref| {m:.3e} (budget {rel:g}*max + {abs_:g})"
    return d / max(m, 1e-30)


@gpu
@pytest.mark.parametrize("n", [B, 5])
@pytest.mark.parametrize("dtype", ["f16", "tf32"])
@pytest.mark.parametrize("wl", sorted(WORKLOADS))
def test_full_size_parity(wl, dtype, n):
    """every buffer and both outputs against the backbone oracle, on a batch-16 engine running n frames.  Budgets as in
    tests/test_backbone_fullsize.py (fp16: 6e-3 of max|ref| against the fp16-emulated oracle, 3e-2 against fp32) and
    tests/test_engine_tf32.py (TF32: 6e-3 of max|ref| + 1e-3 against fp32)"""
    from hyperpose_b200 import capi
    net, H, Wd = WORKLOADS[wl]
    g = getattr(models, net)(0)
    frames = syn.make_frames_u8(40 + n, n, H, Wd)
    eng = capi.Engine(g.to_pack(), (Wd, H), max_batch_size=B, dtype=dtype)
    try:
        eng.infer_u8(frames)
        a, b = eng.read_outputs(n)
        assert a.shape == (n, 19, -(-H // 8), -(-Wd // 8)) and b.shape == (n, 38, -(-H // 8), -(-Wd // 8))
        rel, abs_ = (6e-3, 6e-3) if dtype == "f16" else (6e-3, 1e-3)
        ra, rb, rbufs = torch_ref.run_graph(g, frames, emulate_fp16=dtype == "f16")
        worst = 0.0
        for bi in range(1, len(g.buffers)):          # buffer 0: the stem's patch buffer (the fused u8 stem never writes it)
            try:
                got = eng.debug_read_buffer(bi, n).astype(np.float32).transpose(0, 3, 1, 2)
            except capi.HyperposeError as ex:        # the un-pooled output of a conv with the 2x2 max-pool in its epilogue
                assert dtype == "f16" and ex.status == capi.HP_ERR_UNSUPPORTED, ex
                continue
            ref = rbufs[bi].cpu().numpy()
            worst = max(worst, _cmp(got[:, :ref.shape[1]], ref, rel, abs_, f"{wl} {dtype} buffer {bi} {tuple(ref.shape)}"))
        e = [_cmp(x, r.cpu().numpy().reshape(x.shape), rel, abs_, f"{wl} {dtype} output") for x, r in ((a, ra), (b, rb))]
        if dtype == "f16":
            fa, fb, _ = torch_ref.run_graph(g, frames, emulate_fp16=False)
            e += [_cmp(x, r.cpu().numpy().reshape(x.shape), 3e-2, 1e-3, f"{wl} f16 output vs fp32") for x, r in ((a, fa), (b, fb))]
        print(f"[lw parity] {wl} {dtype} {n}/{B} frames: worst buffer {worst:.2e}, outputs {', '.join(f'{v:.2e}' for v in e)}")
    finally:
        eng.close()


@gpu
@pytest.mark.parametrize("net", sorted(NETS))
def test_int8_pack_matches_model(net):
    """a calibrated INT8 pack at 86 x 92 (odd 43-row and 11-row maps), byte for byte against the CPU model of the INT8 engine"""
    from hyperpose_b200 import capi
    from tests import int8_sim
    N, H, Wd = 2, 86, 92
    g = NETS[net][0](0)
    cal = capi.Engine(g.to_pack(), (Wd, H), max_batch_size=N, dtype="tf32")
    g.set_int8_scales(cal.calibrate(syn.make_frames_u8(100, 2 * N, H, Wd)))
    cal.close()
    frames = syn.make_frames_u8(7, N, H, Wd)
    eng = capi.Engine(g.to_pack(), (Wd, H), max_batch_size=N, dtype="int8")
    try:
        eng.infer_u8(frames)
        conf, paf = eng.read_outputs(N)
        c_ref, p_ref, bufs = int8_sim.run_graph(g, g.act_scales, frames_u8=frames)
        for bi in range(len(g.buffers)):
            got = eng.debug_read_buffer(bi, N)
            want = np.ascontiguousarray(np.asarray(bufs[bi]).transpose(0, 2, 3, 1))
            assert np.array_equal(got, want), f"buffer {bi}: {int((got != want).sum())} bytes differ"
        assert conf.tobytes() == c_ref.tobytes() and paf.tobytes() == p_ref.tobytes()
    finally:
        eng.close()


# ---- kernel instantiations at the graphs' shapes ----
def _kernel_cases():
    from tests.test_engine_kernels import conv_case, pool_case, stem_case
    return [
        stem_case(32, 3, 1, (1, 256, 384)),                                                     # block_1_1: u8 stem, 32 channels
        conv_case("f16", 64, 32, 1, 3, (1, 256, 384), pool=True, kernel="halo<64,pool,pp>"),  # block_1_2 + maxpool_1: K padded 32 -> 64
        conv_case("f16", 64, 32, 1, 3, (1, 342, 368), pool=True, kernel="halo<64,pool,pp>"),  # the same at the zoo size (22 x 46 tiles)
        conv_case("f16", 200, 128, 1, 3, (3, 86, 92), kernel="halo<128>"),                    # block_3_1: n-tiles 128 + 72 of 256
        conv_case("f16", 200, 200, 1, 3, (3, 86, 92), kernel="halo<128,pp>"),                 # block_3_2/3: K = 9 x 256 (200 real)
        conv_case("f16", 384, 200, 1, 3, (3, 43, 46), kernel="halo<128>"),                    # block_4_1 on the 43 x 46 map
        pool_case("f16", 128, 2, "maxpool<2>", shape=(2, 171, 184)),                            # maxpool_2 after the odd 171-row map
        pool_case("f16", 200, 2, "maxpool<2>", shape=(2, 86, 92)),                              # maxpool_3 on 200 channels
        conv_case("f16", 512, 512, 1, 3, (1, 46, 54), res_mode=1, kernel="conv<f16,128,res>"),  # block_5_1_2: relu(conv + res)
    ]


KCASES = _kernel_cases()


@gpu
@pytest.mark.parametrize("case", KCASES, ids=[c.id for c in KCASES])
def test_kernel_at_graph_shape_against_fp64(case, monkeypatch):
    from tests.test_engine_kernels import _run_and_check
    _run_and_check(case, monkeypatch, np.random.default_rng(zlib.crc32(case.id.encode())))


# the kernel of every op (Engine.debug_op_kernel) at batch 16 on an H100 (132 SMs); "none": fused into the previous op's launch
_HEAD = (["conv<f16,128>", "halo<128>", "halo<128>", "conv<f16,128,res>", "halo<128>"] + ["halo<128>"] * 3 + ["conv<f16,128>", "conv<f16,64>"] +
         ["conv<f16,128>", "halo<128>", "conv<f16,128,res>"] * 5 + ["conv<f16,128>", "conv<f16,64>"])
KERNELS = {
    "vggtiny_256x384": ["none", "conv<f16,32,stem3>", "halo<64,pool,pp>", "none", "halo<128>", "halo<128,pool,pp>", "none",
                        "halo<128>", "halo<128,pp>", "halo<128,pp>", "maxpool<2>", "halo<128,pp>", "halo<128,pp>"] + _HEAD,
    "vggtiny_342x368": ["none", "conv<f16,32,stem3>", "halo<64,pool,pp>", "none", "halo<128>", "halo<128>", "maxpool<2>",
                        "halo<128>", "halo<128,pp>", "halo<128,pp>", "maxpool<2>", "halo<128,pp>", "halo<128,pp>"] + _HEAD,
    "resnet18_368x432": ["none", "conv<f16,64,stem7>", "maxpool<3>"] + ["conv<f16,64>", "conv<f16,64,res>"] * 2 +
                        ["conv<f16,128>", "dw_strip<3,2>", "dw_strip<1,2>", "conv<f16,128>", "conv<f16,128,res>", "halo<128>",
                         "conv<f16,128,res>", "halo<128>", "conv<f16,128>", "conv<f16,128,res>", "halo<128,pp>", "conv<f16,128,res>",
                         "halo<128,pp>", "conv<f16,128>", "conv<f16,128,res>"] + _HEAD,
}


@gpu
@pytest.mark.parametrize("wl", sorted(WORKLOADS))
def test_layers_land_on_the_expected_kernels(wl, monkeypatch):
    from hyperpose_b200 import capi
    for k in ("HPB_HALO", "HPB_HALO_NARROW", "HPB_NO_POOL_FUSE", "HPB_NO_STEM3"):
        monkeypatch.delenv(k, raising=False)
    net, H, Wd = WORKLOADS[wl]
    g = getattr(models, net)(0)
    eng = capi.Engine(g.to_pack(), (Wd, H), max_batch_size=B)
    got = [eng.debug_op_kernel(i) for i in range(len(g.ops))]
    eng.close()
    print(f"[lw kernels] {wl}: " + ", ".join(f"{op.name}={k}" for op, k in zip(g.ops, got)))
    assert got == KERNELS[wl]


# ---- pose level ----
def _crowd(seed, n, eng):
    return syn.make_batch_tensors(seed, n, (4, 8), eng.out_h, eng.out_w)


@gpu
@pytest.mark.parametrize("wl", sorted(WORKLOADS))
def test_pipelined_pose_call_and_pool_on_crowd_maps(wl):
    """hp_pose_submit_u8_host / hp_pose_collect (two batches in flight) and hp_pool with synthetic crowd conf / paf written over the
    engine outputs: the same hp_human records as hp_paf_process_host on those tensors"""
    from hyperpose_b200 import capi
    net, H, Wd = WORKLOADS[wl]
    pack = getattr(models, net)(0).to_pack()
    n = 8
    eng = capi.Engine(pack, (Wd, H), max_batch_size=n)
    parser = capi.PafParser(0.05, 0.05)
    parser.set_capacity(peaks_per_part=128, candidates_per_limb=2048, humans=64)
    host = capi.PafParser(0.05, 0.05)
    host.set_capacity(peaks_per_part=128, candidates_per_limb=2048, humans=64)
    crowds = [_crowd(300 + k, n, eng) for k in range(3)]
    devs = [tuple(torch.from_numpy(t).cuda() for t in c) for c in crowds]
    torch.cuda.synchronize()
    frames = [torch.from_numpy(syn.make_frames_u8(60 + k, n, H, Wd)).pin_memory().numpy() for k in range(3)]
    want = [host.process_batch(c, p, cap=64) for c, p in crowds]
    assert sum(len(h) for w in want for h in w) > 3 * n * 2, "vacuous: the crowd maps hold too few people"
    got = []
    for k in range(3):                                                      # one override per batch: collect before moving it
        eng.set_output_override(devs[k][0].data_ptr(), devs[k][1].data_ptr())
        t1 = eng.submit_pose(parser, frames[k])
        t2 = eng.submit_pose(parser, frames[(k + 1) % 3])                   # a second batch in flight on the other slot
        got.append((eng.collect_pose(t1, cap=64), eng.collect_pose(t2, cap=64)))
    for k in range(3):
        for h_got in got[k]:
            assert [h.tobytes() for h in h_got] == [h.tobytes() for h in want[k]], f"{wl}: batch {k} differs from hp_paf_process_host"
    eng.close(); parser.close()
    pool = capi.Pool(pack, (Wd, H), n, devices=[0])
    pool.set_capacity(peaks_per_part=128, candidates_per_limb=2048, humans=64)
    pool.set_output_override([devs[0][0].data_ptr()], [devs[0][1].data_ptr()])
    got = pool.run(np.ascontiguousarray(np.concatenate([frames[0], frames[1]])), cap=64)
    assert [h.tobytes() for h in got] == [h.tobytes() for h in want[0] + want[0]], f"{wl}: hp_pool differs from hp_paf_process_host"
    pool.close(); host.close()


@gpu
def test_reference_cli_runs_a_vggtiny_pack(tmp_path):
    """the reference's examples/cli.cpp, unmodified, on a TinyVGG pack at the model zoo's 368 x 342 (an odd 171-row map and a
    43 x 46 output): the operator runtime over an image folder writes one drawn image per input"""
    from tests.test_reference_examples import _exes, _read_p6_stream, _write_inputs
    exes = _exes()
    folder, _, _ = _write_inputs(tmp_path, 3, 342, 368)
    pack = tmp_path / "vggtiny.pack"
    pack.write_bytes(models.lw_openpose_vggtiny(0).to_pack())
    r = subprocess.run([exes["cli"], f"--model={pack}", "--w=368", "--h=342", "--max_batch_size=2", f"--source={folder}", "--runtime=operator",
                        "--post=paf", "--imshow=false", f"--saving_prefix={tmp_path / 'out'}"], capture_output=True, text=True, timeout=300, cwd=tmp_path)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "3 images got processed" in r.stdout, r.stdout
    outs = sorted(p for p in os.listdir(tmp_path) if p.startswith("out_") and p.endswith(".png"))
    assert len(outs) == 3
    assert _read_p6_stream(tmp_path / outs[0])[0].shape == (342, 368, 3)
