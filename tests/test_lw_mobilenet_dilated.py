"""Lightweight-OpenPose on its default backbone, MobilenetDilated (lw_openpose.py:33-37, backbones.py:201-229), and the dilated
depthwise convolution it needs (the first 512 -> 512 block: 3x3, dilation 2, stride 1, TF 'SAME' over the 5 x 5 window).

A graph holds a dilated op's filter as its 5 x 5 window, the nine taps two pixels apart and zeros between them (Graph.add_dwconv); the
pack stores the taps and the dilation.  So the CPU references (oracle/torch_backbone.py, tests/int8_sim.py), which read Op.weight as a
dense depthwise filter, compute the dilated op as it is: the same window, the same SAME padding (2 per side) and, taps row major, the
same order of the nonzero products -- the zero taps add +-0, which leaves a float sum unchanged.

CPU: every existing graph keeps its exact pack; the pack carries the taps and the dilation in the op record (0 for 1); both references
equal an explicit dilated convolution on one op; the imported graph equals a
plain fp32 PyTorch model written from the reference definition (BatchNorm unfolded, F.conv2d(dilation=2, groups=C) with explicit TF
'SAME' padding) at 64 x 96 and an odd 86 x 92; the importers reject wrong lists; the exporter round-trips.

GPU: the dilated kernels (fp16 TMA and column paths, TF32, INT8) against float64 / the INT8 model at the real shape and at small and
odd ones; a dilated op is never paired with another in the dual-filter launch; malformed dilations are refused when the engine is
created; the whole network at 368 x 432 against the backbone oracle (fp16, TF32; batch 16 and a ragged 5); a calibrated INT8 pack
byte for byte; the pipelined pose call on synthetic crowd maps."""
import copy
import hashlib
import struct
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from hyperpose_b200 import export, models, synthetic as syn, weights as W
from oracle import torch_backbone as torch_ref
from tests import test_lw_backbones as tlb
from tests.test_weights_import import _same_pad, _tl_arrays, _TlReader

NET = "lw_openpose_mobilenet_dilated"
build, Weights, order = models.lw_openpose_mobilenet_dilated, W.LwMobilenetDilatedWeights, W.lw_mobilenet_dilated_layer_order

# sha256 of every existing graph's seed-0 pack before depthwise ops could carry a dilation
PACK_SHA256 = {
    "mobilenet_thin_openpose": "3e8e8c2994945432364f1da1c8668db449ddded368f941a2d900c428f99867b3",     # BASELINE cfg2
    "openpose_vgg19": "67e43f7b6aa7b901e395424d4a61b3ae563d6f9cf718169af85ec8edc725488e",              # cfg3
    "resnet50_lw_openpose": "44e23dbdbf5e47a770bd1009ee80d3ca55e74ef832eddbc43d95933f4f9ba5a9",        # cfg4
    "resnet50_pifpaf": "47421c2ff427f6b281a1430140c0b327edfdfbfc9668c623fdda62227d1afe4c",             # cfg5
    "ppn_resnet18": "6ffde33eee985ac5b825ac69cc654477b77c3106618dc01753251dad746e3bca",
    "ppn_resnet50": "95ebdd64e27b36bbd1cd1db43c5746202c1c9a794a160bbc77c8091000f5dc21",
    "lw_openpose_vggtiny": "ef5a372fea0b46611acb03612e8e3a7a749e44856f7f5251fc05d90da9c35630",
    "lw_openpose_resnet18": "ed9ee633fbe07d7139bfc0062f27dab2caf206eabceb7ba039168f3721634860",
    "tiny_test_net": "01f4fc6fce6b1c9ba83df7d7c538d96bfd5899d5c9363c7e38f9cc8942a580bd",
}


# ================================================ CPU ===========================================================================
@pytest.mark.parametrize("net", sorted(PACK_SHA256))
def test_existing_packs_are_unchanged(net):
    assert hashlib.sha256(getattr(models, net)(seed=0).to_pack()).hexdigest() == PACK_SHA256[net]


def test_pack_carries_the_dilation():
    """the op record's dilation field: 2 on the dilated depthwise op, 0 (= 1) on every other op"""
    g = build(0)
    pack = g.to_pack()
    nb = len(g.buffers)
    fields = [struct.unpack_from("<18I3Q", pack, 72 + 8 * nb + 96 * i) for i in range(len(g.ops))]
    assert [(op.name, f[17]) for op, f in zip(g.ops, fields) if f[17]] == [("convblock_7_dw", 2)]
    op = g.ops[[o.name for o in g.ops].index("convblock_7_dw")]
    assert (op.type, op.R, op.stride, op.cout_g, op.dilation) == (models.OP_DWCONV, 3, 1, 512, 2)
    assert op.weight.shape == (512, 5, 5) and np.array_equal(op.taps(), op.weight[:, ::2, ::2])
    w_off = fields[g.ops.index(op)][18]
    blob0 = 72 + 8 * nb + 96 * len(g.ops)
    assert np.array_equal(np.frombuffer(pack, "<f4", 512 * 9, blob0 + 4 * w_off).reshape(512, 3, 3), op.taps())   # the taps, not the window
    plain = _with_dilation_1(g)
    assert g.flops_per_frame(368, 432) == plain.flops_per_frame(368, 432)     # nine taps per output either way
    assert plain.to_pack() != pack and len(plain.to_pack()) == len(pack)


def _with_dilation_1(g):
    """the same graph with the dilated op undilated (the same nine taps, adjacent)"""
    g = copy.deepcopy(g)
    for op in g.ops:
        op.weight, op.dilation = op.taps(), 1
    return g


def test_references_compute_the_dilated_op():
    """oracle/torch_backbone.py and tests/int8_sim.py on a graph with one dilated op: the dilated convolution, against F.conv2d(dilation=2)
    with explicit TF 'SAME' padding and against the INT8 model's arithmetic written out with tap offsets r*2, t*2"""
    from tests import int8_sim
    rng = np.random.default_rng(3)
    N, C, H, Wd = 2, 16, 9, 11
    g = models.Graph("d", 19, 38, 0)
    a, b = g.add_buffer(C, 0), g.add_buffer(C, 0)
    w = rng.standard_normal((C, 3, 3)).astype(np.float32)
    bias, alpha = rng.standard_normal(C).astype(np.float32), rng.uniform(0, 1, C).astype(np.float32)
    g.add_dwconv(a, b, w, bias, alpha, dilation=2)
    x = rng.standard_normal((N, C, H, Wd))
    frames = np.zeros((N, H, Wd, 3), np.uint8)
    _, _, bufs = torch_ref.run_graph(g, frames, device="cpu", dtype=torch.float64, init={a: x})
    y = F.conv2d(F.pad(torch.from_numpy(x), (2, 2, 2, 2)), torch.from_numpy(w.astype(np.float64)).view(C, 1, 3, 3),
                 torch.from_numpy(bias.astype(np.float64)), dilation=2, groups=C)
    y = torch.where(y > 0, y, y * torch.from_numpy(alpha.astype(np.float64)).view(1, -1, 1, 1))
    assert torch.allclose(bufs[b], y, rtol=1e-12, atol=1e-12)
    s = np.array([0.02, 0.03], np.float32)
    q = rng.integers(-127, 128, (N, C, H, Wd)).astype(np.int8)
    _, _, qb = int8_sim.run_graph(g, s, init={a: q}, N=N, HW=(H, Wd))
    xf = (q.astype(np.float32) * s[0]).astype(np.float32)
    xp = np.zeros((N, C, H + 4, Wd + 4), np.float32); xp[:, :, 2:2 + H, 2:2 + Wd] = xf
    acc = np.zeros((N, C, H, Wd), np.float32)
    for r in range(3):
        for t in range(3):
            acc = (acc + (xp[:, :, 2 * r:2 * r + H, 2 * t:2 * t + Wd] * w[:, r, t].reshape(1, -1, 1, 1)).astype(np.float32)).astype(np.float32)
    v = (acc + bias.reshape(1, -1, 1, 1)).astype(np.float32)
    v = np.where(v > 0, v, (v * alpha.reshape(1, -1, 1, 1)).astype(np.float32)).astype(np.float32)
    assert np.array_equal(qb[b], int8_sim.quantize(v, np.float32(1.0) / s[1]))


@pytest.mark.parametrize("bad", [dict(dilation=3), dict(dilation=2, stride=2), dict(dilation=2, K=1)])
def test_graph_refuses_unsupported_dilations(bad):
    g = models.Graph("x")
    a, b = g.add_buffer(64, 0), g.add_buffer(64, 1 if bad.get("stride") == 2 else 0)
    K = bad.get("K", 3)
    with pytest.raises(AssertionError):
        g.add_dwconv(a, b, np.ones((64, K, K), np.float32), np.zeros(64, np.float32), np.zeros(64, np.float32), stride=bad.get("stride", 1),
                     dilation=bad["dilation"])


def _backbone_reference(r, x):
    """MobilenetDilated_backbone (backbones.py:201-229): conv_block = Conv2d(+bias, relu) + BatchNorm(relu) (the second definition,
    :234-239), then dw_conv_block = DepthwiseConv2d(no bias) + BN(relu), Conv2d 1x1 (no bias) + BN(relu), eleven times"""
    x = F.relu(r.bn(F.relu(r.conv(x, stride=2))))
    for co, st, dil in models.MOBILENET_DILATED_BLOCKS:
        if dil == 1:
            x = r.dwconv(x, st)
        else:
            f = next(r.it)                                                     # [kh, kw, C, 1]
            k = (f.shape[0] - 1) * dil + 1
            x = F.conv2d(_same_pad(x, k, st), torch.from_numpy(f.transpose(2, 3, 0, 1).copy()), None, stride=st, dilation=dil,
                         groups=f.shape[2])
        x = F.relu(r.bn(x))
        x = F.relu(r.bn(r.conv(x, bias=False)))
        assert x.shape[1] == co
    return x


@pytest.mark.parametrize("hw", [(64, 96), (86, 92)])
def test_imported_graph_equals_reference_definition(hw, tmp_path):
    arrays = _tl_arrays(order(), 61)
    tlb._params_npz(tmp_path / "w.npz", arrays)
    g = build(weights=Weights.from_npz(str(tmp_path / "w.npz")))
    assert g.to_pack() == build(weights=Weights(arrays)).to_pack()
    H, Wd = hw
    frames = np.random.default_rng(8).integers(0, 256, (2, H, Wd, 3), dtype=np.uint8)
    conf, paf, _ = torch_ref.run_graph(g, frames, flip_rgb=True, device="cpu")
    x = torch.from_numpy(np.ascontiguousarray((frames.astype(np.float64) / 255).astype(np.float32)[..., ::-1].transpose(0, 3, 1, 2)))
    r = _TlReader(arrays)
    rc, rp = tlb._lw_head_reference(r, _backbone_reference(r, x))
    h8, w8 = -(-H // 8), -(-Wd // 8)
    assert conf.shape == rc.shape == (2, 19, h8, w8) and paf.shape == rp.shape == (2, 38, h8, w8)
    tol = 2e-4 * max(1.0, float(rc.abs().max()), float(rp.abs().max()))
    assert float((conf.cpu() - rc).abs().max()) < tol and float((paf.cpu() - rp).abs().max()) < tol
    # the check sees the dilation: the same weights undilated give other maps
    c1, _, _ = torch_ref.run_graph(_with_dilation_1(g), frames, flip_rgb=True, device="cpu")
    assert float((c1 - conf).abs().max()) > 10 * tol


def test_seeded_graph_has_the_imported_layout():
    g = build(0)
    assert tlb._layout(g) == tlb._layout(build(weights=Weights(_tl_arrays(order(), 3))))
    assert [(o.name, o.dilation) for o in g.ops] == [(o.name, o.dilation) for o in build(weights=Weights(_tl_arrays(order(), 3))).ops]
    assert g.to_pack() == build(0).to_pack() != build(1).to_pack()


def test_graph_shapes():
    g = build(0)
    assert (g.head_type, g.out_down_shift, g.conf_channels, g.paf_channels, g.mean) == (0, 3, 19, 38, (0.0, 0.0, 0.0))
    assert g.ops[-1].out_mode == models.OUT_F32_NCHW_SPLIT and g.ops[-1].split == 19
    dws = [op for op in g.ops if op.type == models.OP_DWCONV]
    assert [(op.R, op.stride, op.cout_g, op.dilation) for op in dws] == [(1, 1, 32, 1)] + [
        (3, st, ci, dil) for (_, st, dil), ci in zip(models.MOBILENET_DILATED_BLOCKS, [32, 64, 128, 128, 256, 256] + [512] * 5)]
    assert all(np.all(op.alpha == 0) for op in g.ops if op.name.startswith("convblock_"))         # every BatchNorm has ReLU
    cpm = next(op for op in g.ops if op.name == "cpm_init")
    assert cpm.weight.shape == (1, 128, 512, 1, 1) and g.buffers[cpm.in_buf] == (512, 3)
    head = [e for e in order() if e[1].split(".")[0] in ("cpm", "init", "ref")]
    assert order()[-len(head):] == head == W.lw_resnet18_layer_order()[-len(head):]       # the shared LW head on 512 channels
    assert len(order()) - len(head) == 2 + 11 * 4                                           # stem conv + BN, eleven separable blocks


def test_importer_rejects_wrong_lists():
    arrays = _tl_arrays(order(), 4)
    with pytest.raises(ValueError):
        Weights(arrays[:-1])
    with pytest.raises(ValueError):
        Weights(arrays + [np.zeros(3, np.float32)])
    bad = list(arrays)
    i = next(k for k, a in enumerate(bad) if a.ndim == 4 and a.shape[3] == 1 and a.shape[2] == 512)   # a 512-channel depthwise filter
    bad[i] = np.zeros((5, 5, 512, 1), np.float32)
    with pytest.raises(ValueError):
        Weights(bad)
    with pytest.raises(ValueError):
        W.MobilenetThinWeights(arrays)


def test_export_round_trips(tmp_path):
    out = tmp_path / f"{NET}.pack"
    assert export.main(["--model", NET, "--out", str(out), "--seed", "3"]) == 0
    assert out.read_bytes() == build(3).to_pack()
    arrays = _tl_arrays(order(), 12)
    tlb._params_npz(tmp_path / "w.npz", arrays)
    out2 = tmp_path / f"{NET}_trained.pack"
    assert export.main(["--model", NET, "--out", str(out2), "--weights", str(tmp_path / "w.npz")]) == 0
    assert out2.read_bytes() == build(weights=Weights(arrays)).to_pack()


# ================================================ GPU ===========================================================================
gpu = pytest.mark.gpu
H0, W0, B = 368, 432, 16          # the published size: 46 x 54 maps at stride 8


# ---- the dilated kernels against float64 (tests/test_engine_kernels.py's checks; its reference reads the dilated op's window) ----
def _dw_case(dtype, C, shape, kernel, env=None, max_batch=None, mixed_pair=False, seed=0):
    """one dilated 3x3 depthwise op (or, mixed_pair: an undilated and a dilated op on the same input, the shape of a dual-filter
    launch) between offset channel ranges"""
    from tests.test_engine_kernels import Case, _graph, _r, _slopes
    rng = np.random.default_rng(seed)
    g = _graph("dwd")
    in_off, out_off = 8, 16
    n = 2 if mixed_pair else 1
    b_in = g.add_buffer(_r(in_off + C + 8, 8), 0)
    b_out = g.add_buffer(_r(out_off + n * C + 8, 8), 0)
    outs = []
    for j in range(n):
        w = (rng.standard_normal((C, 3, 3)) * np.sqrt(2.0 / 9)).astype(np.float32)
        g.add_dwconv(b_in, b_out, w, rng.standard_normal(C).astype(np.float32) * 0.5, _slopes(rng, C), in_ch_off=in_off,
                     out_ch_off=out_off + j * C, dilation=2 if j == n - 1 else 1)
        outs.append((b_out, out_off + j * C, C))
    kernels = kernel if isinstance(kernel, list) else [kernel]
    cid = f"{dtype}-{'+'.join(kernels)}-C{C}-d2-{'x'.join(map(str, shape))}" + (f"-max{max_batch}" if max_batch else "") + \
          (f"-{','.join(f'{k}={v}' for k, v in env.items())}" if env else "")
    return Case(cid, dtype, shape, g, kernels, outs, 9, env=env, mutate=n - 1, max_batch=max_batch)


NO_TMA = {"HPB_NO_DW_TMA": "1"}
DW_CASES = [
    _dw_case("f16", 512, (B, 46, 54), "dw_tma<1,d2>"),                                  # convblock_7_dw at 368 x 432, batch 16
    _dw_case("f16", 512, (5, 46, 54), "dw_tma<1,d2>", max_batch=B),                     # a ragged batch on a batch-16 engine
    _dw_case("f16", 512, (B, 46, 54), "dw_col<d2>", env=NO_TMA),                        # the column path at the same shape
    _dw_case("f16", 512, (5, 46, 54), "dw_col<d2>", env=NO_TMA, max_batch=B),
    _dw_case("f16", 64, (2, 13, 21), "dw_tma<1,d2>"),                                   # odd rows and columns: both phases ragged
    _dw_case("f16", 72, (2, 13, 21), "dw_col<d2>"),                                     # 72 channels: no TMA plan
    _dw_case("f16", 64, (3, 3, 5), "dw_tma<1,d2>"),                                     # a map smaller than one tile and than the window
    _dw_case("f16", 72, (3, 3, 5), "dw_col<d2>"),
    _dw_case("f16", 192, (1, 20, 130), "dw_tma<1,d2>"),                                 # three 64-channel tiles, 44 + 44 + 42 columns
    _dw_case("f16", 64, (2, 13, 21), ["dw_tma<1>", "dw_tma<1,d2>"], mixed_pair=True),   # same input as an undilated op: not paired
    _dw_case("tf32", 512, (5, 46, 54), "dw_f32<d2>", max_batch=B),
    _dw_case("tf32", 64, (2, 13, 21), "dw_f32<d2>"),
    _dw_case("tf32", 72, (3, 3, 5), "dw_f32<d2>"),
]


@gpu
@pytest.mark.parametrize("case", DW_CASES, ids=[c.id for c in DW_CASES])
def test_dilated_kernel_against_fp64(case, monkeypatch):
    from tests import test_engine_kernels as tek
    tek._run_and_check(case, monkeypatch, np.random.default_rng(zlib.crc32(case.id.encode())))


@gpu
@pytest.mark.parametrize("C,shape", [(512, (B, 46, 54)), (512, (5, 46, 54)), (64, (2, 13, 21)), (72, (2, 13, 21)), (64, (3, 3, 5))])
def test_dilated_int8_kernel_matches_model(C, shape):
    """dwconv_c4_kernel<int8_t> with dilation 2, byte for byte against tests/int8_sim.py (batch-16 engine)"""
    from hyperpose_b200 import capi
    from tests import int8_sim
    from tests.test_engine_kernels import _graph, _slopes
    N, H, Wd = shape
    rng = np.random.default_rng(C + N)
    g = _graph("dwd8")
    a, b = g.add_buffer(C + 16, 0), g.add_buffer(C + 24, 0)
    g.add_dwconv(a, b, (rng.standard_normal((C, 3, 3)) * 0.4).astype(np.float32), rng.standard_normal(C).astype(np.float32) * 0.3,
                 _slopes(rng, C), in_ch_off=8, out_ch_off=16, dilation=2)
    g.act_scales = np.array([0.03, 0.02], np.float32)
    eng = capi.Engine(g.to_pack(), (Wd, H), max_batch_size=max(N, B if C == 512 else N), dtype="int8")
    try:
        assert eng.debug_op_kernel(0) == "dw_i8<d2>"
        x = rng.integers(-127, 128, (N, H, Wd, C + 16), dtype=np.int8)
        y0 = rng.integers(-127, 128, (N, H, Wd, C + 24), dtype=np.int8)
        eng.debug_write_buffer(a, x); eng.debug_write_buffer(b, y0)
        eng.debug_run_ops(0, 0, N)
        got = eng.debug_read_buffer(b, N)
    finally:
        eng.close()
    init = {a: x.transpose(0, 3, 1, 2), b: y0.transpose(0, 3, 1, 2)}
    _, _, bufs = int8_sim.run_graph(g, g.act_scales, init=init, N=N, HW=(H, Wd))
    want = np.ascontiguousarray(bufs[b].transpose(0, 2, 3, 1))
    assert np.array_equal(got, want), f"{int((got != want).sum())} bytes differ"
    plain, _, pb = int8_sim.run_graph(_with_dilation_1(g), g.act_scales, init=init, N=N, HW=(H, Wd))
    assert not np.array_equal(np.ascontiguousarray(pb[b].transpose(0, 2, 3, 1)), got)


# ---- the pack is checked when the engine is created ----
def _one_op_graph(kind):
    g = models.Graph("bad", 19, 38, 0)
    a, b = g.add_buffer(64, 0), g.add_buffer(64, 1 if kind == "stride2" else 0)
    w3 = np.ones((64, 3, 3), np.float32) / 9
    z = np.zeros(64, np.float32)
    if kind == "conv":
        g.add_conv(a, b, np.ones((1, 64, 64, 3, 3), np.float32), z, z)
    elif kind == "maxpool":
        b = g.add_buffer(64, 1); g.add_maxpool(a, b, 64)
    else:
        g.add_dwconv(a, b, np.ones((64, 1, 1), np.float32) if kind in ("1x1", "huge") else w3, z, z, stride=2 if kind == "stride2" else 1)
    op = g.ops[-1]
    op.dilation = {"d3": 3, "huge": 0x80000000}.get(kind, 2)
    if op.type == models.OP_DWCONV and op.R == 3:    # the record add_dwconv refuses to make: the window of that dilation around the taps
        win = np.zeros((64, 2 * op.dilation + 1, 2 * op.dilation + 1), np.float32)
        win[:, ::op.dilation, ::op.dilation] = w3
        op.weight = win
    return g


@gpu
@pytest.mark.parametrize("kind", ["d3", "huge", "stride2", "1x1", "conv", "maxpool"])
def test_malformed_dilation_is_refused(kind):
    from tests.test_engine_kernels import _expect_rejected
    _expect_rejected(_one_op_graph(kind), "dilation")


# ---- the whole network at the published size ----
@gpu
@pytest.mark.parametrize("n", [B, 5])
@pytest.mark.parametrize("dtype", ["f16", "tf32"])
def test_full_size_parity(dtype, n):
    """every buffer and both outputs against the backbone oracle on a batch-16 engine running n frames; the budgets of
    tests/test_lw_backbones.py"""
    from hyperpose_b200 import capi
    g = build(0)
    frames = syn.make_frames_u8(40 + n, n, H0, W0)
    eng = capi.Engine(g.to_pack(), (W0, H0), max_batch_size=B, dtype=dtype)
    try:
        eng.infer_u8(frames)
        a, b = eng.read_outputs(n)
        assert a.shape == (n, 19, 46, 54) and b.shape == (n, 38, 46, 54)
        rel, abs_ = (6e-3, 6e-3) if dtype == "f16" else (6e-3, 1e-3)
        ra, rb, rbufs = torch_ref.run_graph(g, frames, emulate_fp16=dtype == "f16")
        worst = 0.0
        for bi in range(1, len(g.buffers)):          # buffer 0: the stem's patch buffer (the fused u8 stem never writes it)
            try:
                got = eng.debug_read_buffer(bi, n).astype(np.float32).transpose(0, 3, 1, 2)
            except capi.HyperposeError as ex:        # a tensor whose consumer runs in the producer's epilogue
                assert dtype == "f16" and ex.status == capi.HP_ERR_UNSUPPORTED, ex
                continue
            ref = rbufs[bi].cpu().numpy()
            worst = max(worst, tlb._cmp(got[:, :ref.shape[1]], ref, rel, abs_, f"{dtype} buffer {bi} {tuple(ref.shape)}"))
        e = [tlb._cmp(x, r.cpu().numpy().reshape(x.shape), rel, abs_, f"{dtype} output") for x, r in ((a, ra), (b, rb))]
        if dtype == "f16":
            fa, fb, _ = torch_ref.run_graph(g, frames, emulate_fp16=False)
            e += [tlb._cmp(x, r.cpu().numpy().reshape(x.shape), 3e-2, 1e-3, "f16 output vs fp32") for x, r in ((a, fa), (b, fb))]
        print(f"[lw dilated parity] {dtype} {n}/{B} frames: worst buffer {worst:.2e}, outputs {', '.join(f'{v:.2e}' for v in e)}")
    finally:
        eng.close()


@gpu
def test_int8_pack_matches_model():
    """a calibrated INT8 pack at 86 x 92 (odd 43-row and 11-row maps), byte for byte against the CPU model of the INT8 engine"""
    from hyperpose_b200 import capi
    from tests import int8_sim
    N, H, Wd = 2, 86, 92
    g = build(0)
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


@gpu
@pytest.mark.parametrize("dtype,env,dilated_kernel", [("f16", {}, "dw_tma<1,d2>"), ("f16", NO_TMA, "dw_col<d2>"), ("tf32", {}, "dw_f32<d2>")])
def test_launch_list(dtype, env, dilated_kernel, monkeypatch):
    """the dilated layer lands on its dilated kernel; no dilated op is in a dual-filter launch"""
    from hyperpose_b200 import capi
    for k in ("HPB_HALO", "HPB_HALO_NARROW", "HPB_NO_POOL_FUSE", "HPB_NO_STEM3", "HPB_NO_DW_TMA", "HPB_NO_DW_DUAL", "HPB_NO_DW1_FUSE"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    g = build(0)
    eng = capi.Engine(g.to_pack(), (W0, H0), max_batch_size=B, dtype=dtype)
    got = [eng.debug_op_kernel(i) for i in range(len(g.ops))]
    eng.close()
    print(f"[lw dilated kernels] {dtype} {env}: " + ", ".join(f"{op.name}={k}" for op, k in zip(g.ops, got)))
    assert [k for op, k in zip(g.ops, got) if op.dilation != 1] == [dilated_kernel]
    assert [op.name for op, k in zip(g.ops, got) if "d2" in k] == ["convblock_7_dw"]
    for i, k in enumerate(got):
        if k == "dw_tma<2>":
            assert g.ops[i].dilation == 1 and g.ops[i + 1].dilation == 1


@gpu
def test_pipelined_pose_call_on_crowd_maps(monkeypatch):
    """hp_pose_submit_u8_host / hp_pose_collect (two batches in flight) and hp_pool on synthetic crowd maps written over the outputs:
    the same hp_human records as hp_paf_process_host (tests/test_lw_backbones.py's check on this network)"""
    monkeypatch.setitem(tlb.WORKLOADS, "mobilenet_dilated_368x432", (NET, H0, W0))
    tlb.test_pipelined_pose_call_and_pool_on_crowd_maps("mobilenet_dilated_368x432")
