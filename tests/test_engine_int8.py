"""The INT8 engine (HP_DTYPE_INT8, data_type::kINT8) against its CPU model (tests/int8_sim.py), byte for byte: every conv kernel
instantiation and helper kernel in one- or two-op graphs, four whole networks with scales from Engine.calibrate, the calibration
itself (bit for bit against an op-by-op replay at the benchmark batches, short chunks and chunk sums included), the packs an INT8
engine refuses, and the pose paths on an INT8 engine.  The networks at the benchmarks' plans are in tests/test_network_ops.py.

The one-op cases also run every conv kernel with more work items than CTAs (the persistent kernel carries its stage ring from one item
to the next), the conf / PAF output conv, and batches shorter than the engine's max_batch: there the frames past N of the input
buffers hold 127, and every byte past frame N, in every buffer and conf / paf plane, must keep its value."""
import os
import struct
import subprocess

import numpy as np
import pytest

from hyperpose_b200 import build as hb, capi, models, synthetic as syn
from tests import int8_sim

gpu = pytest.mark.gpu

BNS = (16, 32, 48, 64, 96, 128)
CONV_KERNELS = {f"conv<i8,{b}>" for b in BNS} | {f"conv<i8,{b},res>" for b in BNS}
BN_OF = {13: 16, 19: 32, 24: 32, 40: 48, 57: 64, 72: 96, 160: 96, 200: 128, 288: 96, 16: 16, 32: 32, 48: 48, 64: 64, 96: 96, 128: 128}
S1, S2, S3 = (2, 13, 21), (3, 5, 7), (1, 40, 72)
MEAN = (0.41, 0.52, 0.37)


def _r(x, m):
    return (x + m - 1) // m * m


def _graph(name):
    return models.Graph(name, conf_channels=19, paf_channels=38, out_down_shift=0, mean=MEAN)


def _nchw(a):
    return np.ascontiguousarray(a.transpose(0, 3, 1, 2))


def _nhwc(a):
    return np.ascontiguousarray(a.transpose(0, 2, 3, 1))


class Case:
    def __init__(self, cid, shape, graph, kernels, scales, fill=None, entry=None, max_batch=None):
        self.id, self.shape, self.graph, self.kernels, self.scales = cid, shape, graph, kernels, np.asarray(scales, np.float32)
        self.fill = fill or {}   # {buffer: (first channel, value)}
        self.entry = entry       # None (buffers written directly) | "u8" | "f32"
        self.max_batch = max_batch or shape[0]   # the engine's max_batch_size; the case runs shape[0] frames
        if self.max_batch != shape[0]:
            self.id += f"-max{self.max_batch}"


def conv_case(cout, cin=64, G=1, R=3, shape=S1, in_off=0, out_off=0, res_mode=0, res_off=0, pad127=False, seed=0, max_batch=None):
    rng = np.random.default_rng(seed)
    g = _graph("conv")
    b_in = g.add_buffer(_r(in_off + G * cin + (16 if in_off else 0), 16), 0)
    b_out = g.add_buffer(_r(out_off + G * cout + 8, 8), 0)
    kw = {}
    scales = [1 / 64, 4 / 127]
    if res_mode:
        kw = dict(res_buf=g.add_buffer(_r(res_off + G * cout + 8, 8), 0), res_ch_off=res_off, res_mode=res_mode)
        scales.append(1 / 50)
    w = (rng.standard_normal((G, cout, cin, R, R)) * np.sqrt(2.0 / (cin * R * R))).astype(np.float32)
    g.add_conv(b_in, b_out, w, rng.standard_normal(G * cout).astype(np.float32) * 0.5, rng.uniform(-0.5, 1.0, G * cout).astype(np.float32),
               in_ch_off=in_off, out_ch_off=out_off, **kw)
    k = f"conv<i8,{BN_OF[cout]}" + (",res>" if res_mode else ">")
    cid = f"{k}-cout{cout}-cin{cin}-G{G}-{R}x{R}-{'x'.join(map(str, shape))}" + (f"-in{in_off}" if in_off else "") + \
          (f"-out{out_off}" if out_off else "") + (f"-res{res_mode}@{res_off}" if res_mode else "") + ("-pad127" if pad127 else "")
    return Case(cid, shape, g, [k], scales, fill={b_in: (in_off + G * cin, 127)} if pad127 else None, max_batch=max_batch)


def split_case(conf, paf, cin, R, shape, max_batch=None, seed=3):
    """the output conv: conf / paf planes of fp32 y, conf channels first"""
    rng = np.random.default_rng(seed)
    g = models.Graph("split", conf_channels=conf, paf_channels=paf, out_down_shift=0, mean=MEAN)
    b_in = g.add_buffer(_r(cin, 16), 0)
    co = conf + paf
    g.add_conv(b_in, 0, (rng.standard_normal((1, co, cin, R, R)) * np.sqrt(2.0 / (cin * R * R))).astype(np.float32),
               rng.standard_normal(co).astype(np.float32) * 0.5, rng.uniform(-0.5, 1.0, co).astype(np.float32),
               out_mode=models.OUT_F32_NCHW_SPLIT, split=conf)
    k = f"conv<i8,{BN_OF[co]}>"
    return Case(f"{k}-split{conf}+{paf}-cin{cin}-{R}x{R}-{'x'.join(map(str, shape))}", shape, g, [k], [1 / 64], max_batch=max_batch)


def stem_case(cout, R, stride, shape, entry, max_batch=None):
    rng = np.random.default_rng(1)
    g = _graph("stem")
    d = 1 if stride == 2 else 0
    col = g.add_buffer(_r(R * R * 3, 64), d)
    g.add_im2col(col, stride=stride, ksize=R)
    out = g.add_buffer(_r(cout + 8, 8), d)
    g.add_conv(col, out, (rng.standard_normal((1, cout, 3, R, R)) * np.sqrt(2.0 / (3 * R * R))).astype(np.float32),
               rng.standard_normal(cout).astype(np.float32) * 0.5, rng.uniform(-0.5, 1.0, cout).astype(np.float32), im2col_input=1)
    k = f"conv<i8,{BN_OF[cout]}>"
    return Case(f"im2col_i8-{entry}-{R}x{R}-s{stride}-{k}-{'x'.join(map(str, shape))}", shape, g, ["im2col_i8", k], [1 / 127, 3 / 127], entry=entry,
                max_batch=max_batch)


def dw_case(C, K, stride, shape=S1, in_off=16, out_off=8, max_batch=None):
    rng = np.random.default_rng(2)
    g = _graph("dw")
    b_in = g.add_buffer(_r(in_off + C + 8, 8), 0)
    b_out = g.add_buffer(_r(out_off + C + 8, 8), 1 if stride == 2 else 0)
    g.add_dwconv(b_in, b_out, (rng.standard_normal((C, K, K)) * np.sqrt(2.0 / (K * K))).astype(np.float32), rng.standard_normal(C).astype(np.float32) * 0.5,
                 rng.uniform(-0.5, 1.0, C).astype(np.float32), stride=stride, in_ch_off=in_off, out_ch_off=out_off)
    return Case(f"dw_i8-C{C}-{K}x{K}-s{stride}-{'x'.join(map(str, shape))}", shape, g, ["dw_i8"], [1 / 64, 3 / 127], max_batch=max_batch)


def pool_case(C, K, shape=S1, in_off=8, out_off=16, max_batch=None):
    g = _graph("pool")
    b_in = g.add_buffer(_r(in_off + C + 8, 8), 0)
    b_out = g.add_buffer(_r(out_off + C + 8, 8), 1)
    g.add_maxpool(b_in, b_out, C, ksize=K)
    g.ops[-1].in_ch_off, g.ops[-1].out_ch_off = in_off, out_off
    return Case(f"maxpool_i8-K{K}-C{C}-{'x'.join(map(str, shape))}", shape, g, ["maxpool_i8"], [0.05, 0.05], max_batch=max_batch)


def _cases():
    cs = []
    for cout, R, shape, cin, in_off in [(13, 3, S1, 64, 0), (24, 1, S2, 64, 0), (40, 7, S1, 64, 0), (57, 3, S3, 128, 0), (72, 1, S1, 192, 64),
                                        (200, 3, S2, 64, 0), (288, 1, S3, 64, 0), (24, 3, S1, 320, 16)]:
        cs.append(conv_case(cout, cin, 1, R, shape, in_off=in_off))
    cs.append(conv_case(40, 128, 3, 3, S2))                        # 3 groups
    cs.append(conv_case(19, 64, 2, 1, S1, out_off=8))              # two 64-channel groups: group 0's k-step reads on into group 1
    cs.append(conv_case(57, 160, 2, 1, S2))                        # groups of 160 channels: the padded k-step of group 0 reads group 1
    cs.append(conv_case(57, 185, 1, 3, S1, pad127=True))           # 185 of 192 channels, the pad channels hold 127
    for i, cout in enumerate(BNS):
        cs.append(conv_case(cout, 64, 1, (3, 1)[i % 2], (S1, S2, S3)[i % 3], res_mode=1 + i % 2, res_off=(0, 8, 16)[i % 3], out_off=(0, 8)[i % 2]))
    for entry in ("u8", "f32"):
        cs.append(stem_case(40, 3, 1, (2, 13, 21), entry))
        cs.append(stem_case(57, 7, 2, (1, 40, 72), entry))
    cs += [dw_case(40, k, s) for k in (1, 3) for s in (1, 2)]
    cs += [pool_case(40, 2), pool_case(24, 3), pool_case(40, 3, shape=S3)]
    # one frame short of max_batch
    cs += [conv_case(40, 64, 1, 3, S1, max_batch=4), conv_case(64, 64, 1, 1, S2, res_mode=2, res_off=8, max_batch=5),
           stem_case(40, 3, 1, (2, 13, 21), "u8", max_batch=3), stem_case(57, 7, 2, (1, 40, 72), "f32", max_batch=2),
           dw_case(40, 3, 1, max_batch=3), dw_case(40, 1, 2, max_batch=3), pool_case(40, 3, max_batch=3)]
    # the conf / PAF output conv: the split inside the one BN 64 n-tile, and in the second BN 96 n-tile
    cs += [split_case(19, 38, 64, 1, S1), split_case(19, 38, 64, 3, S1, max_batch=3), split_case(100, 60, 64, 3, S2, max_batch=4)]
    return cs


CASES = _cases()


def _multi_round():
    """more items than CTAs (136 .. 272), one frame short of max_batch: all 12 conv kernels, grouped layers, concat offsets, ragged
    last n-tiles, odd k-step counts (1 x 1 and 3 x 3 over one 128-channel chunk), and the output conv"""
    cs = []
    for bn, cout, G, R, shape, out_off in [(16, 13, 4, 1, (3, 40, 72), 8), (32, 24, 1, 3, (1, 130, 140), 0), (48, 40, 2, 3, (2, 45, 97), 0),
                                           (64, 57, 1, 1, (2, 97, 99), 8), (96, 288, 1, 1, (1, 70, 97), 0), (128, 200, 1, 1, (1, 60, 149), 8)]:
        cs.append(conv_case(cout, 64, G, R, shape, out_off=out_off, max_batch=shape[0] + 1))
    for i, (cout, G, R, shape) in enumerate([(16, 4, 3, (3, 40, 72)), (32, 2, 1, (2, 45, 97)), (48, 1, 3, (1, 130, 140)), (64, 1, 1, (2, 97, 99)),
                                             (96, 2, 1, (2, 60, 72)), (128, 1, 1, (1, 130, 140))]):
        cs.append(conv_case(cout, 64, G, R, shape, res_mode=1 + i % 2, res_off=(0, 8, 16)[i % 3], out_off=(0, 8)[i % 2], max_batch=shape[0] + 1))
    cs.append(split_case(19, 38, 64, 1, (2, 97, 99), max_batch=3))
    return cs


MULTI = _multi_round()


def _buf_shape(g, bi, N, H, W):
    c, d = g.buffers[bi]
    for _ in range(d):
        H, W = (H + 1) // 2, (W + 1) // 2
    return N, H, W, c


def _int8_graph(g, scales):
    g.act_scales = np.asarray(scales, np.float32)
    return g


def _run_int8_case(case):
    g = _int8_graph(case.graph, case.scales)
    N, H, W = case.shape
    M = case.max_batch
    split = any(op.type == models.OP_CONV and op.out_mode == models.OUT_F32_NCHW_SPLIT for op in g.ops)
    eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=M, dtype="int8")
    try:
        names = [eng.debug_op_kernel(i) for i in range(len(g.ops))]
        assert names == case.kernels, names
        rng = np.random.default_rng(7)
        if split and N < M:   # the planes' frames past N: what a run over all M frames of other contents left there
            for bi in range(len(g.buffers)):
                eng.debug_write_buffer(bi, rng.integers(-127, 128, _buf_shape(g, bi, M, H, W)).astype(np.int8))
            eng.debug_run_ops(0, len(g.ops) - 1, M)
            planes_before = eng.read_outputs(M)
        written = {op.out_buf for op in g.ops if not (op.type == models.OP_CONV and op.out_mode == models.OUT_F32_NCHW_SPLIT)}
        init = {}
        for bi in range(len(g.buffers)):   # every buffer: random bytes (the output channels outside the op must keep theirs)
            a = rng.integers(-127, 128, _buf_shape(g, bi, M, H, W)).astype(np.int8)
            if bi in case.fill:
                a[..., case.fill[bi][0]:] = case.fill[bi][1]
            if bi not in written:
                a[N:] = 127    # input frames past N: an output that reads them comes out wrong
            init[bi] = a
            eng.debug_write_buffer(bi, a)
        if case.entry == "u8":
            frames = syn.make_frames_u8(3, N, H, W)
            eng.infer_u8(frames)
            kw = dict(frames_u8=frames)
        elif case.entry == "f32":
            x = np.random.default_rng(4).uniform(-0.2, 1.2, (N, 3, H, W)).astype(np.float32)
            eng.infer_f32(x)
            kw = dict(f32_input=x)
        else:
            eng.debug_run_ops(0, len(g.ops) - 1, N)
            kw = dict(N=N, HW=(H, W))
        conf, paf, want = int8_sim.run_graph(g, case.scales, init={b: _nchw(a[:N]) for b, a in init.items()}, **kw)
        for bi in range(len(g.buffers)):
            full = eng.debug_read_buffer(bi, M)
            got, ref = full[:N], _nhwc(want[bi])
            bad = np.argwhere(got != ref)
            assert bad.size == 0, f"buffer {bi}: {len(bad)} bytes differ, first at {bad[0].tolist()}: {got[tuple(bad[0])]} != {ref[tuple(bad[0])]}"
            assert full[N:].tobytes() == init[bi][N:].tobytes(), f"buffer {bi} written past frame {N}"
        if split:
            got = eng.read_outputs(M)
            for name, a, ref in zip(("conf", "paf"), got, (conf, paf)):
                bad = np.argwhere(a[:N] != ref)
                assert bad.size == 0, f"{name}: {len(bad)} values differ, first at {bad[0].tolist()}: {a[:N][tuple(bad[0])]} != {ref[tuple(bad[0])]}"
            if N < M:
                for name, a, was in zip(("conf", "paf"), got, planes_before):
                    assert a[N:].tobytes() == was[N:].tobytes(), f"{name} written past frame {N}"
    finally:
        eng.close()


@gpu
@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_int8_kernel(case):
    _run_int8_case(case)


@gpu
@pytest.mark.parametrize("case", MULTI, ids=[c.id for c in MULTI])
def test_int8_kernel_multi_round(case):
    """some CTA runs two or more items, and the item count is not a multiple of the grid"""
    import torch
    from tests.test_engine_kernels import work_items
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    op = case.graph.ops[0]
    _, H, W = case.shape
    items = work_items(case.kernels[0], op, case.shape[0], H, W)
    grid = min(sms, items)
    print(f"[int8 rounds] {case.id}: {items} items on {grid} CTAs")
    assert items > grid and items % grid
    _run_int8_case(case)


@gpu
def test_int8_conv_inventory():
    """the cases above reach all 12 int8 conv kernels (each case's engine is created here: independent of test order)"""
    reached, multi = set(), set()
    for case in CASES + MULTI:
        g = _int8_graph(case.graph, case.scales)
        N, H, W = case.shape
        eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=case.max_batch, dtype="int8")
        names = {n for n in (eng.debug_op_kernel(i) for i in range(len(g.ops))) if n.startswith("conv<")}
        eng.close()
        reached |= names
        if case in MULTI:
            multi |= names
    assert reached == CONV_KERNELS, sorted(CONV_KERNELS - reached)
    assert multi == CONV_KERNELS, sorted(CONV_KERNELS - multi)


# ---- whole networks -------------------------------------------------------------------------------------------------------
NETS = {
    "tiny": (lambda: models.tiny_test_net(1), (2, 64, 96)),
    "vgg19": (lambda: models.openpose_vgg19(0), (2, 368, 656)),
    "mobilenet_thin3": (lambda: models.mobilenet_thin_openpose(0, n_stages=3), (2, 96, 128)),
    "resnet50_lw": (lambda: models.resnet50_lw_openpose(0), (2, 96, 128)),
}


def _calibrated(make, shape, seed=100):
    g = make()
    N, H, W = shape
    cal = capi.Engine(g.to_pack(), (W, H), max_batch_size=N, dtype="tf32")
    g.set_int8_scales(cal.calibrate(syn.make_frames_u8(seed, 2 * N, H, W)))   # twice max_batch: two chunks
    cal.close()
    return g


@gpu
@pytest.mark.parametrize("net", sorted(NETS))
def test_int8_network_matches_model(net):
    make, (N, H, W) = NETS[net]
    g = _calibrated(make, (N, H, W))
    frames = syn.make_frames_u8(7, N, H, W)
    eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=N, dtype="int8")
    try:
        assert capi.lib().hp_engine_dtype(eng._h) == 2
        eng.infer_u8(frames)
        conf, paf = eng.read_outputs(N)
        c_ref, p_ref, bufs = int8_sim.run_graph(g, g.act_scales, frames_u8=frames)
        for bi in range(len(g.buffers)):
            got = eng.debug_read_buffer(bi, N)
            assert np.array_equal(got, _nhwc(bufs[bi])), f"buffer {bi}: {int((got != _nhwc(bufs[bi])).sum())} bytes differ"
        assert conf.tobytes() == c_ref.tobytes() and paf.tobytes() == p_ref.tobytes()
        if net in ("vgg19", "mobilenet_thin3"):   # accuracy against the fp32 engine: reported, not gated (random weights say nothing about a trained model)
            f32 = capi.Engine(make().to_pack(), (W, H), max_batch_size=N, dtype="tf32")
            f32.infer_u8(frames)
            c32, p32 = f32.read_outputs(N)
            f32.close()
            rel = lambda a, b: float(np.abs(a - b).max() / np.abs(b).max())
            print(f"\nINT8 vs TF32 {net} {H}x{W}: conf max rel err {rel(conf, c32):.4f}, paf {rel(paf, p32):.4f}; "
                  f"rms rel conf {float(np.sqrt(((conf - c32) ** 2).mean() / (c32 ** 2).mean())):.4f}, "
                  f"paf {float(np.sqrt(((paf - p32) ** 2).mean() / (p32 ** 2).mean())):.4f}")
    finally:
        eng.close()


@gpu
def test_int8_model_on_the_gpu_matches_the_cpu():
    """int8_sim.run_graph(device="cuda") runs the integer convolutions there (im2col + DGEMM, cuDNN off) and gives the CPU run's
    bytes: MobilenetThin (the im2col stem, grouped convs) and ResNet-50-LW (residual convs) at 64 x 96"""
    kinds = set()
    for name in ("mobilenet_thin_openpose", "resnet50_lw_openpose"):
        g = getattr(models, name)(0)
        frames = syn.make_frames_u8(3, 2, 64, 96)
        g.set_int8_scales(int8_sim.float_absmax(g, frames))
        c0, p0, b0 = int8_sim.run_graph(g, g.act_scales, frames_u8=frames)
        c1, p1, b1 = int8_sim.run_graph(g, g.act_scales, frames_u8=frames, device="cuda")
        for bi, (x, y) in enumerate(zip(b0, b1)):
            assert x.tobytes() == y.tobytes(), f"{name}: buffer {bi}: {int((x != y).sum())} bytes differ"
        assert c0.tobytes() == c1.tobytes() and p0.tobytes() == p1.tobytes(), name
        kinds |= {k for op in g.ops if op.type == models.OP_CONV for k, on in (("grouped", op.groups > 1), ("residual", op.res_mode),
                                                                               ("im2col", op.im2col_input)) if on}
    assert kinds == {"grouped", "residual", "im2col"}, kinds


# ---- calibration ----------------------------------------------------------------------------------------------------------
@gpu
def test_calibration_matches_fp32_reference_and_is_a_running_max():
    from oracle import torch_backbone
    g = models.tiny_test_net(1)
    N, H, W = 2, 64, 96
    fa, fb = syn.make_frames_u8(11, N, H, W), syn.make_frames_u8(12, N, H, W)
    eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=N, dtype="tf32")
    a = eng.calibrate(fa)
    b = eng.calibrate(fb)
    ab = eng.calibrate(fb, a)
    both = eng.calibrate(np.concatenate([fa, fb]))
    eng.close()
    assert np.array_equal(ab, np.maximum(a, b)) and np.array_equal(both, ab)
    ref = np.zeros(len(g.buffers))
    for oi, op in enumerate(g.ops):   # what each op stored, op by op (buffers are written more than once)
        if op.type == models.OP_CONV and op.out_mode == models.OUT_F32_NCHW_SPLIT:
            continue
        _, _, bufs = torch_backbone.run_graph(g, fa, rounding="tf32", device="cpu", upto=oi)
        ref[op.out_buf] = max(ref[op.out_buf], float(bufs[op.out_buf].abs().max()))
    assert np.all(np.abs(a - ref) <= 6e-3 * ref + 1e-3), (a, ref)


CAL_NETS = {"cfg3": ("openpose_vgg19", 368, 656, 16), "cfg4": ("resnet50_lw_openpose", 368, 432, 32),
            "cfg2": ("mobilenet_thin_openpose", 368, 432, 8)}   # tools/bench_int8.py's workloads: graph, H, W, max_batch


def _replay_absmax(g, eng, frames):
    """what calibrate folds, op by op: max |x| of each op's whole output buffer over the frames (infer_u8 first, so that the channels
    other ops write hold what they held when calibrate ran; heads and the split output conv skipped)"""
    n = frames.shape[0]
    eng.infer_u8(frames)
    amax = np.zeros(len(g.buffers), np.float32)
    for i, op in enumerate(g.ops):
        eng.debug_run_ops(i, i, n)
        if op.type in (models.OP_PIFPAF_HEAD, models.OP_PPN_HEAD) or (op.type == models.OP_CONV and op.out_mode == models.OUT_F32_NCHW_SPLIT):
            continue
        amax[op.out_buf] = max(amax[op.out_buf], np.abs(eng.debug_read_buffer(op.out_buf, n, raw=True)).max())
    return amax


def _same_bits(a, b):
    return np.asarray(a, np.float32).tobytes() == np.asarray(b, np.float32).tobytes()


@gpu
@pytest.mark.parametrize("cfg", sorted(CAL_NETS))
def test_calibration_at_benchmark_batch_is_exact(cfg):
    """calibrate on a TF32 engine at the benchmark's max_batch, bit for bit: (a) one full chunk equals the running max of an op-by-op
    replay; (b) a short chunk of n = B - 3 frames ignores frames >= n (they hold 1e30); (c) 2B - 3 frames, a full chunk and a short
    one, equal the element-wise max of the two calibrated apart.  Calibration folds whole buffers, so channels other ops write count
    too: each compared run starts from the buffer contents the other started from."""
    name, H, W, B = CAL_NETS[cfg]
    g = getattr(models, name)(0)
    eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=B, dtype="tf32")
    try:
        frames = syn.make_frames_u8(500, 2 * B - 3, H, W)
        full, n = frames[:B], B - 3
        eng.infer_u8(full)
        a = eng.calibrate(full)
        ra = _replay_absmax(g, eng, full)
        assert _same_bits(a, ra), f"{cfg}: calibrate differs from the replay at buffers {np.flatnonzero(a != ra).tolist()}"
        # (b)
        saved = [eng.debug_read_buffer(bi, B, raw=True) for bi in range(len(g.buffers))]
        for bi, x in enumerate(saved):
            y = x.copy()
            y[n:] = 1e30
            eng.debug_write_buffer(bi, y)
        b = eng.calibrate(full[:n])
        assert (b < 1e29).all(), f"{cfg}: the {n}-frame calibration read frames >= {n} of buffers {np.flatnonzero(b >= 1e29).tolist()}"
        rb = _replay_absmax(g, eng, full[:n])
        assert _same_bits(b, rb), f"{cfg}: the {n}-frame calibration differs from the replay at buffers {np.flatnonzero(b != rb).tolist()}"
        # (c), from the contents (a) started from (channels no op writes, such as a buffer's pad channels, still held 1e30)
        for bi, x in enumerate(saved):
            eng.debug_write_buffer(bi, x)
        first = eng.calibrate(full)
        assert _same_bits(first, a), f"{cfg}: calibrating the same frames from the same contents differs at buffers {np.flatnonzero(first != a).tolist()}"
        last = eng.calibrate(frames[B:])
        assert not _same_bits(last, first), f"{cfg}: two frame sets calibrate alike"
        for bi, x in enumerate(saved):
            eng.debug_write_buffer(bi, x)
        both = eng.calibrate(frames)
        assert _same_bits(both, np.maximum(first, last)), f"{cfg}: chunks combine wrongly at buffers {np.flatnonzero(both != np.maximum(first, last)).tolist()}"
    finally:
        eng.close()


@gpu
def test_calibrate_needs_tf32_engine():
    g = models.tiny_test_net(1)
    eng = capi.Engine(g.to_pack(), (48, 32), max_batch_size=1)
    with pytest.raises(capi.HyperposeError, match="TF32"):
        eng.calibrate(syn.make_frames_u8(1, 1, 32, 48))
    eng.close()


# ---- packs the INT8 engine refuses ------------------------------------------------------------------------------------------
def _create(pack, dtype="int8", size=(48, 32)):
    return capi.Engine(pack, size, max_batch_size=1, dtype=dtype)


@gpu
def test_int8_rejections():
    g = models.tiny_test_net(1)
    with pytest.raises(capi.HyperposeError, match="no INT8 scale table"):
        _create(g.to_pack())
    g.set_int8_scales(np.full(len(g.buffers), 5.0, np.float32))
    good = g.to_pack()
    _create(good).close()
    bad = bytearray(good)
    struct.pack_into("<I", bad, 48, len(g.buffers) - 1)
    with pytest.raises(capi.HyperposeError, match="scale table has"):
        _create(bytes(bad))
    for v in (0.0, -1.0, np.inf, np.nan):
        s = g.act_scales.copy(); s[3] = v
        g.act_scales = s
        with pytest.raises(capi.HyperposeError, match="scale of buffer 3"):
            _create(g.to_pack())
    s = np.full(len(g.buffers), 5.0, np.float32); s[2] = 6.0   # buffer 2 is the max-pool's output
    g.act_scales = s
    with pytest.raises(capi.HyperposeError, match="max-pool op 2"):
        _create(g.to_pack())
    p = models.resnet50_pifpaf(0)
    p.set_int8_scales(np.ones(len(p.buffers), np.float32))
    with pytest.raises(capi.HyperposeError, match="head_type"):
        _create(p.to_pack(), size=(129, 129))
    for dt in ("f16", "tf32"):
        _create(p.to_pack(), dt, size=(129, 129)).close()


@gpu
def test_int8_rejects_inexact_accumulation():
    """a conv summing more than (2^31 - 1) / 127^2 = 133152 products per output could overflow the s32 accumulator"""
    for cin, ok in ((2704, True), (2720, False)):   # 7 x 7 x cin = 132496 / 133280
        g = _graph("k")
        a = g.add_buffer(cin, 0); b = g.add_buffer(16, 0)
        g.add_conv(a, b, np.full((1, 16, cin, 7, 7), 0.01, np.float32), np.zeros(16, np.float32), np.zeros(16, np.float32))
        g.act_scales = np.ones(2, np.float32)
        if ok:
            _create(g.to_pack(), size=(8, 4)).close()
        else:
            with pytest.raises(capi.HyperposeError, match="s32 accumulator"):
                _create(g.to_pack(), size=(8, 4))


# ---- pose paths on an INT8 engine -------------------------------------------------------------------------------------------
@gpu
def test_pose_paths_and_f32_entry_int8():
    import oracle
    import torch
    N, H, W = 2, 64, 96
    g = _calibrated(lambda: models.tiny_test_net(2), (N, H, W), seed=21)
    frames = syn.make_frames_u8(5, N, H, W)
    eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=N, dtype="int8")
    eng.infer_u8(frames)
    c1, p1 = eng.read_outputs(N)
    ct, pt = float(np.quantile(c1[:, :18], 0.97)), float(np.quantile(p1, 0.5))
    parser = capi.PafParser(ct, pt)
    parser.set_capacity(peaks_per_part=1024, candidates_per_limb=1 << 15, humans=128)
    humans = eng.run_pose(parser, frames, cap=128)
    n_h = 0
    for i in range(N):
        want = oracle.oracle_process(c1[i], p1[i], ct, pt, peak_cap=1 << 18, conn_cap=1 << 14)["humans"]
        assert humans[i].tobytes() == want.tobytes()
        n_h += len(want)
    # the CUDA-graph device path equals the host path, replayed twice
    d = torch.from_numpy(frames).cuda()
    for _ in range(2):
        t = eng.submit_pose_device(parser, d.data_ptr(), N)
        got = eng.collect_pose(t, cap=128)
        assert [h.tobytes() for h in got] == [h.tobytes() for h in humans]
    assert eng.pose_stats()["graph_launches"] >= 1
    # the f32 entry: the same as the model run from the same f32 input
    x = np.random.default_rng(9).uniform(-0.1, 1.1, (N, 3, H, W)).astype(np.float32)
    eng.infer_f32(x)
    c2, p2 = eng.read_outputs(N)
    cr, pr, bufs = int8_sim.run_graph(g, g.act_scales, f32_input=x)
    assert c2.tobytes() == cr.tobytes() and p2.tobytes() == pr.tobytes()
    for bi in range(len(g.buffers)):
        assert np.array_equal(eng.debug_read_buffer(bi, N), _nhwc(bufs[bi])), bi
    eng.close(); parser.close()


# ---- the C++ drop-in: data_type::kINT8 and HPB_DTYPE=int8 ----------------------------------------------------------------
@gpu
def test_dropin_selects_int8(tmp_path):
    """hyperpose::dnn::tensorrt built with data_type::kINT8 runs the INT8 engine on a calibrated pack and the TF32 engine on a pack
    without a table; tensorrt_serialized runs INT8 under HPB_DTYPE=int8 and f16 without it.  Which engine ran is read from the bytes
    of its outputs: examples/dtype_probe_b200 pushes one f32 frame through the drop-in, the same frame goes through an Engine of each
    dtype here, and the outputs must equal that dtype's bytes (and differ from the other candidates')."""
    exe = hb.build_dtype_probe()
    if exe is None:
        pytest.skip("the probe is built where the reference headers exist")
    N, H, W = 1, 32, 48
    plain = tmp_path / "plain.pack"
    plain.write_bytes(models.tiny_test_net(1).to_pack())
    cal = tmp_path / "cal.pack"
    cal.write_bytes(_calibrated(lambda: models.tiny_test_net(1), (N, H, W)).to_pack())
    n = 3 * H * W
    x = ((np.arange(n, dtype=np.uint64) * np.uint64(2654435761)) % np.uint64(1024)).astype(np.float32) / np.float32(1024.0)

    def engine_bytes(pack, dtype):
        e = capi.Engine(pack.read_bytes(), (W, H), max_batch_size=1, dtype=dtype)
        e.infer_f32(x.reshape(1, 3, H, W))
        c, p = e.read_outputs(1)
        e.close()
        return c.tobytes() + p.tobytes()

    def probe(pack, mode, dtype_env=None):
        out = tmp_path / f"{pack.stem}-{mode}-{dtype_env}.bin"
        env = {k: v for k, v in os.environ.items() if k != "HPB_DTYPE"}
        if dtype_env:
            env["HPB_DTYPE"] = dtype_env
        r = subprocess.run([exe, str(pack), str(W), str(H), mode, str(out)], capture_output=True, text=True, timeout=120, env=env)
        assert r.returncode == 0, r.stdout + r.stderr
        return out.read_bytes()

    want = {(pk.stem, dt): engine_bytes(pk, dt) for pk in (plain, cal) for dt in ("f16", "tf32")}
    want[("cal", "int8")] = engine_bytes(cal, "int8")
    assert len({want[("cal", d)] for d in ("f16", "tf32", "int8")}) == 3   # the three engines are told apart
    assert probe(cal, "kint8") == want[("cal", "int8")]                  # kINT8 + table: the INT8 engine
    assert probe(plain, "kint8") == want[("plain", "tf32")]              # kINT8, no table: TF32, as before
    assert probe(cal, "kfloat") == want[("cal", "tf32")]                 # the table changes nothing for kFLOAT / kHALF
    assert probe(cal, "khalf") == want[("cal", "f16")]
    assert probe(cal, "serialized", "int8") == want[("cal", "int8")]     # HPB_DTYPE=int8 on tensorrt_serialized
    assert probe(cal, "serialized") == want[("cal", "f16")]              # serialized default: f16
