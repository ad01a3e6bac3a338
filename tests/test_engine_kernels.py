"""Every conv kernel instantiation the engine can launch, and the depthwise / max-pool kernels, one- or two-op graphs at a time,
against a float64 reference of the same op (oracle/torch_backbone.py on the CPU, operands on the engine's fp16 / TF32 grid).

Inputs are random values on the operand grid, of either sign, magnitudes around 1.  Every case asserts which kernel its op launches
(Engine.debug_op_kernel), then checks
  (a) every output element:  |got - ref| <= 2^-11 |ref| + (K + 2) 2^-23 mag + 2^-24
      ref: the float64 result before the engine's final rounding; 2^-11 |ref| is that rounding (half an fp16 / TF32 ulp);
      K: products accumulated per output (R * S * padded cin_g, or K * K for a depthwise op); mag = sum |w x| + |b| (+ |res|),
      from a magnitude pass of the reference; 2^-23 mag per addition allows two fp32 ulps for the tensor core's alignment and
      truncation; 2^-24 covers fp16 subnormals;
  (b) the channels of the output buffer outside the op's range -- a partial n-tile's pad channels included -- keep their bits;
  (b') a case may run N frames on an engine built for max_batch > N (the last, short batch of a video): frames N .. max_batch - 1
      of every input buffer hold NaN, and every byte of those frames, in every buffer and conf / paf plane, must keep its value;
  (c) the bound rejects a wrong reference: with one filter tap zeroed, and with the last output channel's weights replaced by the
      first's, most outputs the mutation changes must break it;
  (d) the worst |got - ref| / bound of the case is printed, with the work items and grid of each conv launch (work_items).
The conf / paf planes of the output conv (OUT_F32_NCHW_SPLIT) hold the unrounded fp32 result: their bound has no 2^-11 |ref| term.
Max-pool is exact and compared bit for bit."""
import copy
import zlib

import numpy as np
import pytest
import torch

from hyperpose_b200 import capi, models
from oracle import torch_backbone

gpu = pytest.mark.gpu

# All conv kernels launch_conv can pick: one per tile width in conv_kernel_bn<T, kRes, kStemR> and halo_kernel's 128-pixel item
# (engine.cu).  A new tile width has to be added here too.
BNS = (16, 32, 48, 64, 96, 128)
CONV_KERNELS = ({f"conv<f16,{b}>" for b in BNS} | {f"conv<f16,{b},res>" for b in BNS} | {f"conv<f16,{b},stem3>" for b in BNS} |
                {f"conv<f16,{b},stem7>" for b in BNS} | {f"conv<tf32,{b}>" for b in BNS} | {f"conv<tf32,{b},res>" for b in BNS} |
                {f"halo<{b}>" for b in BNS} | {f"halo<{b},pool>" for b in BNS})
assert len(CONV_KERNELS) == 48

# tile width the engine picks for each output width the cases use (n-tiles of at most 128 channels, the least padding)
BN_OF = {13: 16, 16: 16, 19: 32, 24: 32, 32: 32, 40: 48, 48: 48, 57: 64, 64: 64, 72: 96, 96: 96, 128: 128, 200: 128, 288: 96}

# (N, H, W): a ragged last 128-pixel tile; tiles that span images; TMA zero-fill on all four borders.  None of them is a
# 3x3 halo shape (their 16 x 8 tile grids waste more than 6 %).
S1, S2, S3 = (2, 13, 21), (3, 5, 7), (1, 40, 72)
HALO0, HALO_RAGGED = (2, 32, 40), (1, 46, 80)   # 16 x 8 tile grid: no waste / 4.3 % waste
MEAN = (0.41, 0.52, 0.37)


def _r(x, m):
    return (x + m - 1) // m * m


class Case:
    def __init__(self, cid, dtype, shape, graph, kernels, outs, K, env=None, stem=False, mutate=0, twin_env=None, fill=None, max_batch=None):
        self.id, self.dtype, self.shape, self.graph, self.kernels, self.outs, self.K = cid, dtype, shape, graph, kernels, outs, K
        self.max_batch = max_batch or shape[0]   # the engine's max_batch_size; the case runs shape[0] frames
        assert self.max_batch >= shape[0]
        # outs: (buffer, first channel, channels), or ("conf" | "paf", 0, channels) for a plane of the split output conv
        self.env = env or {}
        self.stem = stem            # the input is u8 frames (infer_u8, then infer_f32 through the im2col buffer)
        self.mutate = mutate        # op whose weights the wrong references change, or None (max-pool)
        self.twin_env = twin_env    # the same graph under these switches must give the same bytes
        self.fill = fill or {}      # {buffer: (first channel, value)}: channels from there on hold this value


def _graph(name):
    return models.Graph(name, conf_channels=19, paf_channels=38, out_down_shift=0, mean=MEAN)


def _conv_w(rng, G, co, ci, R, S=None):
    S = S or R
    return (rng.standard_normal((G, co, ci, R, S)) * np.sqrt(2.0 / (ci * R * S))).astype(np.float32)


def _slopes(rng, n, monotone=False):
    return rng.uniform(0.0 if monotone else -0.5, 1.0, n).astype(np.float32)


def conv_case(dtype, cout, cin=64, G=1, R=3, shape=S1, in_off=0, out_off=0, res_mode=0, res_off=0, pad_value=None, kernel=None,
              env=None, pool=False, seed=0, S=None, max_batch=None):
    S = S or R
    rng = np.random.default_rng(seed)
    chunk = 64 if dtype == "f16" else 32
    g = _graph("conv")
    in_c = _r(in_off + G * _r(cin, chunk) + (64 if in_off else 0), 8)
    b_in = g.add_buffer(in_c, 0)
    b_out = g.add_buffer(_r(out_off + G * cout + 8, 8), 0)
    kw = {}
    if res_mode:
        kw = dict(res_buf=g.add_buffer(_r(res_off + G * cout + 8, 8), 0), res_ch_off=res_off, res_mode=res_mode)
    g.add_conv(b_in, b_out, _conv_w(rng, G, cout, cin, R, S), rng.standard_normal(G * cout).astype(np.float32) * 0.5,
               _slopes(rng, G * cout, monotone=pool), in_ch_off=in_off, out_ch_off=out_off, **kw)
    kernels, outs = [kernel], [(b_out, out_off, G * cout)]
    if pool:
        b_pool = g.add_buffer(_r(out_off + G * cout + 8, 8), 1)
        g.add_maxpool(b_out, b_pool, G * cout)
        g.ops[-1].in_ch_off = g.ops[-1].out_ch_off = out_off
        kernels, outs = [kernel, "none"], [(b_pool, out_off, G * cout)]
    cid = f"{dtype}-{kernel}-cout{cout}-cin{cin}-G{G}-{R}x{S}-{'x'.join(map(str, shape))}" + (f"-in{in_off}" if in_off else "") + \
          (f"-out{out_off}" if out_off else "") + (f"-res{res_mode}@{res_off}" if res_mode else "") + (f"-{','.join(f'{k}={v}' for k, v in env.items())}" if env else "") + \
          (f"-max{max_batch}" if max_batch and max_batch != shape[0] else "")
    fill = {b_in: (in_off + G * cin, 3e4 if dtype == "f16" else 1e30)} if pad_value else None
    return Case(cid, dtype, shape, g, kernels, outs, R * S * _r(cin, chunk), env=env, mutate=0,
                twin_env={"HPB_NO_POOL_FUSE": "1"} if pool else None, fill=fill, max_batch=max_batch)


def stem_case(cout, R, stride, shape, out_off=0, seed=0, max_batch=None):
    rng = np.random.default_rng(seed)
    g = _graph("stem")
    d = 1 if stride == 2 else 0
    col = g.add_buffer(_r(R * R * 3, 64), d)
    g.add_im2col(col, stride=stride, ksize=R)
    out = g.add_buffer(_r(out_off + cout + 8, 8), d)
    g.add_conv(col, out, _conv_w(rng, 1, cout, 3, R), rng.standard_normal(cout).astype(np.float32) * 0.5, _slopes(rng, cout),
               im2col_input=1, out_ch_off=out_off)
    k = f"conv<f16,{BN_OF[cout]},stem{R}>"
    return Case(f"f16-{k}-cout{cout}-s{stride}-{'x'.join(map(str, shape))}" + (f"-max{max_batch}" if max_batch else ""), "f16", shape, g,
                ["none", k], [(out, out_off, cout)], _r(R * R * 3, 64), stem=True, mutate=1, max_batch=max_batch)


def dw_case(dtype, C, K, stride, kernel, shape=S1, in_off=8, out_off=16, pair=False, seed=0, max_batch=None):
    rng = np.random.default_rng(seed)
    g = _graph("dw")
    b_in = g.add_buffer(_r(in_off + C + 8, 8), 0)
    b_out = g.add_buffer(_r(out_off + (2 if pair else 1) * C + 8, 8), 1 if stride == 2 else 0)
    outs = []
    for j in range(2 if pair else 1):
        w = (rng.standard_normal((C, K, K)) * np.sqrt(2.0 / (K * K))).astype(np.float32)
        g.add_dwconv(b_in, b_out, w, rng.standard_normal(C).astype(np.float32) * 0.5, _slopes(rng, C), stride=stride,
                     in_ch_off=in_off, out_ch_off=out_off + j * C)
        outs.append((b_out, out_off + j * C, C))
    kernels = [kernel, "none"] if pair else [kernel]
    return Case(f"{dtype}-{kernel}-C{C}-{K}x{K}-s{stride}-{'x'.join(map(str, shape))}" + (f"-max{max_batch}" if max_batch else ""), dtype, shape,
                g, kernels, outs, K * K, mutate=0, max_batch=max_batch)


def pool_case(dtype, C, K, kernel, shape=S1, in_off=8, out_off=16, max_batch=None):
    g = _graph("pool")
    b_in = g.add_buffer(_r(in_off + C + 8, 8), 0)
    b_out = g.add_buffer(_r(out_off + C + 8, 8), 1)
    g.add_maxpool(b_in, b_out, C, ksize=K)
    g.ops[-1].in_ch_off, g.ops[-1].out_ch_off = in_off, out_off
    return Case(f"{dtype}-{kernel}-C{C}-{'x'.join(map(str, shape))}" + (f"-max{max_batch}" if max_batch else ""), dtype, shape, g, [kernel],
                [(b_out, out_off, C)], 0, mutate=None, max_batch=max_batch)


def _cases():
    cs = []
    widths = [(13, 3, S1, 64, 0), (24, 1, S2, 64, 0), (40, 7, S1, 64, 0), (57, 3, S3, 128, 0), (72, 1, S1, 192, 64),
              (200, 3, S2, 64, 0), (288, 1, S3, 64, 0)]   # (cout_g, R, shape, cin_g, in_ch_off): odd trailing channels, partial n-tiles
    for dt in ("f16", "tf32"):
        for cout, R, shape, cin, in_off in widths:
            cs.append(conv_case(dt, cout, cin, 1, R, shape, in_off=in_off, kernel=f"conv<{dt},{BN_OF[cout]}>"))
        cs.append(conv_case(dt, 40, 64, 3, 3, S2, kernel=f"conv<{dt},48>"))                       # 3 groups
        cs.append(conv_case(dt, 19, 64 if dt == "f16" else 32, 2, 1, S1, out_off=8, kernel=f"conv<{dt},32>"))   # group 1 starts at channel 27
        cs.append(conv_case(dt, 57, 185, 1, 3 if dt == "f16" else 1, S1, pad_value=True, kernel=f"conv<{dt},64>"))   # 185 of 192 channels
        for i, cout in enumerate(BNS):                                                          # residual epilogues
            cs.append(conv_case(dt, cout, 64, 1, (3, 1)[i % 2], (S1, S2, S3)[i % 3], res_mode=1 + i % 2, res_off=(0, 8, 16)[i % 3],
                                out_off=(0, 8)[i % 2], kernel=f"conv<{dt},{cout},res>"))
    cs.append(conv_case("tf32", 24, 96, 1, 3, S3, kernel="conv<tf32,32>"))                      # three 32-channel chunks
    for i, cout in enumerate((13, 24, 40, 57, 72, 128)):
        cs.append(stem_case(cout, 3, 1, (2, 13, 21)))
        cs.append(stem_case(cout, 3, 2, (2, 27, 41), out_off=8))
        cs.append(stem_case(cout, 7, 2, (1, 40, 72)))
    for i, cout in enumerate((13, 24, 40, 57, 72, 200)):
        cs.append(conv_case("f16", cout, 64, 1, 3, (HALO0, HALO_RAGGED)[i % 2], in_off=(0, 64)[i % 2], out_off=(0, 8)[i % 2],
                            kernel=f"halo<{BN_OF[cout]}>"))
    cs.append(conv_case("f16", 40, 64, 2, 3, HALO0, kernel="halo<48>"))
    cs.append(conv_case("f16", 57, 64, 1, 7, (1, 20, 24), kernel="halo<64>", env={"HPB_HALO": "all"}))
    for i, cout in enumerate(BNS):
        cs.append(conv_case("f16", cout, 64, 1, 3, (HALO0, HALO_RAGGED)[i % 2], out_off=(0, 8)[i % 2], pool=True, kernel=f"halo<{cout},pool>"))
    cs += [dw_case("f16", 40, 3, 2, "dw_strip<3,2>"), dw_case("f16", 48, 1, 1, "dw_strip<1,1>"), dw_case("f16", 40, 1, 2, "dw_strip<1,2>"),
           dw_case("f16", 40, 3, 1, "dw_col"), dw_case("f16", 64, 3, 1, "dw_tma<1>"), dw_case("f16", 192, 3, 1, "dw_tma<1>", shape=(1, 20, 70)),
           dw_case("f16", 64, 3, 1, "dw_tma<2>", pair=True)]
    cs += [dw_case("tf32", 40, k, s, "dw_f32") for k in (1, 3) for s in (1, 2)]
    cs += [pool_case("f16", 40, 2, "maxpool<2>"), pool_case("f16", 40, 3, "maxpool<3>"), pool_case("tf32", 40, 2, "maxpool_f32"),
           pool_case("tf32", 24, 3, "maxpool_f32")]
    return cs


CASES = _cases()


def _engine(case, monkeypatch, env=None):
    for k in ("HPB_HALO", "HPB_NO_POOL_FUSE", "HPB_NO_STEM3", "HPB_NO_DW1_FUSE", "HPB_NO_DW_DUAL", "HPB_NO_DW_TMA"):
        monkeypatch.delenv(k, raising=False)
    for k, v in {**case.env, **(env or {})}.items():
        monkeypatch.setenv(k, v)
    N, H, W = case.shape
    return capi.Engine(case.graph.to_pack(), (W, H), max_batch_size=case.max_batch, dtype=case.dtype)


def _buf_shape(case, bi):
    """a buffer's NHWC shape over all max_batch frames"""
    N, H, W = case.shape
    c, d = case.graph.buffers[bi]
    for _ in range(d):
        H, W = (H + 1) // 2, (W + 1) // 2
    return case.max_batch, H, W, c


def work_items(kernel, op, N, H, W):
    """work items of a conv launch over N frames of an H x W input (engine.cu, launch_conv): conv_wgmma_kernel takes
    ceil(N H W / 128) pixel tiles x groups x n-tiles; the halo kernel T x groups x n-tiles, T = N ceil(H / 16) ceil(W / 8) 16 x 8
    tiles, or ceil(T / 2) tile pairs for the wide item.  A CTA runs items blockIdx.x, + gridDim.x, ... (the ping-pong item hands them
    to its two warpgroups in turn)"""
    args = kernel[kernel.index("<") + 1:-1].split(",")
    if kernel.startswith("conv<"):
        bn, m = int(args[1]), -(-N * H * W // 128)
    else:
        bn, m = int(args[0]), N * -(-H // 16) * -(-W // 8)
        if "wide" in args:
            m = -(-m // 2)
    return m * op.groups * -(-op.cout_g // bn)


def conv_launches(case):
    """[(op, kernel, items, grid)] of the case's conv launches; grid = min(SMs, items)"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    out = []
    for i, (op, k) in enumerate(zip(case.graph.ops, case.kernels)):
        if k.startswith(("conv<", "halo<")):
            _, H, W, _ = _buf_shape(case, op.in_buf)
            items = work_items(k, op, case.shape[0], H, W)
            out.append((i, k, items, min(sms, items)))
    return out


def _on_grid(x, dtype):
    return x.astype(np.float16) if dtype == "f16" else torch_backbone.tf32_round(torch.from_numpy(x.astype(np.float32))).numpy()


def _planes(case):
    return [o for o in case.outs if isinstance(o[0], str)]


def _inputs(case, rng, written=None):
    """NHWC contents of every buffer over all max_batch frames: random operands on the grid, sentinels in the output buffers, NaN in
    the frames past the run's N of every other buffer"""
    N = case.shape[0]
    written = {o[0] for o in case.outs} if written is None else written
    data = {}
    for bi in range(len(case.graph.buffers)):
        shp = _buf_shape(case, bi)
        if bi in written:
            data[bi] = _on_grid(rng.uniform(-1000, 1000, shp), case.dtype)
            continue
        x = rng.standard_normal(shp)
        if case.mutate is None:
            x = -np.abs(x) - 0.25       # all negative: a window padded with zeros instead of -inf is caught at the borders
        if bi in case.fill:
            x[..., case.fill[bi][0]:] = case.fill[bi][1]
        x[N:] = np.nan
        data[bi] = _on_grid(x, case.dtype)
    return data


def _read_all(eng, case, n):
    """n frames of every buffer the engine keeps in memory (a buffer whose consumer runs in the producer's epilogue is never
    written) and, when the case writes them, of the conf / paf planes (NHWC)"""
    out = {}
    for bi in range(len(case.graph.buffers)):
        try:
            out[bi] = eng.debug_read_buffer(bi, n)
        except capi.HyperposeError as e:
            assert e.status == capi.HP_ERR_UNSUPPORTED and "not materialised" in str(e), str(e)
    if _planes(case):
        conf, paf = eng.read_outputs(n)
        out["conf"], out["paf"] = conf.transpose(0, 2, 3, 1), paf.transpose(0, 2, 3, 1)
    return out


def _reference(case, g, data, frames, magnitude=False):
    N = case.shape[0]
    init = {bi: a[:N].astype(np.float64).transpose(0, 3, 1, 2) for bi, a in data.items()}
    conf, paf, bufs = torch_backbone.run_graph(g, frames, device="cpu", dtype=torch.float64, init=init,
                                               rounding="fp16" if case.dtype == "f16" else "tf32", round_stores=False, magnitude=magnitude)
    src = {"conf": conf, "paf": paf}
    return [(src[b] if isinstance(b, str) else bufs[b])[:, off:off + c].numpy().transpose(0, 2, 3, 1) for b, off, c in case.outs]


def _mutants(case):
    """two wrong graphs: one filter tap zeroed (the centre tap; for 1x1 the last 8 input channels), and the last output channel's
    weights replaced by the first's"""
    out = []
    for kind in ("tap", "channel"):
        g = copy.deepcopy(case.graph)
        op = g.ops[case.mutate]
        w = op.weight if op.type == models.OP_CONV else op.weight[None]     # [G, cout, cin, R, S] / [1, C, K, K]
        if kind == "tap":
            if op.type == models.OP_CONV and w.shape[-2:] == (1, 1):
                w[:, :, -8:] = 0
            else:
                w[..., w.shape[-2] // 2, w.shape[-1] // 2] = 0
        else:
            w[-1, -1] = w[-1, 0]
        out.append((kind, g))
    return out


def _run_and_check(case, monkeypatch, rng):
    N, H, W = case.shape
    M = case.max_batch
    eng = _engine(case, monkeypatch)
    assert [eng.debug_op_kernel(i) for i in range(len(case.graph.ops))] == case.kernels
    launches = conv_launches(case)
    data = _inputs(case, rng)
    frames = rng.integers(0, 256, (N, H, W, 3), dtype=np.uint8)
    # the planes' frames past N: what a run over all max_batch frames of other (finite) contents left there
    before = {bi: _on_grid(rng.standard_normal(_buf_shape(case, bi)), case.dtype) for bi in data} if _planes(case) and N < M else None

    def run(entry):
        planes_before = None
        if before is not None:
            for bi, a in before.items():
                eng.debug_write_buffer(bi, a)
            eng.debug_run_ops(0, len(case.graph.ops) - 1, M)
            planes_before = _read_all(eng, case, M)
        for bi, a in data.items():
            eng.debug_write_buffer(bi, a)
        if entry == "u8":
            eng.infer_u8(frames)
        elif entry == "f32":
            x = (frames.astype(np.float64) * (1.0 / 255)).astype(np.float32)[..., ::-1].transpose(0, 3, 1, 2)
            eng.infer_f32(np.ascontiguousarray(x))
        else:
            eng.debug_run_ops(0, len(case.graph.ops) - 1, N)
        full = _read_all(eng, case, M)
        # (b') frames N .. max_batch - 1 keep their bytes
        for b, a in full.items():
            if N < M:
                was = planes_before[b] if isinstance(b, str) else data[b]
                assert a[N:].tobytes() == was[N:].tobytes(), f"{case.id} ({entry}): {b} written past frame {N}"
        return {o[0]: full[o[0]][:N] for o in case.outs}

    runs = {e: run(e) for e in (("u8", "f32") if case.stem else ("ops",))}
    if case.twin_env:
        twin = _engine(case, monkeypatch, case.twin_env)
        eng.close()
        eng = twin
        twin_out = run("ops")
        for b, a in runs["ops"].items():
            assert a.tobytes() == twin_out[b].tobytes(), f"{case.id}: {b} differs under {case.twin_env}"
    eng.close()

    # (b) channels outside the op's range keep their bits
    for entry, got in runs.items():
        for b, a in got.items():
            if isinstance(b, str):
                continue
            keep = np.ones(a.shape[-1], bool)
            for ob, off, c in case.outs:
                if ob == b:
                    keep[off:off + c] = False
            assert a[..., keep].tobytes() == data[b][:N][..., keep].tobytes(), f"{case.id} ({entry}): channels outside the output range were written"

    shown = ", ".join(f"op {i} {k}: {items} items on {grid} CTAs" for i, k, items, grid in launches)
    ref = _reference(case, case.graph, data, frames)
    if case.mutate is None:   # max-pool: exact
        for entry, got in runs.items():
            for (b, off, c), r in zip(case.outs, ref):
                want = r.astype(np.float16 if case.dtype == "f16" else np.float32)
                assert got[b][..., off:off + c].tobytes() == want.tobytes(), f"{case.id}: max-pool differs from the reference"
        print(f"[kernel bound] {case.id}: {case.kernels[0]} bit-exact")
        return 0.0
    mag = _reference(case, case.graph, data, frames, magnitude=True)
    # the fp16 / TF32 buffers hold the result rounded once more (2^-11 |ref|); the conf / paf planes hold it unrounded
    bound = [(0.0 if isinstance(o[0], str) else 2.0 ** -11) * np.abs(r) + (case.K + 2) * 2.0 ** -23 * m + 2.0 ** -24
             for o, r, m in zip(case.outs, ref, mag)]
    worst = 0.0
    for entry, got in runs.items():
        for (b, off, c), r, bd in zip(case.outs, ref, bound):
            g64 = got[b][..., off:off + c].astype(np.float64)
            assert np.isfinite(g64).all(), f"{case.id} ({entry}): non-finite output at {np.argwhere(~np.isfinite(g64))[0].tolist()}"
            ratio = np.abs(g64 - r) / bd
            i = np.unravel_index(np.argmax(ratio), ratio.shape)
            assert ratio[i] <= 1.0, f"{case.id} ({entry}): {b}: |got - ref| = {abs(g64[i] - r[i]):.3e} > bound {bd[i]:.3e} at {i} (got {g64[i]}, ref {r[i]})"
            worst = max(worst, float(ratio.max()))
        # (c) the bound rejects wrong references
        for kind, mg in _mutants(case):
            mref = _reference(case, mg, data, frames)
            changed = broken = 0
            for (b, off, c), r, mr, bd in zip(case.outs, ref, mref, bound):
                g64 = got[b][..., off:off + c].astype(np.float64)
                ch = mr != r
                changed += int(ch.sum())
                broken += int((np.abs(g64 - mr) > bd)[ch].sum())
            assert changed > 0, f"{case.id}: the {kind} mutation changes nothing"
            assert broken > 0.5 * changed, f"{case.id} ({entry}): the bound accepts the {kind}-mutated reference on {changed - broken} of {changed} changed outputs"
    print(f"[kernel bound] {case.id}: {case.kernels} worst |got - ref| / bound {worst:.3f}; {shown}")
    return worst


@gpu
@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_kernel_against_fp64_reference(case, monkeypatch):
    _run_and_check(case, monkeypatch, np.random.default_rng(zlib.crc32(case.id.encode())))


@gpu
def test_cases_reach_every_conv_kernel(monkeypatch):
    """the engines of the cases above, created but not run: together they launch all 48 conv kernels"""
    seen = set()
    for case in CASES:
        eng = _engine(case, monkeypatch)
        seen |= {eng.debug_op_kernel(i) for i in range(len(case.graph.ops))}
        eng.close()
    missing = CONV_KERNELS - seen
    print(f"[kernel inventory] {len(CONV_KERNELS) - len(missing)}/{len(CONV_KERNELS)} conv kernels reached")
    assert not missing, sorted(missing)


@gpu
def test_fused_pointwise_depthwise_is_bit_identical_to_two_launches(monkeypatch):
    """a conv followed by a 1x1 depthwise op: the depthwise stage runs in the conv's epilogue and rounds the tensor in between to
    fp16 exactly as the two launches do, so the output bytes must agree with HPB_NO_DW1_FUSE=1"""
    rng = np.random.default_rng(5)
    g = _graph("conv+dw1")
    a, b, c = g.add_buffer(64, 0), g.add_buffer(48, 0), g.add_buffer(56, 0)
    g.add_conv(a, b, _conv_w(rng, 1, 48, 64, 3), rng.standard_normal(48).astype(np.float32), _slopes(rng, 48))
    g.add_dwconv(b, c, rng.standard_normal((48, 1, 1)).astype(np.float32), rng.standard_normal(48).astype(np.float32), _slopes(rng, 48),
                 out_ch_off=8)
    N, H, W = S1
    x = rng.standard_normal((N, H, W, 64)).astype(np.float16)
    outs = []
    for env, kernels in (({}, ["conv<f16,48>", "none"]), ({"HPB_NO_DW1_FUSE": "1"}, ["conv<f16,48>", "dw_strip<1,1>"])):
        case = Case("dw1", "f16", S1, g, kernels, [], 0, env=env)
        eng = _engine(case, monkeypatch)
        assert [eng.debug_op_kernel(i) for i in range(2)] == kernels
        eng.debug_write_buffer(a, x)
        eng.debug_write_buffer(c, np.full((N, H, W, 56), 7.0, np.float16))
        eng.debug_run_ops(0, 1, N)
        outs.append(eng.debug_read_buffer(c, N))
        eng.close()
    assert outs[0].tobytes() == outs[1].tobytes()
    assert (outs[0][..., :8] == 7.0).all() and np.abs(outs[0][..., 8:]).max() > 0


# ---- pack validation: creating the engine refuses ops whose kernels would address outside their buffers ----

def _expect_rejected(g, what, in_hw=(24, 16)):
    with pytest.raises(capi.HyperposeError) as e:
        capi.Engine(g.to_pack(), in_hw, max_batch_size=1)
    assert e.value.status == capi.HP_ERR_ARG and what in str(e.value), str(e.value)


@gpu
@pytest.mark.parametrize("in_off,out_off,in_c,out_c", [(4, 0, 48, 48), (0, 12, 48, 48), (16, 0, 48, 48), (0, 16, 48, 48)])
def test_maxpool_channel_ranges_are_validated(in_off, out_off, in_c, out_c):
    """misaligned offsets (16-byte / float4 loads) and channel ranges past the buffer"""
    g = _graph("bad pool")
    a = g.add_buffer(in_c, 0); b = g.add_buffer(out_c, 1)
    g.add_maxpool(a, b, 40)
    g.ops[-1].in_ch_off, g.ops[-1].out_ch_off = in_off, out_off
    _expect_rejected(g, "maxpool op 0")


@gpu
@pytest.mark.parametrize("down,head_type", [(1, 0), (0, 1)])
def test_split_output_conv_geometry_is_validated(down, head_type):
    """the conf / paf planes are out_h x out_w: the output conv's input must be at the header's output resolution, head_type 0"""
    rng = np.random.default_rng(0)
    g = _graph("bad split")
    g.head_type = head_type
    a = g.add_buffer(64, down)
    g.add_conv(a, 0, _conv_w(rng, 1, 57, 64, 1), np.zeros(57, np.float32), np.ones(57, np.float32), out_mode=models.OUT_F32_NCHW_SPLIT, split=19)
    _expect_rejected(g, "output conv op 0")


@gpu
@pytest.mark.parametrize("pif_down,paf_down", [(2, 1), (1, 2)])
def test_pifpaf_head_input_resolution_is_validated(pif_down, paf_down):
    """the head kernels read input row y >> 1 for every output row: both inputs must be at out_down_shift"""
    g = models.Graph("bad heads", 85, 171, 1, head_type=1)
    pif = g.add_buffer(344, pif_down); paf = g.add_buffer(688, paf_down)
    g.ops.append(models.Op(models.OP_PIFPAF_HEAD, in_buf=pif, res_buf=paf))
    _expect_rejected(g, "pifpaf head op 0")
