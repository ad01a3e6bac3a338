"""Model graphs + the HPB2PACK writer (host-side logic; numpy only).

The reference's C++ engine consumes .onnx/.uff/.trt files downloaded from Google Drive
(scripts/downloader.py:11-21; none in the tree, no network).  This module rebuilds the same
layer tables from the reference's Python model definitions and serialises them, together with
seeded random-init weights, into the flat pack `hp_engine_create` loads
(hyperpose_b200/csrc/pack_format.h).  A converter from real trained weights only has to fill
`Graph.add_conv(..., weight=..., bias=..., alpha=...)` with the trained arrays.

Graphs:
  * openpose_vgg19  -- hyperpose/Model/backbones.py:447-509 (VGG-19 first 10 convs, 3 max-pools)
                       + hyperpose/Model/openpose/model/openpose.py:36-47 (CPM 512->256->128),
                       :119-154 (init stage), :156-199 (5 refinement stages, 7x7 convs, PReLU).
"""
from __future__ import annotations

import struct
from dataclasses import dataclass, field

import numpy as np

OP_IM2COL3, OP_CONV, OP_MAXPOOL2, OP_DWCONV, OP_PIFPAF_HEAD, OP_PPN_HEAD = 1, 2, 3, 4, 5, 6
OUT_F16_NHWC, OUT_F32_NCHW_SPLIT = 0, 1
PACK_MAGIC = b"HPB2PACK"
PACK_VERSION = 2


@dataclass
class Op:
    type: int
    in_buf: int = 0
    out_buf: int = 0
    in_ch_off: int = 0
    out_ch_off: int = 0
    R: int = 1
    S: int = 1
    groups: int = 1
    cin_g: int = 0
    cout_g: int = 0
    out_mode: int = OUT_F16_NHWC
    split: int = 0
    im2col_input: int = 0
    stride: int = 1
    res_buf: int = 0
    res_ch_off: int = 0
    res_mode: int = 0                  # 1: act(conv + res)   2: act(conv) + res
    weight: np.ndarray | None = None   # [G, cout_g, cin_g, R, S] float32 (OP_DWCONV: [C, K, K]; dilated: the window, see add_dwconv)
    bias: np.ndarray | None = None     # [G*cout_g]
    alpha: np.ndarray | None = None    # [G*cout_g]  PReLU slope; 0 = ReLU, 1 = linear
    name: str = ""
    dilation: int = 1                  # OP_DWCONV: taps this many pixels apart (2 only for 3x3 at stride 1); written as 0 when 1

    def taps(self) -> np.ndarray:
        """the filter as the pack stores it: [G, cout_g, cin_g, R, S], or a depthwise op's [C, K, K] taps (every dilation-th element of
        a dilated op's window)"""
        d = self.dilation
        if self.type != OP_DWCONV or d == 1:
            return self.weight
        off = self.weight.copy()
        off[:, ::d, ::d] = 0
        assert not off.any(), f"{self.name}: a dilated depthwise window holds nonzero values between its taps"
        return self.weight[:, ::d, ::d]


@dataclass
class Graph:
    name: str
    conf_channels: int = 19
    paf_channels: int = 38
    out_down_shift: int = 3
    mean: tuple = (0.0, 0.0, 0.0)
    head_type: int = 0                 # 1: OpenPifPaf fields (pif[17,5,ho,wo] / paf[19,9,ho,wo] in the conf / paf output slots)
                                       # 2: Pose Proposal Network (boxes [6,K,gh,gw] / edges [L,nh,nw,gh,gw] in the conf / paf output slots)
    buffers: list = field(default_factory=list)   # (channels, down_shift)
    ops: list = field(default_factory=list)
    act_scales: np.ndarray | None = None          # INT8 calibration table: one fp32 scale per buffer (set_int8_scales), or None

    def add_buffer(self, channels: int, down_shift: int) -> int:
        assert channels % 8 == 0
        self.buffers.append((channels, down_shift))
        return len(self.buffers) - 1

    def add_im2col(self, out_buf: int, stride: int = 1, ksize: int = 3, name="im2col") -> None:
        self.ops.append(Op(OP_IM2COL3, out_buf=out_buf, R=ksize, S=ksize, stride=stride, name=name))

    def add_dwconv(self, in_buf, out_buf, weight, bias, alpha, stride=1, in_ch_off=0, out_ch_off=0, name="dw", dilation=1) -> None:
        """depthwise KxK conv (K in {1,3}) + bias + PReLU; weight [C, K, K].  dilation 2 (3x3, stride 1): taps 2 pixels apart, TF 'SAME'
        over the 5 x 5 window (2 pixels of padding per side).  A dilated op keeps its filter as that window, [C, (K-1)d+1, (K-1)d+1] with
        zeros between the taps: anything that reads Op.weight as a dense depthwise filter (the CPU references of oracle/ and tests/)
        computes the dilated convolution.  The pack stores the K x K taps and the dilation (Op.taps)."""
        C, K, K2 = weight.shape
        assert K == K2 and K in (1, 3) and C % 8 == 0
        assert dilation == 1 or (dilation == 2 and K == 3 and stride == 1), (dilation, K, stride)
        w = np.ascontiguousarray(weight, np.float32)
        if dilation != 1:
            win = np.zeros((C, (K - 1) * dilation + 1, (K - 1) * dilation + 1), np.float32)
            win[:, ::dilation, ::dilation] = w
            w = win
        self.ops.append(Op(OP_DWCONV, in_buf, out_buf, in_ch_off, out_ch_off, K, K, 1, C, C, stride=stride,
                           weight=w, bias=np.ascontiguousarray(bias, np.float32).reshape(-1),
                           alpha=np.ascontiguousarray(alpha, np.float32).reshape(-1), name=name, dilation=dilation))

    def add_maxpool(self, in_buf: int, out_buf: int, channels: int, name="pool", ksize: int = 2) -> None:
        self.ops.append(Op(OP_MAXPOOL2, in_buf=in_buf, out_buf=out_buf, R=ksize, S=ksize, cout_g=channels, name=name))

    def add_conv(self, in_buf, out_buf, weight, bias, alpha, in_ch_off=0, out_ch_off=0, out_mode=OUT_F16_NHWC, split=0,
                 im2col_input=0, name="conv", res_buf=0, res_ch_off=0, res_mode=0) -> None:
        G, cout_g, cin_g, R, S = weight.shape
        self.ops.append(Op(OP_CONV, in_buf, out_buf, in_ch_off, out_ch_off, R, S, G, cin_g, cout_g, out_mode, split, im2col_input,
                           weight=np.ascontiguousarray(weight, np.float32), bias=np.ascontiguousarray(bias, np.float32).reshape(-1),
                           alpha=np.ascontiguousarray(alpha, np.float32).reshape(-1), name=name,
                           res_buf=res_buf, res_ch_off=res_ch_off, res_mode=res_mode))

    def set_int8_scales(self, absmax) -> None:
        """INT8 scale table from per-buffer max |x| (Engine.calibrate): s = absmax / 127, an all-zero buffer gets 1.  A max-pool works
        on the int8 values, so its input and output buffers need one scale: buffers joined by max-pools share the largest absmax among
        them (a pool's output buffer may also hold other ops' results, e.g. MobilenetThin's concat: none of them is clipped)."""
        a = np.asarray(absmax, np.float32).reshape(-1).copy()
        assert a.size == len(self.buffers), (a.size, len(self.buffers))
        root = list(range(a.size))

        def find(b):
            while root[b] != b:
                root[b] = root[root[b]]
                b = root[b]
            return b
        for op in self.ops:
            if op.type == OP_MAXPOOL2:
                root[find(op.out_buf)] = find(op.in_buf)
        top = {}
        for b in range(a.size):
            top[find(b)] = max(top.get(find(b), np.float32(0)), a[b])
        a = np.array([top[find(b)] for b in range(a.size)], np.float32)
        self.act_scales = np.where(a > 0, a / np.float32(127.0), np.float32(1.0)).astype(np.float32)

    # ---- serialisation (layout of pack_format.h) ----
    def to_pack(self) -> bytes:
        """the pack; with act_scales set, the INT8 scale table follows the blob and the header's reserved[0] counts it"""
        blob = []
        off = 0
        op_recs = []
        for op in self.ops:
            w_off = b_off = a_off = 0
            if op.type in (OP_CONV, OP_DWCONV):
                w = op.taps()
                w_off = off; blob.append(w.reshape(-1)); off += w.size
                b_off = off; blob.append(op.bias); off += op.bias.size
                a_off = off; blob.append(op.alpha); off += op.alpha.size
            op_recs.append(struct.pack("<18I3Q", op.type, op.in_buf, op.out_buf, op.in_ch_off, op.out_ch_off, op.R, op.S, op.groups,
                                       op.cin_g, op.cout_g, op.out_mode, op.split, op.im2col_input, op.stride,
                                       op.res_buf, op.res_ch_off, op.res_mode, 0 if op.dilation == 1 else op.dilation, w_off, b_off, a_off))
        blob_arr = np.concatenate(blob).astype("<f4") if blob else np.zeros(0, "<f4")
        table = b""
        if self.act_scales is not None:
            assert len(self.act_scales) == len(self.buffers), (len(self.act_scales), len(self.buffers))
            table = np.asarray(self.act_scales, "<f4").tobytes()
        hdr = struct.pack("<8s6I3f5IQ", PACK_MAGIC, PACK_VERSION, len(self.buffers), len(self.ops), self.conf_channels,
                          self.paf_channels, self.out_down_shift, *[float(m) for m in self.mean], self.head_type,
                          len(self.buffers) if table else 0, 0, 0, 0, blob_arr.size)
        bufs = b"".join(struct.pack("<2I", c, d) for c, d in self.buffers)
        return hdr + bufs + b"".join(op_recs) + blob_arr.tobytes() + table

    def flops_per_frame(self, in_h: int, in_w: int) -> float:
        total = 0.0
        for op in self.ops:
            if op.type not in (OP_CONV, OP_DWCONV):
                continue
            _, d = self.buffers[op.out_buf if op.type == OP_DWCONV or op.out_mode == OUT_F16_NHWC else op.in_buf]
            h, w = in_h, in_w
            for _ in range(d):
                h, w = (h + 1) // 2, (w + 1) // 2
            if op.type == OP_DWCONV:
                total += 2.0 * h * w * op.cout_g * op.R * op.S
            else:
                total += 2.0 * h * w * op.groups * op.cout_g * op.cin_g * op.R * op.S
        return total


def _he(rng, G, cout, cin, R, S, gain=2.0):
    std = np.sqrt(gain / (cin * R * S))
    return (rng.standard_normal((G, cout, cin, R, S)) * std).astype(np.float32)


def _block_diag(w_a: np.ndarray, w_b: np.ndarray) -> np.ndarray:
    """two [1,co,ci,R,S] branch weights -> one dense [1, co_a+co_b, ci_a+ci_b, R, S] block-diagonal conv"""
    _, ca, ia, R, S = w_a.shape
    _, cb, ib, _, _ = w_b.shape
    w = np.zeros((1, ca + cb, ia + ib, R, S), np.float32)
    w[0, :ca, :ia] = w_a[0]
    w[0, ca:, ia:] = w_b[0]
    return w


def openpose_vgg19(seed: int = 0, n_stages: int = 6, weights=None) -> Graph:
    """OpenPose-COCO on VGG-19 (BASELINE.json config 3).  `weights`: a hyperpose_b200.weights source
    (ListWeights of a trained TensorLayer model, or RandomWeights(seed) -- the default: He-normal, seeded).

    Both branches of a stage (conf: L2, paf: L1) are executed together: their first layers share the
    input and are merged into one conv (cout 256); later layers run as a 2-group conv; the two 1x1
    output convs are fused into one block-diagonal conv writing [conf | paf] straight into the next
    stage's concat buffer (openpose.py:74: concat([features, conf, paf])).
    """
    from .weights import RandomWeights
    ws = weights if weights is not None else RandomWeights(seed)
    g = Graph("openpose_vgg19", 19, 38, 3, mean=tuple(np.array([103.939, 116.779, 123.68]) / 255.0))  # backbones.py:455
    relu = lambda n: np.zeros(n, np.float32)

    def plain(name, co, ci, k):                 # single conv -> ([1,co,ci,k,k], bias)
        w, b = ws.conv(name, co, ci, k)
        return w[None], b

    def pair(prefix, i, co_conf, co_paf, ci, k, mode):
        """layer i of the conf and the paf branch as one conv: 'shared' input (concat along cout), 'grouped'
        (2 groups), 'blockdiag' (different cout per branch, e.g. the 19 / 38-channel outputs); PReLU slopes concatenated"""
        gain = 1.0 if mode == "blockdiag" else 2.0
        wc, bc = ws.conv(f"{prefix}.conf.{i}", co_conf, ci, k, gain)
        wp, bp = ws.conv(f"{prefix}.paf.{i}", co_paf, ci, k, gain)
        al = np.concatenate([ws.prelu(f"{prefix}.conf.{i}", co_conf), ws.prelu(f"{prefix}.paf.{i}", co_paf)])
        if mode == "shared":
            w = np.concatenate([wc, wp], axis=0)[None]
        elif mode == "grouped":
            w = np.stack([wc, wp])
        else:
            w = _block_diag(wc[None], wp[None])
        return w, np.concatenate([bc, bp]), al

    # ---- VGG-19 front (backbones.py:461-476) ----
    b_col = g.add_buffer(64, 0)
    g.add_im2col(b_col)
    cur = g.add_buffer(64, 0)
    g.add_conv(b_col, cur, *plain("conv1_1", 64, 3, 3), relu(64), im2col_input=1, name="conv1_1")
    nxt = g.add_buffer(64, 0)
    g.add_conv(cur, nxt, *plain("conv1_2", 64, 64, 3), relu(64), name="conv1_2")
    cur = g.add_buffer(64, 1); g.add_maxpool(nxt, cur, 64, "maxpool_1")
    for i, (ci, co) in enumerate([(64, 128), (128, 128)]):
        nxt = g.add_buffer(co, 1); g.add_conv(cur, nxt, *plain(f"conv2_{i+1}", co, ci, 3), relu(co), name=f"conv2_{i+1}"); cur = nxt
    nxt = g.add_buffer(128, 2); g.add_maxpool(cur, nxt, 128, "maxpool_2"); cur = nxt
    for i, (ci, co) in enumerate([(128, 256), (256, 256), (256, 256), (256, 256)]):
        nxt = g.add_buffer(co, 2); g.add_conv(cur, nxt, *plain(f"conv3_{i+1}", co, ci, 3), relu(co), name=f"conv3_{i+1}"); cur = nxt
    nxt = g.add_buffer(256, 3); g.add_maxpool(cur, nxt, 256, "maxpool_3"); cur = nxt
    for i, (ci, co) in enumerate([(256, 512), (512, 512)]):
        nxt = g.add_buffer(co, 3); g.add_conv(cur, nxt, *plain(f"conv4_{i+1}", co, ci, 3), relu(co), name=f"conv4_{i+1}"); cur = nxt
    # ---- CPM (openpose.py:36-39) ----
    nxt = g.add_buffer(256, 3); g.add_conv(cur, nxt, *plain("cpm_1", 256, 512, 3), relu(256), name="cpm_1"); cur = nxt
    cat = g.add_buffer(192, 3)   # [features 128 | conf 19 | paf 38 | 7 zero pad]: the refinement stages' input
    g.add_conv(cur, cat, *plain("cpm_2", 128, 256, 3), relu(128), name="cpm_2")
    ta = g.add_buffer(256, 3)
    tb = g.add_buffer(256, 3)
    wide = g.add_buffer(1024, 3)

    def out_conv(in_buf, prefix, i, cin_each, last, name):
        w, b, al = pair(prefix, i, 19, 38, cin_each, 1, "blockdiag")
        if last:
            g.add_conv(in_buf, 0, w, b, al, out_mode=OUT_F32_NCHW_SPLIT, split=19, name=name)
        else:
            g.add_conv(in_buf, cat, w, b, al, out_ch_off=128, name=name)

    # ---- init stage (openpose.py:119-154): 3x(3x3,128) + 1x1x512 + 1x1x{19,38}, PReLU after every conv ----
    g.add_conv(cat, ta, *pair("init", 1, 128, 128, 128, 3, "shared"), name="init_1")
    g.add_conv(ta, tb, *pair("init", 2, 128, 128, 128, 3, "grouped"), name="init_2")
    g.add_conv(tb, ta, *pair("init", 3, 128, 128, 128, 3, "grouped"), name="init_3")
    g.add_conv(ta, wide, *pair("init", 4, 512, 512, 128, 1, "grouped"), name="init_4")
    out_conv(wide, "init", 5, 512, n_stages == 1, "init_out")
    # ---- refinement stages (openpose.py:156-199): 5x(7x7,128) + 1x1x128 + 1x1x{19,38} ----
    for s in range(1, n_stages):
        g.add_conv(cat, ta, *pair(f"ref{s}", 1, 128, 128, 185, 7, "shared"), name=f"ref{s}_1")
        src, dst = ta, tb
        for k in range(2, 6):
            g.add_conv(src, dst, *pair(f"ref{s}", k, 128, 128, 128, 7, "grouped"), name=f"ref{s}_{k}")
            src, dst = dst, src
        g.add_conv(src, dst, *pair(f"ref{s}", 6, 128, 128, 128, 1, "grouped"), name=f"ref{s}_6")
        out_conv(dst, f"ref{s}", 7, 128, s == n_stages - 1, f"ref{s}_out")
    return g


def _bn_fold(rng, n):
    """random inference-time BatchNorm -> (scale, shift): y = scale * x + shift"""
    gamma = rng.uniform(0.8, 1.2, n); beta = rng.normal(0, 0.05, n); mean = rng.normal(0, 0.05, n); var = rng.uniform(0.8, 1.2, n)
    scale = gamma / np.sqrt(var + 1e-5)
    return scale.astype(np.float32), (beta - mean * scale).astype(np.float32)


def _r64(c: int) -> int:
    return (c + 63) // 64 * 64


def mobilenet_thin_openpose(seed: int = 0, n_stages: int = 6, weights=None) -> Graph:
    """OpenPose on MobilenetThin (BASELINE.json config 2): hyperpose/Model/backbones.py:240-297 (3x3/2 stem + 11
    depthwise-separable blocks, three scales concatenated to 1152 channels at stride 8) and
    hyperpose/Model/openpose/model/mbv2_th_openpose.py:106-158 (init + 5 refinement stages of separable blocks).
    Inference-time BatchNorm is folded: depthwise conv + BN (+ReLU) -> one OP_DWCONV; 1x1 conv + BN (+ReLU) -> one OP_CONV.
    The stem is Conv(act=relu) followed by BatchNorm(act=relu) (mbv2_th_openpose.py:160-166), which cannot be folded through
    the inner ReLU: conv(+bias, ReLU) then a 1x1 depthwise affine + ReLU.  The last separable block of a stage is built with
    act=None (:121,:127,:144,:151): BOTH of its BatchNorms are linear.  Both branches of a stage run together (grouped 1x1
    convs, block-diagonal output conv).
    `weights`: a hyperpose_b200.weights.MobilenetThinWeights (trained TensorLayer model); default = seeded random values."""
    rng = np.random.default_rng(seed)
    ws = weights
    g = Graph("mobilenet_thin_openpose", 19, 38, 3, mean=(0.0, 0.0, 0.0))
    relu = lambda n: np.zeros(n, np.float32)
    lin = lambda n: np.ones(n, np.float32)
    dw_w, bn, dw, pw = _sep_helpers(g, rng, ws)
    cur, cur_off, cur_c, cur_d = _mobilenet_stem(g, rng, ws, bn), 0, 32, 1
    cat_c = _r64(1152 + 57)
    cat = g.add_buffer(cat_c, 3)   # [maxpool(block3) 128 | block7 512 | block11 512 | conf 19 | paf 38 | 7 zero]
    # (n_filter, stride) of convblock_1..11 at scale_size 8 (backbones.py:264-275)
    blocks = [(64, 1), (128, 2), (128, 1), (256, 2), (256, 1), (512, 1), (512, 1), (512, 1), (512, 1), (512, 1), (512, 1)]
    for i, (co, st) in enumerate(blocks, start=1):
        d_out = cur_d + (1 if st == 2 else 0)
        t = g.add_buffer(_r64(cur_c), d_out)
        dw(cur, t, cur_c, 3, stride=st, in_off=cur_off, name=f"convblock_{i}_dw", wname=f"convblock_{i}")
        if i in (7, 11):     # concat_list[1] / [2] (backbones.py:288,293): written straight into the concat buffer
            off = 128 if i == 7 else 640
            pw(t, cat, 1, _r64(cur_c), co, out_off=off, cin_real=cur_c, name=f"convblock_{i}_pw", wname=f"convblock_{i}")
            cur, cur_off = cat, off
        else:
            nxt = g.add_buffer(_r64(co), d_out)
            pw(t, nxt, 1, _r64(cur_c), co, cin_real=cur_c, name=f"convblock_{i}_pw", wname=f"convblock_{i}")
            cur, cur_off = nxt, 0
        if i == 3:           # concat_list[0] = maxpool(x) (backbones.py:283)
            g.add_maxpool(cur, cat, 128, "maxpool")
        cur_c, cur_d = co, d_out

    def stage(cin_real, mid, last, name):
        """two branches of 5 separable blocks (mbv2_th_openpose.py:111-158) executed together"""
        C = cat_c
        br_names = [f"{name}.conf", f"{name}.paf"]
        wide = g.add_buffer(2 * C, 3)
        for br in range(2):
            if ws:
                wd = np.zeros((C, 3, 3), np.float32); wd[:cin_real] = dw_w(f"{br_names[br]}.1.dw", cin_real, 3)
                sc = np.ones(C, np.float32); sh = np.zeros(C, np.float32)
                sc[:cin_real], sh[:cin_real] = bn(f"{br_names[br]}.1.dwbn", cin_real)
            else:
                wd = dw_w("", C, 3)
                wd[cin_real:] = 0
                sc, sh = bn("", C)
                sh[cin_real:] = 0
            g.add_dwconv(cat, wide, wd * sc[:, None, None], sh, relu(C), out_ch_off=br * C, name=f"{name}_1_dw{br}")
        a = g.add_buffer(256, 3); b = g.add_buffer(256, 3)
        pw(wide, a, 2, C, 128, cin_real=cin_real, name=f"{name}_1_pw", wname=[f"{n_}.1" for n_ in br_names])
        for k in (2, 3):
            dw(a, b, 256, 3, name=f"{name}_{k}_dw", wname=[(f"{n_}.{k}", 128) for n_ in br_names])
            pw(b, a, 2, 128, 128, name=f"{name}_{k}_pw", wname=[f"{n_}.{k}" for n_ in br_names])
        dw(a, b, 256, 1, name=f"{name}_4_dw", wname=[(f"{n_}.4", 128) for n_ in br_names])
        m = g.add_buffer(2 * mid, 3)
        pw(b, m, 2, 128, mid, name=f"{name}_4_pw", wname=[f"{n_}.4" for n_ in br_names])
        m2 = g.add_buffer(2 * mid, 3)
        # block 5 is separable_block(act=None): its depthwise BatchNorm is linear too
        dw(m, m2, 2 * mid, 1, name=f"{name}_5_dw", act=False, wname=[(f"{n_}.5", mid) for n_ in br_names])
        if ws:
            w = _block_diag(ws.conv(f"{name}.conf.5.pw", 19, mid, 1)[0][None], ws.conv(f"{name}.paf.5.pw", 38, mid, 1)[0][None])
            sc, sh = (np.concatenate(x) for x in zip(bn(f"{name}.conf.5.pwbn", 19), bn(f"{name}.paf.5.pwbn", 38)))
        else:
            w = _block_diag(_he(rng, 1, 19, mid, 1, 1, 1.0), _he(rng, 1, 38, mid, 1, 1, 1.0))
            sc, sh = bn("", 57)
        w = w * sc.reshape(1, 57, 1, 1, 1)
        if last:
            g.add_conv(m2, 0, w, sh, lin(57), out_mode=OUT_F32_NCHW_SPLIT, split=19, name=f"{name}_out")
        else:
            g.add_conv(m2, cat, w, sh, lin(57), out_ch_off=1152, name=f"{name}_out")

    stage(1152, 512, n_stages == 1, "init")
    for s_ in range(1, n_stages):
        stage(1209, 128, s_ == n_stages - 1, f"ref{s_}")
    return g


def _sep_helpers(g, rng, ws):
    """the builders of MobileNet separable blocks (BatchNorm folded) on graph `g` -> (dw_w, bn, dw, pw).  Every tensor comes from `ws` by
    name when a trained model is imported (weights.BnNetWeights), else from the seeded generator `rng`, drawn in call order."""
    relu = lambda n: np.zeros(n, np.float32)
    lin = lambda n: np.ones(n, np.float32)

    def dw_w(name, C, K):
        return ws.dwconv(name, C, K) if ws else (rng.standard_normal((C, K, K)) * np.sqrt(2.0 / (K * K))).astype(np.float32)

    def bn(name, C):
        return ws.bn(name, C) if ws else _bn_fold(rng, C)

    def dw(in_buf, out_buf, C, K, stride=1, in_off=0, out_off=0, name="dw", act=True, wname=None, dilation=1):
        """depthwise conv + BN (+ReLU).  wname: one weight name, or a list of (name, channels) whose depthwise filters / BatchNorms are
        laid side by side"""
        parts = wname if isinstance(wname, list) else [(wname or name, C)]
        if ws:
            w = np.concatenate([dw_w(n_ + ".dw", c_, K) for n_, c_ in parts])
            sc, sh = (np.concatenate(x) for x in zip(*[bn(n_ + ".dwbn", c_) for n_, c_ in parts]))
        else:
            w = dw_w(name, C, K); sc, sh = bn(name, C)
        g.add_dwconv(in_buf, out_buf, w * sc[:, None, None], sh, relu(C) if act else lin(C), stride=stride, in_ch_off=in_off, out_ch_off=out_off,
                     name=name, dilation=dilation)

    def pw(in_buf, out_buf, groups, cin_g, cout_g, act=True, out_off=0, cin_real=None, name="pw", wname=None, **kw):
        """wname: None (random), one name (groups == 1) or one name per group"""
        if ws:
            names = wname if isinstance(wname, list) else [wname]
            w = np.zeros((groups, cout_g, cin_g, 1, 1), np.float32)
            scs, shs = [], []
            for gi, n_ in enumerate(names):
                ci = cin_real if cin_real is not None else cin_g
                w[gi, :, :ci] = ws.conv(n_ + ".pw", cout_g, ci, 1)[0]
                sc_, sh_ = bn(n_ + ".pwbn", cout_g); scs.append(sc_); shs.append(sh_)
            sc, sh = np.concatenate(scs), np.concatenate(shs)
        else:
            w = _he(rng, groups, cout_g, cin_g, 1, 1, 2.0 if act else 1.0)
            if cin_real is not None:
                w[:, :, cin_real:] = 0
            sc, sh = bn(name, groups * cout_g)
        w = w * sc.reshape(groups, cout_g, 1, 1, 1)
        g.add_conv(in_buf, out_buf, w, sh, relu(groups * cout_g) if act else lin(groups * cout_g), out_ch_off=out_off, name=name, **kw)

    return dw_w, bn, dw, pw


def _mobilenet_stem(g, rng, ws, bn):
    """conv_block(32, 3, strides=2) of MobilenetThin / MobilenetDilated (the second `conv_block` of backbones.py, :234-239): conv 3x3/2
    3->32 (+bias, ReLU), then BatchNorm(ReLU) as a 1x1 depthwise affine.  `bn`: _sep_helpers' BatchNorm source.  -> the 32-channel
    output buffer at stride 2 (64 channels wide)"""
    relu = lambda n: np.zeros(n, np.float32)
    b_col = g.add_buffer(64, 1); g.add_im2col(b_col, stride=2)
    b0 = g.add_buffer(64, 1)
    if ws:
        w0, bias0 = ws.conv("convblock_0.conv", 32, 3, 3)
        w0 = w0[None]
    else:
        w0, bias0 = _he(rng, 1, 32, 3, 3, 3), (rng.standard_normal(32) * 0.05).astype(np.float32)
    g.add_conv(b_col, b0, w0, bias0, relu(32), im2col_input=1, name="convblock_0")
    sc, sh = bn("convblock_0.bn", 32)
    b0b = g.add_buffer(64, 1)
    g.add_dwconv(b0, b0b, sc.reshape(32, 1, 1), sh, relu(32), name="convblock_0_bn")
    return b0b


def _resnet50_body(g, rng, ws, cur, cur_c, cur_d, layout):
    """the 16 bottleneck blocks of Resnet50_backbone (backbones.py:598-698).  BatchNorm folded; the residual add runs in the conv
    epilogue (relu(conv3 + res)).  A stride-2 block computes its 3x3 (and its 1x1 projection) at stride 1 and sub-samples with a
    one-hot depthwise 3x3/2 (centre tap of the TF-SAME window) / 1x1/2 op -- exact.  Returns (buffer, channels, down_shift)."""
    relu = lambda n: np.zeros(n, np.float32)
    lin = lambda n: np.ones(n, np.float32)

    def conv_bn(in_buf, out_buf, ci, co, k, act=True, name="c", gain=None, wname=None, **kw):
        if ws:
            w = ws.conv(wname[0], co, ci, k)[0][None]
            sc, sh = ws.bn(wname[1], co)
        else:
            w = _he(rng, 1, co, ci, k, k, gain if gain is not None else (2.0 if act else 1.0))
            sc, sh = _bn_fold(rng, co)
        g.add_conv(in_buf, out_buf, w * sc.reshape(1, co, 1, 1, 1), sh, relu(co) if act else lin(co), name=name, **kw)

    def subsample(in_buf, out_buf, C, centre3: bool, name):
        w = np.zeros((C, 3, 3), np.float32) if centre3 else np.ones((C, 1, 1), np.float32)
        if centre3:
            w[:, 1, 1] = 1.0
        g.add_dwconv(in_buf, out_buf, w, np.zeros(C, np.float32), lin(C), stride=2, name=name)

    for bi, (nf, nblk, st0) in enumerate(layout, start=1):
        for k in range(1, nblk + 1):
            st = st0 if k == 1 else 1
            name = f"block_{bi}_{k}"
            d_out = cur_d + (1 if st == 2 else 0)
            # residual path (backbones.py:676-682)
            if st != 1 or cur_c != 4 * nf:
                src = cur
                if st == 2:
                    src = g.add_buffer(_r64(cur_c), d_out); subsample(cur, src, cur_c, False, f"{name}_ds_sub")
                res = g.add_buffer(4 * nf, d_out)
                conv_bn(src, res, cur_c, 4 * nf, 1, act=False, name=f"{name}_ds", gain=0.5, wname=(f"{name}.ds_conv1", f"{name}.ds_bn1"))
            else:
                res = cur
            a = g.add_buffer(_r64(nf), cur_d); conv_bn(cur, a, cur_c, nf, 1, name=f"{name}_conv1", wname=(f"{name}.conv1", f"{name}.bn1"))
            b = g.add_buffer(_r64(nf), cur_d); conv_bn(a, b, nf, nf, 3, name=f"{name}_conv2", wname=(f"{name}.conv2", f"{name}.bn2"))
            if st == 2:
                b2 = g.add_buffer(_r64(nf), d_out); subsample(b, b2, nf, True, f"{name}_conv2_sub"); b = b2
            out = g.add_buffer(4 * nf, d_out)
            # (random init: small gain on the residual branch, like a trained net's near-zero last gamma: keeps the
            #  activations of 16 stacked blocks inside the fp16 range)
            conv_bn(b, out, nf, 4 * nf, 1, act=True, name=f"{name}_conv3", gain=0.1, res_buf=res, res_mode=1,
                    wname=(f"{name}.conv3", f"{name}.bn3"))   # relu(x + res)
            cur, cur_c, cur_d = out, 4 * nf, d_out
    return cur, cur_c, cur_d


def resnet50_lw_openpose(seed: int = 0, weights=None) -> Graph:
    """Lightweight-OpenPose head on ResNet-50 at stride 8 (BASELINE.json config 4):
    hyperpose/Model/backbones.py:587-698 (7x7/2 stem, 3x3/2 max-pool, 16 bottleneck blocks; block_3_1 / block_4_1 keep
    stride 1 when scale_size == 8, :598-601) + hyperpose/Model/openpose/model/lw_openpose.py:106-191 (CPM, init stage,
    one refinement stage with residual blocks).  BatchNorm folded; residual adds run in the conv epilogue
    (ResNet: relu(conv + res); LW blocks: relu(bn(conv)) + res).
    `weights`: a hyperpose_b200.weights.Resnet50LwWeights (trained TensorLayer model); default = seeded random values."""
    rng = np.random.default_rng(seed)
    ws = weights
    g = Graph("resnet50_lw_openpose", 19, 38, 3, mean=(0.0, 0.0, 0.0))
    relu = lambda n: np.zeros(n, np.float32)

    col = g.add_buffer(192, 1); g.add_im2col(col, stride=2, ksize=7)
    c1 = g.add_buffer(64, 1)
    if ws:
        w = ws.conv("conv1", 64, 3, 7)[0][None]; sc, sh = ws.bn("bn1", 64)
    else:
        w = _he(rng, 1, 64, 3, 7, 7); sc, sh = _bn_fold(rng, 64)
    g.add_conv(col, c1, w * sc.reshape(1, 64, 1, 1, 1), sh, relu(64), im2col_input=1, name="conv1+bn1")
    x = g.add_buffer(64, 2); g.add_maxpool(c1, x, 64, "maxpool_1", ksize=3)
    # (n_filter, blocks, stride of the first block) at scale_size 8
    cur, cur_c, cur_d = _resnet50_body(g, rng, ws, x, 64, 2, [(64, 3, 1), (128, 4, 2), (256, 6, 1), (512, 3, 1)])
    _lw_head(g, rng, ws, cur, cur_c)
    return g


def _lw_head(g, rng, ws, cur, cur_c):
    """the LightWeightOpenPose head on a stride-8 backbone output `cur` of `cur_c` channels (lw_openpose.py:106-191): CPM, init stage,
    one refinement stage with residual blocks (relu(bn(conv)) + res in the conv epilogue), conf / paf into the split outputs.
    Layer names (cpm.*, init.*, ref.b{k}.*) are those of weights._lw_head_order, for every backbone."""
    relu = lambda n: np.zeros(n, np.float32)
    lin = lambda n: np.ones(n, np.float32)
    b_ = lambda n: (rng.standard_normal(n) * 0.05).astype(np.float32)

    def lw_conv(in_buf, out_buf, ci, co, k, act=True, name="c", wname=None, **kw):      # Conv2d(+bias, relu)
        if ws:
            w, b = ws.conv(wname, co, ci, k); w = w[None]
        else:
            w, b = _he(rng, 1, co, ci, k, k, 2.0 if act else 1.0), b_(co)
        g.add_conv(in_buf, out_buf, w, b, relu(co) if act else lin(co), name=name, **kw)

    def lw_block(in_buf, out_buf, ci, co, k, name, wname=None, **kw):                   # conv_block: Conv2d(+bias) + BN + relu (lw_openpose.py:193-199)
        if ws:
            w, b = ws.conv(wname, co, ci, k); w = w[None]; sc, sh = ws.bn(wname + ".bn", co)
        else:
            w = _he(rng, 1, co, ci, k, k); sc, sh = _bn_fold(rng, co); b = b_(co)
        g.add_conv(in_buf, out_buf, w * sc.reshape(1, co, 1, 1, 1), sh + b * sc, relu(co), name=name, **kw)

    def head_pair(in_buf, wide_buf, out_spec, prefix, name_mid, name_out):
        """conf_block / paf_block (lw_openpose.py:131-143,166-177): 1x1x512 (relu) + 1x1x{19,38} each; the two 512-channel convs
        share their input (one conv, cout 1024), the two output convs form one block-diagonal conv"""
        if ws:
            (wc1, bc1), (wp1, bp1) = ws.conv(f"{prefix}.conf.1", 512, 128, 1), ws.conv(f"{prefix}.paf.1", 512, 128, 1)
            w1, b1 = np.concatenate([wc1, wp1], axis=0)[None], np.concatenate([bc1, bp1])
            (wc2, bc2), (wp2, bp2) = ws.conv(f"{prefix}.conf.2", 19, 512, 1), ws.conv(f"{prefix}.paf.2", 38, 512, 1)
            w2, b2 = _block_diag(wc2[None], wp2[None]), np.concatenate([bc2, bp2])
        else:
            w1, b1 = np.concatenate([_he(rng, 1, 512, 128, 1, 1), _he(rng, 1, 512, 128, 1, 1)], axis=1), b_(1024)
        g.add_conv(in_buf, wide_buf, w1, b1, relu(1024), name=name_mid)
        if not ws:
            w2, b2 = _block_diag(_he(rng, 1, 19, 512, 1, 1, 1.0), _he(rng, 1, 38, 512, 1, 1, 1.0)), b_(57)
        g.add_conv(wide_buf, out_spec[0], w2, b2, lin(57), name=name_out, **out_spec[1])

    # ---- CPM (lw_openpose.py:106-121) ----
    t0 = g.add_buffer(128, 3); lw_conv(cur, t0, cur_c, 128, 1, name="cpm_init", wname="cpm.init")
    t1 = g.add_buffer(128, 3); lw_block(t0, t1, 128, 128, 3, "cpm_b1", wname="cpm.b1")
    t2 = g.add_buffer(128, 3); lw_block(t1, t2, 128, 128, 3, "cpm_b2", wname="cpm.b2")
    t3 = g.add_buffer(128, 3); lw_block(t2, t3, 128, 128, 3, "cpm_b3", wname="cpm.b3", res_buf=t0, res_mode=2)          # x + main_block(x)
    cat = g.add_buffer(192, 3)                                                                            # [cpm 128 | conf 19 | paf 38 | 7]
    lw_conv(t3, cat, 128, 128, 3, name="cpm_end", wname="cpm.end")
    # ---- init stage (:123-149) ----
    i1 = g.add_buffer(128, 3); lw_conv(cat, i1, 128, 128, 3, name="init_1", wname="init.1")
    i2 = g.add_buffer(128, 3); lw_conv(i1, i2, 128, 128, 3, name="init_2", wname="init.2")
    i3 = g.add_buffer(128, 3); lw_conv(i2, i3, 128, 128, 3, name="init_3", wname="init.3")
    wide = g.add_buffer(1024, 3)
    head_pair(i3, wide, (cat, dict(out_ch_off=128)), "init", "init_4", "init_out")
    # ---- refinement stage (:151-191): 5 residual blocks, then 1x1x512 + 1x1x{19,38} ----
    src, ci = cat, 185
    for k in range(1, 6):
        r0 = g.add_buffer(128, 3)
        if ws:
            w, b = ws.conv(f"ref.b{k}.init", 128, ci, 1)
            w = w[None]
        else:
            w, b = _he(rng, 1, 128, ci, 1, 1), b_(128)
        g.add_conv(src, r0, w, b, relu(128), name=f"ref_b{k}_init")
        r1 = g.add_buffer(128, 3); lw_block(r0, r1, 128, 128, 3, f"ref_b{k}_c1", wname=f"ref.b{k}.c1")
        r2 = g.add_buffer(128, 3); lw_block(r1, r2, 128, 128, 3, f"ref_b{k}_c2", wname=f"ref.b{k}.c2", res_buf=r0, res_mode=2)
        src, ci = r2, 128
    wide2 = g.add_buffer(1024, 3)
    head_pair(src, wide2, (0, dict(out_mode=OUT_F32_NCHW_SPLIT, split=19)), "ref", "ref_4", "ref_out")


# (block name, n_filter) of vggtiny_backbone at scale_size 8 (backbones.py:343-365); "pool" is MaxPool2d(2, 2, 'SAME')
VGGTINY_LAYERS = [("block_1_1", 32), ("block_1_2", 64), "pool", ("block_2_1", 128), ("block_2_2", 128), "pool",
                  ("block_3_1", 200), ("block_3_2", 200), ("block_3_3", 200), "pool", ("block_4_1", 384), ("block_4_2", 384)]


def lw_openpose_vggtiny(seed: int = 0, weights=None) -> Graph:
    """Lightweight-OpenPose on TinyVGG (the model of the reference's quick start, export_pb.py --model_type=LightweightOpenpose
    --model_backbone=Vggtiny): vggtiny_backbone(scale_size=8) (backbones.py:343-391: nine 3x3 Conv2d(+bias) + BatchNorm(relu) blocks,
    three 2x2 'SAME' max-pools with ceil output, 384 channels at stride 8), then the LW head (_lw_head).  BatchNorm folded.
    A 32- or 200-channel tensor lives in a buffer rounded up to 64 channels, whose zero pad channels the next conv reads as its
    padded K.  `weights`: a hyperpose_b200.weights.LwVggtinyWeights; default = seeded random values."""
    rng = np.random.default_rng(seed)
    ws = weights
    g = Graph("lw_openpose_vggtiny", 19, 38, 3, mean=(0.0, 0.0, 0.0))
    col = g.add_buffer(64, 0); g.add_im2col(col)
    cur, cur_c, cur_d, n_pool = col, 3, 0, 0
    for layer in VGGTINY_LAYERS:
        if layer == "pool":
            n_pool += 1
            nxt = g.add_buffer(_r64(cur_c), cur_d + 1); g.add_maxpool(cur, nxt, cur_c, f"maxpool_{n_pool}")
            cur, cur_d = nxt, cur_d + 1
            continue
        name, co = layer
        if ws:
            w, b = ws.conv(name, co, cur_c, 3); w = w[None]; sc, sh = ws.bn(name + ".bn", co)
        else:
            w = _he(rng, 1, co, cur_c, 3, 3); b = (rng.standard_normal(co) * 0.05).astype(np.float32); sc, sh = _bn_fold(rng, co)
        nxt = g.add_buffer(_r64(co), cur_d)
        g.add_conv(cur, nxt, w * sc.reshape(1, co, 1, 1, 1), sh + b * sc, np.zeros(co, np.float32), im2col_input=int(cur == col), name=name)
        cur, cur_c = nxt, co
    _lw_head(g, rng, ws, cur, cur_c)
    return g


def lw_openpose_resnet18(seed: int = 0, weights=None) -> Graph:
    """Lightweight-OpenPose on ResNet-18: Resnet18_backbone(scale_size=8) (backbones.py:512-585: 7x7/2 stem, 3x3/2 max-pool, blocks
    2_1 .. 5_1; at scale 8 blocks 4_1 and 5_1 keep stride 1, so 512 channels at stride 8), then the LW head (_lw_head).  Blocks as in
    ppn_resnet18 (_resnet18_body).  `weights`: a hyperpose_b200.weights.LwResnet18Weights; default = seeded random values."""
    rng = np.random.default_rng(seed)
    ws = weights
    g = Graph("lw_openpose_resnet18", 19, 38, 3, mean=(0.0, 0.0, 0.0))
    cur, cur_c, cur_d = _resnet18_body(g, rng, ws, *_ppn_stem(g, rng, ws), RESNET18_STRIDES_8)
    _lw_head(g, rng, ws, cur, cur_c)
    return g


# (n_filter, stride, dilation) of the eleven dw_conv_blocks of MobilenetDilated_backbone (backbones.py:201-229; scale_size is forced to 8,
# so the two `strides` variables there are (1, 1))
MOBILENET_DILATED_BLOCKS = [(64, 1, 1), (128, 2, 1), (128, 1, 1), (256, 2, 1), (256, 1, 1), (512, 1, 1), (512, 1, 2), (512, 1, 1),
                            (512, 1, 1), (512, 1, 1), (512, 1, 1)]


def lw_openpose_mobilenet_dilated(seed: int = 0, weights=None) -> Graph:
    """Lightweight-OpenPose on its default backbone, MobilenetDilated_backbone (lw_openpose.py:33-37, backbones.py:201-229): the
    MobilenetThin stem (_mobilenet_stem), eleven dw_conv_blocks -- DepthwiseConv2d (no bias) + BatchNorm(relu), Conv2d 1x1 (no bias) +
    BatchNorm(relu) -- down to stride 8 with 512 channels, the first 512 -> 512 block's depthwise conv dilated by 2, then the LW head
    (_lw_head).  BatchNorm folded.  `weights`: a hyperpose_b200.weights.LwMobilenetDilatedWeights; default = seeded random values."""
    rng = np.random.default_rng(seed)
    ws = weights
    g = Graph("lw_openpose_mobilenet_dilated", 19, 38, 3, mean=(0.0, 0.0, 0.0))
    _, bn, dw, pw = _sep_helpers(g, rng, ws)
    cur, cur_c, cur_d = _mobilenet_stem(g, rng, ws, bn), 32, 1
    for i, (co, st, dil) in enumerate(MOBILENET_DILATED_BLOCKS, start=1):
        d_out = cur_d + (1 if st == 2 else 0)
        t = g.add_buffer(_r64(cur_c), d_out)
        dw(cur, t, cur_c, 3, stride=st, name=f"convblock_{i}_dw", wname=f"convblock_{i}", dilation=dil)
        nxt = g.add_buffer(_r64(co), d_out)
        pw(t, nxt, 1, _r64(cur_c), co, cin_real=cur_c, name=f"convblock_{i}_pw", wname=f"convblock_{i}")
        cur, cur_c, cur_d = nxt, co, d_out
    _lw_head(g, rng, ws, cur, cur_c)
    return g


def resnet50_pifpaf(seed: int = 0, weights=None) -> Graph:
    """OpenPifPaf on ResNet-50 (BASELINE.json config 5): hyperpose/Model/pifpaf/model.py:41-51 (Resnet50_backbone(use_pool=False,
    scale_size=32): 7x7/2 stem, NO max-pool, stride-2 first blocks in stages 2-4 => stride 16), :215-281 (two 1x1 heads to
    17*5*4 and 19*9*4 channels, pixel-shuffle x2, sigmoid / softplus) -> fields at stride 8, cropped to 2*h16 - 1 (49 for 385).
    Input normalisation (x - mean) / std (model.py:38-39,58): the mean is subtracted in the patch gather, 1/std is folded
    into the stem weights.  `weights`: a hyperpose_b200.weights.Resnet50PifPafWeights; default = seeded random values."""
    rng = np.random.default_rng(seed)
    ws = weights
    mean = (0.485, 0.456, 0.406); std = np.array([0.229, 0.224, 0.225], np.float32)
    g = Graph("resnet50_pifpaf", 85, 171, 4, mean=mean, head_type=1)
    relu = lambda n: np.zeros(n, np.float32)
    lin = lambda n: np.ones(n, np.float32)

    col = g.add_buffer(192, 1); g.add_im2col(col, stride=2, ksize=7)
    c1 = g.add_buffer(64, 1)
    if ws:
        w = ws.conv("conv1", 64, 3, 7)[0][None] / std.reshape(1, 1, 3, 1, 1); sc, sh = ws.bn("bn1", 64)
    else:
        w = _he(rng, 1, 64, 3, 7, 7) / std.reshape(1, 1, 3, 1, 1); sc, sh = _bn_fold(rng, 64)
    g.add_conv(col, c1, w * sc.reshape(1, 64, 1, 1, 1), sh, relu(64), im2col_input=1, name="conv1+bn1")
    cur, cur_c, cur_d = _resnet50_body(g, rng, ws, c1, 64, 1, [(64, 3, 1), (128, 4, 2), (256, 6, 2), (512, 3, 2)])
    # heads (model.py:229,262): 1x1 conv + bias, no activation
    pif_raw = g.add_buffer(512, 4); paf_raw = g.add_buffer(768, 4)
    if ws:
        (wpif, bpif), (wpaf, bpaf) = ws.conv("pif_head", 340, 2048, 1), ws.conv("paf_head", 684, 2048, 1)
        wpif, wpaf = wpif[None], wpaf[None]
    else:
        wpif, bpif = _he(rng, 1, 340, 2048, 1, 1, 0.5), (rng.standard_normal(340) * 0.1).astype(np.float32)
    g.add_conv(cur, pif_raw, wpif, bpif, lin(340), name="pif_head")
    if not ws:
        wpaf, bpaf = _he(rng, 1, 684, 2048, 1, 1, 0.5), (rng.standard_normal(684) * 0.1).astype(np.float32)
    g.add_conv(cur, paf_raw, wpaf, bpaf, lin(684), name="paf_head")
    g.ops.append(Op(OP_PIFPAF_HEAD, in_buf=pif_raw, res_buf=paf_raw, name="pifpaf_heads"))
    return g


PPN_K, PPN_L, PPN_NH, PPN_NW = 18, 17, 9, 9     # pose_proposal/model.py:14-15 defaults: key points, limbs, 9 x 9 neighbourhood


def _ppn_stem(g, rng, ws):
    """7x7/2 conv (no bias) + BN + ReLU, then the 3x3/2 max-pool: (buffer, channels, down_shift) at stride 4"""
    col = g.add_buffer(192, 1); g.add_im2col(col, stride=2, ksize=7)
    c1 = g.add_buffer(64, 1)
    if ws:
        w = ws.conv("conv1", 64, 3, 7)[0][None]; sc, sh = ws.bn("bn1", 64)
    else:
        w = _he(rng, 1, 64, 3, 7, 7); sc, sh = _bn_fold(rng, 64)
    g.add_conv(col, c1, w * sc.reshape(1, 64, 1, 1, 1), sh, np.zeros(64, np.float32), im2col_input=1, name="conv1+bn1")
    x = g.add_buffer(64, 2); g.add_maxpool(c1, x, 64, "maxpool_1", ksize=3)
    return x, 64, 2


def _ppn_head(g, rng, ws, cur, cur_c, cur_d):
    """pose_proposal/model.py:43-79: add_block_1 / add_block_2 (3x3 conv + bias, BN, leaky ReLU 0.1 = PReLU with every slope 0.1),
    add_block_3 (1x1 conv + bias to 6K + L*nh*nw channels), then OP_PPN_HEAD (sigmoid + restore_coor, :84-93,:111-119)"""
    n_out = 6 * PPN_K + PPN_L * PPN_NH * PPN_NW
    leaky = lambda n: np.full(n, 0.1, np.float32)
    for i, ci in ((1, cur_c), (2, 512)):
        if ws:
            w, b = ws.conv(f"add{i}", 512, ci, 3); w = w[None]; sc, sh = ws.bn(f"add{i}.bn", 512)
        else:
            w = _he(rng, 1, 512, ci, 3, 3); b = (rng.standard_normal(512) * 0.05).astype(np.float32); sc, sh = _bn_fold(rng, 512)
        nxt = g.add_buffer(512, cur_d)
        g.add_conv(cur, nxt, w * sc.reshape(1, 512, 1, 1, 1), sh + b * sc, leaky(512), name=f"add_block_{i}")
        cur = nxt
    raw = g.add_buffer((n_out + 7) // 8 * 8, cur_d)      # 1485 -> 1488 channels
    if ws:
        w, b = ws.conv("add3", n_out, 512, 1); w = w[None]
    else:
        w = _he(rng, 1, n_out, 512, 1, 1, 1.0); b = (rng.standard_normal(n_out) * 0.1).astype(np.float32)
    g.add_conv(cur, raw, w, b, np.ones(n_out, np.float32), name="add_block_3")
    g.ops.append(Op(OP_PPN_HEAD, in_buf=raw, R=PPN_NH, S=PPN_NW, groups=PPN_L, cout_g=PPN_K, name="ppn_head"))


def ppn_resnet18(seed: int = 0, weights=None) -> Graph:
    """Pose Proposal Network on ResNet-18 (the default backbone of hyperpose/Model/pose_proposal/model.py:39-42):
    Resnet18_backbone(scale_size=32) (backbones.py:512-585: 7x7/2 stem, 3x3/2 max-pool, blocks 2_1 .. 5_1; block_5_2 exists only
    with `pretraining`, :535-536,:552, so it is not built), stride 32, 512 channels, then the PPN head (_ppn_head).
    A block is relu(bn(conv3x3(relu(bn(conv3x3/s(x))))) + res) with res = bn(conv1x1/s(x)) when it down-samples.  A stride-2 conv
    runs at stride 1 and a one-hot depthwise op sub-samples it (exact, see _resnet50_body).  BatchNorm folded.
    `weights`: a hyperpose_b200.weights.Ppn18Weights; default = seeded random values."""
    rng = np.random.default_rng(seed)
    ws = weights
    g = Graph("ppn_resnet18", 6 * PPN_K, PPN_L * PPN_NH * PPN_NW, 5, mean=(0.0, 0.0, 0.0), head_type=2)
    cur, cur_c, cur_d = _resnet18_body(g, rng, ws, *_ppn_stem(g, rng, ws), [st for _, _, st, _ in RESNET18_BLOCKS])
    _ppn_head(g, rng, ws, cur, cur_c, cur_d)
    return g


def _resnet18_body(g, rng, ws, cur, cur_c, cur_d, strides):
    """blocks 2_1 .. 5_1 of Resnet18_backbone (RESNET18_BLOCKS) with the given stride per block, from the stem output `cur`.
    BatchNorm folded; relu(x + res) in the conv epilogue.  Returns (buffer, channels, down_shift)."""
    relu = lambda n: np.zeros(n, np.float32)
    lin = lambda n: np.ones(n, np.float32)

    def conv_bn(in_buf, out_buf, ci, co, k, act, name, gain, **kw):
        if ws:
            w = ws.conv(f"{name}.conv", co, ci, k)[0][None]; sc, sh = ws.bn(f"{name}.bn", co)
        else:
            w = _he(rng, 1, co, ci, k, k, gain); sc, sh = _bn_fold(rng, co)
        g.add_conv(in_buf, out_buf, w * sc.reshape(1, co, 1, 1, 1), sh, relu(co) if act else lin(co), name=name, **kw)

    def subsample(in_buf, out_buf, C, centre3, name):
        w = np.zeros((C, 3, 3), np.float32) if centre3 else np.ones((C, 1, 1), np.float32)
        if centre3:
            w[:, 1, 1] = 1.0
        g.add_dwconv(in_buf, out_buf, w, np.zeros(C, np.float32), lin(C), stride=2, name=name)

    for (name, nf, _, ds), st in zip(RESNET18_BLOCKS, strides):
        d_out = cur_d + (1 if st == 2 else 0)
        a = g.add_buffer(nf, cur_d)
        conv_bn(cur, a, cur_c, nf, 3, True, f"{name}_1", 2.0)
        if st == 2:
            a2 = g.add_buffer(nf, d_out); subsample(a, a2, nf, True, f"{name}_1_sub"); a = a2
        if ds:
            src = cur
            if st == 2:
                src = g.add_buffer(cur_c, d_out); subsample(cur, src, cur_c, False, f"{name}_ds_sub")
            res = g.add_buffer(nf, d_out)
            conv_bn(src, res, cur_c, nf, 1, False, f"{name}_ds", 1.0)
        else:
            res = cur
        out = g.add_buffer(nf, d_out)
        conv_bn(a, out, nf, nf, 3, True, f"{name}_2", 0.5, res_buf=res, res_mode=1)    # relu(x + res)
        cur, cur_c, cur_d = out, nf, d_out
    return cur, cur_c, cur_d


# (block name, n_filter, stride, is_down_sample) of Resnet18_backbone(scale_size=32) (backbones.py:529-535)
RESNET18_BLOCKS = [("block_2_1", 64, 1, False), ("block_2_2", 64, 1, False), ("block_3_1", 128, 2, True), ("block_3_2", 128, 1, False),
                   ("block_4_1", 256, 2, True), ("block_4_2", 256, 1, False), ("block_5_1", 512, 2, True)]
# the strides at scale_size 8: blocks 4_1 and 5_1 keep stride 1 (backbones.py:520-523)
RESNET18_STRIDES_8 = (1, 1, 2, 1, 1, 1, 1)


def ppn_resnet50(seed: int = 0, weights=None) -> Graph:
    """Pose Proposal Network on ResNet-50 (the model zoo's ppn-resnet50-V2-HW=384x384, scripts/downloader.py:15):
    Resnet50_backbone(scale_size=32, use_pool=True) (backbones.py:587-698: 7x7/2 stem, 3x3/2 max-pool, 16 bottleneck blocks with
    stride-2 first blocks in stages 3-5), stride 32, 2048 channels, then the PPN head (_ppn_head).  BatchNorm folded.
    `weights`: a hyperpose_b200.weights.Ppn50Weights; default = seeded random values."""
    rng = np.random.default_rng(seed)
    ws = weights
    g = Graph("ppn_resnet50", 6 * PPN_K, PPN_L * PPN_NH * PPN_NW, 5, mean=(0.0, 0.0, 0.0), head_type=2)
    x, c, d = _ppn_stem(g, rng, ws)
    cur, cur_c, cur_d = _resnet50_body(g, rng, ws, x, c, d, [(64, 3, 1), (128, 4, 2), (256, 6, 2), (512, 3, 2)])
    _ppn_head(g, rng, ws, cur, cur_c, cur_d)
    return g


def tiny_test_net(seed: int = 0) -> Graph:
    """small graph exercising every op type / conv variant (tests only need seconds):
    im2col conv, 3x3, maxpool, merged + grouped 7x7, 185->192 padded input, block-diagonal split output."""
    rng = np.random.default_rng(seed)
    g = Graph("tiny", 19, 38, 1, mean=(0.4, 0.45, 0.5))
    relu = lambda n: np.zeros(n, np.float32)
    prelu = lambda n: rng.uniform(0.1, 0.4, n).astype(np.float32)
    b_ = lambda n: (rng.standard_normal(n) * 0.05).astype(np.float32)
    b0 = g.add_buffer(64, 0); g.add_im2col(b0)
    b1 = g.add_buffer(64, 0); g.add_conv(b0, b1, _he(rng, 1, 64, 3, 3, 3), b_(64), relu(64), im2col_input=1, name="c1")
    b2 = g.add_buffer(64, 1); g.add_maxpool(b1, b2, 64)
    cat = g.add_buffer(192, 1)
    g.add_conv(b2, cat, _he(rng, 1, 128, 64, 3, 3), b_(128), relu(128), name="c2")
    ta = g.add_buffer(256, 1); tb = g.add_buffer(256, 1)
    w = _block_diag(_he(rng, 1, 19, 128, 1, 1, 1.0), _he(rng, 1, 38, 128, 1, 1, 1.0))
    g.add_conv(cat, ta, np.concatenate([_he(rng, 1, 128, 128, 3, 3), _he(rng, 1, 128, 128, 3, 3)], axis=1), b_(256), prelu(256), name="m1")
    g.add_conv(ta, cat, w, b_(57), prelu(57), out_ch_off=128, name="o1")
    g.add_conv(cat, ta, np.concatenate([_he(rng, 1, 128, 185, 7, 7), _he(rng, 1, 128, 185, 7, 7)], axis=1), b_(256), prelu(256), name="r1")
    g.add_conv(ta, tb, _he(rng, 2, 128, 128, 7, 7), b_(256), prelu(256), name="r2")
    g.add_conv(tb, ta, _he(rng, 2, 128, 128, 1, 1), b_(256), prelu(256), name="r3")
    g.add_conv(ta, 0, w.copy(), b_(57), prelu(57), out_mode=OUT_F32_NCHW_SPLIT, split=19, name="out")
    return g
