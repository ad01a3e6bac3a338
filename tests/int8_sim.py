"""CPU model of the INT8 engine's arithmetic (HP_DTYPE_INT8), exact to the byte.

Symmetric quantization: buffer b holds int8 q in [-127, 127] standing for q * s_b.  Every step is the engine's, in the same order and
with the same rounding:
  * weights: s_w[o] = max |W[o]| / 127 (1 for an all-zero row), q_w = clamp(rint(W / s_w), -127, 127), mul[o] = s_in * s_w[o];
  * conv: the integer convolution in float64 (exact: every operand and every partial sum is an integer of magnitude at most
    127^2 K < 2^31 < 2^53, so any summation order gives the same sum; run_graph(device="cuda") computes it there as an
    im2col + DGEMM with cuDNN off, since cuDNN's FFT and Winograd algorithms are not exact), cast to float32, then
    v = acc * mul + bias, residual r = q_r * s_res (mode 1: act(v + r), mode 2: act(v) + r), act(y) = y > 0 ? y : y * alpha, each a
    separately rounded float32 operation; NHWC outputs store clamp(rint(y * (1 / s_out)), -127, 127), the conf / PAF outputs y;
  * im2col: the fp32 normalised input (u8 * factor in double, to float32, minus the mean; or the f32 entry minus the mean), quantized
    with the im2col buffer's scale;
  * max-pool: on the int8 values;
  * depthwise: per tap x = q * s_in, acc = acc + x * w from 0, taps row major then by column; + bias, PReLU, quantize.
Buffers are [N, C, H, W] int8 arrays."""
import numpy as np
import torch
import torch.nn.functional as F

from hyperpose_b200 import models

f32 = np.float32


def quantize(y, inv_s):
    """float32 y -> int8 clamp(rint(y * inv_s), -127, 127), the product rounded to float32 first"""
    p = (np.asarray(y, f32) * f32(inv_s)).astype(f32)
    return np.clip(np.rint(p), -127, 127).astype(np.int8)


def quantize_weights(weight):
    """[O, ...] float32 -> (q [O, ...] int8, s_w [O] float32): one scale per output channel"""
    w = np.asarray(weight, f32)
    flat = w.reshape(w.shape[0], -1)
    amax = np.abs(flat).max(axis=1)
    sw = np.where(amax > 0, amax / f32(127.0), f32(1.0)).astype(f32)
    q = np.clip(np.rint((flat / sw[:, None]).astype(f32)), -127, 127).astype(np.int8)
    return q.reshape(w.shape), sw


def float_absmax(g: models.Graph, frames_u8, factor=1.0 / 255):
    """per-buffer max |x| of a float32 run of g (oracle/torch_backbone, CPU), for Graph.set_int8_scales where no GPU calibrates: the
    final buffer contents, and for the im2col buffer (which that run does not fill with patches) max |x| of the normalised frames"""
    from oracle import torch_backbone
    _, _, bufs = torch_backbone.run_graph(g, frames_u8, factor=factor, device="cpu", rounding="tf32")
    a = np.array([float(b.abs().max()) for b in bufs], f32)
    x = (frames_u8.astype(np.float64) * factor).astype(f32)[..., ::-1] - np.asarray(g.mean, f32)
    for op in g.ops:
        if op.type == models.OP_IM2COL3:
            a[op.out_buf] = np.abs(x).max()
    return a


def _same_pad_before(n, k, stride):
    out = (n + stride - 1) // stride
    return max((out - 1) * stride + k - n, 0) // 2


def _shape(g, bi, H, W):
    c, d = g.buffers[bi]
    for _ in range(d):
        H, W = (H + 1) // 2, (W + 1) // 2
    return c, H, W


def _int_conv(x, qw, G, R, S, im2col, device):
    """the integer convolution of int8 x [N, C, H, W] (for im2col: [N, R S cin, H, W], k = (r S + s) cin + c) with int8 qw
    [G co, ci, R, S] in float64 on `device` -> float64 numpy [N, G co, H, W]"""
    w = torch.from_numpy(qw.astype(np.float64)).to(device)
    with torch.backends.cudnn.flags(enabled=False):
        if im2col:
            xt = torch.from_numpy(x.astype(np.float64)).to(device)
            acc = torch.einsum("nkhw,ok->nohw", xt, w.permute(0, 2, 3, 1).reshape(w.shape[0], -1))
        else:
            acc = F.conv2d(torch.from_numpy(x.astype(np.float64)).to(device), w, padding=(R // 2, S // 2), groups=G)
    return acc.cpu().numpy()


def run_graph(g: models.Graph, act_scales, frames_u8=None, f32_input=None, factor=1.0 / 255, flip_rgb=True, init=None, N=None, HW=None,
              device="cpu"):
    """-> (conf, paf, bufs).  Input: u8 frames [N, H, W, 3] (BGR), or f32_input [N, 3, H, W] (the f32 entry: already scaled), or
    neither (graphs without an im2col op: N and HW=(H, W) give the geometry).  init: {buffer: int8 [N, C, H, W]} starting contents.
    device: where the integer convolutions run (the rest stays on the CPU); the result is the same bytes on any device."""
    s = np.asarray(act_scales, f32)
    if frames_u8 is not None:
        N, H, W, _ = frames_u8.shape
    elif f32_input is not None:
        N, _, H, W = f32_input.shape
    else:
        H, W = HW
    bufs = []
    for bi in range(len(g.buffers)):
        c, h, w = _shape(g, bi, H, W)
        bufs.append(np.array(init[bi], np.int8) if init is not None and bi in init else np.zeros((N, c, h, w), np.int8))
    conf = paf = None
    for op in g.ops:
        if op.type == models.OP_IM2COL3:
            if frames_u8 is not None:
                x = (frames_u8.astype(np.float64) * factor).astype(f32)
                if flip_rgb:
                    x = x[..., ::-1]
                x = np.ascontiguousarray(x.transpose(0, 3, 1, 2))
            else:
                x = np.asarray(f32_input, f32)
            x = (x - np.asarray(g.mean, f32).reshape(1, 3, 1, 1)).astype(f32)
            R, st = op.R or 3, op.stride or 1
            C, OH, OW = _shape(g, op.out_buf, H, W)
            ph, pw = _same_pad_before(H, R, st), _same_pad_before(W, R, st)
            xp = np.zeros((N, 3, H + 2 * R, W + 2 * R), f32)
            xp[:, :, R:R + H, R:R + W] = x
            col = np.zeros((N, C, OH, OW), f32)
            for r in range(R):
                for t in range(R):
                    h0, w0 = R - ph + r, R - pw + t
                    patch = xp[:, :, h0:h0 + st * (OH - 1) + 1:st, w0:w0 + st * (OW - 1) + 1:st]
                    col[:, (r * R + t) * 3:(r * R + t) * 3 + 3] = patch
            bufs[op.out_buf] = quantize(col, f32(1.0) / s[op.out_buf])
        elif op.type == models.OP_MAXPOOL2:
            x = torch.from_numpy(bufs[op.in_buf][:, op.in_ch_off:op.in_ch_off + op.cout_g].astype(np.float64))
            K = op.R if op.R else 2
            pads = []
            for dim in (x.shape[3], x.shape[2]):
                out = (dim + 1) // 2
                total = max((out - 1) * 2 + K - dim, 0)
                pads += [total // 2, total - total // 2]
            y = F.max_pool2d(F.pad(x, pads, value=-1000.0), K, 2)
            bufs[op.out_buf][:, op.out_ch_off:op.out_ch_off + op.cout_g] = y.numpy().astype(np.int8)
        elif op.type == models.OP_CONV:
            G, co, ci, R, S = op.weight.shape
            qw, sw = quantize_weights(op.weight.reshape(G * co, ci, R, S))
            mul = (s[op.in_buf] * sw).astype(f32)
            if op.im2col_input:
                acc = _int_conv(bufs[op.in_buf][:, :R * S * ci], qw, G, R, S, True, device)
            else:
                acc = _int_conv(bufs[op.in_buf][:, op.in_ch_off:op.in_ch_off + G * ci], qw, G, R, S, False, device)
            v = acc.astype(f32) * mul.reshape(1, -1, 1, 1)
            v = (v + op.bias.astype(f32).reshape(1, -1, 1, 1)).astype(f32)
            if op.res_mode:
                r = (bufs[op.res_buf][:, op.res_ch_off:op.res_ch_off + G * co].astype(f32) * s[op.res_buf]).astype(f32)
            if op.res_mode == 1:
                v = (v + r).astype(f32)
            v = np.where(v > 0, v, (v * op.alpha.astype(f32).reshape(1, -1, 1, 1)).astype(f32)).astype(f32)
            if op.res_mode == 2:
                v = (v + r).astype(f32)
            if op.out_mode == models.OUT_F32_NCHW_SPLIT:
                conf, paf = np.ascontiguousarray(v[:, :op.split]), np.ascontiguousarray(v[:, op.split:])
            else:
                bufs[op.out_buf][:, op.out_ch_off:op.out_ch_off + G * co] = quantize(v, f32(1.0) / s[op.out_buf])
        elif op.type == models.OP_DWCONV:
            C, K, _ = op.weight.shape
            st = op.stride or 1
            x = (bufs[op.in_buf][:, op.in_ch_off:op.in_ch_off + C].astype(f32) * s[op.in_buf]).astype(f32)
            _, h, w = x.shape[1:]
            _, OH, OW = _shape(g, op.out_buf, H, W)
            ph, pw = _same_pad_before(h, K, st), _same_pad_before(w, K, st)
            xp = np.zeros((N, C, h + 2 * K, w + 2 * K), f32)
            xp[:, :, K:K + h, K:K + w] = x
            acc = np.zeros((N, C, OH, OW), f32)
            for r in range(K):
                for t in range(K):
                    h0, w0 = K - ph + r, K - pw + t
                    patch = xp[:, :, h0:h0 + st * (OH - 1) + 1:st, w0:w0 + st * (OW - 1) + 1:st]
                    acc = (acc + (patch * op.weight[:, r, t].astype(f32).reshape(1, -1, 1, 1)).astype(f32)).astype(f32)
            y = (acc + op.bias.astype(f32).reshape(1, -1, 1, 1)).astype(f32)
            y = np.where(y > 0, y, (y * op.alpha.astype(f32).reshape(1, -1, 1, 1)).astype(f32)).astype(f32)
            bufs[op.out_buf][:, op.out_ch_off:op.out_ch_off + C] = quantize(y, f32(1.0) / s[op.out_buf])
        else:
            raise ValueError(f"the INT8 engine has no op type {op.type}")
    return conf, paf, bufs
