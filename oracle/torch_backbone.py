"""oracle/torch_backbone.py -- plain PyTorch executor for hyperpose_b200.models.Graph.  TEST INFRASTRUCTURE ONLY
(tests, and the CPU-baseline / --impl reference legs of bench.py, where it stands in for the conv stage on the host cores:
the reference runs its convs in TensorRT on a GPU, src/tensorrt.cpp:387-396, and has no CPU implementation of them).

The backbone is a floating-point kernel, so its checker is a torch reference of the same ops
(F.conv2d / max_pool2d / PReLU), as the reference's TensorRT FP32 engine would compute them.
`emulate_fp16=True` additionally rounds weights and stored activations to fp16 exactly where the
engine does (fp16 operands, fp32 accumulation), which isolates kernel bugs from precision.

For per-kernel error bounds the same executor runs in float64 (`dtype`) from given buffer contents (`init`), with the operand
grid of either engine (`rounding` "fp16" | "tf32"), optionally without rounding the stored results (`round_stores=False`: the
caller's bound accounts for the engine's final rounding), and as a magnitude pass (`magnitude=True`: |weights|, |bias|, |inputs|,
linear activations, so that every output holds sum |w x| + |b| (+ |res|), the scale of its accumulation error)."""
import numpy as np
import torch
import torch.nn.functional as F

from hyperpose_b200 import models


def tf32_round(t: torch.Tensor) -> torch.Tensor:
    """round to nearest, ties away from zero, onto the TF32 grid (8-bit exponent, 10-bit mantissa) -- cvt.rna.tf32.f32 and the
    engine's host-side tf32_round; the value is taken through fp32 first, as the engine holds it"""
    i = t.float().contiguous().view(torch.int32)
    r = torch.where((i & 0x7f800000) == 0x7f800000, i, (i + 0x1000) & -0x2000)
    return r.view(torch.float32).to(t.dtype)


def run_graph(g: models.Graph, frames_u8: np.ndarray, factor=1.0 / 255, flip_rgb=True, emulate_fp16=False, device="cuda",
              upto=None, dtype=torch.float32, init=None, rounding=None, round_stores=True, magnitude=False):
    """-> (conf, paf, buffers), the buffers as [N, C, H, W] tensors of `dtype`.
    init: {buffer index: array [N, C, H, W]}, the starting contents of those buffers (the others start as zeros).
    rounding: None | "fp16" | "tf32" -- the engine's operand grid: conv weights, the normalised u8 input and every stored
    activation are rounded onto it (emulate_fp16=True is rounding="fp16"); round_stores=False leaves the stored activations
    unrounded.  The u8 normalisation is computed in fp32, as the engine does, before it is rounded and widened to `dtype`."""
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    if emulate_fp16:
        rounding = "fp16"
    assert rounding in (None, "fp16", "tf32"), rounding
    grid = {None: lambda t: t, "fp16": lambda t: t.half().to(t.dtype), "tf32": tf32_round}[rounding]
    q = grid if round_stores else (lambda t: t)
    m = torch.abs if magnitude else (lambda t: t)
    N, H, W, _ = frames_u8.shape
    bufs = []
    for bi, (c, d) in enumerate(g.buffers):
        h, w = H, W
        for _ in range(d):
            h, w = (h + 1) // 2, (w + 1) // 2
        if init is not None and bi in init:
            b = torch.as_tensor(np.asarray(init[bi]), device=device).to(dtype).clone()
            assert tuple(b.shape) == (N, c, h, w), (bi, tuple(b.shape), (N, c, h, w))
            bufs.append(m(b))
        else:
            bufs.append(torch.zeros(N, c, h, w, device=device, dtype=dtype))
    conf = paf = None
    img, img_stride = None, 1

    def t_(a):
        return torch.from_numpy(np.asarray(a)).to(device)

    def act(y, alpha):
        if magnitude:
            return y
        a = t_(alpha).to(dtype).view(1, -1, 1, 1)
        return torch.where(y > 0, y, y * a)

    def same_pad(x, k, stride):
        """TF 'SAME': out = ceil(in/stride); pad_before = total // 2"""
        pads = []
        for dim in (x.shape[3], x.shape[2]):   # F.pad order: W first, then H
            out = (dim + stride - 1) // stride
            total = max((out - 1) * stride + k - dim, 0)
            pads += [total // 2, total - total // 2]
        return F.pad(x, pads)

    for oi, op in enumerate(g.ops):
        if upto is not None and oi > upto:
            break
        if op.type == models.OP_IM2COL3:
            x = (frames_u8.astype(np.float64) * factor).astype(np.float32)          # data.cpp:48
            if flip_rgb:
                x = x[..., ::-1]
            x = torch.from_numpy(np.ascontiguousarray(x.transpose(0, 3, 1, 2))).to(device)
            x = x - torch.tensor(g.mean, dtype=torch.float32, device=device).view(1, 3, 1, 1)
            img, img_stride = m(grid(x).to(dtype)), op.stride
            if op.stride == 1:
                bufs[op.out_buf][:, :3] = img
        elif op.type == models.OP_MAXPOOL2:
            x = bufs[op.in_buf][:, op.in_ch_off:op.in_ch_off + op.cout_g]
            K = op.R if op.R else 2
            # TF SAME max-pool: pad with -inf (window clipped at the border)
            pads = []
            for dim in (x.shape[3], x.shape[2]):
                out = (dim + 1) // 2
                total = max((out - 1) * 2 + K - dim, 0)
                pads += [total // 2, total - total // 2]
            xp = F.pad(x, pads, value=float("-inf"))
            bufs[op.out_buf][:, op.out_ch_off:op.out_ch_off + op.cout_g] = F.max_pool2d(xp, K, 2)
        elif op.type == models.OP_CONV:
            G, co, ci, R, S = op.weight.shape
            w = m(grid(t_(op.weight.reshape(G * co, ci, R, S))).to(dtype))
            bias = m(t_(op.bias).to(dtype))
            if op.im2col_input:
                y = F.conv2d(same_pad(img, R, img_stride), w, bias, stride=img_stride)
            else:
                x = bufs[op.in_buf][:, op.in_ch_off:op.in_ch_off + G * ci]
                y = F.conv2d(x, w, bias, padding=(R // 2, S // 2), groups=G)
            res = bufs[op.res_buf][:, op.res_ch_off:op.res_ch_off + G * co] if op.res_mode else None
            if op.res_mode == 1:
                y = y + res
            y = act(y, op.alpha)
            if op.res_mode == 2:
                y = y + res
            if op.out_mode == models.OUT_F32_NCHW_SPLIT:
                conf, paf = y[:, :op.split].contiguous(), y[:, op.split:].contiguous()
            else:
                bufs[op.out_buf][:, op.out_ch_off:op.out_ch_off + G * co] = q(y)
        elif op.type == models.OP_PIFPAF_HEAD:
            def head(raw, fields, comps, is_paf):
                x = raw[:, :fields * comps * 4]
                b, c, h, w = x.shape
                x = x.reshape(b, c // 4, 2, 2, h, w).permute(0, 1, 4, 2, 5, 3).reshape(b, c // 4, 2 * h, 2 * w)   # pifpaf/utils.py:371-379
                x = x[:, :, :2 * h - 1, :2 * w - 1].reshape(b, fields, comps, 2 * h - 1, 2 * w - 1).clone()
                gy, gx = torch.meshgrid(torch.arange(2 * h - 1, device=device), torch.arange(2 * w - 1, device=device), indexing="ij")
                x[:, :, 0] = torch.sigmoid(x[:, :, 0])
                for cx in ((1, 3) if is_paf else (1,)):
                    x[:, :, cx] += gx
                for cy in ((2, 4) if is_paf else (2,)):
                    x[:, :, cy] += gy
                for cs in ((7, 8) if is_paf else (4,)):
                    x[:, :, cs] = F.softplus(x[:, :, cs])
                return x
            conf = head(bufs[op.in_buf], 17, 5, False)
            paf = head(bufs[op.res_buf], 19, 9, True)
        elif op.type == models.OP_DWCONV:
            C, K, _ = op.weight.shape
            x = bufs[op.in_buf][:, op.in_ch_off:op.in_ch_off + C]
            w = m(t_(op.weight.reshape(C, 1, K, K)).to(dtype))      # depthwise weights stay fp32 in the engine
            y = F.conv2d(same_pad(x, K, op.stride), w, m(t_(op.bias).to(dtype)), stride=op.stride, groups=C)
            bufs[op.out_buf][:, op.out_ch_off:op.out_ch_off + C] = q(act(y, op.alpha))
    return conf, paf, bufs
