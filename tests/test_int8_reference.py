"""The INT8 scale table in the model pack, and the CPU model of the INT8 engine's arithmetic (tests/int8_sim.py) -- no GPU."""
import ctypes as C
import hashlib
import struct

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from hyperpose_b200 import capi, models
from tests import int8_sim

# sha256 of to_pack() for seed 0, as written before packs could carry a scale table: a pack without one must not change
PACK_SHA256 = {
    "openpose_vgg19": "67e43f7b6aa7b901e395424d4a61b3ae563d6f9cf718169af85ec8edc725488e",
    "mobilenet_thin_openpose": "3e8e8c2994945432364f1da1c8668db449ddded368f941a2d900c428f99867b3",
    "resnet50_lw_openpose": "44e23dbdbf5e47a770bd1009ee80d3ca55e74ef832eddbc43d95933f4f9ba5a9",
    "resnet50_pifpaf": "47421c2ff427f6b281a1430140c0b327edfdfbfc9668c623fdda62227d1afe4c",
}


@pytest.mark.parametrize("name", sorted(PACK_SHA256))
def test_pack_without_scales_unchanged(name):
    g = getattr(models, name)(0)
    assert g.act_scales is None
    assert hashlib.sha256(g.to_pack()).hexdigest() == PACK_SHA256[name]


def test_scale_table_round_trip():
    g = models.tiny_test_net(0)
    plain = g.to_pack()
    rng = np.random.default_rng(3)
    g.set_int8_scales(rng.uniform(0.5, 20.0, len(g.buffers)).astype(np.float32))
    packed = g.to_pack()
    n = len(g.buffers)
    assert len(packed) == len(plain) + 4 * n
    assert struct.unpack_from("<I", packed, 48)[0] == n                  # reserved[0] = n_act_scales
    assert packed[:48] == plain[:48] and packed[52:len(plain)] == plain[52:]
    assert np.array_equal(np.frombuffer(packed[len(plain):], "<f4"), g.act_scales)
    g.act_scales = None
    assert g.to_pack() == plain


def test_pack_int8_calibrated_query():
    L = capi.lib()
    q = lambda b: L.hp_pack_int8_calibrated(b, len(b))
    g = models.tiny_test_net(0)
    assert q(g.to_pack()) == 0
    g.set_int8_scales(np.ones(len(g.buffers), np.float32))
    p = g.to_pack()
    assert q(p) == 1
    assert q(p[:-4]) == 0                                                   # table cut short
    assert L.hp_pack_int8_calibrated(None, 0) == 0


def _graph():
    return models.Graph("t", conf_channels=8, paf_channels=8, out_down_shift=0)


@pytest.mark.parametrize("name", ["openpose_vgg19", "mobilenet_thin_openpose"])
def test_set_int8_scales_ties_pools(name):
    """buffers joined by max-pools share one scale, from the largest absmax among them; every other buffer keeps absmax / 127"""
    g = getattr(models, name)(0)
    rng = np.random.default_rng(5)
    absmax = rng.uniform(0.5, 50.0, len(g.buffers)).astype(np.float32)
    absmax[-1] = 0.0
    g.set_int8_scales(absmax)
    pools = [op for op in g.ops if op.type == models.OP_MAXPOOL2]
    assert pools
    tied = {b for op in pools for b in (op.in_buf, op.out_buf)}
    for op in pools:
        s = g.act_scales[op.out_buf]
        assert s == g.act_scales[op.in_buf]
        assert s >= np.float32(absmax[op.in_buf]) / np.float32(127.0) and s >= np.float32(absmax[op.out_buf]) / np.float32(127.0)
        assert any(s == np.float32(absmax[b]) / np.float32(127.0) for b in tied)
    for b in range(len(g.buffers)):
        if b not in tied:
            want = np.float32(1.0) if absmax[b] == 0 else np.float32(absmax[b]) / np.float32(127.0)
            assert g.act_scales[b] == want
    # a chain in, pool, out: the three share the largest of the three absmax values
    h = _graph()
    x = h.add_buffer(16, 0); y = h.add_buffer(16, 1); z = h.add_buffer(16, 2)
    h.add_maxpool(x, y, 16); h.add_maxpool(y, z, 16)
    h.set_int8_scales(np.array([2.0, 9.0, 4.0], np.float32))
    assert h.act_scales.tolist() == [np.float32(9.0) / np.float32(127.0)] * 3


def test_unit_scales_equal_plain_convolution():
    """integer data, integer weights whose rows reach +-127 (so s_w = 1), unit scales, linear activation: the model is the convolution"""
    rng = np.random.default_rng(0)
    g = _graph()
    a = g.add_buffer(32, 0); b = g.add_buffer(48, 0)
    w = rng.integers(-2, 3, (2, 16, 16, 3, 3)).astype(np.float32)
    w[:, :, 0, 0, 0] = 127.0                                   # reads input channels 0 and 16, which stay zero
    g.add_conv(a, b, w, np.zeros(32, np.float32), np.ones(32, np.float32), out_ch_off=8)
    x = (rng.integers(-1, 2, (2, 32, 7, 9)) * (rng.random((2, 32, 7, 9)) < 0.3)).astype(np.int8)
    x[:, [0, 16]] = 0
    _, _, bufs = int8_sim.run_graph(g, np.ones(2, np.float32), init={a: x}, N=2, HW=(7, 9))
    ref = F.conv2d(torch.from_numpy(x.astype(np.float64)), torch.from_numpy(w.reshape(32, 16, 3, 3).astype(np.float64)), padding=1, groups=2).numpy()
    assert np.abs(ref).max() <= 127
    assert np.array_equal(bufs[b][:, 8:40], ref.astype(np.int8))
    assert not bufs[b][:, :8].any() and not bufs[b][:, 40:].any()


def test_quantize_rounding_cases():
    y = np.array([0.5, 1.5, 2.5, -0.5, -1.5, -2.5, 126.5, 127.5, 300.0, -127.6, -1e30, 1e30], np.float32)
    assert int8_sim.quantize(y, 1.0).tolist() == [0, 2, 2, 0, -2, -2, 126, 127, 127, -127, -127, 127]
    # the product y * inv_s is rounded to float32 before rint: 0.1f * 25 is 2.5000000372... exactly but 2.5 in float32, a tie -> 2
    assert int8_sim.quantize(np.float32(0.1), 25.0).tolist() == 2
    q, sw = int8_sim.quantize_weights(np.array([[[[1.0, -2.0], [0.5, 254.0]]], [[[0.0, 0.0], [0.0, 0.0]]]], np.float32))
    assert sw.tolist() == [2.0, 1.0]
    assert q.reshape(2, 4).tolist() == [[0, -1, 0, 127], [0, 0, 0, 0]]   # 0.5 / 2 = 0.25 and 1 / 2 = 0.5 round to 0, -2 / 2 = -1


def test_hand_computed_conv_epilogue():
    """one 1x1 conv on one pixel, every step written out: negative PReLU slope, both residual modes, the clamp"""
    g = _graph()
    a = g.add_buffer(16, 0); r = g.add_buffer(16, 0); o = g.add_buffer(16, 0)
    w = np.zeros((1, 2, 16, 1, 1), np.float32)
    w[0, 0, 0] = 0.5; w[0, 0, 1] = -1.0    # s_w = 1/127: q = 64 (63.5 rounds to even), -127
    w[0, 1, 0] = 2.0                       # s_w = 2/127: q = 127
    bias = np.array([0.25, -100.0], np.float32)
    alpha = np.array([0.5, -0.25], np.float32)
    scales = np.array([0.5, 0.125, 2.0], np.float32)
    x = np.zeros((1, 16, 1, 1), np.int8); x[0, 0] = 3; x[0, 1] = 2
    res = np.zeros((1, 16, 1, 1), np.int8); res[0, 0] = -8; res[0, 1] = 100
    for mode in (1, 2):
        g.ops = []
        g.add_conv(a, o, w, bias, alpha, res_buf=r, res_mode=mode)
        _, _, bufs = int8_sim.run_graph(g, scales, init={a: x, r: res}, N=1, HW=(1, 1))
        f = np.float32
        sw0, sw1 = f(1.0) / f(127.0), f(2.0) / f(127.0)
        acc0, acc1 = 64 * 3 + (-127) * 2, 127 * 3                       # -62, 381
        v0 = f(f(acc0) * f(f(0.5) * sw0)) + f(0.25)
        v1 = f(f(acc1) * f(f(0.5) * sw1)) - f(100.0)
        r0, r1 = f(-8) * f(0.125), f(100) * f(0.125)
        act = lambda v, al: v if v > 0 else f(v * f(al))
        y0 = act(f(v0 + r0), 0.5) if mode == 1 else f(act(v0, 0.5) + r0)
        y1 = act(f(v1 + r1), -0.25) if mode == 1 else f(act(v1, -0.25) + r1)
        want = [int(np.clip(np.rint(f(y * f(f(1.0) / f(2.0)))), -127, 127)) for y in (y0, y1)]
        assert bufs[o][0, :2, 0, 0].tolist() == want
        assert want[1] > 0   # the negative slope turned the negative pre-activation positive
