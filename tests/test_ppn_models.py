"""Pose Proposal Network graphs (CPU): structure against the reference definitions (pose_proposal/model.py:14-119,
backbones.py:512-698), trained-weight import against a plain PyTorch model written from those definitions, pack round trip and
the exporter."""
import struct

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from hyperpose_b200 import export, models, weights as W
from oracle import torch_backbone as torch_ref
from tests.ppn_head_ref import ppn_head_ref
from tests.test_weights_import import _resnet50_reference, _tl_arrays, _TlReader

N_OUT = 6 * 18 + 17 * 9 * 9


def _head_op(g):
    ops = [op for op in g.ops if op.type == models.OP_PPN_HEAD]
    assert len(ops) == 1 and g.ops[-1] is ops[0]
    return ops[0]


def _down(n, d):
    for _ in range(d):
        n = (n + 1) // 2
    return n


@pytest.mark.parametrize("builder", [models.ppn_resnet18, models.ppn_resnet50])
def test_graph_outputs_and_head(builder):
    g = builder(0)
    assert (g.head_type, g.out_down_shift, g.conf_channels, g.paf_channels) == (2, 5, 108, 1377)
    head = _head_op(g)
    assert (head.cout_g, head.groups, head.R, head.S) == (18, 17, 9, 9)
    c, d = g.buffers[head.in_buf]
    assert c == 1488 and d == 5 and _down(384, d) == 12                  # 12 x 12 grid for 384 x 384
    last = g.ops[-2]
    assert last.type == models.OP_CONV and last.out_buf == head.in_buf and last.weight.shape == (1, N_OUT, 512, 1, 1)
    add1, add2 = g.ops[-4], g.ops[-3]
    assert add1.weight.shape[1:4] == (512, 512 if builder is models.ppn_resnet18 else 2048, 3) and add2.weight.shape[1:4] == (512, 512, 3)
    for op in (add1, add2):                                              # leaky ReLU, slope 0.1
        assert np.all(op.alpha == np.float32(0.1))
    assert np.all(last.alpha == 1.0)                                     # linear


def test_resnet18_blocks_mirror_the_backbone():
    """Resnet18_backbone(scale_size=32): blocks 2_1 .. 5_1 only (block_5_2 exists only with `pretraining`, backbones.py:535-536,552);
    blocks 3_1, 4_1, 5_1 are stride 2 with a 1x1 projection shortcut"""
    g = models.ppn_resnet18(0)
    names = [op.name for op in g.ops]
    blocks = sorted({n[:9] for n in names if n.startswith("block_")})
    assert blocks == ["block_2_1", "block_2_2", "block_3_1", "block_3_2", "block_4_1", "block_4_2", "block_5_1"]
    assert not any(n.startswith("block_5_2") for n in names)
    subs = sorted(op.name for op in g.ops if op.type == models.OP_DWCONV and op.stride == 2)
    assert subs == sorted([f"block_{s}_1_{k}" for s in (3, 4, 5) for k in ("1_sub", "ds_sub")])
    assert sorted(n for n in names if n.endswith("_ds")) == ["block_3_1_ds", "block_4_1_ds", "block_5_1_ds"]
    # stem at stride 2, max-pool to 4, then 8 / 16 / 32
    downs = {op.name: g.buffers[op.out_buf][1] for op in g.ops if op.type in (models.OP_CONV, models.OP_MAXPOOL2)}
    assert downs["conv1+bn1"] == 1 and downs["maxpool_1"] == 2
    assert [downs[f"block_{s}_2"] for s in ("2_2", "3_2", "4_2", "5_1")] == [2, 3, 4, 5]
    assert sum(op.type == models.OP_CONV and op.res_mode == 1 for op in g.ops) == 7


def test_resnet50_backbone_is_the_pooled_stride32_body():
    g = models.ppn_resnet50(0)
    convs = [op for op in g.ops if op.type == models.OP_CONV and op.name.endswith("_conv3")]
    assert len(convs) == 16                                              # 3 + 4 + 6 + 3 bottlenecks
    assert any(op.type == models.OP_MAXPOOL2 and op.R == 3 for op in g.ops)
    assert g.buffers[convs[-1].out_buf] == (2048, 5)


def _reference_ppn(r, feat, in_h, in_w):
    """pose_proposal/model.py:43-119 on `feat`: add_block_1/2 (conv + bias, BatchNorm, leaky ReLU 0.1), add_block_3 ->
    (raw, (boxes, edges) after sigmoid, split, reshape and restore_coor)"""
    for _ in range(2):
        feat = F.leaky_relu(r.bn(r.conv(feat)), 0.1)
    raw = r.conv(feat)
    x = torch.sigmoid(raw.double())
    K, L = 18, 17
    n, _, hout, wout = x.shape
    pc, pi, px, py, pw, ph = (x[:, t * K:(t + 1) * K] for t in range(6))
    pe = x[:, 6 * K:].reshape(n, L, 9, 9, hout, wout)
    gx, gy = torch.meshgrid(torch.arange(wout, dtype=torch.float64), torch.arange(hout, dtype=torch.float64), indexing="xy")
    px, py = (px + gx) * (in_w / wout), (py + gy) * (in_h / hout)
    pw, ph = pw * in_w, ph * in_h
    return raw, (torch.cat([pc, pi, px, py, pw, ph], 1).numpy(), pe.reshape(n, -1, hout, wout).numpy())


def _resnet18_reference(r, x):
    x = F.relu(r.bn(r.conv(x, stride=2, bias=False)))
    pads = []
    for n in (x.shape[3], x.shape[2]):                                   # MaxPool2d(3, 2, 'SAME')
        total = max((-(-n // 2) - 1) * 2 + 3 - n, 0)
        pads += [total // 2, total - total // 2]
    x = F.max_pool2d(F.pad(x, pads, value=float("-inf")), 3, 2)
    for _, nf, st, ds in models.RESNET18_BLOCKS:                          # Res_block: main_block, then down_sample (backbones.py:564-582)
        y = F.relu(r.bn(r.conv(x, stride=st, bias=False)))
        y = r.bn(r.conv(y, bias=False))
        res = r.bn(r.conv(x, stride=st, bias=False)) if ds else x
        x = F.relu(y + res)
    return x


@pytest.mark.parametrize("net", ["ppn_resnet18", "ppn_resnet50"])
def test_import_equals_reference_definition(net):
    order = W.ppn_resnet18_layer_order() if net == "ppn_resnet18" else W.ppn_resnet50_layer_order()
    arrays = _tl_arrays(order, 51)
    ws = (W.Ppn18Weights if net == "ppn_resnet18" else W.Ppn50Weights)(arrays)
    g = getattr(models, net)(weights=ws)
    H, Wd = 96, 160
    frames = np.random.default_rng(7).integers(0, 256, (2, H, Wd, 3), dtype=np.uint8)
    _, _, bufs = torch_ref.run_graph(g, frames, flip_rgb=True, device="cpu")
    raw = bufs[_head_op(g).in_buf][:, :N_OUT]
    x = torch.from_numpy(np.ascontiguousarray((frames.astype(np.float64) / 255).astype(np.float32)[..., ::-1].transpose(0, 3, 1, 2)))
    r = _TlReader(arrays)
    if net == "ppn_resnet18":
        feat = _resnet18_reference(r, x)
    else:
        feat = _resnet50_reference(r, x, [(64, 3, 1), (128, 4, 2), (256, 6, 2), (512, 3, 2)], True, 1e-5)
    raw_r, (box_r, edge_r) = _reference_ppn(r, feat, H, Wd)
    r.done()
    assert raw.shape == raw_r.shape == (2, N_OUT, 3, 5)
    tol = 3e-4 * max(1.0, float(raw_r.abs().max()))
    assert float((raw - raw_r).abs().max()) < tol
    # the head op's formulas (OP_PPN_HEAD) on the same raw tensor equal sigmoid + split + reshape + restore_coor of model.py
    box, edge = ppn_head_ref(raw_r.double().numpy(), 18, 17 * 81, H, Wd)
    assert box.shape == box_r.shape == (2, 108, 3, 5) and edge.shape == edge_r.shape == (2, 1377, 3, 5)
    np.testing.assert_allclose(box, box_r, rtol=1e-12, atol=1e-300)
    np.testing.assert_allclose(edge, edge_r, rtol=1e-12, atol=1e-300)


def test_leaky_slope_is_not_the_tensorlayer_prelu_sigmoid():
    """add_block_1/2 use tl.act.leaky_relu(alpha=0.1): a fixed slope, not a PRelu weight -- no alpha array in all_weights"""
    assert not any(kind == "prelu" for kind, *_ in W.ppn_resnet18_layer_order() + W.ppn_resnet50_layer_order())


def test_importers_reject_wrong_lists():
    arrays = _tl_arrays(W.ppn_resnet18_layer_order(), 3)
    with pytest.raises(ValueError):
        W.Ppn18Weights(arrays[:-1])
    with pytest.raises(ValueError):
        W.Ppn50Weights(arrays)


def test_head_ref_matches_restore_coor_layout():
    """the float64 head restatement on a tiny hand-made raw tensor: channel t*K + k, grid offsets along x / y"""
    K, E = 18, 2
    raw = np.zeros((1, 6 * K + E, 2, 3))
    box, edge = ppn_head_ref(raw, K, E, 64, 96)
    assert box.shape == (1, 108, 2, 3) and edge.shape == (1, 2, 2, 3) and np.all(edge == 0.5)
    np.testing.assert_allclose(box[0, 2 * K], [[16, 48, 80], [16, 48, 80]])      # (0.5 + gx) * 96 / 3
    np.testing.assert_allclose(box[0, 3 * K], [[16, 16, 16], [48, 48, 48]])      # (0.5 + gy) * 64 / 2
    assert np.all(box[0, 4 * K:5 * K] == 48) and np.all(box[0, 5 * K:] == 32)


@pytest.mark.parametrize("builder", [models.ppn_resnet18, models.ppn_resnet50])
def test_pack_round_trip(builder):
    g = builder(1)
    pack = g.to_pack()
    magic, ver, nb, nops, cc, cp, shift = struct.unpack_from("<8s6I", pack, 0)
    head_type = struct.unpack_from("<I", pack, 8 + 24 + 12)[0]
    assert (magic, nb, nops, cc, cp, shift, head_type) == (models.PACK_MAGIC, len(g.buffers), len(g.ops), 108, 1377, 5, 2)
    rec = struct.unpack_from("<18I3Q", pack, 72 + 8 * nb + 96 * (nops - 1))
    assert rec[0] == models.OP_PPN_HEAD and rec[9] == 18 and rec[7] == 17 and rec[5:7] == (9, 9)
    assert pack == builder(1).to_pack()                                  # deterministic per seed


@pytest.mark.parametrize("net", ["ppn_resnet18", "ppn_resnet50"])
def test_export_writes_a_pack(tmp_path, net):
    out = tmp_path / f"{net}.pack"
    assert export.main(["--model", net, "--out", str(out), "--seed", "2"]) == 0
    assert out.read_bytes() == getattr(models, net)(2).to_pack()
    order = W.ppn_resnet18_layer_order() if net == "ppn_resnet18" else W.ppn_resnet50_layer_order()
    arrays = _tl_arrays(order, 9)
    npz = tmp_path / "w.npz"
    params = np.empty(len(arrays), object)
    params[:] = arrays
    np.savez(npz, params=params)
    out2 = tmp_path / f"{net}_trained.pack"
    assert export.main(["--model", net, "--out", str(out2), "--weights", str(npz)]) == 0
    ws = (W.Ppn18Weights if net == "ppn_resnet18" else W.Ppn50Weights)(arrays)
    assert out2.read_bytes() == getattr(models, net)(weights=ws).to_pack()
