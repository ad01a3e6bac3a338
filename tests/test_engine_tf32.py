"""The data_type::kFLOAT engine (include/hyperpose/operator/dnn/tensorrt.hpp:14-22,48,61): fp32 activations in HBM,
wgmma kind tf32 (conv_wgmma_kernel<float, ...>), fp32 helper kernels -- hp_engine_create_ex(..., HP_DTYPE_TF32).

Checker: oracle/torch_backbone.py in plain fp32 (TF32 off in torch).  Tolerance, stated here as the contract asks: TF32 keeps a
10-bit mantissa on the conv operands (weights and activations rounded to nearest by their producers), everything else is fp32,
so every buffer and both outputs must sit within
        max|diff| <= 6e-3 * max|ref| + 1e-3
of the fp32 reference (measured values are printed; the f16 engine's budget against the same reference is 3e-2)."""
import numpy as np
import pytest

from hyperpose_b200 import capi, models, synthetic as syn
from oracle import torch_backbone

pytestmark = pytest.mark.gpu

REL, ABS = 6e-3, 1e-3


def _cmp(got, ref, what, rel=REL, abs_=ABS):
    d = float(np.abs(got - ref).max())
    m = float(np.abs(ref).max())
    assert np.isfinite(got).all(), what
    assert d <= rel * m + abs_, f"{what}: max|diff| {d:.3e} vs max|ref| {m:.3e}"
    return d / max(m, 1e-30)


def _run(g, H, W, N, seed, skip0=True):
    frames = syn.make_frames_u8(seed, N, H, W)
    eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=N, dtype="tf32")
    assert capi.lib().hp_engine_dtype(eng._h) == 1
    eng.infer_u8(frames)
    a, b = eng.read_outputs(N)
    ra, rb, rbufs = torch_backbone.run_graph(g, frames, emulate_fp16=False)
    worst = 0.0
    for bi in range(1 if skip0 else 0, len(g.buffers)):
        got = eng.debug_read_buffer(bi, N)
        assert got.dtype == np.float32
        ref = rbufs[bi].cpu().numpy()
        worst = max(worst, _cmp(got.transpose(0, 3, 1, 2)[:, :ref.shape[1]], ref, f"{g.name} buffer {bi}"))
    ea = _cmp(a, ra.cpu().numpy().reshape(a.shape), f"{g.name} output a")
    eb = _cmp(b, rb.cpu().numpy().reshape(b.shape), f"{g.name} output b")
    print(f"[tf32] {g.name} {H}x{W} batch {N}: worst buffer rel err {worst:.2e}, outputs {ea:.2e} / {eb:.2e} (vs torch fp32)")
    return eng, frames, (a, b)


@pytest.mark.parametrize("hw,N", [((64, 80), 2), ((50, 70), 3), ((16, 24), 1)])
def test_tiny_net_every_layer_tf32(hw, N):
    """every op type incl. ragged sizes: im2col gather, 3x3 / 1x1 / grouped / residual convs, depthwise, max-pools, NCHW-split output"""
    eng, _, _ = _run(models.tiny_test_net(1), hw[0], hw[1], N, 3)
    eng.close()


def test_openpose_vgg19_at_368x656_tf32():
    """BASELINE cfg3 network at the benchmarked resolution through the kFLOAT engine"""
    eng, frames, (conf, paf) = _run(models.openpose_vgg19(0), 368, 656, 2, 21)
    # and it is a different arithmetic from the kHALF engine, not an alias of it
    e16 = capi.Engine(models.openpose_vgg19(0).to_pack(), (656, 368), max_batch_size=2)
    e16.infer_u8(frames)
    c16, p16 = e16.read_outputs(2)
    assert not np.array_equal(c16, conf)
    d = float(np.abs(c16 - conf).max()) / float(np.abs(conf).max())
    assert d < 3e-2
    print(f"[tf32] f16 engine vs tf32 engine on the same frames: {d:.2e} of max|conf|")
    e16.close(); eng.close()


def test_mobilenet_thin_tf32():
    eng, _, _ = _run(models.mobilenet_thin_openpose(0, n_stages=3), 96, 128, 2, 4)
    eng.close()


def test_resnet50_lw_openpose_tf32():
    eng, _, _ = _run(models.resnet50_lw_openpose(0), 96, 128, 2, 6)
    eng.close()


def test_resnet50_pifpaf_tf32():
    eng, _, _ = _run(models.resnet50_pifpaf(0), 129, 129, 2, 8)
    eng.close()


def test_f32_nchw_entry_and_pose_call_tf32():
    """tensorrt::inference(const std::vector<float>&, n) and hp_pose_run_u8_host on a kFLOAT engine"""
    import oracle
    g = models.tiny_test_net(2)
    H, W, N = 32, 48, 2
    frames = syn.make_frames_u8(5, N, H, W)
    eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=N, dtype="tf32")
    eng.infer_u8(frames)
    c1, p1 = eng.read_outputs(N)
    x = (frames.astype(np.float64) / 255.0).astype(np.float32)[..., ::-1].transpose(0, 3, 1, 2)   # data.cpp:21-51
    eng.infer_f32(np.ascontiguousarray(x))
    c2, p2 = eng.read_outputs(N)
    assert np.allclose(c1, c2, atol=1e-5) and np.allclose(p1, p2, atol=1e-5)
    ct, pt = float(np.quantile(c1[:, :18], 0.97)), float(np.quantile(p1, 0.5))
    parser = capi.PafParser(ct, pt)
    parser.set_capacity(peaks_per_part=1024, candidates_per_limb=1 << 15, humans=128)
    humans = eng.run_pose(parser, frames, cap=128)
    for i in range(N):
        assert humans[i].tobytes() == oracle.oracle_process(c1[i], p1[i], ct, pt, peak_cap=1 << 18, conn_cap=1 << 14)["humans"].tobytes()
    eng.close(); parser.close()
