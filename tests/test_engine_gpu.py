"""GPU tests of the DNN engine (wgmma implicit-GEMM convs) against a plain PyTorch fp32 reference.

Tolerances (written here, as the contract asks):
  * vs the torch reference with fp16 rounding emulated at the same points: max |diff| <= 2e-3 * max|ref| + 2e-3
    (only fp32 summation-order differences remain);
  * vs the pure fp32 reference: reported, and bounded by 3e-2 * max|ref| (fp16 operand rounding through
    ~40 layers; the reference engine is documented FP32, the north_star sets parser parity on identical
    tensors and leaves the backbone budget to be stated -- this is it)."""
import os

import numpy as np
import pytest

import oracle
from hyperpose_b200 import capi, models, synthetic as syn
from oracle import torch_backbone as torch_ref

pytestmark = pytest.mark.gpu


def _err(a, b):
    return float(np.abs(a - b).max()), float(np.abs(b).max())


def _check(got, ref, rel, abs_, what):
    d, m = _err(got, ref)
    assert d <= rel * m + abs_, f"{what}: max|diff| {d:.3e} vs max|ref| {m:.3e}"
    return d, m


@pytest.mark.parametrize("hw,N", [((64, 80), 2), ((50, 70), 3), ((16, 24), 1)])
def test_tiny_net_every_layer(hw, N):
    """every op type / conv variant, incl. ragged sizes (tile padding, TMA zero-fill borders, ceil max-pool)"""
    H, W = hw
    g = models.tiny_test_net(1)
    frames = syn.make_frames_u8(3, N, H, W)
    eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=N)
    eng.infer_u8(frames)
    conf, paf = eng.read_outputs(N)
    rconf, rpaf, rbufs = torch_ref.run_graph(g, frames, emulate_fp16=True)
    for bi in range(len(g.buffers)):
        try:
            got = eng.debug_read_buffer(bi, N).astype(np.float32).transpose(0, 3, 1, 2)
        except capi.HyperposeError as ex:
            # the output of a conv whose 2x2 max-pool / 1x1 depthwise op runs in its epilogue is never written; the buffer that
            # follows is compared like every other one, which checks the two together
            assert ex.status == capi.HP_ERR_UNSUPPORTED, ex
            continue
        ref = rbufs[bi].cpu().numpy()
        if bi == 0:   # im2col buffer: compare its centre tap (k = 4*3 + c) with the normalised image
            if not os.environ.get("HPB_NO_STEM3"):
                # fused 3x3 stem: the patches never leave shared memory, this buffer is not written; buffer 1 (the first conv's
                # output) checks the stem, test_f32_nchw_entry_matches_u8_entry the im2col kernel
                assert not got.any()
                continue
            got = got[:, 12:15]
            ref = ref[:, :3]
        # the concat buffer is overwritten by later ops in both executors identically
        _check(got, ref, 2e-3, 2e-3, f"buffer {bi}")
    _check(conf, rconf.cpu().numpy(), 2e-3, 2e-3, "conf")
    _check(paf, rpaf.cpu().numpy(), 2e-3, 2e-3, "paf")
    fconf, fpaf, _ = torch_ref.run_graph(g, frames, emulate_fp16=False)
    _check(conf, fconf.cpu().numpy(), 3e-2, 1e-3, "conf vs fp32")
    _check(paf, fpaf.cpu().numpy(), 3e-2, 1e-3, "paf vs fp32")
    eng.close()


def test_openpose_vgg19_small_resolution():
    """the full 56-op OpenPose-VGG19 graph (BASELINE config 3 architecture) at 96x128, batch 2"""
    g = models.openpose_vgg19(0)
    H, W, N = 96, 128, 2
    frames = syn.make_frames_u8(2, N, H, W)
    eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=N)
    assert (eng.out_h, eng.out_w, eng.c_conf, eng.c_paf) == (12, 16, 19, 38)
    eng.infer_u8(frames)
    conf, paf = eng.read_outputs(N)
    rconf, rpaf, _ = torch_ref.run_graph(g, frames, emulate_fp16=True)
    _check(conf, rconf.cpu().numpy(), 5e-3, 2e-3, "conf (fp16-emulated ref)")
    _check(paf, rpaf.cpu().numpy(), 5e-3, 2e-3, "paf (fp16-emulated ref)")
    fconf, fpaf, _ = torch_ref.run_graph(g, frames, emulate_fp16=False)
    d1, m1 = _check(conf, fconf.cpu().numpy(), 3e-2, 1e-3, "conf vs fp32")
    d2, m2 = _check(paf, fpaf.cpu().numpy(), 3e-2, 1e-3, "paf vs fp32")
    print(f"fp16-operand budget: conf {d1:.2e}/{m1:.2e}  paf {d2:.2e}/{m2:.2e}")
    eng.close()


@pytest.mark.parametrize("hw,N", [((96, 128), 2), ((72, 88), 1)])
def test_mobilenet_thin_openpose(hw, N):
    """BASELINE config 2 architecture (MobilenetThin + separable-block heads): depthwise 3x3/1x1 (stride 1/2, TF SAME),
    stride-2 stem, three-scale concat, grouped 1x1 convs -- every buffer and both outputs vs torch"""
    H, W = hw
    g = models.mobilenet_thin_openpose(0, n_stages=3)
    frames = syn.make_frames_u8(4, N, H, W)
    eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=N)
    eng.infer_u8(frames)
    conf, paf = eng.read_outputs(N)
    rconf, rpaf, rbufs = torch_ref.run_graph(g, frames, emulate_fp16=True)
    for bi in range(1, len(g.buffers)):
        try:
            got = eng.debug_read_buffer(bi, N).astype(np.float32).transpose(0, 3, 1, 2)
        except capi.HyperposeError as ex:
            # the output of a conv whose 2x2 max-pool / 1x1 depthwise op runs in its epilogue is never written; the buffer that
            # follows is compared like every other one, which checks the two together
            assert ex.status == capi.HP_ERR_UNSUPPORTED, ex
            continue
        _check(got, rbufs[bi].cpu().numpy(), 4e-3, 4e-3, f"buffer {bi}")
    _check(conf, rconf.cpu().numpy(), 4e-3, 4e-3, "conf")
    _check(paf, rpaf.cpu().numpy(), 4e-3, 4e-3, "paf")
    fconf, fpaf, _ = torch_ref.run_graph(g, frames, emulate_fp16=False)
    d1, m1 = _check(conf, fconf.cpu().numpy(), 3e-2, 2e-3, "conf vs fp32")
    d2, m2 = _check(paf, fpaf.cpu().numpy(), 3e-2, 2e-3, "paf vs fp32")
    print(f"mobilenet-thin fp16 budget: conf {d1:.2e}/{m1:.2e} paf {d2:.2e}/{m2:.2e}")
    eng.close()


@pytest.mark.parametrize("hw,N", [((96, 128), 2), ((72, 104), 1)])
def test_resnet50_lw_openpose(hw, N):
    """BASELINE config 4 architecture (ResNet-50 stride 8 + Lightweight-OpenPose head): 7x7/2 stem, 3x3/2 max-pool,
    bottleneck residual epilogues (both add orders), exact stride-2 sub-sampling -- every buffer and both outputs vs torch"""
    H, W = hw
    g = models.resnet50_lw_openpose(0)
    frames = syn.make_frames_u8(6, N, H, W)
    eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=N)
    eng.infer_u8(frames)
    conf, paf = eng.read_outputs(N)
    rconf, rpaf, rbufs = torch_ref.run_graph(g, frames, emulate_fp16=True)
    for bi in range(1, len(g.buffers)):
        try:
            got = eng.debug_read_buffer(bi, N).astype(np.float32).transpose(0, 3, 1, 2)
        except capi.HyperposeError as ex:
            # the output of a conv whose 2x2 max-pool / 1x1 depthwise op runs in its epilogue is never written; the buffer that
            # follows is compared like every other one, which checks the two together
            assert ex.status == capi.HP_ERR_UNSUPPORTED, ex
            continue
        _check(got, rbufs[bi].cpu().numpy(), 6e-3, 6e-3, f"buffer {bi}")
    _check(conf, rconf.cpu().numpy(), 6e-3, 6e-3, "conf")
    _check(paf, rpaf.cpu().numpy(), 6e-3, 6e-3, "paf")
    fconf, fpaf, _ = torch_ref.run_graph(g, frames, emulate_fp16=False)
    d1, m1 = _check(conf, fconf.cpu().numpy(), 3e-2, 2e-3, "conf vs fp32")
    d2, m2 = _check(paf, fpaf.cpu().numpy(), 3e-2, 2e-3, "paf vs fp32")
    print(f"resnet50-lw fp16 budget: conf {d1:.2e}/{m1:.2e} paf {d2:.2e}/{m2:.2e}")
    eng.close()


def test_resnet50_pifpaf_fields_and_decode():
    """BASELINE config 5: ResNet-50 (stride 16, no max-pool) + PIF/PAF heads (pixel shuffle, crop, sigmoid/softplus, index grid)
    vs torch, then the engine's own device-resident fields through the CUDA decoder vs the reference decoder (oracle/_ref)."""
    g = models.resnet50_pifpaf(0)
    H = W = 129
    N = 2
    frames = syn.make_frames_u8(8, N, H, W)
    eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=N)
    assert (eng.out_h, eng.out_w, eng.c_conf, eng.c_paf) == (17, 17, 85, 171)
    eng.infer_u8(frames)
    pif, paf = eng.read_outputs(N)
    rpif, rpaf, _ = torch_ref.run_graph(g, frames, emulate_fp16=True)
    _check(pif.reshape(N, 17, 5, 17, 17), rpif.cpu().numpy(), 8e-3, 8e-3, "pif fields")
    _check(paf.reshape(N, 19, 9, 17, 17), rpaf.cpu().numpy(), 8e-3, 8e-3, "paf fields")
    if oracle.pifpaf_ref_available():
        # Random weights regress coordinates far outside the image; the reference then indexes its high-resolution map with
        # negative values cast to size_t (postprocessor.cpp:693,741 -- undefined behaviour, observed to fabricate people).
        # Both decoders therefore get the same fields with the regressed coordinates clipped into the map.
        pf = pif.reshape(N, 17, 5, 17, 17).copy(); pa = paf.reshape(N, 19, 9, 17, 17).copy()
        pf[:, :, 1:3] = np.clip(pf[:, :, 1:3], 0.0, 16.0); pa[:, :, 1:5] = np.clip(pa[:, :, 1:5], 0.0, 16.0)
        dec = capi.PifPafParser(H, W, 0.1)
        got = dec.process_batch(pf, pa)
        for i in range(N):
            want = oracle.ref_pifpaf_process(pf[i], pa[i], H, W, 0.1)
            assert got[i].tobytes() == want.tobytes(), (len(got[i]), len(want))
        dec.close()
    eng.close()


def test_f32_nchw_entry_matches_u8_entry():
    """tensorrt::inference(const std::vector<float>&, n): pre-scaled NCHW floats give the same outputs"""
    g = models.tiny_test_net(2)
    H, W, N = 32, 48, 2
    frames = syn.make_frames_u8(5, N, H, W)
    eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=N)
    eng.infer_u8(frames)
    c1, p1 = eng.read_outputs(N)
    x = (frames.astype(np.float64) / 255.0).astype(np.float32)[..., ::-1].transpose(0, 3, 1, 2)   # data.cpp:21-51
    eng.infer_f32(np.ascontiguousarray(x))
    c2, p2 = eng.read_outputs(N)
    assert np.allclose(c1, c2, atol=2e-3) and np.allclose(p1, p2, atol=2e-3)
    eng.close()


def test_batch_overflow_is_an_error():
    g = models.tiny_test_net(0)
    eng = capi.Engine(g.to_pack(), (32, 32), max_batch_size=2)
    with pytest.raises(capi.HyperposeError) as e:
        eng.infer_u8(np.zeros((3, 32, 32, 3), np.uint8))
    assert e.value.status == capi.HP_ERR_BATCH     # std::logic_error in the reference (tensorrt.cpp:439-443)
    eng.close()


def test_end_to_end_pose_call_matches_oracle_on_the_engines_own_tensors():
    """hp_pose_run_u8_host: frames -> humans with conf/paf staying on the device; parse parity is defined on
    identical input tensors, so the oracle runs on the engine's conf/paf read back to the host.  Random weights
    give structureless maps, so conf_thresh is set at a high quantile of the engine's own output."""
    g = models.tiny_test_net(4)
    H, W, N = 64, 96, 4
    frames = syn.make_frames_u8(9, N, H, W)
    eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=N)
    eng.infer_u8(frames)
    conf, paf = eng.read_outputs(N)
    ct = float(np.quantile(conf[:, :18], 0.97))
    pt = float(np.quantile(paf, 0.5))
    parser = capi.PafParser(ct, pt)
    parser.set_capacity(peaks_per_part=1024, candidates_per_limb=1 << 15, humans=128)
    humans = eng.run_pose(parser, frames, cap=128)
    total_peaks = 0
    for i in range(N):
        orc = oracle.oracle_process(conf[i], paf[i], ct, pt, peak_cap=1 << 18, conn_cap=1 << 14)
        total_peaks += len(orc["peaks"])
        assert humans[i].tobytes() == orc["humans"].tobytes()
    assert total_peaks > 20, "vacuous: no peaks at this threshold"
    eng.close(); parser.close()


def test_output_override_hook_and_profile():
    """bench-only hook: synthetic tensors copied over the outputs after the last conv; per-op event profile"""
    import torch
    g = models.tiny_test_net(4)
    H, W, N = 64, 96, 2
    frames = syn.make_frames_u8(9, N, H, W)
    eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=N)
    conf, paf = syn.make_batch_tensors(3, N, (1, 3), eng.out_h, eng.out_w)
    dc, dp = torch.from_numpy(conf).cuda(), torch.from_numpy(paf).cuda()
    torch.cuda.synchronize()
    eng.set_output_override(dc.data_ptr(), dp.data_ptr())
    eng.set_profiling(True)
    parser = capi.PafParser()
    humans = eng.run_pose(parser, frames)
    eng.set_profiling(False)
    for i in range(N):
        assert humans[i].tobytes() == oracle.oracle_process(conf[i], paf[i])["humans"].tobytes()
    ms, ty, fl, runs = eng.get_profile()
    assert runs == 1 and len(ms) == len(g.ops) and ms[ty == models.OP_CONV].sum() > 0
    eng.close(); parser.close()


@pytest.mark.parametrize("src_hw,keep", [((90, 150), False), ((128, 192), False), ((200, 120), True), ((48, 200), True), ((64, 96), False)])
def test_gpu_frame_resize_bit_exact_vs_oracle(src_hw, keep):
    """A1: the resize step of tensorrt::inference (cv::resize INTER_LINEAR / non_scaling_resize) on the GPU,
    bit-exact against the oracle restatement that is pinned to cv2 (tests/test_oracle_cv_pin.py)"""
    g = models.tiny_test_net(0)
    H, W = 64, 96
    eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=2)
    rng = np.random.default_rng(5)
    frames = [rng.integers(0, 256, (src_hw[0], src_hw[1], 3), dtype=np.uint8) for _ in range(2)]
    for i, f in enumerate(frames):
        eng.stage_frame(i, f, keep_ratio=keep)
    got = eng.debug_read_frames(2)
    for i, f in enumerate(frames):
        want = oracle.resize_linear_u8(f, H, W, letterbox=keep)
        assert np.array_equal(got[i], want), f"frame {i}: {np.abs(got[i].astype(int) - want.astype(int)).max()}"
    eng.infer_staged(2)
    c1, p1 = eng.read_outputs(2)
    eng.infer_u8(got)
    c2, p2 = eng.read_outputs(2)
    assert np.array_equal(c1, c2) and np.array_equal(p1, p2)
    eng.close()


def test_full_size_batch_permutation_invariance():
    """size-independent property at the full BASELINE cfg3 size (368x656, batch 16): frames are independent, so permuting
    the batch permutes the outputs bit-for-bit -- exercises im2col tiles that straddle row and image boundaries and the
    ragged last pixel tile at full scale."""
    g = models.openpose_vgg19(0, n_stages=2)
    H, W, N = 368, 656, 16
    frames = syn.make_frames_u8(12, N, H, W)
    eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=N)
    eng.infer_u8(frames)
    c1, p1 = eng.read_outputs(N)
    perm = np.random.default_rng(1).permutation(N)
    eng.infer_u8(frames[perm])
    c2, p2 = eng.read_outputs(N)
    assert np.array_equal(c1[perm], c2) and np.array_equal(p1[perm], p2)
    # a smaller batch through the same engine (different tile / unit counts) gives the same per-frame result
    eng.infer_u8(frames[:5])
    c3, p3 = eng.read_outputs(5)
    assert np.array_equal(c1[:5], c3) and np.array_equal(p1[:5], p3)
    assert np.isfinite(c1).all() and np.abs(c1).max() > 0
    eng.close()


def test_fused_3x3_stem_kernel_matches_im2col_path():
    """3x3 stems: the fused u8 stem (default; warpgroup 0 of conv_wgmma_kernel gathers the patches straight from the u8 frames)
    == the im2col-buffer path (HPB_NO_STEM3), on an odd-sized input (partial tiles, all four borders)"""
    import subprocess, sys, textwrap
    code = textwrap.dedent('''
        import numpy as np, sys
        sys.path.insert(0, %r)
        from hyperpose_b200 import capi, models, synthetic as syn
        g = models.tiny_test_net(1)
        fr = syn.make_frames_u8(3, 2, 50, 70)
        e = capi.Engine(g.to_pack(), (70, 50), max_batch_size=2)
        e.infer_u8(fr); c, p = e.read_outputs(2)
        np.save(sys.argv[1], np.concatenate([c.ravel(), p.ravel()]))
    ''') % os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    import tempfile
    outs = []
    for env in ({}, {"HPB_NO_STEM3": "1"}):
        with tempfile.NamedTemporaryFile(suffix=".npy") as f:
            r = subprocess.run([sys.executable, "-c", code, f.name], env={**os.environ, **env}, capture_output=True, text=True, timeout=300)
            assert r.returncode == 0, r.stderr
            outs.append(np.load(f.name))
    # the two paths feed the same fp16 patch values to the same MMA shape: results agree to fp32 summation order
    assert np.allclose(outs[0], outs[1], rtol=0, atol=1e-4 * np.abs(outs[0]).max())


def test_halo_box_kernel_matches_im2col_kernels():
    """conv_halo_kernel (one TMA halo box per 16 x 8-pixel tile serves every filter tap through shifted wgmma descriptors)
    == the per-tap im2col-mode kernels, on ragged sizes (partial tiles on the right / bottom, all four zero-padded borders,
    grouped and 7x7 layers with HPB_HALO=all)"""
    import subprocess, sys, tempfile, textwrap
    code = textwrap.dedent('''
        import numpy as np, sys
        sys.path.insert(0, %r)
        from hyperpose_b200 import capi, models, synthetic as syn
        outs = []
        for (h, w, n) in ((50, 70, 3), (64, 80, 2), (16, 24, 1)):
            e = capi.Engine(models.tiny_test_net(1).to_pack(), (w, h), max_batch_size=n)
            e.infer_u8(syn.make_frames_u8(3, n, h, w)); c, p = e.read_outputs(n)
            outs += [c.ravel(), p.ravel()]
            e.close()
        e = capi.Engine(models.openpose_vgg19(0).to_pack(), (104, 72), max_batch_size=2)
        e.infer_u8(syn.make_frames_u8(5, 2, 72, 104)); c, p = e.read_outputs(2)
        outs += [c.ravel(), p.ravel()]
        np.save(sys.argv[1], np.concatenate(outs))
    ''') % os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    outs = []
    for env in ({"HPB_HALO": "0"}, {"HPB_HALO": "all"}, {}):
        with tempfile.NamedTemporaryFile(suffix=".npy") as f:
            r = subprocess.run([sys.executable, "-c", code, f.name], env={**os.environ, **env}, capture_output=True, text=True, timeout=600)
            assert r.returncode == 0, r.stderr
            outs.append(np.load(f.name))
    m = np.abs(outs[0]).max()
    assert m > 0
    # same fp16 operands, same fp32 accumulator; only the order of the k-steps differs (chunk-major instead of tap-major)
    # (through ~40 layers with fp16 activations the re-ordered sums differ by a few fp16 roundings)
    assert np.abs(outs[1] - outs[0]).max() <= 2e-3 * m, np.abs(outs[1] - outs[0]).max() / m
    assert np.abs(outs[2] - outs[0]).max() <= 2e-3 * m


def test_max_pool_fused_into_the_halo_epilogue_is_bit_identical(monkeypatch):
    """conv (halo kernel) -> 2x2 max-pool with the pool taken in the conv's epilogue (on the raw accumulators, before bias / ReLU /
    rounding -- all monotone) against the two separate launches (HPB_NO_POOL_FUSE=1): every materialised buffer and both outputs
    must be the same BYTES; the un-pooled buffer is the one that is no longer written."""
    g = models.openpose_vgg19(0, n_stages=2)
    H, W, N = 112, 136, 3                  # 112 = 7 x 16, 136 = 17 x 8: interior, edge and corner tiles; even sizes
    frames = syn.make_frames_u8(17, N, H, W)

    def run():
        eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=N)
        eng.infer_u8(frames)
        outs = eng.read_outputs(N)
        bufs = {}
        for bi in range(1, len(g.buffers)):
            try:
                bufs[bi] = eng.debug_read_buffer(bi, N).tobytes()
            except capi.HyperposeError as ex:
                assert ex.status == capi.HP_ERR_UNSUPPORTED
        eng.close()
        return outs, bufs

    fused_outs, fused = run()
    monkeypatch.setenv("HPB_NO_POOL_FUSE", "1")
    plain_outs, plain = run()
    assert len(plain) == len(g.buffers) - 1 and len(fused) == len(plain) - 1, "exactly one buffer (conv1_2's un-pooled output) is fused away"
    for bi, b in fused.items():
        assert b == plain[bi], f"buffer {bi} differs between the fused and the two-launch form"
    assert fused_outs[0].tobytes() == plain_outs[0].tobytes() and fused_outs[1].tobytes() == plain_outs[1].tobytes()


def test_fused_depthwise_forms_are_bit_identical(monkeypatch):
    """MobilenetThin-OpenPose: (a) the 1x1 "depthwise" ops (per-channel affine + ReLU) applied in the preceding conv's epilogue, with the
    fp16 rounding of the tensor in between kept, and (b) the two depthwise 3x3 convs of a stage's first block served by one dual
    launch -- against the plain one-launch-per-op form (HPB_NO_DW1_FUSE / HPB_NO_DW_DUAL): identical bytes in both outputs."""
    g = models.mobilenet_thin_openpose(0, n_stages=3)
    H, W, N = 96, 128, 2
    frames = syn.make_frames_u8(19, N, H, W)

    def run():
        eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=N)
        launches0 = eng.launch_count
        eng.infer_u8(frames)
        outs = eng.read_outputs(N)
        n = eng.launch_count - launches0
        eng.close()
        return outs, n

    fused, n_fused = run()
    monkeypatch.setenv("HPB_NO_DW1_FUSE", "1")
    monkeypatch.setenv("HPB_NO_DW_DUAL", "1")
    plain, n_plain = run()
    assert n_fused < n_plain, (n_fused, n_plain)
    assert fused[0].tobytes() == plain[0].tobytes() and fused[1].tobytes() == plain[1].tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("hw,N", [((96, 128), 2), ((368, 432), 3), ((200, 1040), 1)])
def test_tma_tiled_depthwise_kernel_is_bit_identical(monkeypatch, hw, N):
    """MobilenetThin-OpenPose with the 3x3 / stride-1 depthwise layers of >= 64 channels on dwconv3_tma_kernel (input tiles with their
    halo staged by TMA, single and dual filter sets) against the per-lane-load kernels (HPB_NO_DW_TMA): every activation buffer and both
    outputs must be the same BYTES.  368x432 has ragged bottom tiles (46 rows); 200x1040 is wider than one 62-column tile at every
    resolution (520 / 260 / 130 columns: several x tiles with ragged right edges)."""
    g = models.mobilenet_thin_openpose(0, n_stages=2)
    H, W = hw
    frames = syn.make_frames_u8(23, N, H, W)

    def run():
        eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=N)
        eng.infer_u8(frames)
        outs = eng.read_outputs(N)
        bufs = {}
        for bi in range(1, len(g.buffers)):
            try:
                bufs[bi] = eng.debug_read_buffer(bi, N).tobytes()
            except capi.HyperposeError as ex:
                assert ex.status == capi.HP_ERR_UNSUPPORTED
        eng.close()
        return outs, bufs

    tiled_outs, tiled = run()
    monkeypatch.setenv("HPB_NO_DW_TMA", "1")
    plain_outs, plain = run()
    assert tiled.keys() == plain.keys()
    for bi, b in tiled.items():
        assert b == plain[bi], f"buffer {bi} ({g.buffers[bi]}) differs between the TMA-tiled and the per-lane-load depthwise kernels"
    assert tiled_outs[0].tobytes() == plain_outs[0].tobytes() and tiled_outs[1].tobytes() == plain_outs[1].tobytes()
