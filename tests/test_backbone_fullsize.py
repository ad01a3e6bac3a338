"""Backbone parity AT THE BENCHMARKED SIZES (VERDICT round 1, "what's weak" item 1).

Every network of the BASELINE configs runs at its full input size through the engine and through the backbone oracle
(oracle/torch_backbone.py: plain PyTorch fp32, TF32 off), and EVERY activation buffer plus both outputs are compared:

  * against the oracle with fp16 rounding emulated where the engine rounds (fp16 operands, fp32 accumulation):
        max|diff| <= 5e-3 * max|ref| + 5e-3            (summation order and a few fp16 ulps are all that is left)
  * against pure fp32:  max|diff| <= 3e-2 * max|ref|   (the fp16-operand budget; measured values are printed and
        recorded in DESIGN.md section 4)

Large-image behaviours this covers that the small-resolution tests cannot: im2col tiles wrapping over rows and images at
W = 656, the 16x8 halo grid at 368x656, the many-wave 7x7 layers, the u8 stem at 656 columns.

Pose-level check (what fp16 does to the OUTPUT of the path): the same frames through fp32 torch -> CPU oracle parser and
through the engine -> GPU parser, thresholds at quantiles of the fp32 maps; peak-set and human-set agreement asserted."""
import numpy as np
import pytest

import oracle
from hyperpose_b200 import capi, models, synthetic as syn
from oracle import torch_backbone

pytestmark = pytest.mark.gpu


def _cmp(got, ref, rel, abs_, what):
    d = float(np.abs(got - ref).max())
    m = float(np.abs(ref).max())
    assert np.isfinite(got).all(), f"{what}: non-finite values"
    assert d <= rel * m + abs_, f"{what}: max|diff| {d:.3e} vs max|ref| {m:.3e} (budget {rel:g}*max + {abs_:g})"
    return d, m


def _every_buffer(g, eng, frames, N, rel, abs_, skip=()):
    """engine buffers (fp16 NHWC) vs the fp16-emulated oracle, all of them; returns the worst relative error"""
    _, _, rbufs = torch_backbone.run_graph(g, frames, emulate_fp16=True)
    worst = 0.0
    for bi in range(len(g.buffers)):
        if bi in skip:
            continue
        try:
            got = eng.debug_read_buffer(bi, N).astype(np.float32).transpose(0, 3, 1, 2)
        except capi.HyperposeError as ex:
            # the un-pooled output of a conv whose 2x2 max-pool runs in its epilogue is never written; the pooled buffer that
            # follows is compared like every other one, which checks conv + pool together
            assert ex.status == capi.HP_ERR_UNSUPPORTED, ex
            continue
        ref = rbufs[bi].cpu().numpy()
        c = ref.shape[1]
        d, m = _cmp(got[:, :c], ref, rel, abs_, f"{g.name} buffer {bi} {tuple(ref.shape)}")
        worst = max(worst, d / max(m, 1e-30))
    return worst


def _run(g, H, W, N, seed, rel16, rel32, im2col_buf0=True):
    frames = syn.make_frames_u8(seed, N, H, W)
    eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=N)
    eng.infer_u8(frames)
    a, b = eng.read_outputs(N)
    # buffer 0 is the im2col / stem patch buffer: the fused stems never write it
    worst = _every_buffer(g, eng, frames, N, rel16, rel16, skip=(0,) if im2col_buf0 else ())
    ra, rb, _ = torch_backbone.run_graph(g, frames, emulate_fp16=True)
    ra, rb = ra.cpu().numpy().reshape(a.shape), rb.cpu().numpy().reshape(b.shape)
    _cmp(a, ra, rel16, rel16, f"{g.name} output a (fp16-emulated oracle)")
    _cmp(b, rb, rel16, rel16, f"{g.name} output b (fp16-emulated oracle)")
    fa, fb, _ = torch_backbone.run_graph(g, frames, emulate_fp16=False)
    fa, fb = fa.cpu().numpy().reshape(a.shape), fb.cpu().numpy().reshape(b.shape)
    d1, m1 = _cmp(a, fa, rel32, 1e-3, f"{g.name} output a vs fp32")
    d2, m2 = _cmp(b, fb, rel32, 1e-3, f"{g.name} output b vs fp32")
    print(f"[fullsize] {g.name} {H}x{W} batch {N}: worst buffer rel err vs fp16-emulated oracle {worst:.2e}; "
          f"vs fp32: a {d1:.2e}/{m1:.2e} = {d1 / m1:.2e}, b {d2:.2e}/{m2:.2e} = {d2 / m2:.2e}")
    eng.close()
    return frames, (a, b), (fa, fb)


def test_openpose_vgg19_six_stages_at_368x656():
    """BASELINE cfg3: the full 56-op graph at the benchmarked resolution, batch 3 (tiles straddle image boundaries)"""
    _run(models.openpose_vgg19(0), 368, 656, 3, 21, 5e-3, 3e-2)


def test_mobilenet_thin_openpose_at_368x432():
    """BASELINE cfg2 at full size (6 stages)"""
    _run(models.mobilenet_thin_openpose(0), 368, 432, 2, 22, 5e-3, 3e-2)


def test_resnet50_lw_openpose_at_368x432():
    """BASELINE cfg4 at full size"""
    _run(models.resnet50_lw_openpose(0), 368, 432, 2, 23, 6e-3, 3e-2)


def test_resnet50_pifpaf_at_385x385():
    """BASELINE cfg5 at full size (49x49 fields)"""
    _run(models.resnet50_pifpaf(0), 385, 385, 2, 24, 8e-3, 3e-2)


def _peak_set(peaks):
    return {(int(p["part_id"]), int(p["x"]), int(p["y"])) for p in peaks}


def test_pose_level_agreement_fp16_engine_vs_fp32_backbone():
    """frames -> fp32 torch backbone -> CPU oracle parser   vs   frames -> fp16 engine -> GPU parser (hp_pose_run_u8_host).
    Random-init weights give structureless maps, so the thresholds sit at quantiles of the fp32 maps (as in
    test_end_to_end_pose_call...).  Parser parity on IDENTICAL tensors is bit-exact (test_paf_gpu.py); this measures what the
    fp16 operand rounding of the backbone does to the result: peaks that sit within the fp16 budget of the threshold or of a
    neighbouring local maximum may flip on these structureless maps (a worst case: every pixel is near a threshold or a
    tie; trained heat-maps have isolated peaks).  Asserted: Jaccard of the peak sets >= 0.85
    and human counts within 10 % -- the measured values are printed."""
    g = models.openpose_vgg19(0)
    H, W, N = 368, 656, 2
    frames = syn.make_frames_u8(31, N, H, W)
    fconf, fpaf, _ = torch_backbone.run_graph(g, frames, emulate_fp16=False)
    fconf, fpaf = fconf.cpu().numpy(), fpaf.cpu().numpy()
    ct = float(np.quantile(fconf[:, :18], 0.985))
    pt = float(np.quantile(fpaf, 0.5))
    eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=N)
    parser = capi.PafParser(ct, pt)
    parser.set_capacity(peaks_per_part=2048, candidates_per_limb=1 << 16, humans=256)
    humans = eng.run_pose(parser, frames, cap=256)
    inter = union = n_ref_h = n_got_h = 0
    for i in range(N):
        ref = oracle.oracle_process(fconf[i], fpaf[i], ct, pt, peak_cap=1 << 18, conn_cap=1 << 15)
        got_peaks = _peak_set(parser.debug_peaks(i))
        ref_peaks = _peak_set(ref["peaks"])
        inter += len(got_peaks & ref_peaks)
        union += len(got_peaks | ref_peaks)
        n_ref_h += len(ref["humans"])
        n_got_h += len(humans[i])
    jac = inter / max(union, 1)
    print(f"[pose-level] peaks: {inter} common of {union} (Jaccard {jac:.4f}); humans fp32-oracle {n_ref_h} vs fp16-engine {n_got_h} "
          f"(conf_thresh {ct:.4g}, paf_thresh {pt:.4g})")
    assert union > 200, "vacuous: too few peaks at this threshold"
    assert jac >= 0.85, f"peak-set agreement {jac:.3f}"
    assert abs(n_ref_h - n_got_h) <= max(2, 0.1 * max(n_ref_h, n_got_h)), (n_ref_h, n_got_h)
    eng.close(); parser.close()
