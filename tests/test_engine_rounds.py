"""Conv launches in the regimes the one-tile cases of tests/test_engine_kernels.py never reach, on its harness (_run_and_check:
every output against float64 within its bound, the channels outside the op keep their bits, the bound rejects two wrong references):

  * more than one work item per CTA.  The conv kernels are persistent (item = blockIdx.x, + gridDim.x, ... with gridDim.x =
    min(SMs, items)) and carry the stage ring's slot and phase, the accumulator reset and the last k-step's stage hand-back from one
    item to the next.  Every instantiation of CONV_KERNELS and the wide / ping-pong halo items runs a launch in which some CTA takes
    two or more items and the item count is not a multiple of the grid; in every family some CTA takes three or more items of an odd
    number of k-steps, so that consecutive items start on different ring slots and phases.  The cases cover grouped layers, concat
    output offsets and ragged last n-tiles.
  * a batch shorter than the engine's max_batch (the last batch of a video).  The tensor maps span max_batch frames, so a load past
    frame N reads real data (NaN here) and a store past it lands in frame N: nothing but the kernels' own masks keeps those frames.
    Every multi-round case runs N = max_batch - 1 frames, and so do small cases of every kernel family: conv, residual, both stems
    through both entries, every halo item with both epilogues, the depthwise and max-pool kernels.
  * the conf / PAF output conv (OUT_F32_NCHW_SPLIT): planar fp32 stores into two outputs, split inside an n-tile or in a later one,
    checked without the output-rounding term of the bound.
  * filter shapes no model uses yet: 5 x 5 on both kernels (and every halo item that takes it), 1 x 7 and 7 x 1.
The last tests check that the engine refuses filters its kernels do not compute."""
import zlib

import numpy as np
import pytest

from hyperpose_b200 import models
from tests.test_engine_kernels import (BNS, CONV_KERNELS, HALO0, MEAN, S1, S2, Case, _conv_w, _engine, _expect_rejected, _graph, _r,
                                       _run_and_check, _slopes, conv_case, conv_launches, dw_case, pool_case, stem_case)

gpu = pytest.mark.gpu

NONE = {"HPB_HALO": "none"}   # 3 x 3 shapes the automatic rule would move to the halo kernel stay on conv_wgmma_kernel
ALL = {"HPB_HALO": "all"}
REG = {"HPB_HALO_REG_EPILOGUE": "1"}
NARROW = {"HPB_HALO_NARROW": "1"}
WIDE = "halo<128,wide>"
PP_KERNELS = {"halo<64,pp>", "halo<128,pp>", "halo<64,pool,pp>", "halo<128,pool,pp>"}
ALL_KERNELS = CONV_KERNELS | {WIDE} | PP_KERNELS


def _short(c, max_batch=None):
    """the case on an engine built for one frame more than it runs (or for max_batch)"""
    N = c.shape[0]
    c.max_batch = max_batch or N + 1
    c.id += f"-max{c.max_batch}"
    return c


def _twin(c, env):
    c.twin_env = env
    return c


def split_case(dtype, conf, paf, cin, R, shape, linear=False, max_batch=None, seed=0):
    """the output conv: conf channels [0, conf) and paf channels [conf, conf + paf) into the engine's fp32 NCHW planes"""
    rng = np.random.default_rng(seed)
    chunk = 64 if dtype == "f16" else 32
    g = models.Graph("split", conf_channels=conf, paf_channels=paf, out_down_shift=0, mean=MEAN)
    b_in = g.add_buffer(_r(_r(cin, chunk), 8), 0)
    co = conf + paf
    g.add_conv(b_in, 0, _conv_w(rng, 1, co, cin, R), rng.standard_normal(co).astype(np.float32) * 0.5,
               np.ones(co, np.float32) if linear else _slopes(rng, co), out_mode=models.OUT_F32_NCHW_SPLIT, split=conf)
    bn = {57: 64, 160: 96}[co]
    k = f"conv<{dtype},{bn}>"
    cid = f"{dtype}-{k}-split{conf}+{paf}-cin{cin}-{R}x{R}-{'linear' if linear else 'prelu'}-{'x'.join(map(str, shape))}" + \
          (f"-max{max_batch}" if max_batch else "")
    return Case(cid, dtype, shape, g, [k], [("conf", 0, conf), ("paf", 0, paf)], R * R * _r(cin, chunk), max_batch=max_batch)


# ---- more than one item per CTA (each also one frame short of max_batch) ------------------------------------------------------
def _multi_round():
    cs = []
    # (BN, cout_g, groups, R, shape, out_off): 136 .. 272 items
    plain = [(16, 13, 4, 1, (3, 40, 72), 8), (32, 24, 1, 3, (1, 130, 140), 0), (48, 40, 2, 3, (2, 45, 97), 0),
             (64, 57, 1, 1, (2, 97, 99), 8), (96, 288, 1, 1, (1, 70, 97), 0), (128, 200, 1, 1, (1, 60, 149), 8)]
    res = [(16, 16, 4, 3, (3, 40, 72)), (32, 32, 2, 1, (2, 45, 97)), (48, 48, 1, 3, (1, 130, 140)), (64, 64, 1, 1, (2, 97, 99)),
           (96, 96, 2, 1, (2, 60, 72)), (128, 128, 1, 1, (1, 130, 140))]
    for dt in ("f16", "tf32"):
        cin = 64 if dt == "f16" else 32
        for bn, cout, G, R, shape, out_off in plain:
            cs.append(_short(conv_case(dt, cout, cin, G, R, shape, out_off=out_off, kernel=f"conv<{dt},{bn}>", env=NONE)))
        for i, (bn, cout, G, R, shape) in enumerate(res):
            cs.append(_short(conv_case(dt, cout, cin, G, R, shape, res_mode=1 + i % 2, res_off=(0, 8, 16)[i % 3], out_off=(0, 8)[i % 2],
                                       kernel=f"conv<{dt},{bn},res>", env=NONE)))
    for i, cout in enumerate((13, 24, 40, 57, 72, 128)):
        stride = (1, 2)[i % 2]
        shape3 = (2, 150, 120) if i == 0 else ((1, 130, 140) if stride == 1 else ((2, 180, 194) if cout == 57 else (1, 260, 280)))
        cs.append(_short(stem_case(cout, 3, stride, shape3, out_off=(0, 8)[i % 2])))
        cs.append(_short(stem_case(cout, 7, 2, (2, 300, 240) if i == 0 else (1, 260, 280))))
    # the halo kernel: 16 x 8 tiles, 144 .. 300 items
    for i, (cout, G) in enumerate(((13, 2), (24, 1), (40, 1), (57, 1), (72, 1), (200, 1))):
        bn = {13: 16, 24: 32, 40: 48, 57: 64, 72: 96, 200: 128}[cout]
        shape = (2, 64, 72) if cout == 200 else (3, 64, 96)
        cs.append(_short(_twin(conv_case("f16", cout, 64, G, 3, shape, out_off=(0, 8)[i % 2], kernel=f"halo<{bn}>"), REG)))
    for i, bn in enumerate(BNS):   # max_batch 4: below the ping-pong item's two items per CTA
        cs.append(_short(conv_case("f16", bn, 64, 2 if bn == 16 else 1, 3, (3, 64, 96), out_off=(0, 8)[i % 2], pool=True,
                                   kernel=f"halo<{bn},pool>")))
    cs.append(_short(_twin(conv_case("f16", 128, 64, 6, 3, (3, 46, 82), kernel=WIDE, env=ALL), NARROW)))   # 99 tiles: odd
    cs.append(_short(_twin(conv_case("f16", 64, 64, 3, 3, (3, 46, 82), kernel="halo<64,pp>", env=ALL), NARROW)))
    # the default rule: four chunks / a fused pool, and two items per CTA at max_batch
    cs.append(_short(_twin(conv_case("f16", 128, 256, 1, 3, (5, 46, 82), kernel="halo<128,pp>"), NARROW), max_batch=9))
    cs.append(_short(_twin(conv_case("f16", 64, 64, 1, 3, (2, 128, 144), pool=True, kernel="halo<64,pool,pp>"), NARROW)))
    cs.append(_short(_twin(conv_case("f16", 128, 64, 1, 3, (3, 64, 96), pool=True, out_off=8, kernel="halo<128,pool,pp>"), NARROW), max_batch=6))
    cs += [split_case(dt, 19, 38, 64, 1, (2, 97, 99), max_batch=3) for dt in ("f16", "tf32")]   # the conf / PAF output conv
    return cs


MULTI = _multi_round()


# ---- short batches of every kernel family, on small maps ----------------------------------------------------------------------
def _short_batch():
    cs = []
    for dt in ("f16", "tf32"):
        cs.append(_short(conv_case(dt, 40, 64, 1, 3, S1, kernel=f"conv<{dt},48>", env=NONE), 4))
        cs.append(_short(conv_case(dt, 64, 64, 1, 3, S2, res_mode=1, res_off=8, kernel=f"conv<{dt},64,res>", env=NONE), 5))
    cs.append(_short(stem_case(40, 3, 1, (2, 13, 21)), 3))
    cs.append(_short(stem_case(24, 3, 2, (1, 27, 41), out_off=8), 2))
    cs.append(_short(stem_case(57, 7, 2, (1, 40, 72)), 2))
    cs.append(_short(_twin(conv_case("f16", 40, 64, 1, 3, HALO0, kernel="halo<48>"), REG), 3))
    cs.append(_short(_twin(conv_case("f16", 128, 64, 1, 3, (1, 46, 80), out_off=8, kernel="halo<128>"), REG), 2))
    cs.append(_short(_twin(conv_case("f16", 64, 64, 1, 3, (1, 46, 80), pool=True, kernel="halo<64,pool>"), REG), 3))
    # 33 tiles: the last item's second tile is frame 1's first, inside the max_batch buffer
    cs.append(_short(_twin(conv_case("f16", 128, 64, 1, 3, (1, 46, 82), kernel=WIDE, env=ALL), REG), 2))
    cs.append(_short(_twin(conv_case("f16", 128, 128, 1, 7, (1, 46, 82), kernel=WIDE, env=ALL), REG), 2))
    cs.append(_short(_twin(conv_case("f16", 64, 64, 1, 3, (1, 46, 82), kernel="halo<64,pp>", env=ALL), REG), 3))
    # the ping-pong item chosen for 16 frames (768 items), launched for one
    cs.append(_short(_twin(conv_case("f16", 64, 64, 1, 3, (1, 64, 96), pool=True, kernel="halo<64,pool,pp>"), REG), 16))
    cs += [_short(dw_case("f16", 40, 3, 2, "dw_strip<3,2>"), 3), _short(dw_case("f16", 48, 1, 1, "dw_strip<1,1>"), 3),
           _short(dw_case("f16", 40, 1, 2, "dw_strip<1,2>"), 3), _short(dw_case("f16", 40, 3, 1, "dw_col"), 3),
           _short(dw_case("f16", 64, 3, 1, "dw_tma<1>"), 3), _short(dw_case("f16", 64, 3, 1, "dw_tma<2>", pair=True), 3)]
    cs += [_short(dw_case("tf32", 40, k, s, "dw_f32"), 3) for k, s in ((1, 1), (3, 2))]
    cs += [_short(pool_case("f16", 40, 2, "maxpool<2>"), 3), _short(pool_case("f16", 40, 3, "maxpool<3>"), 3),
           _short(pool_case("tf32", 40, 2, "maxpool_f32"), 3), _short(pool_case("tf32", 24, 3, "maxpool_f32", shape=S2), 4)]
    return cs


SHORT = _short_batch()


# ---- the conf / PAF output conv -----------------------------------------------------------------------------------------------
def _split_cases():
    cs = []
    for dt in ("f16", "tf32"):
        cs += [split_case(dt, 19, 38, 64, 1, S1, max_batch=3),                 # split inside the one BN 64 n-tile
               split_case(dt, 19, 38, 64, 3, S2, linear=True),
               split_case(dt, 100, 60, 64, 1, S1, linear=True, max_batch=4),   # BN 96: the split in the second n-tile
               split_case(dt, 100, 60, 64, 3, S2)]
    return cs


SPLIT = _split_cases()


# ---- filter shapes ------------------------------------------------------------------------------------------------------------
def _filter_cases():
    cs = []
    for dt in ("f16", "tf32"):
        cs.append(conv_case(dt, 40, 64, 1, 5, S1, kernel=f"conv<{dt},48>", env=NONE))
        cs.append(conv_case(dt, 24, 64, 1, 1, S1, S=7, kernel=f"conv<{dt},32>", env=NONE))
        cs.append(conv_case(dt, 24, 64, 1, 7, S2, S=1, kernel=f"conv<{dt},32>", env=NONE))
    cs.append(_twin(conv_case("f16", 40, 64, 1, 5, HALO0, kernel="halo<48>", env=ALL), REG))
    cs.append(_twin(conv_case("f16", 64, 64, 1, 5, (1, 46, 82), pool=True, kernel="halo<64,pool>", env=ALL), REG))
    cs.append(_twin(conv_case("f16", 128, 64, 1, 5, (1, 46, 82), kernel=WIDE, env=ALL), NARROW))
    return cs


FILTERS = _filter_cases()


def _seed(case):
    return np.random.default_rng(zlib.crc32(case.id.encode()))


def _main_launch(case):
    """(op, kernel, items, grid) of the case's conv launch"""
    (launch,) = conv_launches(case)
    return launch


@gpu
@pytest.mark.parametrize("case", MULTI, ids=[c.id for c in MULTI])
def test_multi_round_launch_against_fp64_reference(case, monkeypatch):
    _, kernel, items, grid = _main_launch(case)
    assert items > grid and items % grid, f"{case.id}: {kernel} runs {items} items on {grid} CTAs"
    _run_and_check(case, monkeypatch, _seed(case))


@gpu
@pytest.mark.parametrize("case", SHORT, ids=[c.id for c in SHORT])
def test_short_batch_against_fp64_reference(case, monkeypatch):
    _run_and_check(case, monkeypatch, _seed(case))


@gpu
@pytest.mark.parametrize("case", SPLIT, ids=[c.id for c in SPLIT])
def test_split_output_conv_against_fp64_reference(case, monkeypatch):
    _run_and_check(case, monkeypatch, _seed(case))


@gpu
@pytest.mark.parametrize("case", FILTERS, ids=[c.id for c in FILTERS])
def test_filter_shape_against_fp64_reference(case, monkeypatch):
    _run_and_check(case, monkeypatch, _seed(case))


def _families():
    """kernel family -> the multi-round cases of it"""
    fam = {}
    for c in MULTI:
        k = c.kernels[0] if c.kernels[0] != "none" else c.kernels[1]
        key = k.split("<")[0] + "<" + ",".join(a for a in k[k.index("<") + 1:-1].split(",") if not a.isdigit()) + ">"
        fam.setdefault(key, []).append(c)
    return fam


@gpu
def test_cases_reach_every_conv_kernel_multi_round_and_short(monkeypatch):
    """the engines of the cases above, created but not run: every conv kernel runs in some multi-round case and in some short batch,
    and every kernel family has a case whose busiest CTA takes three or more items of an odd number of k-steps"""
    seen = {"multi-round": set(), "short-batch": set()}
    for case in MULTI + SHORT + SPLIT + FILTERS:
        eng = _engine(case, monkeypatch)
        names = [eng.debug_op_kernel(i) for i in range(len(case.graph.ops))]
        eng.close()
        assert names == case.kernels, (case.id, names)
        conv = {k for k in names if k.startswith(("conv<", "halo<"))}
        if case.max_batch > case.shape[0]:
            seen["short-batch"] |= conv
        if any(items > grid for _, _, items, grid in conv_launches(case)):
            seen["multi-round"] |= conv
    for what, got in seen.items():
        print(f"[kernel inventory] {what}: {len(got & ALL_KERNELS)}/{len(ALL_KERNELS)} conv kernels")
        assert ALL_KERNELS <= got, (what, sorted(ALL_KERNELS - got))
    fams = _families()
    for key, cases in sorted(fams.items()):
        best = [(c.id, items, grid, c.K // (32 if c.dtype == "tf32" else 64)) for c in cases for _, _, items, grid in conv_launches(c)]
        three = [b for b in best if b[1] > 2 * b[2] and b[3] % 2]
        print(f"[kernel inventory] {key}: {len(cases)} multi-round cases; three or more items, odd k-steps: {[b[0] for b in three]}")
        assert three, (key, best)
    assert len(fams) == 11, sorted(fams)


# ---- filters the kernels do not compute ---------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("R,S,cin,cout,G", [(2, 2, 64, 16, 1), (4, 1, 64, 16, 1), (1, 4, 64, 16, 1), (0, 0, 64, 16, 1), (3, 3, 64, 0, 1),
                                            (3, 3, 0, 16, 1), (3, 3, 64, 16, 0)])
def test_conv_filters_the_kernels_do_not_compute_are_rejected(R, S, cin, cout, G):
    """an even filter would be padded R / 2 before the image instead of "SAME"'s (R - 1) / 2; an empty filter or channel range
    leaves the epilogue nothing to store but the accumulators' old contents.  Creating the engine must fail."""
    g = _graph("bad filter")
    a = g.add_buffer(64, 0)
    b = g.add_buffer(16, 0)
    g.add_conv(a, b, np.ones((G, cout, cin, R, S), np.float32), np.zeros(G * cout, np.float32), np.zeros(G * cout, np.float32))
    _expect_rejected(g, "conv op 0")
