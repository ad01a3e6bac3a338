"""The halo kernel's wide work item (two 16 x 8 tiles x one 128-channel n-tile, every weight tile shared by both tiles) against the
128-pixel item (HPB_HALO_NARROW=1) byte for byte, and against the float64 reference of tests/test_engine_kernels.py within its bound.

HPB_HALO=all takes the wide item wherever it exists, so these shapes run it whatever the default rule picks at their batch size:
OpenPose's refinement map 46 x 82 (33 tiles per frame; the right column of tiles is 2 pixels wide, the bottom row 14 high) with
7 x 7 filters in two groups of 128 and with 185 of 192 input channels into 256 outputs (two n-tiles); one frame (fewer items than
SMs, an odd tile count); three frames (99 tiles: the last item has one tile, and pairs straddle frames); and a 3 x 3 layer on a map
whose partial tiles are 5 pixels wide and 5 high.  The last test checks the default rule on the benchmark's own graph."""
import zlib

import numpy as np
import pytest

from hyperpose_b200 import capi, models
from tests import test_engine_kernels
from tests.test_engine_kernels import _run_and_check, conv_case

WIDE = "halo<128,wide>"


def _wide_case(cout, cin, G, R, shape, mutants=True, **kw):
    c = conv_case("f16", cout, cin, G, R, shape, kernel=WIDE, env={"HPB_HALO": "all"}, **kw)
    c.twin_env = {"HPB_HALO_NARROW": "1"}   # the same graph on the 128-pixel item must give the same bytes
    c.mutants = mutants
    return c


CASES = [
    _wide_case(128, 128, 2, 7, (2, 46, 82)),                    # two groups of 128 -> 128, 66 tiles
    # 185 of 192 channels (3 chunks), two n-tiles.  With 9408 products per output, one zeroed tap of 49 moves most outputs by less
    # than the bound, so this case skips the wrong-reference check; the byte comparison with the 128-pixel item still applies
    _wide_case(256, 185, 1, 7, (2, 46, 82), mutants=False, pad_value=True),
    _wide_case(128, 128, 2, 7, (1, 46, 82)),                    # batch 1: 17 items per group, the last with one tile
    _wide_case(128, 128, 1, 7, (3, 46, 82), out_off=8),         # 99 tiles: odd count, pairs across frames
    _wide_case(200, 128, 1, 3, (2, 37, 45)),                    # 3 x 3, partial n-tile, 5-pixel partial tiles right and bottom
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_wide_item_against_narrow_item_and_fp64_reference(case, monkeypatch):
    if not case.mutants:
        monkeypatch.setattr(test_engine_kernels, "_mutants", lambda case: [])
    _run_and_check(case, monkeypatch, np.random.default_rng(zlib.crc32(case.id.encode())))


@pytest.mark.gpu
def test_default_rule_for_the_benchmark_refinement_convs(monkeypatch):
    """OpenPose-VGG19 at 368 x 656, batch 16 (bench.py's cfg3): every 7 x 7 refinement conv takes the wide item, and
    HPB_HALO_NARROW=1 puts them all back on the 128-pixel item"""
    monkeypatch.delenv("HPB_HALO", raising=False)
    g = models.openpose_vgg19(0)
    ref7 = [i for i, o in enumerate(g.ops) if o.name.startswith("ref") and o.R == 7]
    assert len(ref7) == 25
    for narrow, want in ((False, WIDE), (True, "halo<128>")):
        if narrow:
            monkeypatch.setenv("HPB_HALO_NARROW", "1")
        else:
            monkeypatch.delenv("HPB_HALO_NARROW", raising=False)
        eng = capi.Engine(g.to_pack(), (656, 368), max_batch_size=16)
        got = {g.ops[i].name: eng.debug_op_kernel(i) for i in ref7}
        eng.close()
        assert got == {g.ops[i].name: want for i in ref7}
