"""Which conv kernel the engine's default rule picks for the layer shapes of the benchmarked networks, each case checked against the
float64 reference of tests/test_engine_kernels.py: layers of two or more 64-channel chunks at the 46 x 82 map of OpenPose's refinement
stages go to the halo-box kernel (several rounds of CTAs, the ragged 2-column right and 14-row bottom tiles), a one-chunk 3x3 layer and a layer whose 16 x 8 tile grid
wastes most of a 25 x 25 map stay on the im2col kernel."""
import zlib

import numpy as np
import pytest

from tests.test_engine_kernels import _run_and_check, conv_case

REF = (3, 46, 82)   # 3 frames of the refinement stages' map: 89 128-pixel tiles per n-tile / group, more than one round of CTAs

CASES = [
    conv_case("f16", 128, 128, 2, 7, REF, kernel="halo<128>"),                        # two groups of 128 -> 128
    conv_case("f16", 256, 185, 1, 3, REF, pad_value=True, kernel="halo<128>"),        # 185 of 192 channels (3 chunks), two n-tiles
    conv_case("f16", 64, 64, 1, 3, (8, 46, 54), kernel="conv<f16,64>"),               # one chunk
    conv_case("f16", 128, 128, 1, 3, (32, 25, 25), kernel="conv<f16,128>"),           # the 16 x 8 grid wastes 64 % of the map
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_default_rule_kernel_against_fp64_reference(case, monkeypatch):
    _run_and_check(case, monkeypatch, np.random.default_rng(zlib.crc32(case.id.encode())))
