"""The halo kernel's ping-pong item (one 16 x 8 tile x one n-tile per consumer warpgroup, the two warpgroups taking turns on the tensor
pipe) against the 128-pixel item (HPB_HALO_NARROW=1) byte for byte, and against the float64 reference of tests/test_engine_kernels.py
within its bound.

The default rule gives the ping-pong item to 3 x 3 layers of BN 64 / 128 with four or more 64-channel chunks or a fused max-pool,
when the launch has at least two items per CTA, so the cases below are sized above that (132 SMs: 264 items); HPB_HALO=all takes it
for BN 64 at any size.  The cases: 64 -> 64 with the 2x2 max-pool fused, on a 94 x 164 map (even, but partial tiles right and
bottom); 64 -> 128 pooled (one chunk); 256 -> 256 at 92 x 164 (four chunks, partial tiles right and bottom); 512 -> 512 at 46 x 82
(eight chunks: the four-slot box ring wraps many times); the grouped 128 -> 128 of init_2, pooled into a concat buffer at channel
offset 8 (330 items: half the CTAs get an odd number); and, forced, a 64 -> 64 launch of 33 items (fewer than SMs, an odd count).
The last test checks the default rule on the benchmark's own graph."""
import zlib

import numpy as np
import pytest

from hyperpose_b200 import capi, models
from tests.test_engine_kernels import _run_and_check, conv_case


def _pp_case(cout, cin, G, shape, env=None, **kw):
    bn = 64 if cout <= 64 else 128
    kernel = f"halo<{bn},pool,pp>" if kw.get("pool") else f"halo<{bn},pp>"
    c = conv_case("f16", cout, cin, G, 3, shape, kernel=kernel, env=env, **kw)
    c.twin_env = {"HPB_HALO_NARROW": "1"}   # the same graph on the 128-pixel item must give the same bytes
    return c


CASES = [
    _pp_case(64, 64, 1, (3, 94, 164), pool=True),               # 378 items, pooled epilogue per m64 block, partial tiles
    _pp_case(128, 64, 1, (8, 64, 80), pool=True),               # one chunk, 320 items
    _pp_case(256, 256, 1, (2, 92, 164)),                        # four chunks, two n-tiles, 504 items
    _pp_case(512, 512, 1, (3, 46, 82)),                         # eight chunks, four n-tiles, 396 items
    _pp_case(128, 128, 2, (5, 46, 82), out_off=8, pool=True),   # grouped (init_2), concat offset; 330 items
    _pp_case(64, 64, 1, (1, 46, 82), env={"HPB_HALO": "all"}),  # 33 items: fewer than SMs, one warpgroup of the last CTA idle
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_pingpong_item_against_narrow_item_and_fp64_reference(case, monkeypatch):
    _run_and_check(case, monkeypatch, np.random.default_rng(zlib.crc32(case.id.encode())))


@pytest.mark.gpu
def test_default_rule_for_the_benchmark_trunk_convs(monkeypatch):
    """OpenPose-VGG19 at 368 x 656, batch 16 (bench.py's cfg3): the 3 x 3 halo layers of 256 or more input channels and those with a
    fused max-pool take the ping-pong item, conv2_1, conv3_1 and init_1 ... init_3 keep the 128-pixel item, and HPB_HALO_NARROW=1 puts
    them all on the 128-pixel item"""
    monkeypatch.delenv("HPB_HALO", raising=False)
    g = models.openpose_vgg19(0)
    trunk = [i for i, o in enumerate(g.ops) if o.type == models.OP_CONV and o.R == 3 and o.name != "conv1_1"]
    assert len(trunk) == 14
    got = {}
    for narrow in (False, True):
        if narrow:
            monkeypatch.setenv("HPB_HALO_NARROW", "1")
        else:
            monkeypatch.delenv("HPB_HALO_NARROW", raising=False)
        eng = capi.Engine(g.to_pack(), (656, 368), max_batch_size=16)
        got[narrow] = {g.ops[i].name: eng.debug_op_kernel(i) for i in trunk}
        eng.close()
    pp = {n for n, k in got[False].items() if k.endswith(",pp>")}
    assert pp == {"conv1_2", "conv2_2", "conv3_2", "conv3_3", "conv3_4", "conv4_1", "conv4_2", "cpm_1", "cpm_2"}, got[False]
    assert {n for n, k in got[False].items() if ",pool" in k} == {"conv1_2", "conv2_2", "conv3_4"}, got[False]
    assert got[True] == {n: k.replace(",pp>", ">") for n, k in got[False].items()}
