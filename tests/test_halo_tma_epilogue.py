"""The halo kernel's TMA-store epilogue (the fp16 tile staged in shared memory, then one TMA box per 64-channel slice) against the
register epilogue (HPB_HALO_REG_EPILOGUE=1: per-thread global stores) byte for byte, and against the float64 reference of
tests/test_engine_kernels.py within its bound; every case also asserts which epilogue each engine runs (Engine.debug_op_epilogue).

The cases cover each work item with and without the fused 2x2 max-pool: the 128-pixel item (HPB_HALO_NARROW=1), the wide item
(HPB_HALO=all: 7 x 7 and 3 x 3), and the ping-pong item at BN 64 and 128 (the default rule, or HPB_HALO=all below its size
threshold).  The maps leave partial tiles at the right and bottom edges (46 x 82: tiles of 14 rows and 2 columns; pooled 23 x 41),
the outputs go to a concat channel offset, a grouped layer writes two groups, the 200-channel layer's second n-tile holds 72 real
channels (the channels past them must keep their bits, check (b) of _run_and_check), and one frame / 99 tiles give the wide item an
odd tile count.  Plans the TMA store cannot express keep the register epilogue: a grouped layer whose groups are not whole
n-tiles, an output channel offset that is not a multiple of 8, and a channel count that is not.  The last tests check that every
halo layer of the benchmark's graphs and of the Lightweight-OpenPose TinyVGG / ResNet-18 graphs takes the TMA store."""
import zlib

import numpy as np
import pytest

from bench import WORKLOADS
from hyperpose_b200 import capi, models
from tests.test_engine_kernels import HALO0, HALO_RAGGED, _engine, _run_and_check, conv_case

REG = {"HPB_HALO_REG_EPILOGUE": "1"}
ALL = {"HPB_HALO": "all"}
NARROW = {"HPB_HALO_NARROW": "1", **ALL}   # every eligible shape on the halo kernel, all of it on the 128-pixel item
WIDE = "halo<128,wide>"


def _case(kernel, cout, cin, G, R, shape, env=None, **kw):
    c = conv_case("f16", cout, cin, G, R, shape, kernel=kernel, env=env, **kw)
    c.twin_env = REG   # the register epilogue must give the same bytes
    return c


CASES = [
    _case("halo<128>", 128, 128, 1, 3, (2, 46, 82), env=NARROW),                          # partial tiles right and bottom
    _case("halo<64,pool>", 64, 64, 1, 3, (3, 46, 82), env=NARROW, pool=True),             # pooled 23 x 41: partial pooled boxes
    _case("halo<128,pool>", 128, 64, 1, 3, (1, 36, 52), env=NARROW, pool=True, out_off=8),   # batch 1, concat offset
    _case("halo<128>", 200, 64, 1, 3, (1, 46, 80), out_off=8),                            # n-tiles of 128 + 72 real channels
    _case(WIDE, 128, 128, 1, 7, (3, 46, 82), env=ALL, out_off=8),                         # 99 tiles: odd count, pairs across frames
    _case(WIDE, 128, 128, 2, 7, (1, 46, 82), env=ALL),                                    # batch 1, two groups, odd tile count
    _case(WIDE, 200, 128, 1, 3, (2, 37, 45), env=ALL),                                    # 3 x 3, partial n-tile, 5-pixel edge tiles
    _case("halo<64,pool,pp>", 64, 64, 1, 3, (3, 94, 164), pool=True),                     # 378 items
    _case("halo<128,pool,pp>", 128, 128, 2, 3, (5, 46, 82), out_off=8, pool=True),        # grouped (init_2), concat offset
    _case("halo<128,pp>", 256, 256, 1, 3, (2, 92, 164)),                                  # four chunks, two n-tiles, 16 KiB staging slot
    _case("halo<64,pp>", 64, 64, 1, 3, (1, 46, 82), env=ALL),                             # 33 items, two staging slots per warpgroup
]

FALLBACK = [
    conv_case("f16", 40, 64, 2, 3, HALO0, kernel="halo<48>"),                  # groups of 40 channels in n-tiles of 48
    conv_case("f16", 64, 64, 1, 3, HALO0, out_off=4, kernel="halo<64>"),       # channel offset 4: not 16-byte aligned
    conv_case("f16", 57, 64, 1, 3, HALO_RAGGED, in_off=64, out_off=8, kernel="halo<64>"),   # 57 channels: a ragged 16-byte unit
]
for _c in FALLBACK:
    _c.twin_env = REG


def _epilogues(case, monkeypatch, env=None):
    eng = _engine(case, monkeypatch, env)
    try:
        return [eng.debug_op_epilogue(i) for i in range(len(case.graph.ops))]
    finally:
        eng.close()


def _clear_env(monkeypatch):
    for k in ("HPB_HALO_REG_EPILOGUE", "HPB_HALO_NARROW"):
        monkeypatch.delenv(k, raising=False)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_tma_epilogue_against_register_epilogue_and_fp64_reference(case, monkeypatch):
    _clear_env(monkeypatch)
    _run_and_check(case, monkeypatch, np.random.default_rng(zlib.crc32(case.id.encode())))
    _clear_env(monkeypatch)
    assert _epilogues(case, monkeypatch)[0] == "tma"
    assert _epilogues(case, monkeypatch, REG)[0] == "reg"


@pytest.mark.gpu
@pytest.mark.parametrize("case", FALLBACK, ids=[c.id for c in FALLBACK])
def test_plans_the_tma_store_cannot_express_keep_the_register_epilogue(case, monkeypatch):
    _clear_env(monkeypatch)
    _run_and_check(case, monkeypatch, np.random.default_rng(zlib.crc32(case.id.encode())))
    _clear_env(monkeypatch)
    assert _epilogues(case, monkeypatch)[0] == "reg"


def _halo_epilogues(graph, H, W, B, monkeypatch):
    """-> ({halo op name: epilogue}, {epilogues of the other ops}) of `graph` at H x W, batch B"""
    _clear_env(monkeypatch)
    monkeypatch.delenv("HPB_HALO", raising=False)
    g = getattr(models, graph)(seed=0)
    eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=B)
    try:
        halo = {g.ops[i].name: eng.debug_op_epilogue(i) for i in range(len(g.ops)) if eng.debug_op_kernel(i).startswith("halo<")}
        other = {eng.debug_op_epilogue(i) for i in range(len(g.ops)) if not eng.debug_op_kernel(i).startswith("halo<")}
    finally:
        eng.close()
    return g, halo, other


@pytest.mark.gpu
@pytest.mark.parametrize("workload", ["cfg2", "cfg3", "cfg4", "cfg5"])
def test_every_benchmark_halo_layer_takes_the_tma_store(workload, monkeypatch):
    """bench.py's graphs at their benchmark sizes: every op on the halo kernel runs the TMA-store epilogue (cfg3: all 3 x 3 trunk,
    cpm and init layers and the 25 wide-item 7 x 7 refinement convs)"""
    wl = WORKLOADS[workload]
    g, halo, other = _halo_epilogues(wl["graph"], wl["in_h"], wl["in_w"], wl["batch"], monkeypatch)
    assert other <= {"reg"}
    assert all(v == "tma" for v in halo.values()), halo
    if workload == "cfg3":
        trunk = {o.name for o in g.ops if o.type == models.OP_CONV and o.R == 3 and o.name != "conv1_1"}
        assert len(trunk) == 14 and trunk <= set(halo), sorted(halo)
        assert sum(1 for n in halo if n.startswith("ref")) == 25, sorted(halo)


@pytest.mark.gpu
@pytest.mark.parametrize("graph,H,W", [("lw_openpose_vggtiny", 256, 384), ("lw_openpose_resnet18", 368, 432)])
def test_every_lightweight_openpose_halo_layer_takes_the_tma_store(graph, H, W, monkeypatch):
    """TinyVGG's 200-channel layers (n-tiles of 128 + 72 into 256-channel buffers) included"""
    _, halo, other = _halo_epilogues(graph, H, W, 16, monkeypatch)
    assert other <= {"reg"} and halo
    assert all(v == "tma" for v in halo.values()), halo
