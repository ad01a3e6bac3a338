"""The im2col conv kernel's TMA-store epilogue (the fp16 m64 block staged in shared memory, then one TMA box per 64-channel slice)
against the register epilogue (HPB_CONV_REG_EPILOGUE=1: per-thread global stores) byte for byte, and against the float64 reference of
tests/test_engine_kernels.py within its bound; every case also asserts which epilogue the engine runs (Engine.debug_op_conv_epilogue).

The cases cover BN 64 and 128, 1x1 and 3x3, a grouped 1x1 layer into a concat channel offset, a 200-channel layer whose second n-tile
holds 72 real channels (the channels past them must keep their bits, check (b) of _run_and_check), residual modes 1 and 2, pixel
counts that leave a partial last tile, and batches below max_batch (check (b'): frames past N keep every byte).  The fused u8 stem and
the fused 1x1 depthwise stage (post_w) are compared with the register epilogue separately.  The 57-channel concat writes of the
OpenPose heads keep the register epilogue: the TMA store clips a box only in 16-byte units of channels."""
import zlib

import numpy as np
import pytest

from bench import WORKLOADS
from hyperpose_b200 import capi, models
from tests.test_engine_kernels import S1, S3, _buf_shape, _conv_w, _engine, _graph, _run_and_check, _slopes, conv_case, stem_case

REG = {"HPB_CONV_REG_EPILOGUE": "1"}


def _case(kernel, cout, cin, G, R, shape, **kw):
    c = conv_case("f16", cout, cin, G, R, shape, kernel=kernel, **kw)
    c.twin_env = REG   # the register epilogue must give the same bytes
    return c


CASES = [
    _case("conv<f16,64>", 64, 64, 1, 3, S1),                                        # 546 pixels: a partial last tile
    _case("conv<f16,64>", 64, 128, 1, 1, (3, 20, 24)),                              # 1x1, 1440 pixels
    _case("conv<f16,128>", 128, 128, 2, 1, (2, 20, 30), out_off=8),                  # grouped 1x1 (init_4, ref*_6), concat offset
    _case("conv<f16,128>", 128, 128, 2, 1, (2, 16, 16), max_batch=4),                # whole tiles, batch below max_batch
    _case("conv<f16,128>", 128, 64, 1, 1, S1, max_batch=3),                         # partial last tile, batch below max_batch
    _case("conv<f16,128>", 200, 64, 1, 1, S3, out_off=8),                           # n-tiles of 128 + 72 real channels
    _case("conv<f16,128,res>", 128, 64, 1, 1, S3, res_mode=1, res_off=8, out_off=8),
    _case("conv<f16,64,res>", 64, 64, 1, 3, S1, res_mode=2, res_off=16),
    _case("conv<f16,64,res>", 64, 64, 1, 1, (2, 16, 16), res_mode=1, max_batch=3),
]

FALLBACK = [
    _case("conv<f16,64>", 57, 256, 1, 1, S3, out_off=128),   # the heads' 57 channels into the concat buffer: a ragged 16-byte unit
    _case("conv<f16,64>", 64, 64, 1, 1, S1, out_off=4),      # channel offset 4: not 16-byte aligned
    _case("conv<f16,96>", 96, 64, 1, 1, S1),                 # no TMA form at BN 96
]


def _clear_env(monkeypatch):
    monkeypatch.delenv("HPB_CONV_REG_EPILOGUE", raising=False)


def _epilogues(case, monkeypatch, env=None):
    eng = _engine(case, monkeypatch, env)
    try:
        return [eng.debug_op_conv_epilogue(i) for i in range(len(case.graph.ops))]
    finally:
        eng.close()


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


@pytest.mark.gpu
@pytest.mark.parametrize("cout,R,stride,shape,max_batch", [(64, 3, 1, (2, 13, 21), 3), (128, 3, 2, (2, 27, 41), None), (64, 7, 2, (1, 40, 72), None)])
def test_fused_stem_tma_epilogue(cout, R, stride, shape, max_batch, monkeypatch):
    """the fused u8 stem (conv1_1 of cfg3): within the fp64 bound, and the same bytes as the register epilogue from u8 frames"""
    _clear_env(monkeypatch)
    case = stem_case(cout, R, stride, shape, max_batch=max_batch)
    _run_and_check(case, monkeypatch, np.random.default_rng(zlib.crc32(case.id.encode())))
    assert _epilogues(case, monkeypatch)[1] == "tma"
    N, H, W = shape
    frames = np.random.default_rng(3).integers(0, 256, (N, H, W, 3), dtype=np.uint8)
    out_buf = case.outs[0][0]
    got = []
    for env in (None, REG):
        _clear_env(monkeypatch)
        eng = _engine(case, monkeypatch, env)
        eng.debug_write_buffer(out_buf, np.full(_buf_shape(case, out_buf), 7.0, np.float16))
        eng.infer_u8(frames)
        got.append(eng.debug_read_buffer(out_buf, case.max_batch))
        eng.close()
    assert got[0].tobytes() == got[1].tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("cout", [64, 128])
def test_fused_pointwise_depthwise_through_the_tma_store(cout, monkeypatch):
    """a conv followed by a 1x1 depthwise op (post_w in the epilogue) into a channel offset: the TMA store gives the bytes of the
    register epilogue and of the two separate launches"""
    rng = np.random.default_rng(11)
    g = _graph("conv+dw1")
    a, b, c = g.add_buffer(64, 0), g.add_buffer(cout, 0), g.add_buffer(cout + 16, 0)
    g.add_conv(a, b, _conv_w(rng, 1, cout, 64, 1), rng.standard_normal(cout).astype(np.float32), _slopes(rng, cout))
    g.add_dwconv(b, c, rng.standard_normal((cout, 1, 1)).astype(np.float32), rng.standard_normal(cout).astype(np.float32), _slopes(rng, cout),
                 out_ch_off=8)
    N, H, W = S3
    x = rng.standard_normal((N, H, W, 64)).astype(np.float16)
    outs = []
    for env, want in (({}, "tma"), (REG, "reg"), ({"HPB_NO_DW1_FUSE": "1"}, "tma")):
        _clear_env(monkeypatch)
        monkeypatch.delenv("HPB_NO_DW1_FUSE", raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=N)
        assert eng.debug_op_kernel(1) == ("dw_strip<1,1>" if "HPB_NO_DW1_FUSE" in env else "none")
        assert eng.debug_op_conv_epilogue(0) == want
        eng.debug_write_buffer(a, x)
        eng.debug_write_buffer(c, np.full((N, H, W, cout + 16), 7.0, np.float16))
        eng.debug_run_ops(0, 1, N)
        outs.append(eng.debug_read_buffer(c, N))
        eng.close()
    assert outs[0].tobytes() == outs[1].tobytes() == outs[2].tobytes()
    assert (outs[0][..., :8] == 7.0).all() and (outs[0][..., 8 + cout:] == 7.0).all() and np.abs(outs[0][..., 8:8 + cout]).max() > 0


def _want_tma(g, kern, i):
    """does op i take the TMA store by engine.cu's rule (set_conv_tma_store)?  An fp16 im2col-kernel op at BN 64 / 128 with an NHWC
    output whose channel offset, channel count and row stride are multiples of 8, and whose groups are whole n-tiles.  A fused 1x1
    depthwise op (kernel "none" after the conv) moves the output to its own."""
    op = g.ops[i]
    if not kern[i].startswith(("conv<f16,64", "conv<f16,128")) or op.out_mode != models.OUT_F16_NHWC:
        return False
    bn = int(kern[i].split(",")[1].rstrip(">"))
    out = g.ops[i + 1] if i + 1 < len(g.ops) and g.ops[i + 1].type == models.OP_DWCONV and kern[i + 1] == "none" else op
    return (out.out_ch_off % 8 == 0 and g.buffers[out.out_buf][0] % 8 == 0 and (op.groups * op.cout_g) % 8 == 0 and
            (op.groups == 1 or op.cout_g % bn == 0))


@pytest.mark.gpu
@pytest.mark.parametrize("workload", ["cfg2", "cfg3", "cfg4", "cfg5"])
def test_every_eligible_benchmark_conv_takes_the_tma_store(workload, monkeypatch):
    """bench.py's graphs at their benchmark sizes: every im2col-kernel op the TMA store can address runs it, every other op the
    register epilogue (cfg3: conv1_1, init_4 and ref1_6 .. ref5_6 take it; the 57-channel head convs do not)"""
    _clear_env(monkeypatch)
    wl = WORKLOADS[workload]
    g = getattr(models, wl["graph"])(seed=0)
    eng = capi.Engine(g.to_pack(), (wl["in_w"], wl["in_h"]), max_batch_size=wl["batch"])
    try:
        kern = [eng.debug_op_kernel(i) for i in range(len(g.ops))]
        epi = {g.ops[i].name: eng.debug_op_conv_epilogue(i) for i in range(len(g.ops))}
    finally:
        eng.close()
    want = {op.name: "tma" if _want_tma(g, kern, i) else "reg" for i, op in enumerate(g.ops)}
    assert epi == want, {n: (epi[n], want[n]) for n in epi if epi[n] != want[n]}
    assert "tma" in epi.values()
    if workload == "cfg3":
        assert {n for n, v in epi.items() if v == "tma"} == {"conv1_1", "init_4"} | {f"ref{s}_6" for s in range(1, 6)}, epi


@pytest.mark.gpu
def test_tf32_engine_keeps_the_register_epilogue(monkeypatch):
    _clear_env(monkeypatch)
    case = conv_case("tf32", 128, 64, 1, 1, S1, kernel="conv<tf32,128>")
    assert _epilogues(case, monkeypatch)[0] == "reg"
