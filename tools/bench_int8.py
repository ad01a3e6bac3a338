"""fp16 vs INT8 engine on bench.py's workloads (cfg3, cfg4, cfg2: shapes and batches as bench.py), on the device-resident CUDA-graph
pose path (hp_pose_submit_u8_device / hp_pose_collect, two batches in flight) with synthetic crowd tensors over the network outputs,
as bench.py does.  The INT8 scales come from a TF32-engine calibration on one batch of frames of another seed.

Per workload the two engines alternate in one process, three rounds each, every round after >= 2 s of the same steps.  Reported:
frames/s, conv kernel ms per step (the engine's per-op CUDA-event profile, direct launches), algorithmic TOPS over the 1,979 TOPS
dense INT8 figure of the H100 SXM data sheet, and the card name and power limit (nvidia-smi, read only).

    python tools/bench_int8.py [--steps 30] [--workloads cfg3,cfg4,cfg2]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hyperpose_b200 import capi, models, synthetic as syn  # noqa: E402

WORKLOADS = {   # bench.py's WORKLOADS: graph, input size, batch, GFLOP per frame
    "cfg3": ("openpose_vgg19", 368, 656, 16, 484.6e9),
    "cfg2": ("mobilenet_thin_openpose", 368, 432, 8, 22.3e9),
    "cfg4": ("resnet50_lw_openpose", 368, 432, 32, 136.7e9),
}
DATASHEET_INT8_TOPS = 1979.0   # H100 SXM data sheet, dense INT8


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=20)
        return q.stdout.strip()
    except Exception:
        return torch.cuda.get_device_name(0)


def setup(graph_name, H, W, B):
    g = getattr(models, graph_name)(0)
    cal = capi.Engine(g.to_pack(), (W, H), max_batch_size=B, dtype="tf32")
    g.set_int8_scales(cal.calibrate(syn.make_frames_u8(500, B, H, W)))
    cal.close()
    pack = g.to_pack()
    engines = {dt: capi.Engine(pack, (W, H), max_batch_size=B, dtype=dt) for dt in ("f16", "int8")}
    e = engines["f16"]
    conf, paf = syn.make_batch_tensors(1000, B, (10, 20), e.out_h, e.out_w)
    d_conf, d_paf = torch.from_numpy(np.ascontiguousarray(conf)).cuda(), torch.from_numpy(np.ascontiguousarray(paf)).cuda()
    frames = [torch.from_numpy(syn.make_frames_u8(2 + i, B, H, W)).cuda() for i in range(6)]
    parsers = {}
    for dt, eng in engines.items():
        eng.set_output_override(d_conf.data_ptr(), d_paf.data_ptr())
        p = capi.PafParser(0.05, 0.05)
        p.set_capacity(peaks_per_part=128, candidates_per_limb=2048, humans=128)
        parsers[dt] = p
    return g, engines, parsers, frames, (d_conf, d_paf)


def run_steps(eng, parser, frames, B, n):
    pend = None
    for i in range(n):
        t = eng.submit_pose_device(parser, frames[i % len(frames)].data_ptr(), B)
        if pend is not None:
            eng.collect_pose(pend, cap=128)
        pend = t
    eng.collect_pose(pend, cap=128)


def timed(eng, parser, frames, B, steps):
    t_end = time.perf_counter() + 2.0
    while time.perf_counter() < t_end:   # >= 2 s preload
        run_steps(eng, parser, frames, B, 5)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    run_steps(eng, parser, frames, B, steps)
    torch.cuda.synchronize()
    return B * steps / (time.perf_counter() - t0)


def conv_ms(g, eng, frames, B):
    st = eng.device_outputs()[2]
    for i in range(5):
        eng.infer_u8_device(frames[i % len(frames)].data_ptr(), B, st)
    eng.sync()
    eng.set_profiling(True)
    for i in range(20):
        eng.infer_u8_device(frames[i % len(frames)].data_ptr(), B, st)
    eng.sync()
    ms, ty, _, _ = eng.get_profile()
    eng.set_profiling(False)
    return float(ms[ty == models.OP_CONV].sum()), float(ms.sum()), {op.name: round(float(m), 4) for op, m in zip(g.ops, ms)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--workloads", default="cfg3,cfg4,cfg2")
    ap.add_argument("--layers", action="store_true", help="also print per-op ms of both engines")
    a = ap.parse_args()
    print(json.dumps({"card": card()}))
    for wl in a.workloads.split(","):
        name, H, W, B, flops = WORKLOADS[wl]
        g, engines, parsers, frames, _keep = setup(name, H, W, B)
        fps = {dt: [] for dt in engines}
        for _ in range(3):
            for dt in ("f16", "int8"):
                fps[dt].append(round(timed(engines[dt], parsers[dt], frames, B, a.steps), 1))
        res = {"workload": wl, "batch": B, "fps": fps}
        for dt, eng in engines.items():
            c, tot, per = conv_ms(g, eng, frames, B)
            res[f"{dt}_conv_ms_per_step"] = round(c, 3)
            res[f"{dt}_engine_ms_per_step"] = round(tot, 3)
            res[f"{dt}_conv_tops"] = round(flops * B / (c * 1e-3) / 1e12, 1)
            if a.layers:
                res[f"{dt}_layers"] = per
        res["int8_conv_tops_over_datasheet"] = round(res["int8_conv_tops"] / DATASHEET_INT8_TOPS, 3)
        print(json.dumps(res))
        for e in engines.values():
            e.close()
        for p in parsers.values():
            p.close()
    print(json.dumps({"card": card()}))


if __name__ == "__main__":
    main()
