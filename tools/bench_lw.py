"""Lightweight-OpenPose throughput on TinyVGG, ResNet-18 and MobilenetDilated: lw_openpose_vggtiny at 256 x 384 (the reference's
published size) and 342 x 368 (the model zoo's TinyVGG-V2-HW=342x368), lw_openpose_resnet18 and lw_openpose_mobilenet_dilated (the
published "LightweightOpenPose (Dilated MobileNet)") at 368 x 432; fp16 engine, batch 16.

The path is device-resident and pipelined: u8 frames already in HBM -> hp_pose_submit_u8_device / hp_pose_collect (CUDA-graph replay
of convs + PAF parse + record copy, two batches in flight).  Random weights give structureless maps, so synthetic crowd tensors
(4-8 people per frame) are copied over the outputs through the output override, as bench.py does: the parser does real work.

One JSON line per workload: frames/s of three rounds (CUDA events around `--steps` steps after a >= 2 s warm-up; the workloads
alternate inside a round), conv ms per step (the engine's per-op CUDA-event profile, a separate run), the algorithmic GFLOP per
frame from the graph, and the card, its power limit and the SM clock read by nvidia-smi right after the timed rounds.
--per-op adds every op's kernel (Engine.debug_op_kernel) and its time per step.  The MobilenetDilated line also carries the time of its
dilated depthwise layer next to the same layer run undilated (the same graph with dilation 1, profiled on its own engine).

    python tools/bench_lw.py [--steps 50] [--per-op]"""
import argparse
import copy
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hyperpose_b200 import capi, models, synthetic as syn  # noqa: E402

B = 16
HCAP = 64
WORKLOADS = [("lw_vggtiny", "lw_openpose_vggtiny", 256, 384), ("lw_vggtiny", "lw_openpose_vggtiny", 342, 368),
             ("lw_resnet18", "lw_openpose_resnet18", 368, 432), ("lw_mobilenet_dilated", "lw_openpose_mobilenet_dilated", 368, 432)]


def smi():
    """card name, power limit (W), SM clock and its maximum (MHz), read only"""
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True, timeout=20)
    name, plim, sm, smax = [x.strip() for x in q.stdout.strip().split(",")]
    return {"card": name, "power_limit_w": float(plim), "sm_mhz": float(sm), "sm_max_mhz": float(smax)}


class Workload:
    def __init__(self, label, net, H, W, seed, graph=None):
        self.label, self.H, self.W = label, H, W
        self.g = graph if graph is not None else getattr(models, net)(0)
        self.eng = capi.Engine(self.g.to_pack(), (W, H), max_batch_size=B)
        self.parser = capi.PafParser(0.05, 0.05)
        self.parser.set_capacity(peaks_per_part=128, candidates_per_limb=2048, humans=HCAP)
        conf, paf = syn.make_batch_tensors(seed, B, (4, 8), self.eng.out_h, self.eng.out_w)
        self.d_conf, self.d_paf = torch.from_numpy(conf).cuda(), torch.from_numpy(paf).cuda()
        torch.cuda.synchronize()
        self.eng.set_output_override(self.d_conf.data_ptr(), self.d_paf.data_ptr())
        self.frames = [torch.from_numpy(syn.make_frames_u8(seed + i, B, H, W)).cuda() for i in range(4)]
        self.st = torch.cuda.ExternalStream(self.eng.device_outputs()[2])
        self.pending = None

    def step(self, i):
        t = self.eng.submit_pose_device(self.parser, self.frames[i % len(self.frames)].data_ptr(), B)
        if self.pending is not None:
            self.eng.collect_pose(self.pending, cap=HCAP)
        self.pending = t

    def drain(self):
        h = self.eng.collect_pose(self.pending, cap=HCAP) if self.pending is not None else None
        self.pending = None
        return h

    def timed(self, steps):
        t_end, i = time.perf_counter() + 2.0, 0
        while time.perf_counter() < t_end:
            self.step(i); i += 1
        self.drain()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(self.st)
        for i in range(steps):
            self.step(i)
        self.drain()
        b.record(self.st)
        torch.cuda.synchronize()
        return B * steps / (a.elapsed_time(b) * 1e-3)

    def profile(self):
        eng = self.eng
        for i in range(5):
            eng.infer_u8_device(self.frames[i % 4].data_ptr(), B, self.st.cuda_stream)
        eng.sync()
        eng.set_profiling(True)
        for i in range(20):
            eng.infer_u8_device(self.frames[i % 4].data_ptr(), B, self.st.cuda_stream)
        eng.sync()
        ms, ty, _, _ = eng.get_profile()
        eng.set_profiling(False)
        return ms, ty

    def close(self):
        self.eng.close()
        self.parser.close()


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--per-op", action="store_true", help="every op's kernel and time per step")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_lw measures on the GPU: no CUDA device")
    wls = [Workload(label, net, H, W, 500 + 10 * k) for k, (label, net, H, W) in enumerate(WORKLOADS)]
    humans = []
    for w in wls:
        w.step(0)
        humans.append([len(h) for h in w.drain()])
    fps = [[] for _ in wls]
    for _ in range(3):
        for k, w in enumerate(wls):
            fps[k].append(round(w.timed(a.steps), 1))
    clocks = smi()
    for k, w in enumerate(wls):
        ms, ty = w.profile()
        res = {"workload": w.label, "input": [w.H, w.W], "output": [w.eng.out_h, w.eng.out_w], "batch": B, "dtype": "f16",
               "api": "hp_pose_submit_u8_device / hp_pose_collect (device-resident frames, two batches in flight)",
               "fps": fps[k], "fps_median": float(np.median(fps[k])), "humans_per_frame": [min(humans[k]), max(humans[k])],
               "conv_ms_per_step": round(float(ms[ty == models.OP_CONV].sum()), 3), "engine_ms_per_step": round(float(ms.sum()), 3),
               "gflop_per_frame": round(w.g.flops_per_frame(w.H, w.W) / 1e9, 2), **clocks}
        dilated = [i for i, op in enumerate(w.g.ops) if op.dilation != 1]
        if dilated:
            plain = copy.deepcopy(w.g)
            for op in plain.ops:
                op.weight, op.dilation = op.taps(), 1
            pw = Workload(w.label, None, w.H, w.W, 900, graph=plain)
            pms, _ = pw.profile()
            res["dilated_layers"] = [{"op": w.g.ops[i].name, "kernel": w.eng.debug_op_kernel(i), "ms": round(float(ms[i]), 4),
                                      "undilated_kernel": pw.eng.debug_op_kernel(i), "undilated_ms": round(float(pms[i]), 4)} for i in dilated]
            pw.close()
        if a.per_op:
            res["per_op"] = [{"op": op.name, "kernel": w.eng.debug_op_kernel(i), "ms": round(float(ms[i]), 4)} for i, op in enumerate(w.g.ops)]
        print(json.dumps(res))
    for w in wls:
        w.close()


if __name__ == "__main__":
    main()
