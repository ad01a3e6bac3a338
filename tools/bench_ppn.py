"""Pose Proposal Network throughput: ppn_resnet18 and ppn_resnet50 at 384 x 384, batch 16, f16 and TF32 engines.

Three paths over the same crowd override, each timed per network and precision:
  * two_call: u8 frames already in HBM -> hp_engine_infer_u8_device -> hp_ppn_process_device_strided on the engine's two output slots
    (no copy) -> hp_ppn_fetch, all on the engine's stream; one batch at a time (hp_ppn_fetch synchronises the device);
  * pipelined_device: the same frames through hp_pose_submit_ppn_u8_device / hp_pose_collect, two tickets in flight (network, parse
    and record D2H replayed from one CUDA graph per ticket);
  * pipelined_frames_1280x720: page-locked 1280 x 720 host frames through hp_pose_submit_ppn_frames_u8_host / hp_pose_collect (H2D on
    the copy stream, one batched resize to 384 x 384 on the GPU), two tickets in flight.
Random weights give structureless maps, so synthetic crowd tensors (synthetic.make_ppn_tensors, 4-8 people per frame) are copied over
the outputs through the output override, as bench.py does for the PAF workloads: the parser does real work.  The first batch of each
pipelined path is checked against the two-call path's records.

Reported per network and precision: frames/s of each path (>= `--steps` batches after a >= 2 s warm-up; two_call between CUDA events,
the pipelined paths by the host clock from the first submit to the last collect; three rounds, paths and precisions alternating), conv
ms per step and ppn_head_kernel ms per step (the engine's per-op CUDA-event profile), parse ms per batch (CUDA events around
hp_ppn_process_device_strided alone), and the card name and power limit (nvidia-smi, read only).

    python tools/bench_ppn.py [--steps 50] [--nets ppn_resnet18,ppn_resnet50]"""
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

H = W = 384
B = 16
CAM_H, CAM_W = 720, 1280
PATHS = ("two_call", "pipelined_device", "pipelined_frames_1280x720")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=20)
        return q.stdout.strip()
    except Exception:
        return torch.cuda.get_device_name(0)


class Path:
    """one engine + parser over the same crowd tensors"""

    def __init__(self, pack, dtype, d_box, d_edge):
        self.eng = capi.Engine(pack, (W, H), max_batch_size=B, dtype=dtype)
        self.eng.set_output_override(d_box.data_ptr(), d_edge.data_ptr())
        self.st = self.eng.device_outputs()[2]
        self.parser = capi.PoseProposalParser((W, H))
        self.pipe_parser = capi.PoseProposalParser((W, H))
        self.p = capi.ppn_engine_pointers(self.eng)

    def parse(self):
        p = self.p
        self.parser.process_device(*p["ptrs"], B, p["K"], p["gh"], p["gw"], 17, 9, 9, stream=self.st,
                                   box_frame_stride=p["box_frame_stride"], edge_frame_stride=p["edge_frame_stride"])

    def step(self, d_frames):
        self.eng.infer_u8_device(d_frames.data_ptr(), B, self.st)
        self.parse()
        return self.parser.fetch(B, 256)

    def submit_device(self, d_frames):
        return self.eng.submit_pose_device(self.pipe_parser, d_frames.data_ptr(), B)

    def submit_camera(self, cam_frames):
        return self.eng.submit_pose_frames(self.pipe_parser, cam_frames)

    def collect(self, ticket):
        return self.eng.collect_pose(ticket, 256)

    def close(self):
        self.eng.close()
        self.parser.close()
        self.pipe_parser.close()


def timed(path, frames, steps):
    t_end = time.perf_counter() + 2.0
    i = 0
    while time.perf_counter() < t_end:
        path.step(frames[i % len(frames)]); i += 1
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for i in range(steps):
        path.step(frames[i % len(frames)])
    b.record()
    torch.cuda.synchronize()
    return B * steps / (a.elapsed_time(b) * 1e-3)


def timed_pipelined(path, submit, inputs, steps):
    """two tickets in flight: submit batch i, then collect batch i - 1"""
    def run(n, warm_until=None):
        pending = []
        i = 0
        while (i < n) if warm_until is None else (time.perf_counter() < warm_until):
            pending.append(submit(inputs[i % len(inputs)])); i += 1
            if len(pending) == 2:
                path.collect(pending.pop(0))
        for t in pending:
            path.collect(t)
    run(0, time.perf_counter() + 2.0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    run(steps)   # (the last collect waits for the last batch's records)
    return B * steps / (time.perf_counter() - t0)


def same_humans(a, b):
    return len(a) == len(b) and all(len(x) == len(y) and x.tobytes() == y.tobytes() for x, y in zip(a, b))


def profile(g, path, frames):
    eng = path.eng
    for i in range(5):
        eng.infer_u8_device(frames[i % len(frames)].data_ptr(), B, path.st)
    eng.sync()
    eng.set_profiling(True)
    for i in range(20):
        eng.infer_u8_device(frames[i % len(frames)].data_ptr(), B, path.st)
    eng.sync()
    ms, ty, _, _ = eng.get_profile()
    eng.set_profiling(False)
    conv = float(ms[ty == models.OP_CONV].sum())
    head = float(ms[ty == models.OP_PPN_HEAD].sum())
    # the parse alone, on the outputs the last run left (the crowd tensors)
    for _ in range(5):
        path.parse()
    s = torch.cuda.ExternalStream(path.st)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(s)
    n = 50
    for _ in range(n):
        path.parse()
    b.record(s)
    torch.cuda.synchronize()
    return conv, head, a.elapsed_time(b) / n, float(ms.sum())


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--nets", default="ppn_resnet18,ppn_resnet50")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ppn measures on the GPU"
    print(json.dumps({"card": card()}))
    ts = [syn.make_ppn_tensors(2000 + i, (4, 8)) for i in range(B)]
    d_box = torch.from_numpy(np.ascontiguousarray(np.stack([np.stack(t[:6]) for t in ts]).reshape(B, -1, 12, 12))).cuda()
    d_edge = torch.from_numpy(np.ascontiguousarray(np.stack([t[6] for t in ts]).reshape(B, -1, 12, 12))).cuda()
    frames = [torch.from_numpy(syn.make_frames_u8(10 + i, B, H, W)).cuda() for i in range(4)]
    # page-locked camera-size frames (the resize kernel brings them to the network size)
    cams = [[torch.from_numpy(f).pin_memory().numpy() for f in syn.make_frames_u8(20 + i, B, CAM_H, CAM_W)] for i in range(2)]
    for net in a.nets.split(","):
        g = getattr(models, net)(0)
        pack = g.to_pack()
        paths = {dt: Path(pack, dt, d_box, d_edge) for dt in ("f16", "tf32")}
        humans = paths["f16"].step(frames[0])
        for dt, p in paths.items():   # the pipelined calls return the two-call path's records
            want = p.step(frames[0])
            assert same_humans(p.collect(p.submit_device(frames[0])), want), (net, dt, "pipelined_device")
            assert same_humans(p.collect(p.submit_camera(cams[0])), want), (net, dt, "pipelined_frames")
        humans = [len(h) for h in humans]
        fps = {path: {dt: [] for dt in paths} for path in PATHS}
        for _ in range(3):
            for dt, p in paths.items():
                fps["two_call"][dt].append(round(timed(p, frames, a.steps), 1))
                fps["pipelined_device"][dt].append(round(timed_pipelined(p, p.submit_device, frames, a.steps), 1))
                fps["pipelined_frames_1280x720"][dt].append(round(timed_pipelined(p, p.submit_camera, cams, a.steps), 1))
        res = {"net": net, "input": [H, W], "batch": B, "humans_per_frame": [min(humans), max(humans)], "fps": fps,
               "median_fps": {path: {dt: float(np.median(v)) for dt, v in d.items()} for path, d in fps.items()}}
        for dt, p in paths.items():
            conv, head, parse, tot = profile(g, p, frames)
            res[dt] = {"conv_ms_per_step": round(conv, 3), "ppn_head_kernel_ms": round(head, 4), "parse_ms": round(parse, 4),
                       "engine_ms_per_step": round(tot, 3), "conv_tflops": round(g.flops_per_frame(H, W) * B / (conv * 1e-3) / 1e12, 1)}
        print(json.dumps(res))
        for p in paths.values():
            p.close()
    print(json.dumps({"card": card()}))


if __name__ == "__main__":
    main()
