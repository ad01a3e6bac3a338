"""Pose Proposal Network throughput: ppn_resnet18 and ppn_resnet50 at 384 x 384, batch 16, f16 and TF32 engines.

The path is device-resident: u8 frames already in HBM -> hp_engine_infer_u8_device -> hp_ppn_process_device_strided on the engine's
two output slots (no copy) -> hp_ppn_fetch, all on the engine's stream.  Random weights give structureless maps, so synthetic crowd
tensors (synthetic.make_ppn_tensors, 4-8 people per frame) are copied over the outputs through the output override, as bench.py does
for the PAF workloads: the parser does real work.

Reported per network and precision: frames/s (CUDA events around >= `--steps` steps after a >= 2 s warm-up, three rounds, the two
precisions alternating), conv ms per step and ppn_head_kernel ms per step (the engine's per-op CUDA-event profile), parse ms per batch
(CUDA events around hp_ppn_process_device_strided alone), and the card name and power limit (nvidia-smi, read only).

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
        self.p = capi.ppn_engine_pointers(self.eng)

    def parse(self):
        p = self.p
        self.parser.process_device(*p["ptrs"], B, p["K"], p["gh"], p["gw"], 17, 9, 9, stream=self.st,
                                   box_frame_stride=p["box_frame_stride"], edge_frame_stride=p["edge_frame_stride"])

    def step(self, d_frames):
        self.eng.infer_u8_device(d_frames.data_ptr(), B, self.st)
        self.parse()
        return self.parser.fetch(B, 256)

    def close(self):
        self.eng.close()
        self.parser.close()


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
    for net in a.nets.split(","):
        g = getattr(models, net)(0)
        pack = g.to_pack()
        paths = {dt: Path(pack, dt, d_box, d_edge) for dt in ("f16", "tf32")}
        humans = [len(h) for h in paths["f16"].step(frames[0])]
        fps = {dt: [] for dt in paths}
        for _ in range(3):
            for dt, p in paths.items():
                fps[dt].append(round(timed(p, frames, a.steps), 1))
        res = {"net": net, "input": [H, W], "batch": B, "humans_per_frame": [min(humans), max(humans)], "fps": fps}
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
