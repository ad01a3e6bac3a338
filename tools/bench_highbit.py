"""16-bit frames through the pipelined pose calls: the depth reduction fused into the batched resize, against 8-bit frames of the same
content and against the reduction a user runs today as a separate pass.

Workloads: bench_yuv.py's (bench.py's cfg2, cfg3, cfg4 and cfg5: graph, network size, batch; fp16 engine; synthetic crowd maps or
PIF/PAF fields copied over the network's outputs so the parser does real work), 720p and 1080p.  Each round alternates, in one process:
  p016-dev    submit_pose_yuv420_16_device(bits 16) on P016 frames in an NVDEC-like surface (pitch 2 * width rounded up to 256 bytes,
              luma rows to 16, the UV plane after the luma surface);
  nv12-dev    submit_pose_yuv420_device on the same content reduced to NV12 (what P016 reduces to), in an NVDEC-like surface;
  p016-torch  the P016 surface reduced by a torch pass (round half to even, as convertTo) into a packed NV12 buffer on the engine
              stream, then submit_pose_yuv420_device: what a user without the fused call does on the device.
Two batches in flight in every arm.  One JSON line per workload: frames/s of every arm in each round (host clock over `--steps` batches
after `--warmup` batches; each batch ends in a collect, which waits for it), the device time per batch of the resize kernel in each arm
and of the torch pass (torch.profiler with CUDA activities, runs of their own), and the card and its power limit read by nvidia-smi in
the same process.

    python tools/bench_highbit.py [--steps 30] [--warmup 10] [--rounds 3] [--workloads cfg2,cfg3,cfg4,cfg5] [--out FILE]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from bench_frames import WORKLOADS, smi  # noqa: E402
from bench_yuv import SETS, SOURCES, Workload as YuvWorkload  # noqa: E402
from hyperpose_b200 import capi  # noqa: E402


def nvdec_surfaces(rng, h, w):
    """(P016 surface int16 [rows * 3/2, pitch16], its record, NV12 surface u8 [rows * 3/2, pitch8] of the reduced content, its record)
    of one h x w frame, both on the device; the P016 samples are MSB-aligned 16-bit words (bits = 16)"""
    rows = (h + 15) // 16 * 16
    p16, p8 = (2 * w + 255) // 256 * 256, (w + 255) // 256 * 256
    s16 = rng.integers(0, 1 << 16, (rows + rows // 2, p16 // 2), dtype=np.uint16)
    s8 = np.zeros((rows + rows // 2, p8), np.uint8)
    s8[:, :w] = np.minimum(np.rint(s16[:, :w] / 256.0), 255).astype(np.uint8)
    t16, t8 = torch.from_numpy(s16.view(np.int16)).cuda(), torch.from_numpy(s8).cuda()
    a, b = t16.data_ptr(), t8.data_ptr()
    return (t16, capi.FrameYUV420_16(a, a + rows * p16, a + rows * p16 + 2, h, w, p16, p16, 2, 16),
            t8, capi.FrameYUV420(b, b + rows * p8, b + rows * p8 + 1, h, w, p8, p8, 2))


def reduce_torch(src, out):
    """convertTo(CV_8U, 1/256) of int16-stored 16-bit samples as torch int32 ops: (v + 127 + ((v >> 8) & 1)) >> 8, saturated"""
    v = src.to(torch.int32) & 0xFFFF
    out.copy_(((v + 127 + ((v >> 8) & 1)) >> 8).clamp_(max=255))


class Workload(YuvWorkload):
    """bench_yuv's engine, parser and output override, with P016 surfaces, the NV12 of their content and the torch pass's buffers"""

    def __init__(self, key):
        super().__init__(key)
        rng = np.random.default_rng(11)
        self.p016, self.nv12_same, self.packed = {}, {}, {}
        for (h, w) in SOURCES:
            s = (h, w)
            sets = [[nvdec_surfaces(rng, h, w) for _ in range(self.B)] for _ in range(SETS)]
            self.p016[s] = [[(t16, r16) for t16, r16, _, _ in fs] for fs in sets]
            self.nv12_same[s] = [[(t8, r8) for _, _, t8, r8 in fs] for fs in sets]
            packed = []
            for _ in range(SETS):
                bufs = []
                for _ in range(self.B):
                    o = torch.empty((h * 3 // 2, w), dtype=torch.uint8, device="cuda")
                    p = o.data_ptr()
                    bufs.append((o, capi.FrameYUV420(p, p + h * w, p + h * w + 1, h, w, w, w, 2)))
                packed.append(bufs)
            self.packed[s] = packed
        torch.cuda.synchronize()

    def reduced_by_torch(self, s, i):
        """p016-torch: both planes of every P016 frame reduced by torch into a packed NV12 buffer on the engine stream (ordered before
        the batch's resize), then the NV12 call"""
        k = i % SETS
        h, w = s
        rows = (h + 15) // 16 * 16
        with torch.cuda.stream(self.stream):
            for (t16, _), (o, _) in zip(self.p016[s][k], self.packed[s][k]):
                reduce_torch(t16[:h, :w], o[:h])
                reduce_torch(t16[rows:rows + h // 2, :w], o[h:])
        return self.eng.submit_pose_yuv420_device(self.parser, [r for _, r in self.packed[s][k]])

    def arms(self):
        e, p = self.eng, self.parser
        out = {}
        for s in SOURCES:
            tag = f"{s[1]}x{s[0]}"
            out[f"p016-dev-{tag}"] = (lambda s: lambda i: e.submit_pose_yuv420_16_device(p, [r for _, r in self.p016[s][i % SETS]]))(s)
            out[f"nv12-dev-{tag}"] = (lambda s: lambda i: e.submit_pose_yuv420_device(p, [r for _, r in self.nv12_same[s][i % SETS]]))(s)
            out[f"p016-torch-{tag}"] = (lambda s: lambda i: self.reduced_by_torch(s, i))(s)
        return out

    def torch_pass_ms(self, arm_name, n=20):
        """device time per batch of the torch kernels (everything but the project's own) in arm `arm_name`"""
        arm = self.arms()[arm_name]
        self.run(arm, 4)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            self.run(arm, n)
            torch.cuda.synchronize()
        return sum(k.device_time_total for k in prof.key_averages() if "at::native" in k.key) / 1e3 / n

    def check(self):
        """the three arms give the same network-size frames"""
        for s in SOURCES:
            tag = f"{s[1]}x{s[0]}"
            got = []
            for a in ("p016-dev", "nv12-dev", "p016-torch"):
                t = self.arms()[f"{a}-{tag}"](0)
                self.eng.collect_pose(t, cap=self.hcap)
                got.append(self.eng.debug_read_slot_frames(t, self.B))
            assert all(np.array_equal(g, got[0]) for g in got[1:]), f"{self.key} {tag}: the arms' frames differ"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--workloads", default="cfg2,cfg3,cfg4,cfg5")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_highbit: no CUDA device")
    for key in args.workloads.split(","):
        assert key in WORKLOADS, key
        w = Workload(key)
        w.check()
        arms = w.arms()
        fps = {name: [] for name in arms}
        for r in range(args.rounds):
            for name, arm in arms.items():
                w.run(arm, args.warmup)
                fps[name].append(round(args.steps * w.B / w.run(arm, args.steps), 1))
        tags = [f"{s[1]}x{s[0]}" for s in SOURCES]
        kernels = {"p016-dev": "resize_frames_yuv420_16_kernel", "nv12-dev": "resize_frames_yuv420_kernel",
                   "p016-torch": "resize_frames_yuv420_kernel"}
        res = {"workload": key, "net": f"{w.H}x{w.W}", "batch": w.B, "fps": fps,
               "fps_median": {k: float(np.median(v)) for k, v in fps.items()},
               "resize_ms_per_batch": {f"{a}-{t}": round(w.kernel_ms(f"{a}-{t}", kern), 4) for t in tags for a, kern in kernels.items()},
               "torch_pass_ms_per_batch": {t: round(w.torch_pass_ms(f"p016-torch-{t}"), 4) for t in tags},
               **smi()}
        line = json.dumps(res)
        print(line, flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(line + "\n")
        w.close()
        del w
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
