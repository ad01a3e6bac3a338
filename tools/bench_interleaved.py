"""Interleaved frames through the pipelined pose calls: the conversion fused into the batched resize, against BGR frames.

Workloads: bench_frames.py's (bench.py's cfg2, cfg3, cfg4 and cfg5: graph, network size, batch; fp16 engine; synthetic crowd maps or
PIF/PAF fields copied over the network's outputs so the parser does real work).  Sources: 1280x720 and 1920x1080.  Each round
alternates, in one process:
  bgr-host    submit_pose_frames on page-locked BGR frames (3 bytes per pixel uploaded);
  yuyv-host   submit_pose_interleaved on page-locked YUYV frames (2 bytes per pixel uploaded), what a V4L2 webcam delivers;
  bgr-dev     submit_pose_frames_device on packed BGR frames in device memory;
  bgra-dev    submit_pose_interleaved_device on BGRA surfaces in device memory, pitch rounded up to 256 bytes as NvBufSurface does;
  bgrp-dev    submit_pose_interleaved_device on BGR surfaces in device memory with a pitch rounded up to 512 bytes (cudaMallocPitch).
Two batches in flight in every arm.  One JSON line per workload: frames/s of every arm in each of three rounds (host clock over
`--steps` batches after `--warmup` batches; each batch ends in a collect, which waits for it), the H2D megabytes per batch of the host
arms, the device time per batch of the resize kernels (torch.profiler with CUDA activities, runs of their own: the BGR kernel in
bgr-dev, the interleaved kernel in bgra-dev, yuyv-host and bgrp-dev), and the card and its power limit read by nvidia-smi in the same
process.

    python tools/bench_interleaved.py [--steps 30] [--warmup 10] [--workloads cfg2,cfg3,cfg4,cfg5] [--out FILE]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from bench_frames import smi  # noqa: E402
from bench_yuv import SETS, SOURCES, Workload as YuvWorkload  # noqa: E402
from hyperpose_b200 import capi  # noqa: E402


def surface(rng, h, w, bpp, align):
    """(device surface u8 [h, pitch], pitch): random bytes, rows padded to `align` bytes"""
    pitch = (w * bpp + align - 1) // align * align
    return torch.from_numpy(rng.integers(0, 256, (h, pitch), dtype=np.uint8)).cuda(), pitch


class Workload(YuvWorkload):
    """bench_yuv's engine, parser, output override and BGR frames, plus the interleaved inputs"""

    def __init__(self, key):
        super().__init__(key)
        B = self.B
        rng = np.random.default_rng(8)
        pinned = lambda a: torch.from_numpy(a).pin_memory().numpy()
        self.yuyv_host, self.bgra_recs, self.bgrp_recs, self._surfs = {}, {}, {}, []
        for (h, w) in SOURCES:
            s = (h, w)
            self.yuyv_host[s] = [[pinned(rng.integers(0, 256, (h, w, 2), dtype=np.uint8)) for _ in range(B)] for _ in range(SETS)]
            for recs, fmt, bpp, align in ((self.bgra_recs, "bgra", 4, 256), (self.bgrp_recs, "bgr", 3, 512)):
                surfs = [[surface(rng, h, w, bpp, align) for _ in range(B)] for _ in range(SETS)]
                self._surfs.append(surfs)
                recs[s] = [[capi.FrameInterleaved(t.data_ptr(), h, w, pitch, capi.PIXEL_FORMATS[fmt]) for t, pitch in fs] for fs in surfs]
        torch.cuda.synchronize()

    def arms(self):
        e, p = self.eng, self.parser
        out = {}
        for s in SOURCES:
            tag = f"{s[1]}x{s[0]}"
            out[f"bgr-host-{tag}"] = (lambda s: lambda i: e.submit_pose_frames(p, self.bgr_host[s][i % SETS]))(s)
            out[f"yuyv-host-{tag}"] = (lambda s: lambda i: e.submit_pose_interleaved(p, self.yuyv_host[s][i % SETS], "yuyv"))(s)
            out[f"bgr-dev-{tag}"] = (lambda s: lambda i: e.submit_pose_frames_device(
                p, [(t.data_ptr(), s[0], s[1]) for t in self.bgr_dev[s][i % SETS]]))(s)
            out[f"bgra-dev-{tag}"] = (lambda s: lambda i: e.submit_pose_interleaved_device(p, self.bgra_recs[s][i % SETS]))(s)
            out[f"bgrp-dev-{tag}"] = (lambda s: lambda i: e.submit_pose_interleaved_device(p, self.bgrp_recs[s][i % SETS]))(s)
        return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--workloads", default="cfg2,cfg3,cfg4,cfg5")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_interleaved: no CUDA device")
    for key in args.workloads.split(","):
        w = Workload(key)
        arms = w.arms()
        fps = {name: [] for name in arms}
        for r in range(args.rounds):
            for name, arm in arms.items():
                w.run(arm, args.warmup)
                fps[name].append(round(args.steps * w.B / w.run(arm, args.steps), 1))
        tags = [f"{s[1]}x{s[0]}" for s in SOURCES]
        kernel = "resize_frames_interleaved_kernel"
        res = {"workload": key, "net": f"{w.H}x{w.W}", "batch": w.B, "fps": fps,
               "fps_median": {k: float(np.median(v)) for k, v in fps.items()},
               "h2d_mb_per_batch": {f"{t}-{fmt}": round(w.B * s[0] * s[1] * m / 1e6, 2)
                                    for t, s in zip(tags, SOURCES) for fmt, m in (("bgr", 3), ("yuyv", 2))},
               "resize_ms_per_batch": {**{f"bgr-{t}": round(w.kernel_ms(f"bgr-dev-{t}", "resize_frames_u8c3_kernel"), 4) for t in tags},
                                       **{f"{a}-{t}": round(w.kernel_ms(f"{a}-{t}", kernel), 4)
                                          for t in tags for a in ("bgra-dev", "yuyv-host", "bgrp-dev")}},
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
