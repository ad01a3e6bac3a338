"""YUV 4:2:0 video frames through the pipelined pose calls: the colour conversion fused into the batched resize, against BGR frames and
against the conversion a user runs today as a separate pass.

Workloads: bench_frames.py's (bench.py's cfg2, cfg3, cfg4 and cfg5: graph, network size, batch; fp16 engine; synthetic crowd maps or
PIF/PAF fields copied over the network's outputs so the parser does real work).  Sources: 1280x720 and 1920x1080.  Each round
alternates, in one process:
  bgr-dev    submit_pose_frames_device on BGR frames in device memory;
  nv12-dev   submit_pose_yuv420_device on NV12 frames in device memory, pitched as NVDEC writes them (pitch rounded up to 256 bytes,
             luma rows to 16, the UV plane after the luma surface);
  nv12-torch the same NV12 frames converted to BGR by a torch pass of the same integer formula on the engine stream, then
             submit_pose_frames_device: what a user without the fused call does;
  bgr-host   submit_pose_frames on page-locked BGR frames;
  nv12-host  submit_pose_yuv420 on page-locked NV12 frames (cv2's packed layout).
Two batches in flight in every arm.  One JSON line per workload: frames/s of every arm in each of three rounds (host clock over
`--steps` batches after `--warmup` batches; each batch ends in a collect, which waits for it), the H2D megabytes per batch of the host
arms, the device time per batch of the BGR and YUV resize kernels (torch.profiler with CUDA activities, separate runs of arms bgr-dev
and nv12-dev), and the card and its power limit read by nvidia-smi in the same process.

    python tools/bench_yuv.py [--steps 30] [--warmup 10] [--workloads cfg2,cfg3,cfg4,cfg5] [--out FILE]"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from bench_frames import WORKLOADS, smi  # noqa: E402
from hyperpose_b200 import capi, models, synthetic as syn  # noqa: E402

SOURCES = [(720, 1280), (1080, 1920)]
SETS = 2   # distinct batches per input, alternated


def nv12_surface(rng, h, w):
    """(surface u8 [rows * 3/2, pitch], rows, pitch): an NV12 frame of h x w in an NVDEC-like surface"""
    pitch, rows = (w + 255) // 256 * 256, (h + 15) // 16 * 16
    s = rng.integers(0, 256, (rows + rows // 2, pitch), dtype=np.uint8)
    return s, rows, pitch


def nv12_to_bgr_torch(surf, h, w, rows, out):
    """cv::cvtColor(COLOR_YUV2BGR_NV12) as torch int32 ops on a device surface, into out u8 [h, w, 3]"""
    y = surf[:h, :w].to(torch.int32)
    uv = surf[rows:rows + h // 2, :w].to(torch.int32).view(h // 2, w // 2, 2)
    u = (uv[..., 0] - 128).repeat_interleave(2, 0).repeat_interleave(2, 1)
    v = (uv[..., 1] - 128).repeat_interleave(2, 0).repeat_interleave(2, 1)
    yy = (y - 16).clamp_min(0) * 1220542 + (1 << 19)
    out[..., 0] = ((yy + 2116026 * u) >> 20).clamp(0, 255)
    out[..., 1] = ((yy - 852492 * v - 409993 * u) >> 20).clamp(0, 255)
    out[..., 2] = ((yy + 1673527 * v) >> 20).clamp(0, 255)


class Workload:
    def __init__(self, key):
        graph, self.H, self.W, self.B, persons, self.pifpaf = WORKLOADS[key]
        self.key = key
        self.eng = capi.Engine(getattr(models, graph)(seed=0).to_pack(), (self.W, self.H), max_batch_size=self.B)
        e, B = self.eng, self.B
        self.hcap = 128 if self.pifpaf else 64
        if self.pifpaf:
            self.parser = capi.PifPafParser(self.H, self.W, 0.1)
            fl = [syn.make_pifpaf_fields(1000 + i, persons, e.out_h, e.out_w) for i in range(B)]
            conf = np.stack([f[0] for f in fl]).reshape(B, 85, e.out_h, e.out_w)
            paf = np.stack([f[1] for f in fl]).reshape(B, 171, e.out_h, e.out_w)
        else:
            self.parser = capi.PafParser(0.05, 0.05)
            self.parser.set_capacity(peaks_per_part=128, candidates_per_limb=2048, humans=self.hcap)
            conf, paf = syn.make_batch_tensors(1000, B, persons, e.out_h, e.out_w)
        self.d_conf, self.d_paf = torch.from_numpy(conf).cuda(), torch.from_numpy(paf).cuda()
        e.set_output_override(self.d_conf.data_ptr(), self.d_paf.data_ptr())
        self.stream = torch.cuda.ExternalStream(e.device_outputs()[2])
        rng = np.random.default_rng(7)
        pinned = lambda a: torch.from_numpy(a).pin_memory().numpy()
        self.bgr_host, self.nv12_host, self.bgr_dev, self.nv12_dev, self.nv12_recs, self.bgr_tmp = {}, {}, {}, {}, {}, {}
        for (h, w) in SOURCES:
            s = (h, w)
            self.bgr_host[s] = [[pinned(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)) for _ in range(B)] for _ in range(SETS)]
            self.nv12_host[s] = [[pinned(rng.integers(0, 256, (h * 3 // 2, w), dtype=np.uint8)) for _ in range(B)] for _ in range(SETS)]
            self.bgr_dev[s] = [[torch.from_numpy(f).cuda() for f in fs] for fs in self.bgr_host[s]]
            surf = [[nv12_surface(rng, h, w) for _ in range(B)] for _ in range(SETS)]
            self.nv12_dev[s] = [[(torch.from_numpy(a).cuda(), rows, pitch) for a, rows, pitch in fs] for fs in surf]
            self.nv12_recs[s] = [[capi.FrameYUV420(t.data_ptr(), t.data_ptr() + rows * pitch, t.data_ptr() + rows * pitch + 1, h, w, pitch,
                                                   pitch, 2) for t, rows, pitch in fs] for fs in self.nv12_dev[s]]
            self.bgr_tmp[s] = [[torch.empty((h, w, 3), dtype=torch.uint8, device="cuda") for _ in range(B)] for _ in range(SETS)]
        torch.cuda.synchronize()

    def converted(self, s, i):
        """nv12-torch: the separate conversion pass on the engine stream (ordered before the batch's resize), then the BGR call"""
        k = i % SETS
        with torch.cuda.stream(self.stream):
            for (surf, rows, _), out in zip(self.nv12_dev[s][k], self.bgr_tmp[s][k]):
                nv12_to_bgr_torch(surf, s[0], s[1], rows, out)
        return self.eng.submit_pose_frames_device(self.parser, [(t.data_ptr(), s[0], s[1]) for t in self.bgr_tmp[s][k]])

    def arms(self):
        e, p = self.eng, self.parser
        out = {}
        for s in SOURCES:
            tag = f"{s[1]}x{s[0]}"
            out[f"bgr-dev-{tag}"] = (lambda s: lambda i: e.submit_pose_frames_device(
                p, [(t.data_ptr(), s[0], s[1]) for t in self.bgr_dev[s][i % SETS]]))(s)
            out[f"nv12-dev-{tag}"] = (lambda s: lambda i: e.submit_pose_yuv420_device(p, self.nv12_recs[s][i % SETS]))(s)
            out[f"nv12-torch-{tag}"] = (lambda s: lambda i: self.converted(s, i))(s)
            out[f"bgr-host-{tag}"] = (lambda s: lambda i: e.submit_pose_frames(p, self.bgr_host[s][i % SETS]))(s)
            out[f"nv12-host-{tag}"] = (lambda s: lambda i: e.submit_pose_yuv420(p, self.nv12_host[s][i % SETS], "nv12"))(s)
        return out

    def run(self, arm, n):
        """n batches of one arm, two in flight.  Returns seconds."""
        e = self.eng
        t0 = time.perf_counter()
        pend = None
        for i in range(n):
            t = arm(i)
            if pend is not None:
                e.collect_pose(pend, cap=self.hcap)
            pend = t
        e.collect_pose(pend, cap=self.hcap)
        return time.perf_counter() - t0

    def kernel_ms(self, arm_name, kernel, n=20):
        """device time per batch of `kernel` in arm `arm_name`"""
        arm = self.arms()[arm_name]
        self.run(arm, 4)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            self.run(arm, n)
            torch.cuda.synchronize()
        ev = [k for k in prof.key_averages() if kernel in k.key]
        assert ev and n - 2 <= ev[0].count <= n, [(k.key, k.count) for k in ev]   # (the trace may miss a launch at either end)
        return ev[0].device_time_total / 1e3 / ev[0].count

    def close(self):
        self.eng.set_output_override(0, 0)
        self.eng.close(); self.parser.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--workloads", default="cfg2,cfg3,cfg4,cfg5")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_yuv: no CUDA device")
    for key in args.workloads.split(","):
        w = Workload(key)
        arms = w.arms()
        fps = {name: [] for name in arms}
        for r in range(args.rounds):
            for name, arm in arms.items():
                w.run(arm, args.warmup)
                fps[name].append(round(args.steps * w.B / w.run(arm, args.steps), 1))
        tags = [f"{s[1]}x{s[0]}" for s in SOURCES]
        res = {"workload": key, "net": f"{w.H}x{w.W}", "batch": w.B, "fps": fps,
               "fps_median": {k: float(np.median(v)) for k, v in fps.items()},
               "h2d_mb_per_batch": {f"{t}-{fmt}": round(w.B * s[0] * s[1] * m / 1e6, 2)
                                    for t, s in zip(tags, SOURCES) for fmt, m in (("bgr", 3), ("nv12", 1.5))},
               "resize_ms_per_batch": {**{f"bgr-{t}": round(w.kernel_ms(f"bgr-dev-{t}", "resize_frames_u8c3_kernel"), 4) for t in tags},
                                       **{f"nv12-{t}": round(w.kernel_ms(f"nv12-dev-{t}", "resize_frames_yuv420_kernel"), 4) for t in tags}},
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
