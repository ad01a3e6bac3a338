"""Rotated frames through the pipelined pose calls: cv::rotate fused into the batched resize, against the same content upright and
against the rotation a user runs today as a separate pass.

Workloads: bench_frames.py's (bench.py's cfg2, cfg3, cfg4 and cfg5: graph, network size, batch; fp16 engine; synthetic crowd maps or
PIF/PAF fields copied over the network's outputs so the parser does real work).  Sources: portrait phone video, 1080x1920 content stored
as 1920x1080 and 720x1280 content stored as 1280x720, with a 90-degree clockwise rotation to apply.  Each round alternates, in one
process:
  nv12-upright   submit_pose_yuv420_device on the same content already upright (a portrait NVDEC-like surface);
  nv12-rot       submit_pose_yuv420_device(rotation=90) on the stored NV12 frames in an NVDEC-like surface (pitch rounded up to 256
                 bytes, 2048 for 1920 columns; luma rows to 16; the UV plane after the luma surface);
  nv12-torch     the stored frames rotated by a torch rot90 pass of both planes into an upright NV12 buffer on the engine stream, then
                 submit_pose_yuv420_device: what a user without the fused call does on the device;
  nv12-host-up   submit_pose_yuv420 on page-locked upright NV12 frames (cv2's packed layout);
  nv12-host-rot  submit_pose_yuv420(rotation=90) on page-locked stored NV12 frames;
  bgra-upright   submit_pose_interleaved_device on upright BGRA surfaces, pitch rounded up to 256 bytes as NvBufSurface does;
  bgra-rot       submit_pose_interleaved_device(rotation=90) on stored BGRA surfaces, pitched alike.
Two batches in flight in every arm.  One JSON line per workload: frames/s of every arm in each of three rounds (host clock over
`--steps` batches after `--warmup` batches; each batch ends in a collect, which waits for it), the device time per batch of the resize
kernel in the device arms and of the torch pass (torch.profiler with CUDA activities, runs of their own), and the card and its power
limit read by nvidia-smi in the same process.

    python tools/bench_rotated.py [--steps 30] [--warmup 10] [--workloads cfg2,cfg3,cfg4,cfg5] [--out FILE]"""
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
from bench_interleaved import surface  # noqa: E402
from bench_yuv import SETS, Workload as YuvWorkload  # noqa: E402
from hyperpose_b200 import capi  # noqa: E402

STORED = [(720, 1280), (1080, 1920)]   # stored (rows, columns); the content is the transpose, turned 90 degrees clockwise


def nvdec_surface(y, uv):
    """(device surface, record) of an NV12 frame (luma y [h, w], interleaved chroma uv [h/2, w]) in an NVDEC-like surface"""
    h, w = y.shape
    pitch, rows = (w + 255) // 256 * 256, (h + 15) // 16 * 16
    s = np.zeros((rows + rows // 2, pitch), np.uint8)
    s[:h, :w], s[rows:rows + h // 2, :w] = y, uv
    t = torch.from_numpy(s).cuda()
    p = t.data_ptr()
    return t, capi.FrameYUV420(p, p + rows * pitch, p + rows * pitch + 1, h, w, pitch, pitch, 2)


def rot_cw(a):
    """a [h, w, ...] turned 90 degrees clockwise"""
    return np.ascontiguousarray(np.rot90(a, -1))


class Workload(YuvWorkload):
    """bench_yuv's engine, parser and output override, with the rotated and upright inputs"""

    def __init__(self, key):
        super().__init__(key)
        B = self.B
        rng = np.random.default_rng(9)
        pinned = lambda a: torch.from_numpy(a).pin_memory().numpy()
        self.rot_dev, self.up_dev, self.torch_in, self.torch_out = {}, {}, {}, {}
        self.rot_host, self.up_host, self.bgra_rot, self.bgra_up, self._keep = {}, {}, {}, {}, []
        for (h, w) in STORED:
            s = (h, w)
            rot_recs, up_recs, tin, tout, rot_host, up_host = [], [], [], [], [], []
            for _ in range(SETS):
                rr, ur, ti, to, rh, uh = [], [], [], [], [], []
                for _ in range(B):
                    y = rng.integers(0, 256, (h, w), dtype=np.uint8)
                    uv = rng.integers(0, 256, (h // 2, w // 2, 2), dtype=np.uint8)
                    yu, uvu = rot_cw(y), rot_cw(uv)
                    t, rec = nvdec_surface(y, uv.reshape(h // 2, w))
                    tu, recu = nvdec_surface(yu, uvu.reshape(w // 2, h))
                    rr.append(rec); ur.append(recu); self._keep += [t, tu]
                    ti.append((t, rec))
                    o = torch.empty((w * 3 // 2, h), dtype=torch.uint8, device="cuda")   # upright packed NV12, pitch h
                    p = o.data_ptr()
                    to.append((o, capi.FrameYUV420(p, p + w * h, p + w * h + 1, w, h, h, h, 2)))
                    rh.append(pinned(np.concatenate([y, uv.reshape(h // 2, w)])))
                    uh.append(pinned(np.concatenate([yu, uvu.reshape(w // 2, h)])))
                rot_recs.append(rr); up_recs.append(ur); tin.append(ti); tout.append(to); rot_host.append(rh); up_host.append(uh)
            self.rot_dev[s], self.up_dev[s], self.torch_in[s], self.torch_out[s] = rot_recs, up_recs, tin, tout
            self.rot_host[s], self.up_host[s] = rot_host, up_host
            for recs, hh, ww in ((self.bgra_rot, h, w), (self.bgra_up, w, h)):
                surfs = [[surface(rng, hh, ww, 4, 256) for _ in range(B)] for _ in range(SETS)]
                self._keep.append(surfs)
                recs[s] = [[capi.FrameInterleaved(t.data_ptr(), hh, ww, pitch, capi.PIXEL_FORMATS["bgra"]) for t, pitch in fs]
                           for fs in surfs]
        torch.cuda.synchronize()

    def rotated_by_torch(self, s, i):
        """nv12-torch: both planes of every stored frame turned by torch.rot90 into an upright NV12 buffer on the engine stream (ordered
        before the batch's resize), then the upright call"""
        k = i % SETS
        h, w = s
        rows = (h + 15) // 16 * 16
        with torch.cuda.stream(self.stream):
            for (t, _), (o, _) in zip(self.torch_in[s][k], self.torch_out[s][k]):
                o[:w].copy_(torch.rot90(t[:h, :w], -1, (0, 1)))
                o[w:].view(w // 2, h // 2, 2).copy_(torch.rot90(t[rows:rows + h // 2, :w].view(h // 2, w // 2, 2), -1, (0, 1)))
        return self.eng.submit_pose_yuv420_device(self.parser, [r for _, r in self.torch_out[s][k]])

    def arms(self):
        e, p = self.eng, self.parser
        out = {}
        for s in STORED:
            tag = f"{s[0]}x{s[1]}"   # content width x height (portrait)
            out[f"nv12-upright-{tag}"] = (lambda s: lambda i: e.submit_pose_yuv420_device(p, self.up_dev[s][i % SETS]))(s)
            out[f"nv12-rot-{tag}"] = (lambda s: lambda i: e.submit_pose_yuv420_device(p, self.rot_dev[s][i % SETS], rotation=90))(s)
            out[f"nv12-torch-{tag}"] = (lambda s: lambda i: self.rotated_by_torch(s, i))(s)
            out[f"nv12-host-up-{tag}"] = (lambda s: lambda i: e.submit_pose_yuv420(p, self.up_host[s][i % SETS], "nv12"))(s)
            out[f"nv12-host-rot-{tag}"] = (lambda s: lambda i: e.submit_pose_yuv420(p, self.rot_host[s][i % SETS], "nv12", rotation=90))(s)
            out[f"bgra-upright-{tag}"] = (lambda s: lambda i: e.submit_pose_interleaved_device(p, self.bgra_up[s][i % SETS]))(s)
            out[f"bgra-rot-{tag}"] = (lambda s: lambda i: e.submit_pose_interleaved_device(p, self.bgra_rot[s][i % SETS], rotation=90))(s)
        return out

    def torch_pass_ms(self, arm_name, n=20):
        """device time per batch of the torch kernels (everything but the project's own) in arm `arm_name`"""
        arm = self.arms()[arm_name]
        self.run(arm, 4)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            self.run(arm, n)
            torch.cuda.synchronize()
        return sum(k.device_time_total for k in prof.key_averages() if "at::native" in k.key) / 1e3 / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--workloads", default="cfg2,cfg3,cfg4,cfg5")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_rotated: no CUDA device")
    for key in args.workloads.split(","):
        assert key in WORKLOADS, key
        w = Workload(key)
        arms = w.arms()
        fps = {name: [] for name in arms}
        for r in range(args.rounds):
            for name, arm in arms.items():
                w.run(arm, args.warmup)
                fps[name].append(round(args.steps * w.B / w.run(arm, args.steps), 1))
        tags = [f"{s[0]}x{s[1]}" for s in STORED]
        kernels = {"nv12-upright": "resize_frames_yuv420_kernel", "nv12-rot": "resize_frames_yuv420_kernel",
                   "nv12-host-rot": "resize_frames_yuv420_kernel", "bgra-upright": "resize_frames_interleaved_kernel",
                   "bgra-rot": "resize_frames_interleaved_kernel"}
        res = {"workload": key, "net": f"{w.H}x{w.W}", "batch": w.B, "fps": fps,
               "fps_median": {k: float(np.median(v)) for k, v in fps.items()},
               "resize_ms_per_batch": {f"{a}-{t}": round(w.kernel_ms(f"{a}-{t}", kern), 4) for t in tags for a, kern in kernels.items()},
               "torch_pass_ms_per_batch": {t: round(w.torch_pass_ms(f"nv12-torch-{t}"), 4) for t in tags},
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
