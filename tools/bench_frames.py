"""Camera-size frames through the pipelined pose calls: what the on-device resize costs against frames already at the network size.

Workloads: bench.py's cfg2, cfg3, cfg4 and cfg5 (graph, network size, batch), fp16 engine, synthetic crowd maps (cfg5: PIF/PAF
fields) copied over the network's outputs as bench.py does, so the parser does real work.  Sources: 640x360, 1280x720 and
1920x1080 BGR frames, page-locked host memory and device memory.  Each round alternates, in one process:
  (a)      submit_pose on page-locked network-size frames, two batches in flight: the upper bound;
  (b-host) submit_pose_frames on page-locked camera-size frames, two batches in flight;
  (b-dev)  submit_pose_frames_device on camera-size frames in device memory, two batches in flight;
  (c)      the per-frame path: N x stage_frame + infer_staged + parse on the device + fetch, one batch at a time.
One JSON line per workload: frames/s of every arm in each of three rounds (host clock over `--steps` batches after `--warmup`
batches; every batch ends in a collect or fetch, which waits for it), the H2D megabytes per batch, the resize kernel's ms per batch
(torch.profiler with CUDA activities, a separate run of arm b-host), and the card and its power limit read by nvidia-smi in the
same process.

    python tools/bench_frames.py [--steps 30] [--warmup 10] [--workloads cfg2,cfg3,cfg4,cfg5] [--out FILE]"""
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

# bench.py's WORKLOADS: (graph, in_h, in_w, batch, persons, pifpaf)
WORKLOADS = {"cfg2": ("mobilenet_thin_openpose", 368, 432, 8, (1, 5), False),
             "cfg3": ("openpose_vgg19", 368, 656, 16, (10, 20), False),
             "cfg4": ("resnet50_lw_openpose", 368, 432, 32, (10, 20), False),
             "cfg5": ("resnet50_pifpaf", 385, 385, 16, (2, 8), True)}
SOURCES = [(360, 640), (720, 1280), (1080, 1920)]
SETS = 2   # distinct batches per input, alternated


def smi():
    """card name and power limit (W), read only"""
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True, timeout=20)
    name, plim = [x.strip() for x in q.stdout.strip().split(",")]
    return {"card": name, "power_limit_w": float(plim)}


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
        torch.cuda.synchronize()
        e.set_output_override(self.d_conf.data_ptr(), self.d_paf.data_ptr())
        rng = np.random.default_rng(7)
        pinned = lambda a: torch.from_numpy(a).pin_memory().numpy()
        self.net = [pinned(syn.make_frames_u8(2 + i, B, self.H, self.W)) for i in range(SETS)]
        self.host = {s: [[pinned(rng.integers(0, 256, (s[0], s[1], 3), dtype=np.uint8)) for _ in range(B)] for _ in range(SETS)]
                     for s in SOURCES}
        self.dev = {s: [[torch.from_numpy(f).cuda() for f in fs] for fs in self.host[s]] for s in SOURCES}
        torch.cuda.synchronize()
        self.dev_tab = {s: [[(t.data_ptr(), s[0], s[1]) for t in ts] for ts in self.dev[s]] for s in SOURCES}

    def arms(self):
        e, p = self.eng, self.parser
        out = {"a": lambda i: e.submit_pose(p, self.net[i % SETS])}
        for s in SOURCES:
            tag = f"{s[1]}x{s[0]}"
            out[f"b-host-{tag}"] = (lambda s: lambda i: e.submit_pose_frames(p, self.host[s][i % SETS]))(s)
            out[f"b-dev-{tag}"] = (lambda s: lambda i: e.submit_pose_frames_device(p, self.dev_tab[s][i % SETS]))(s)
            out[f"c-{tag}"] = (lambda s: ("sync", lambda i: self.staged(self.host[s][i % SETS])))(s)
        return out

    def staged(self, frames):
        e, p = self.eng, self.parser
        for k, f in enumerate(frames):
            e.stage_frame(k, f)
        e.infer_staged(len(frames))
        d_conf, d_paf, st = e.device_outputs()
        if self.pifpaf:
            p.process_device(d_conf, d_paf, len(frames), e.out_h, e.out_w, st)
        else:
            p.process_device(d_conf, d_paf, len(frames), e.c_conf, e.c_paf, e.out_h, e.out_w, st)
        return p.fetch(len(frames), self.hcap)

    def run(self, arm, n):
        """n batches of one arm; two in flight for the pipelined arms.  Returns seconds."""
        e = self.eng
        t0 = time.perf_counter()
        if isinstance(arm, tuple):
            for i in range(n):
                arm[1](i)
        else:
            pend = None
            for i in range(n):
                t = arm(i)
                if pend is not None:
                    e.collect_pose(pend, cap=self.hcap)
                pend = t
            e.collect_pose(pend, cap=self.hcap)
        return time.perf_counter() - t0

    def resize_ms(self, s, n=20):
        """the resize kernel's device time per batch, arm b-host at source size s"""
        arm = self.arms()[f"b-host-{s[1]}x{s[0]}"]
        self.run(arm, 4)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            self.run(arm, n)
            torch.cuda.synchronize()
        ev = [k for k in prof.key_averages() if "resize_frames_u8c3_kernel" in k.key]
        assert ev and ev[0].count == n, [(k.key, k.count) for k in ev]
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
        raise SystemExit("bench_frames: no CUDA device")
    for key in args.workloads.split(","):
        w = Workload(key)
        arms = w.arms()
        fps = {name: [] for name in arms}
        for r in range(args.rounds):
            for name, arm in arms.items():
                w.run(arm, args.warmup)
                fps[name].append(round(args.steps * w.B / w.run(arm, args.steps), 1))
        card = smi()
        res = {"workload": key, "net": f"{w.H}x{w.W}", "batch": w.B, "fps": fps,
               "fps_median": {k: float(np.median(v)) for k, v in fps.items()},
               "h2d_mb_per_batch": {"a": w.B * w.H * w.W * 3 / 1e6,
                                    **{f"{s[1]}x{s[0]}": w.B * s[0] * s[1] * 3 / 1e6 for s in SOURCES}},
               "resize_ms_per_batch": {f"{s[1]}x{s[0]}": round(w.resize_ms(s), 4) for s in SOURCES},
               **card}
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
