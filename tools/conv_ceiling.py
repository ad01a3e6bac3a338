"""What cuBLAS and cuDNN achieve on the conv shapes of one bench.py workload, next to the engine's own per-op times.

One JSON line per distinct conv shape (map size, filter, groups, channels) of the workload's graph at its benchmark batch size:
  ours   : mean CUDA-event time of the graph's ops of that shape inside the engine (tools/layer_times.py) and their kernels;
  cublas : torch.matmul in fp16 on the equivalent GEMM, [G, M, K] x [G, K, N] with M = batch * H * W, K = R * S * cin_g, N = cout_g,
           fp32 accumulation throughout (allow_fp16_reduced_precision_reduction = False);
  cudnn  : torch.nn.functional.conv2d, fp16 channels_last, the same groups and "SAME" padding.
The libraries get the engine's padded input channels (a multiple of 64: the 185-channel refinement input runs as 192), so all three
do the same work; TFLOP/s are quoted on the layer's algorithmic FLOPs (real channels), as DESIGN.md and bench.py do.  The card's name,
power limit and SM clock are read in the same run and printed on every line.

    python tools/conv_ceiling.py [--workload cfg3] [--iters 20]
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from layer_times import WORKLOADS, op_times  # noqa: E402
from hyperpose_b200 import models  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True)
    name, plim, sm, smmax = [s.strip() for s in q.stdout.strip().split(",")]
    return {"gpu": name, "power_limit_w": float(plim), "sm_clock_mhz": int(sm), "sm_clock_max_mhz": int(smmax)}


def event_ms(fn, iters, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--workload", default="cfg3", choices=sorted(WORKLOADS))
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction = False
    torch.backends.cudnn.benchmark = True
    wl = WORKLOADS[args.workload]
    B = wl["batch"]
    g, ops = op_times(args.workload)

    shapes = {}
    for op, (name, kernel, ms) in zip(g.ops, ops):
        if op.type != models.OP_CONV or op.im2col_input:
            continue
        h, w = wl["in_h"], wl["in_w"]
        for _ in range(g.buffers[op.in_buf][1]):
            h, w = (h + 1) // 2, (w + 1) // 2
        cin_pad = -(-op.cin_g // 64) * 64
        key = (h, w, op.R, op.S, op.groups, op.cin_g, cin_pad, op.cout_g, kernel)   # a fused pool epilogue is a shape of its own
        shapes.setdefault(key, []).append((name, kernel, ms))

    dev = torch.device("cuda")
    for (h, w, R, S, G, cin, cin_pad, cout, _), members in shapes.items():
        flop = 2.0 * B * h * w * G * cout * cin * R * S
        ours_ms = sum(m[2] for m in members) / len(members)
        M, K, N = B * h * w, R * S * cin_pad, cout
        a = torch.randn(G, M, K, device=dev, dtype=torch.float16)
        b = torch.randn(G, K, N, device=dev, dtype=torch.float16)
        cublas_ms = event_ms(lambda: torch.matmul(a, b), args.iters)
        del a, b
        x = torch.randn(B, G * cin_pad, h, w, device=dev, dtype=torch.float16).to(memory_format=torch.channels_last)
        wt = torch.randn(G * cout, cin_pad, R, S, device=dev, dtype=torch.float16).to(memory_format=torch.channels_last)
        cudnn_ms = event_ms(lambda: F.conv2d(x, wt, padding=(R // 2, S // 2), groups=G), args.iters)
        del x, wt
        torch.cuda.empty_cache()
        tf = lambda ms: round(flop / (ms * 1e-3) / 1e12, 1)
        print(json.dumps({"workload": args.workload, "shape": {"H": h, "W": w, "R": R, "S": S, "groups": G, "cin_g": cin, "cin_g_run": cin_pad,
                                                               "cout_g": cout, "batch": B},
                          "ops": [m[0] for m in members], "kernels": sorted({m[1] for m in members}), "gflop": round(flop / 1e9, 2),
                          "gemm_MKN": [M, K, N],
                          "ours_ms": round(ours_ms, 4), "ours_tflops": tf(ours_ms),
                          "cublas_ms": round(cublas_ms, 4), "cublas_tflops": tf(cublas_ms),
                          "cudnn_ms": round(cudnn_ms, 4), "cudnn_tflops": tf(cudnn_ms), **card()}), flush=True)


if __name__ == "__main__":
    main()
