"""Where the halo kernel's time goes on a bench.py graph's halo layers (cfg3: the VGG trunk, cpm_*, init_* and the 7x7 refinement
convs), from an instrumented build: builds the library with -DHPB_HALO_PHASES into a temporary directory, runs every halo layer of
the graph on its own at the benchmark batch, and prints per layer the consumer warpgroups' clock64 cycles split into waiting for the
halo box (A late), waiting for a weight tile (B late), waiting in wgmma_wait, the epilogue (accumulators to the output or to the
staging buffer), waiting for the other warpgroup's turn (ping-pong item only), waiting for a staging buffer the previous TMA store
still reads, and the rest (issuing MMAs, descriptors, barrier arrives).  Set HPB_HALO_NARROW=1 for the 128-pixel item."""
import argparse
import json
import os
import sys
import tempfile
import ctypes as C

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import WORKLOADS  # noqa: E402
from hyperpose_b200 import build as hb, capi, models, synthetic as syn  # noqa: E402

PHASES = ["total", "a_wait", "b_wait", "mma_wait", "epilogue", "turn_wait", "stage_wait"]   # HALO_PH_* order (conv_wgmma.cuh)


def read_phases(L, reset=True):
    out = np.zeros(len(PHASES), np.uint64)
    capi.check(L.hp_debug_halo_phases(out.ctypes.data_as(C.c_void_p), len(PHASES), 1 if reset else 0))
    return out.astype(np.float64)


def main():
    ap = argparse.ArgumentParser(description=__doc__)
    ap.add_argument("--workload", default="cfg3", choices=sorted(WORKLOADS))
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--build-dir", help="where the instrumented library is built (default: a new temporary directory)")
    args = ap.parse_args()
    capi.LIB_PATH = hb.build(out_dir=args.build_dir or tempfile.mkdtemp(prefix="halo_phases_"), defines=("HPB_HALO_PHASES",))
    L = capi.lib()
    L.hp_debug_halo_phases.argtypes = [C.c_void_p, C.c_int, C.c_int]
    wl = WORKLOADS[args.workload]
    H, W, B = wl["in_h"], wl["in_w"], wl["batch"]
    g = getattr(models, wl["graph"])(seed=0)
    eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=B)
    frames = torch.from_numpy(syn.make_frames_u8(2, B, H, W)).cuda()
    st = torch.cuda.Stream()
    for _ in range(3):
        eng.infer_u8_device(frames.data_ptr(), B, st.cuda_stream)
    torch.cuda.synchronize()
    print(f"# {torch.cuda.get_device_name()}, {args.workload} batch {B}, HPB_HALO_NARROW={os.environ.get('HPB_HALO_NARROW')}; "
          "share of consumer-warpgroup cycles")
    print(f"{'layer':<12} {'kernel':<18} {'k-steps':>7} {'Mclk/wg':>8} " + " ".join(f"{p:>9}" for p in PHASES[1:]) + f" {'rest':>6}")
    rows = []
    for i, o in enumerate(g.ops):
        k = eng.debug_op_kernel(i)
        if not k.startswith("halo<"):
            continue
        eng.debug_run_ops(i, i, B)   # warm
        read_phases(L)
        for _ in range(args.reps):
            eng.debug_run_ops(i, i, B)
        ph = read_phases(L)
        tot = ph[0]
        share = ph[1:] / tot
        ksteps = o.R * o.R * ((o.cin_g + 63) // 64)
        ctas = torch.cuda.get_device_properties(0).multi_processor_count
        rows.append({"op": o.name, "kernel": k, "ksteps_per_item": ksteps, **{p: round(float(s), 4) for p, s in zip(PHASES[1:], share)}})
        print(f"{o.name:<12} {k:<18} {ksteps:>7} {tot / args.reps / (2 * ctas) / 1e6:>8.3f} " +
              " ".join(f"{s:>9.1%}" for s in share) + f" {1 - share.sum():>6.1%}")
    eng.close()
    print(json.dumps({"workload": args.workload, "HPB_HALO_NARROW": os.environ.get("HPB_HALO_NARROW"), "gpu": torch.cuda.get_device_name(),
                      "layers": rows}))


if __name__ == "__main__":
    main()
