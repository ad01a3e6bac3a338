"""Per-op CUDA-event times of one bench.py workload's graph (engine only, 40 profiled steps after warm-up) and the kernel each op
launches, as one JSON line.  Used to compare kernel variants selected by environment switches (HPB_HALO, HPB_NO_STEM3,
HPB_NO_POOL_FUSE, ...): run it once per setting and compare the lines."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import WORKLOADS  # noqa: E402
from hyperpose_b200 import capi, models, synthetic as syn  # noqa: E402

ap = argparse.ArgumentParser(description=__doc__)
ap.add_argument("--workload", default="cfg3", choices=sorted(WORKLOADS))
ap.add_argument("--steps", type=int, default=40)
args = ap.parse_args()

wl = WORKLOADS[args.workload]
H, W, B = wl["in_h"], wl["in_w"], wl["batch"]
g = getattr(models, wl["graph"])(seed=0)
eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=B)
sets = [torch.from_numpy(syn.make_frames_u8(2 + i, B, H, W)).cuda() for i in range(6)]
st = torch.cuda.Stream()
for i in range(5):
    eng.infer_u8_device(sets[i % 6].data_ptr(), B, st.cuda_stream)
torch.cuda.synchronize()
eng.set_profiling(True)
for i in range(args.steps):
    eng.infer_u8_device(sets[i % 6].data_ptr(), B, st.cuda_stream)
torch.cuda.synchronize()
ms, ty, fl, runs = eng.get_profile()
ops = [[o.name, eng.debug_op_kernel(i), round(float(m), 4)] for i, (o, m) in enumerate(zip(g.ops, ms))]
print(json.dumps({"workload": args.workload, "HPB_HALO": os.environ.get("HPB_HALO"), "gpu": torch.cuda.get_device_name(),
                  "sum_ms": round(float(ms.sum()), 4), "ops": ops}))
eng.close()
