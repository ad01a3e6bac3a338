"""Per-op CUDA-event times of the cfg3 graph (engine only, 40 profiled steps after warm-up); one line per op.
Used to compare kernel variants selected by environment switches (HPB_HALO, HPB_NO_STEM3, HPB_NO_POOL_FUSE, ...)."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hyperpose_b200 import capi, models, synthetic as syn  # noqa: E402

H, W, B = 368, 656, 16
g = models.openpose_vgg19(0)
eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=B)
sets = [torch.from_numpy(syn.make_frames_u8(2 + i, B, H, W)).cuda() for i in range(6)]
st = torch.cuda.Stream()
for i in range(5):
    eng.infer_u8_device(sets[i % 6].data_ptr(), B, st.cuda_stream)
torch.cuda.synchronize()
eng.set_profiling(True)
for i in range(40):
    eng.infer_u8_device(sets[i % 6].data_ptr(), B, st.cuda_stream)
torch.cuda.synchronize()
ms, ty, fl, runs = eng.get_profile()
names = [o.name for o in g.ops]
out = {n: round(float(m), 4) for n, m in zip(names, ms)}
out["_sum"] = round(float(ms.sum()), 4)
print(json.dumps(out))
