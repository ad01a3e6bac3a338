"""Phase timing of paf_limbs_kernel on the bench's crowd tensors (HPB_PAF_TIMING=1): where the 120 us go."""
import os, sys
os.environ["HPB_PAF_TIMING"] = "1"
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hyperpose_b200 import capi, synthetic as syn
N, HF, WF = 16, 46, 82
conf, paf = syn.make_batch_tensors(1000, N, (10, 20), HF, WF)
dc, dp = torch.from_numpy(conf).cuda(), torch.from_numpy(paf).cuda()
p = capi.PafParser(); p.set_capacity(128, 2048, 64)
for _ in range(5):
    p.process_device(dc.data_ptr(), dp.data_ptr(), N, 19, 38, HF, WF)
torch.cuda.synchronize()
cta, asm = p.debug_timing(N)
t0 = cta[:, :, 0].min()
rel = (cta.astype(np.int64) - int(t0)) / 1e3
a = (asm.astype(np.int64) - int(t0)) / 1e3
print("CTA start   (us) min/max", rel[:, :, 0].min(), rel[:, :, 0].max())
print("ordered     (us) mean dur", (rel[:, :, 1] - rel[:, :, 0]).mean())
print("candidates  (us) mean dur", (rel[:, :, 2] - rel[:, :, 1]).mean(), "max", (rel[:, :, 2] - rel[:, :, 1]).max())
print("matched     (us) mean dur", (rel[:, :, 3] - rel[:, :, 2]).mean(), "max", (rel[:, :, 3] - rel[:, :, 2]).max())
print("limb phase end (us) per frame max", rel[:, :, 3].max(axis=1).round(1))
print("assembly start", a[:, 0].round(1))
print("assembly dur  ", (a[:, 1] - a[:, 0]).round(1), "path (2 component-parallel, 1 sequential):", (asm[:, 1] & 3).tolist())
print("  of which staged / labelled / grouped / lanes / output (us, mean over the frames on the component-parallel path):",
      [round(float(x), 2) for x in ((a[:, 2] - a[:, 0]).mean(), (a[:, 3] - a[:, 2]).mean(), (a[:, 4] - a[:, 3]).mean(), (a[:, 5] - a[:, 4]).mean(), (a[:, 1] - a[:, 5]).mean())])
print("kernel span (us)", a[:, 1].max())
h = p.fetch(N, 64); print("humans", [len(x) for x in h])
