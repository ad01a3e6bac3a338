"""Writes an HPB2PACK model pack (the file `tensorrt(tensorrt_serialized{path}, ...)` / `hp_engine_create` load):

    python -m hyperpose_b200.export --model openpose_vgg19 --out vgg19.pack [--weights trained.npz] [--seed 0]
                                    [--int8-calibration frames.npy [--factor F] [--no-flip-rgb]]

`--weights` is a TensorLayer `save_weights(format="npz")` file of the reference's model of that architecture -- OpenPose-VGG19 (also
the name-keyed `npz_dict` form), MobilenetThin-OpenPose, LightWeightOpenPose on ResNet-50 / TinyVGG / ResNet-18 / MobilenetDilated, PifPaf on ResNet-50, Pose Proposal Networks
on ResNet-18 / ResNet-50; hyperpose_b200/weights.py
spells out the all_weights order of each, BatchNorm statistics are folded.  Without it the pack holds seeded random weights, which is
what the benchmarks and tests use (no trained model can be downloaded offline).  Replaces the .onnx / .uff / .trt files of
include/hyperpose/utility/model.hpp:13-32 (SURVEY.md 8f rank 1).

`--int8-calibration` adds the INT8 scale table that data_type::kINT8 needs: the network runs on those frames (u8 NHWC BGR at the
network size, a .npy of shape [N, H, W, 3]) on a TF32 engine, and every activation buffer gets scale max |x| / 127 (TensorRT's
min-max calibration).  That step runs on the GPU.  The first layer's scale depends on how the frames are normalised: calibrate with
the `factor` and `flip_rgb` the engine will be created with (--factor, --no-flip-rgb; the defaults are the tensorrt constructor's,
1/255 and BGR -> RGB)."""
from __future__ import annotations

import argparse

import numpy as np

from . import models, weights


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--model", default="openpose_vgg19",
                    choices=["openpose_vgg19", "mobilenet_thin_openpose", "resnet50_lw_openpose", "lw_openpose_vggtiny", "lw_openpose_resnet18",
                             "lw_openpose_mobilenet_dilated", "resnet50_pifpaf", "ppn_resnet18", "ppn_resnet50", "tiny_test_net"])
    ap.add_argument("--out", required=True)
    ap.add_argument("--weights", default=None, help="TensorLayer save_weights(format='npz') file of the same architecture")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--int8-calibration", default=None, metavar="FRAMES.npy",
                    help="u8 [N,H,W,3] frames at the network size: adds the INT8 scale table (runs on the GPU)")
    ap.add_argument("--factor", type=float, default=1.0 / 255,
                    help="input scaling of the calibration run; must match the engine's `factor` (default 1/255)")
    ap.add_argument("--no-flip-rgb", action="store_true", help="calibrate without the BGR -> RGB swap (an engine created with flip_rgb=false)")
    a = ap.parse_args(argv)
    if a.weights:
        loaders = {"openpose_vgg19": weights.ListWeights, "mobilenet_thin_openpose": weights.MobilenetThinWeights,
                   "resnet50_lw_openpose": weights.Resnet50LwWeights, "lw_openpose_vggtiny": weights.LwVggtinyWeights,
                   "lw_openpose_resnet18": weights.LwResnet18Weights, "lw_openpose_mobilenet_dilated": weights.LwMobilenetDilatedWeights,
                   "resnet50_pifpaf": weights.Resnet50PifPafWeights,
                   "ppn_resnet18": weights.Ppn18Weights, "ppn_resnet50": weights.Ppn50Weights}
        if a.model not in loaders:
            ap.error(f"--weights: no trained-weight layout for {a.model}")
        g = getattr(models, a.model)(weights=loaders[a.model].from_npz(a.weights))
    else:
        g = getattr(models, a.model)(a.seed)
    if a.int8_calibration:
        from . import capi
        frames = np.load(a.int8_calibration)
        if frames.dtype != np.uint8 or frames.ndim != 4 or frames.shape[3] != 3:
            ap.error(f"--int8-calibration: expected u8 [N,H,W,3] frames, got {frames.dtype} {frames.shape}")
        eng = capi.Engine(g.to_pack(), (frames.shape[2], frames.shape[1]), max_batch_size=min(8, frames.shape[0]), factor=a.factor,
                          flip_rgb=not a.no_flip_rgb, dtype="tf32")
        g.set_int8_scales(eng.calibrate(frames))
        eng.close()
    blob = g.to_pack()
    with open(a.out, "wb") as f:
        f.write(blob)
    print(f"{a.out}: {g.name}, {len(g.ops)} ops, {len(blob) / 1e6:.1f} MB")
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
