"""Trained-weight import (SURVEY.md 8f rank 1, the exporter side of the model pack) for the four networks of the BASELINE configs:

  * OpenPose-VGG19            hyperpose/Model/openpose/model/openpose.py + backbones.py:447-509      -> ListWeights
  * MobilenetThin-OpenPose    openpose/model/mbv2_th_openpose.py + backbones.py:233-297              -> MobilenetThinWeights
  * LW-OpenPose on ResNet-50  openpose/model/lw_openpose.py + backbones.py:587-698                   -> Resnet50LwWeights
  * LW-OpenPose on TinyVGG    openpose/model/lw_openpose.py + backbones.py:343-391                   -> LwVggtinyWeights
  * LW-OpenPose on ResNet-18  openpose/model/lw_openpose.py + backbones.py:512-585                   -> LwResnet18Weights
  * LW-OpenPose on MobilenetDilated (its default backbone) lw_openpose.py + backbones.py:201-229  -> LwMobilenetDilatedWeights
  * PifPaf on ResNet-50       pifpaf/model.py:41-281 + backbones.py:587-698                          -> Resnet50PifPafWeights
  * PPN on ResNet-18 / -50    pose_proposal/model.py:14-119 + backbones.py:512-698                   -> Ppn18Weights / Ppn50Weights

The reference saves a trained model with TensorLayer's `Model.save_weights(path, format="npz")`: an ORDERED list of
arrays = `model.all_weights`, i.e. layer-creation order; most layers carry auto-generated names
(openpose.py:36-39,126-149), so position -- not name -- is the stable key, exactly how `tl.files.load_and_assign_npz`
restores them.  The `*_layer_order()` functions spell that order out with the array shapes (TensorFlow layouts:
Conv2d filters HWIO, biases [O], DepthwiseConv2d filters [kh, kw, C, 1], BatchNorm beta / gamma / moving_mean / moving_var,
PRelu alpha with `in_channels` elements); the weight classes consume such a list, checking every shape, and hand the tensors
out by the names the graph builders of models.py use.  tests/test_weights_import.py checks every network's (branch-merged,
BatchNorm-folded) graph against a plain PyTorch model written straight from the reference definition.

VGG layer names: `conv1_1 .. conv4_2`, `cpm_1/2`, `init.{conf|paf}.{1..5}` and `ref{1..5}.{conf|paf}.{1..7}`.
"""
from __future__ import annotations

import numpy as np


def openpose_vgg19_layer_order(n_stages: int = 6, n_conf: int = 19, n_paf: int = 38):
    """[(kind, name, cout, cin, k)] in `all_weights` order; kind 'conv' contributes (filters, biases), 'prelu' (alpha,)."""
    order = []
    vgg = [("conv1_1", 64, 3), ("conv1_2", 64, 64), ("conv2_1", 128, 64), ("conv2_2", 128, 128), ("conv3_1", 256, 128),
           ("conv3_2", 256, 256), ("conv3_3", 256, 256), ("conv3_4", 256, 256), ("conv4_1", 512, 256), ("conv4_2", 512, 512)]
    for name, co, ci in vgg:                                     # backbones.py:461-476 (ReLU inside the Conv2d: no extra weight)
        order.append(("conv", name, co, ci, 3))
    order += [("conv", "cpm_1", 256, 512, 3), ("conv", "cpm_2", 128, 256, 3)]   # openpose.py:36-39

    def stage(prefix, cin, layers):
        for branch, cout_last in (("conf", n_conf), ("paf", n_paf)):            # conf_block is created before paf_block (:126,:138)
            c_prev = cin
            for i, (co, k) in enumerate(layers, start=1):
                co = cout_last if co is None else co
                order.append(("conv", f"{prefix}.{branch}.{i}", co, c_prev, k))
                order.append(("prelu", f"{prefix}.{branch}.{i}", co, 0, 0))     # tl.layers.PRelu after every conv
                c_prev = co

    stage("init", 128, [(128, 3), (128, 3), (128, 3), (512, 1), (None, 1)])     # openpose.py:119-154
    for s in range(1, n_stages):                                                # openpose.py:156-199
        stage(f"ref{s}", 128 + n_conf + n_paf, [(128, 7)] * 5 + [(128, 1), (None, 1)])
    return order


class RandomWeights:
    """He-normal convs, small biases, PReLU slopes in [0.1, 0.4) -- what bench.py and the tests run on (no trained
    weights can be fetched offline).  Deterministic per (seed, layer name)."""

    def __init__(self, seed: int = 0):
        self.seed = seed

    def _rng(self, name: str, salt: int):
        return np.random.default_rng([self.seed, salt] + [ord(c) for c in name])

    def conv(self, name, cout, cin, k, gain=2.0):
        r = self._rng(name, 1)
        w = (r.standard_normal((cout, cin, k, k)) * np.sqrt(gain / (cin * k * k))).astype(np.float32)
        return w, (r.standard_normal(cout) * 0.05).astype(np.float32)

    def prelu(self, name, c):
        return self._rng(name, 2).uniform(0.1, 0.4, c).astype(np.float32)


class ListWeights:
    """An `all_weights`-ordered list of arrays (TensorFlow layouts) for openpose_vgg19."""

    def __init__(self, arrays, n_stages: int = 6):
        arrays = [np.asarray(a) for a in arrays]
        self._conv, self._prelu = {}, {}
        it = iter(arrays)
        for kind, name, co, ci, k in openpose_vgg19_layer_order(n_stages):
            try:
                if kind == "conv":
                    f, b = next(it), next(it)
                    if f.shape != (k, k, ci, co) or b.size != co:
                        raise ValueError(f"{name}: expected filters {(k, k, ci, co)} + {co} biases, got {f.shape} / {b.shape}")
                    self._conv[name] = (np.ascontiguousarray(f.transpose(3, 2, 0, 1)).astype(np.float32), b.reshape(co).astype(np.float32))
                else:
                    a = next(it)
                    if a.size != co:
                        raise ValueError(f"{name}: expected {co} PRelu slopes, got shape {a.shape}")
                    # TensorLayer 2.2.3 (requirements.txt:6) constrains the slope: PRelu.build creates
                    # `alpha_var_constrained = tf.nn.sigmoid(alpha_var)` and forward computes relu(x) - sigmoid(alpha) * relu(-x);
                    # the SAVED array is the raw variable (init ~N(0, 0.05) => slope ~0.5), so the slope the pack needs is sigmoid(alpha).
                    self._prelu[name] = (1.0 / (1.0 + np.exp(-a.reshape(co).astype(np.float64)))).astype(np.float32)
            except StopIteration:
                raise ValueError(f"weight list ends before {kind} {name}") from None
        if next(it, None) is not None:
            raise ValueError("weight list is longer than the model")

    @classmethod
    def from_npz(cls, path: str, n_stages: int = 6):
        """Either TensorLayer weight file of the reference:
          * `save_weights(format="npz")` / `tl.files.save_npz`: one object array under the key 'params', in all_weights order
            (hyperpose/Model/train.py:582);
          * `save_weights(format="npz_dict")` / `tl.files.save_npz_dict`: one entry per weight, keyed by the weight's name
            `<layer name>/<filters|biases|alpha>:0` (train.py:319, eval.py:109) -> `from_name_dict`."""
        # npz_dict files need no pickle; only the legacy `params` object array does.  Unpickling executes code from the file:
        # it is re-opened with allow_pickle=True only for that key, and only a file you trust should be passed here.
        z = np.load(path, allow_pickle=False)
        if "params" in z.files:
            z = np.load(path, allow_pickle=True)
            return cls(list(z["params"]), n_stages)
        return cls.from_name_dict({k: z[k] for k in z.files}, n_stages)

    @classmethod
    def from_name_dict(cls, named: dict, n_stages: int = 6):
        """Name-keyed weights -> the all_weights order.  The VGG layers carry explicit names (`conv1_1` .. `conv4_2`,
        backbones.py:461-476); every other layer of the model is created without a name (openpose.py:36-39,126-149) and gets
        TensorLayer's automatic `<class>_<counter>` (`conv2d_7`, `prelu_3`), the counter running in creation order per layer
        class -- so within a class, ascending counter == creation order, which is all that is needed to line the entries up
        with `openpose_vgg19_layer_order`.  Shapes are checked entry by entry by the constructor."""
        import re
        layers = {}
        for key, arr in named.items():
            # only the three weight kinds of the model; anything else in the file (optimizer slots, counters) is ignored
            if not key.endswith(("/filters:0", "/biases:0", "/alpha:0")):
                continue
            lname = key.split("/")[0]
            layers.setdefault(lname, []).append(np.asarray(arr))

        def split(lname):      # (filters, biases) of a conv layer | (alpha,) of a PRelu
            arrs = layers[lname]
            four = [a for a in arrs if a.ndim == 4]
            one = [a for a in arrs if a.ndim != 4]
            if len(four) == 1 and len(one) == 1:
                return [four[0], one[0]]
            if not four and len(one) == 1:
                return [one[0]]
            raise ValueError(f"layer {lname}: cannot tell filters / biases / alpha apart ({[a.shape for a in arrs]})")

        def counter(lname):
            m = re.search(r"_(\d+)$", lname)
            return int(m.group(1)) if m else 0

        order = openpose_vgg19_layer_order(n_stages)
        vgg_names = [name for kind, name, *_ in order if kind == "conv" and name.startswith("conv") and "." not in name]
        unnamed_conv = sorted((n for n in layers if n not in vgg_names and any(a.ndim == 4 for a in layers[n])), key=counter)
        unnamed_prelu = sorted((n for n in layers if n not in vgg_names and all(a.ndim != 4 for a in layers[n])), key=counter)
        ci, pi = iter(unnamed_conv), iter(unnamed_prelu)
        out = []
        try:
            for kind, name, *_ in order:
                if kind == "conv":
                    out += split(name if name in vgg_names else next(ci))
                else:
                    out += split(next(pi))
        except (StopIteration, KeyError) as e:
            raise ValueError(f"name-keyed weight file does not hold the layers of OpenPose-VGG19 with {n_stages} stages ({e!r})") from None
        if next(ci, None) is not None or next(pi, None) is not None:
            raise ValueError("name-keyed weight file holds more conv / PRelu layers than the model")
        return cls(out, n_stages)

    def conv(self, name, cout, cin, k, gain=2.0):
        w, b = self._conv[name]
        assert w.shape == (cout, cin, k, k), (name, w.shape)
        return w, b

    def prelu(self, name, c):
        return self._prelu[name]


# ------------------------------------------------------------------------------------------------------------------------
# Networks with BatchNorm (MobilenetThin-OpenPose, ResNet50 + LW-OpenPose, ResNet50-PifPaf).
# TensorLayer 2.2.3 layer weights in `all_weights` order: Conv2d -> filters HWIO [, biases]; DepthwiseConv2d -> filters
# [kh, kw, C, 1]; BatchNorm -> beta, gamma, moving_mean, moving_var (BatchNorm.build creates them in that order; the moving
# statistics are non-trainable but part of all_weights / of a saved model); epsilon 1e-5.
# ------------------------------------------------------------------------------------------------------------------------
BN_EPS = 1e-5


def _sep_block(order, name, cin, cout, k):
    """separable_block (backbones.py:241-248, mbv2_th_openpose.py:170-177): DepthwiseConv2d(no bias), BN, Conv2d 1x1 (no bias), BN"""
    order += [("dwconv", f"{name}.dw", cin, 0, k), ("bn", f"{name}.dwbn", cin, 0, 0),
              ("conv_nobias", f"{name}.pw", cout, cin, 1), ("bn", f"{name}.pwbn", cout, 0, 0)]


def mobilenet_thin_layer_order(n_stages: int = 6, n_conf: int = 19, n_paf: int = 38):
    """[(kind, name, cout, cin, k)] in all_weights order of MobilenetThinOpenpose (mbv2_th_openpose.py:36-44: backbone, init_stage,
    refinement_stage_1..5; inside a stage conf_block before paf_block, :111-128,:141-156)."""
    order = [("conv", "convblock_0.conv", 32, 3, 3), ("bn", "convblock_0.bn", 32, 0, 0)]         # conv_block (backbones.py:233-239)
    chans = [32, 64, 128, 128, 256, 256, 512, 512, 512, 512, 512, 512]                            # backbones.py:264-275
    for i in range(1, 12):
        _sep_block(order, f"convblock_{i}", chans[i - 1], chans[i], 3)

    def stage(prefix, cin, mid):
        for branch, n_out in (("conf", n_conf), ("paf", n_paf)):
            for k, (ci, co, ks) in enumerate([(cin, 128, 3), (128, 128, 3), (128, 128, 3), (128, mid, 1), (mid, n_out, 1)], start=1):
                _sep_block(order, f"{prefix}.{branch}.{k}", ci, co, ks)

    stage("init", 1152, 512)
    for s in range(1, n_stages):
        stage(f"ref{s}", 1152 + n_conf + n_paf, 128)
    return order


def load_params_npz(path: str):
    """`Model.save_weights(format="npz")`: one object array under 'params' in all_weights order (hyperpose/Model/train.py:582).
    Unpickling executes code from the file: pass only files you trust."""
    z = np.load(path, allow_pickle=False)
    if "params" not in z.files:
        raise ValueError("expected a TensorLayer save_weights(format='npz') file (key 'params'); the name-keyed npz_dict files of the "
                         "BatchNorm networks carry auto-generated layer names and are not supported")
    return list(np.load(path, allow_pickle=True)["params"])


class BnNetWeights:
    """An `all_weights`-ordered list of arrays for a network described by a layer order with kinds
    conv / conv_nobias / dwconv / bn / prelu (see the *_layer_order functions); hands the tensors out by name in the layouts
    models.py uses: conv -> ([cout, cin, k, k], bias | None), dwconv -> [C, k, k], bn -> folded (scale, shift)."""

    def __init__(self, arrays, order, eps: float = BN_EPS):
        arrays = [np.asarray(a) for a in arrays]
        self._conv, self._dw, self._bn, self._prelu = {}, {}, {}, {}
        it = iter(arrays)

        def take(name, what, shape):
            try:
                a = next(it)
            except StopIteration:
                raise ValueError(f"weight list ends before {what} of {name}") from None
            if tuple(a.shape) != tuple(shape) and a.size == int(np.prod(shape)) and a.ndim <= 1:
                a = a.reshape(shape)
            if tuple(a.shape) != tuple(shape):
                raise ValueError(f"{name}: expected {what} of shape {tuple(shape)}, got {a.shape}")
            return a.astype(np.float32)

        for kind, name, co, ci, k in order:
            if kind in ("conv", "conv_nobias"):
                f = take(name, "filters (HWIO)", (k, k, ci, co))
                b = take(name, "biases", (co,)) if kind == "conv" else None
                self._conv[name] = (np.ascontiguousarray(f.transpose(3, 2, 0, 1)), b)
            elif kind == "dwconv":
                f = take(name, "depthwise filters [kh, kw, C, 1]", (k, k, co, 1))
                self._dw[name] = np.ascontiguousarray(f[:, :, :, 0].transpose(2, 0, 1))
            elif kind == "bn":
                beta, gamma, mean, var = (take(name, w, (co,)) for w in ("beta", "gamma", "moving_mean", "moving_var"))
                if np.any(var < 0):
                    raise ValueError(f"{name}: negative moving_var")
                scale = (gamma.astype(np.float64) / np.sqrt(var.astype(np.float64) + eps))
                self._bn[name] = (scale.astype(np.float32), (beta.astype(np.float64) - mean.astype(np.float64) * scale).astype(np.float32))
            elif kind == "prelu":
                a = take(name, "PRelu alpha", (co,))
                self._prelu[name] = (1.0 / (1.0 + np.exp(-a.astype(np.float64)))).astype(np.float32)   # TensorLayer constrains the slope by a sigmoid
            else:
                raise ValueError(kind)
        if next(it, None) is not None:
            raise ValueError("weight list is longer than the model")

    def conv(self, name, cout, cin, k):
        w, b = self._conv[name]
        assert w.shape == (cout, cin, k, k), (name, w.shape, (cout, cin, k, k))
        return w, b

    def dwconv(self, name, C, k):
        w = self._dw[name]
        assert w.shape == (C, k, k), (name, w.shape)
        return w

    def bn(self, name, C):
        sc, sh = self._bn[name]
        assert sc.shape == (C,), (name, sc.shape)
        return sc, sh

    def prelu(self, name, C):
        return self._prelu[name]


class MobilenetThinWeights(BnNetWeights):
    def __init__(self, arrays, n_stages: int = 6):
        super().__init__(arrays, mobilenet_thin_layer_order(n_stages))

    @classmethod
    def from_npz(cls, path: str, n_stages: int = 6):
        return cls(load_params_npz(path), n_stages)


def _resnet50_order(order, layout):
    """Resnet50_backbone (backbones.py:587-698): conv1 (no bias), bn1, then the bottleneck blocks; inside a Basic_block the
    `downsample` attribute is created before `main_block` (:660-675), so its conv / bn come first in all_weights"""
    order += [("conv_nobias", "conv1", 64, 3, 7), ("bn", "bn1", 64, 0, 0)]
    cin = 64
    for bi, (nf, nblk, st0) in enumerate(layout, start=1):
        for k in range(1, nblk + 1):
            st = st0 if k == 1 else 1
            name = f"block_{bi}_{k}"
            if st != 1 or cin != 4 * nf:
                order += [("conv_nobias", f"{name}.ds_conv1", 4 * nf, cin, 1), ("bn", f"{name}.ds_bn1", 4 * nf, 0, 0)]
            order += [("conv_nobias", f"{name}.conv1", nf, cin, 1), ("bn", f"{name}.bn1", nf, 0, 0),
                      ("conv_nobias", f"{name}.conv2", nf, nf, 3), ("bn", f"{name}.bn2", nf, 0, 0),
                      ("conv_nobias", f"{name}.conv3", 4 * nf, nf, 1), ("bn", f"{name}.bn3", 4 * nf, 0, 0)]
            cin = 4 * nf


def resnet50_lw_layer_order(n_conf: int = 19, n_paf: int = 38):
    """all_weights order of LightWeightOpenPose on Resnet50_backbone(scale_size=8) (lw_openpose.py:33-45: backbone, cpm_stage,
    init_stage, refine_stage1; :106-191 for the stages)"""
    order = []
    _resnet50_order(order, [(64, 3, 1), (128, 4, 2), (256, 6, 1), (512, 3, 1)])
    _lw_head_order(order, 2048, n_conf, n_paf)
    return order


def _lw_head_order(order, cin, n_conf: int = 19, n_paf: int = 38):
    """cpm_stage, init_stage, refine_stage1 of LightWeightOpenPose (lw_openpose.py:106-191), created after the backbone; `cin` is the
    backbone's out_channels (the CPM init_layer's input)"""
    blk = lambda name, ci, co, k: [("conv", name, co, ci, k), ("bn", name + ".bn", co, 0, 0)]   # conv_block: Conv2d(+bias) + BatchNorm
    order += [("conv", "cpm.init", 128, cin, 1)] + blk("cpm.b1", 128, 128, 3) + blk("cpm.b2", 128, 128, 3) + blk("cpm.b3", 128, 128, 3)
    order += [("conv", "cpm.end", 128, 128, 3)]
    order += [("conv", f"init.{i}", 128, 128, 3) for i in (1, 2, 3)]
    order += [("conv", "init.conf.1", 512, 128, 1), ("conv", "init.conf.2", n_conf, 512, 1), ("conv", "init.paf.1", 512, 128, 1), ("conv", "init.paf.2", n_paf, 512, 1)]
    for k in range(1, 6):
        order += [("conv", f"ref.b{k}.init", 128, 128 + n_conf + n_paf if k == 1 else 128, 1)] + blk(f"ref.b{k}.c1", 128, 128, 3) + blk(f"ref.b{k}.c2", 128, 128, 3)
    order += [("conv", "ref.conf.1", 512, 128, 1), ("conv", "ref.conf.2", n_conf, 512, 1), ("conv", "ref.paf.1", 512, 128, 1), ("conv", "ref.paf.2", n_paf, 512, 1)]


def lw_vggtiny_layer_order(n_conf: int = 19, n_paf: int = 38):
    """all_weights order of LightWeightOpenPose(backbone=vggtiny_backbone) (lw_openpose.py:33-45): vggtiny_backbone(scale_size=8)
    (backbones.py:343-391: per block a Conv2d with biases, then its BatchNorm), cpm_stage on 384 channels, init_stage, refine_stage1"""
    from .models import VGGTINY_LAYERS
    order, cin = [], 3
    for layer in VGGTINY_LAYERS:
        if layer != "pool":
            name, co = layer
            order += [("conv", name, co, cin, 3), ("bn", name + ".bn", co, 0, 0)]
            cin = co
    _lw_head_order(order, cin, n_conf, n_paf)
    return order


def lw_resnet18_layer_order(n_conf: int = 19, n_paf: int = 38):
    """all_weights order of LightWeightOpenPose(backbone=Resnet18_backbone) (lw_openpose.py:33-45): Resnet18_backbone(scale_size=8)
    (the stride does not change a weight: the same arrays as _resnet18_order), cpm_stage on 512 channels, init_stage, refine_stage1"""
    order = []
    _resnet18_order(order)
    _lw_head_order(order, 512, n_conf, n_paf)
    return order


def lw_mobilenet_dilated_layer_order(n_conf: int = 19, n_paf: int = 38):
    """all_weights order of LightWeightOpenPose on its default MobilenetDilated_backbone (lw_openpose.py:33-37, backbones.py:201-229):
    conv_block(32, 3) -- Conv2d(+bias) then BatchNorm --, eleven dw_conv_blocks as separable blocks (the dilation changes no weight's
    shape), cpm_stage on 512 channels, init_stage, refine_stage1"""
    from .models import MOBILENET_DILATED_BLOCKS
    order = [("conv", "convblock_0.conv", 32, 3, 3), ("bn", "convblock_0.bn", 32, 0, 0)]
    cin = 32
    for i, (co, _, _) in enumerate(MOBILENET_DILATED_BLOCKS, start=1):
        _sep_block(order, f"convblock_{i}", cin, co, 3)
        cin = co
    _lw_head_order(order, 512, n_conf, n_paf)
    return order


def resnet50_pifpaf_layer_order(n_pos: int = 17, n_limbs: int = 19):
    """all_weights order of the PifPaf model (pifpaf/model.py:41-51): Resnet50_backbone(use_pool=False, scale_size=32), pif_head, paf_head
    (one 1x1 Conv2d with bias each, :229,:262)"""
    order = []
    _resnet50_order(order, [(64, 3, 1), (128, 4, 2), (256, 6, 2), (512, 3, 2)])
    order += [("conv", "pif_head", n_pos * 5 * 4, 2048, 1), ("conv", "paf_head", n_limbs * 9 * 4, 2048, 1)]
    return order


def _ppn_head_order(order, cin, K: int = 18, L: int = 17, nh: int = 9, nw: int = 9):
    """PoseProposal's add_layer_1 / add_layer_2 (Conv2d 3x3 with bias, BatchNorm) and add_layer_3 (Conv2d 1x1 with bias),
    pose_proposal/model.py:43-79, created after the backbone"""
    order += [("conv", "add1", 512, cin, 3), ("bn", "add1.bn", 512, 0, 0), ("conv", "add2", 512, 512, 3), ("bn", "add2.bn", 512, 0, 0),
              ("conv", "add3", 6 * K + L * nh * nw, 512, 1)]


def _resnet18_order(order):
    """Resnet18_backbone (backbones.py:512-585): conv_1_1 (no bias), bn_1_1, then the blocks; inside a Res_block `main_block` is
    created before `down_sample` (:564-576), so the shortcut's conv / bn come last"""
    from .models import RESNET18_BLOCKS
    order += [("conv_nobias", "conv1", 64, 3, 7), ("bn", "bn1", 64, 0, 0)]
    cin = 64
    for name, nf, _, ds in RESNET18_BLOCKS:
        order += [("conv_nobias", f"{name}_1.conv", nf, cin, 3), ("bn", f"{name}_1.bn", nf, 0, 0),
                  ("conv_nobias", f"{name}_2.conv", nf, nf, 3), ("bn", f"{name}_2.bn", nf, 0, 0)]
        if ds:
            order += [("conv_nobias", f"{name}_ds.conv", nf, cin, 1), ("bn", f"{name}_ds.bn", nf, 0, 0)]
        cin = nf


def ppn_resnet18_layer_order():
    """all_weights order of PoseProposal on Resnet18_backbone(scale_size=32) (backbones.py:512-585), then the PPN head"""
    order = []
    _resnet18_order(order)
    _ppn_head_order(order, 512)
    return order


def ppn_resnet50_layer_order():
    """all_weights order of PoseProposal on Resnet50_backbone(scale_size=32, use_pool=True) (backbones.py:587-698)"""
    order = []
    _resnet50_order(order, [(64, 3, 1), (128, 4, 2), (256, 6, 2), (512, 3, 2)])
    _ppn_head_order(order, 2048)
    return order


class Ppn18Weights(BnNetWeights):
    def __init__(self, arrays):
        super().__init__(arrays, ppn_resnet18_layer_order())

    @classmethod
    def from_npz(cls, path: str):
        return cls(load_params_npz(path))


class Ppn50Weights(BnNetWeights):
    def __init__(self, arrays):
        super().__init__(arrays, ppn_resnet50_layer_order())

    @classmethod
    def from_npz(cls, path: str):
        return cls(load_params_npz(path))


class Resnet50LwWeights(BnNetWeights):
    def __init__(self, arrays):
        super().__init__(arrays, resnet50_lw_layer_order())

    @classmethod
    def from_npz(cls, path: str):
        return cls(load_params_npz(path))


class LwVggtinyWeights(BnNetWeights):
    def __init__(self, arrays):
        super().__init__(arrays, lw_vggtiny_layer_order())

    @classmethod
    def from_npz(cls, path: str):
        return cls(load_params_npz(path))


class LwResnet18Weights(BnNetWeights):
    def __init__(self, arrays):
        super().__init__(arrays, lw_resnet18_layer_order())

    @classmethod
    def from_npz(cls, path: str):
        return cls(load_params_npz(path))


class LwMobilenetDilatedWeights(BnNetWeights):
    def __init__(self, arrays):
        super().__init__(arrays, lw_mobilenet_dilated_layer_order())

    @classmethod
    def from_npz(cls, path: str):
        return cls(load_params_npz(path))


class Resnet50PifPafWeights(BnNetWeights):
    """(the PifPaf backbone is built with BatchNorm epsilon 1e-4, pifpaf/model.py:42)"""

    def __init__(self, arrays):
        super().__init__(arrays, resnet50_pifpaf_layer_order(), eps=1e-4)

    @classmethod
    def from_npz(cls, path: str):
        return cls(load_params_npz(path))
