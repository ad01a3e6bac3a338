"""The networks the benchmarks time, built exactly as their benchmarks build them (graph, input size, max_batch, dtype, seed-0 weights,
synthetic.make_frames_u8 frames), checked launch by launch with the per-element bound of tests/test_engine_kernels.py.

The engine picks its plans from max_batch (the halo work item, the items per persistent CTA, whether the step runs with programmatic
dependent launch), so the launch sequence the benchmarks time is only seen at their batch sizes.

  1. every op against float64, and the whole run against an op-by-op replay.  infer_u8 runs B frames and every buffer (its memory as it
     stands: a buffer whose final content a fused epilogue never stores may still carry earlier ops' results) and both outputs are
     hashed per frame.  Then the ops run again one launch group at a time (debug_run_ops): a group is an op and
     the ops its launch covers (kernel "none": the im2col op of a fused u8 stem, a max-pool fused into the halo epilogue, a 1x1
     depthwise op fused into a conv epilogue, the second op of a dw_tma<2> pair; on the TF32 engine the im2col op and the conv that
     reads it are one group too, checked from the frames).  Before a group runs, its output channels hold a NaN sentinel (channels it
     also reads keep theirs), and so do both conf / PAF planes when it writes them; afterwards
       (a) frames 0, 1 and B - 1 of every output are within
               |got - ref| <= 2^-11 |ref| + (K + 2) 2^-23 mag + 2^-24
           of a float64 reference computed from the engine's own inputs (oracle/torch_backbone.run_graph on the group's ops, operands
           on the engine's grid, stores unrounded, mag from its magnitude pass).  K = R S (cin_g rounded up to 64, 32 on TF32), or the
           tap count of a depthwise op.  The conf / PAF planes of the split output conv hold the unrounded fp32 result: no 2^-11 term.
           A group with a fused 1x1 depthwise op rounds the tensor in between to fp16 (bit for bit as two launches do), an error of at
           most 2^-11 |y| on each input y of the depthwise stage; carried through its weight w that is 2^-11 |w y| <= 2^-11 mag, added
           to the bound.  A fused max-pool takes the max of values within their bounds, so the pooled bound is the conv's on the
           pooled magnitudes, as in the kernel suite's pool cases.  A stand-alone max-pool is exact and compared bit for bit.  The
           OpenPifPaf and PPN head ops are checked with their own suites' float64 references, within 2^-20 |ref| + 2^-40.
           Frames are independent: frames 0 and 1 cover the tiles that straddle two images, B - 1 the last, ragged tile;
       (b) the channels of every output buffer outside the group's ranges keep their bits (all B frames);
       (c) the bound rejects a wrong reference: for the first op of every conv kernel name, filter taps zeroed (_tap_mutant) change
           frame 0's outputs, and more than half of the changed outputs break the bound;
     and after the last group every buffer and both outputs, all B frames, are byte-identical to the whole run.  The kernels are
     deterministic; the two runs differ only in launch order on the stream (no host synchronisation between the whole run's kernels,
     PDL where the engine uses it), so a kernel that exits before its stores land, or reads before its producer finished, shows here.
     One line per group is printed: kernels, epilogue, work items / CTAs of each conv launch, worst |got - ref| / bound.
  2. a short batch at the benchmark plans: after a full run, frames N' = B/2 + 1 .. B - 1 of every buffer hold NaN, and infer_u8 on
     N' frames must reproduce the full run's frames < N' byte for byte and leave every byte of frames >= N' as it was.
  3. the pipelined pose call (submit_pose / collect_pose, a captured CUDA graph; OpenPifPaf with SMs reserved for the decoder) computes
     every buffer and both outputs byte for byte as infer_u8 does.
  4. the frame resize at camera sizes: every case of make_golden.RESIZE_CASES, with and without keep_ratio, bit-exact against the
     oracle (pinned to cv2 by sha), and a mixed batch whose staging regions grow between frames.
The INT8 configs are tools/bench_int8.py's engines (cfg3, cfg4, cfg2 at their batches), with the scales it uses: a TF32 engine of
the same max_batch calibrates one batch of seed-500 frames.  The INT8 engine launches every op on its own (its im2col op is a group,
whose patch buffer, pad channels included, is an output; the stem conv reads the patches), and its kernels are specified to the
byte, so tests 1 and 2 hold it to tests/int8_sim.py exactly rather than within a bound:
  1. the sentinel is -128 (quantize_i8 clamps to +-127, so no kernel stores it; the conf / PAF planes keep NaN), and
       (a) every output byte and every conf / PAF value of frames 0, 1 and B - 1 equals int8_sim.run_graph on the group's ops, from
           the engine's own inputs and the buffers' scales (the integer convolutions on the GPU: float64, exact in any order);
       (c) an exact comparison passes vacuously only on outputs that do not depend on the inputs: every output holds >= 16
           distinct values, and for the first op of every conv kernel name the tap-mutated reference changes >= 1 % of frame 0's
           outputs.  The printed line gives the distinct values and the fraction of int8 outputs at +-127.
     (b) and the whole-run identity are as above.
  2. frames >= N' hold -128.
The CPU tests at the end check the harness itself: chaining the per-group references over the reference's own buffers reproduces
run_graph of the whole graph exactly, and the per-group int8_sim references reproduce int8_sim.run_graph byte for byte."""
import copy
import hashlib
import os
import time

import numpy as np
import pytest
import torch

import oracle
from hyperpose_b200 import capi, models, synthetic as syn
from oracle import torch_backbone
from tests import int8_sim
from tests.golden.make_golden import RESIZE_CASES, sha
from tests.ppn_head_ref import ppn_head_ref
from tests.test_engine_kernels import _r, work_items
from tests.test_pifpaf_stages import _head_ref

gpu = pytest.mark.gpu

# (id, graph, H, W, max_batch, dtype) as bench.py (cfg2 .. cfg5 and its TF32 line), tools/bench_lw.py and tools/bench_ppn.py build them
CONFIGS = [("cfg3", "openpose_vgg19", 368, 656, 16, "f16"), ("cfg3-tf32", "openpose_vgg19", 368, 656, 16, "tf32"),
           ("cfg2", "mobilenet_thin_openpose", 368, 432, 8, "f16"), ("cfg4", "resnet50_lw_openpose", 368, 432, 32, "f16"),
           ("cfg5", "resnet50_pifpaf", 385, 385, 16, "f16"),
           ("lw_vggtiny-256x384", "lw_openpose_vggtiny", 256, 384, 16, "f16"), ("lw_vggtiny-342x368", "lw_openpose_vggtiny", 342, 368, 16, "f16"),
           ("lw_resnet18", "lw_openpose_resnet18", 368, 432, 16, "f16"),
           ("lw_mobilenet_dilated", "lw_openpose_mobilenet_dilated", 368, 432, 16, "f16"),
           ("ppn_resnet18", "ppn_resnet18", 384, 384, 16, "f16"), ("ppn_resnet18-tf32", "ppn_resnet18", 384, 384, 16, "tf32"),
           ("ppn_resnet50", "ppn_resnet50", 384, 384, 16, "f16"), ("ppn_resnet50-tf32", "ppn_resnet50", 384, 384, 16, "tf32"),
           # tools/bench_int8.py: the INT8 engine, its scales calibrated on seed-500 frames by a TF32 engine of the same max_batch
           ("cfg3-int8", "openpose_vgg19", 368, 656, 16, "int8"), ("cfg4-int8", "resnet50_lw_openpose", 368, 432, 32, "int8"),
           ("cfg2-int8", "mobilenet_thin_openpose", 368, 432, 8, "int8")]
CFG = {c[0]: c for c in CONFIGS}
INT8 = [c[0] for c in CONFIGS if c[5] == "int8"]
FRAME_SEED = 2
CAL_SEED = 500
HEADS = (models.OP_PIFPAF_HEAD, models.OP_PPN_HEAD)


# ---- launch groups and their float64 reference (no GPU) ---------------------------------------------------------------------
def _op_reads(op):
    """[(buffer, first channel, channels)] op reads from activation buffers (an im2col op reads the frames; the conv after it, the
    patches)"""
    if op.type == models.OP_CONV:
        out = [(op.in_buf, 0, op.R * op.S * op.cin_g)] if op.im2col_input else [(op.in_buf, op.in_ch_off, op.groups * op.cin_g)]
        return out + ([(op.res_buf, op.res_ch_off, op.groups * op.cout_g)] if op.res_mode else [])
    if op.type in (models.OP_DWCONV, models.OP_MAXPOOL2):
        return [(op.in_buf, op.in_ch_off, op.cout_g)]
    if op.type == models.OP_PIFPAF_HEAD:
        return [(op.in_buf, 0, None), (op.res_buf, 0, None)]
    if op.type == models.OP_PPN_HEAD:
        return [(op.in_buf, 0, None)]
    return []


def _op_writes(op):
    """[(buffer | "conf" | "paf", first channel, channels)] op writes; None channels: the whole buffer"""
    if op.type == models.OP_IM2COL3:
        return [(op.out_buf, 0, None)]
    if op.type in HEADS or (op.type == models.OP_CONV and op.out_mode == models.OUT_F32_NCHW_SPLIT):
        return [("conf", 0, None), ("paf", 0, None)]
    return [(op.out_buf, op.out_ch_off, op.groups * op.cout_g if op.type == models.OP_CONV else op.cout_g)]


class Group:
    """ops first .. last of graph g: one launch (and on the f16 / TF32 engines, the im2col op with the conv that reads it)"""

    def __init__(self, g, first, last, dtype):
        self.first, self.last, self.dtype = first, last, dtype
        self.ops = g.ops[first:last + 1]
        made = set()
        self.reads = []
        for op in self.ops:
            self.reads += [r for r in _op_reads(op) if r[0] not in made and r not in self.reads]
            made |= {w[0] for w in _op_writes(op)}
        self.in_bufs = sorted({r[0] for r in self.reads})
        # checked outputs: what no later op of the group reads (a fused op's input is never stored, nor the patches of a fused stem);
        # on the INT8 engine the im2col op is a group of its own, and its patch buffer, pad channels included, is an output
        self.outs = []
        for i, op in enumerate(self.ops):
            later = {r[0] for o in self.ops[i + 1:] for r in _op_reads(o)}
            self.outs += [w for w in _op_writes(op) if w[0] not in later]
        self.out_bufs = sorted({o[0] for o in self.outs if not isinstance(o[0], str)})
        self.stem = self.ops[0].type == models.OP_IM2COL3
        self.head = self.ops[-1].type in HEADS
        self.pool = self.ops[-1].type == models.OP_MAXPOOL2 and len(self.ops) == 1
        self.conv = next((i for i, op in enumerate(self.ops) if op.type == models.OP_CONV), None)
        self.dw1 = self.conv is not None and self.ops[-1].type == models.OP_DWCONV   # a 1x1 depthwise op in a conv's epilogue (a stem's too)
        chunk = {"f16": 64, "tf32": 32, "int8": 128}[dtype]
        lead = self.ops[self.conv] if self.conv is not None else self.ops[0]
        if self.conv is not None and lead.im2col_input:   # the patch channels, as the kernel suite's stem cases count them
            self.K = _r(lead.R * lead.S * 3, 64)
        elif self.conv is not None:
            self.K = lead.R * lead.S * _r(lead.cin_g, chunk)
        else:
            self.K = lead.R * lead.S
        # the sub-graph: the group's ops over the buffers they touch, renumbered
        used = sorted({b for op in self.ops for b, _, _ in _op_reads(op) + _op_writes(op) if not isinstance(b, str)})
        remap = {b: i for i, b in enumerate(used)}
        sg = copy.copy(g)
        sg.buffers = [g.buffers[b] for b in used]
        sg.ops = []
        for op in self.ops:
            o = copy.copy(op)
            o.in_buf, o.out_buf, o.res_buf = remap.get(op.in_buf, 0), remap.get(op.out_buf, 0), remap.get(op.res_buf, 0)
            sg.ops.append(o)
        self.graph, self.used = sg, used

    def reference(self, init, frames, magnitude=False, graph=None, device="cpu"):
        """float64 run of the group's ops from buffer contents init {buffer: [N, C, H, W]} and u8 frames [N, H, W, 3], stores not
        rounded -> ({buffer: [N, C, H, W] tensor} of every buffer the ops touch, conf, paf)"""
        init = {self.used.index(b): a for b, a in init.items() if b in self.used}
        conf, paf, bufs = torch_backbone.run_graph(graph or self.graph, frames, device=device, dtype=torch.float64, init=init,
                                                   rounding="fp16" if self.dtype == "f16" else "tf32", round_stores=False, magnitude=magnitude)
        return {b: bufs[i] for i, b in enumerate(self.used)}, conf, paf

    def reference_int8(self, scales, init, frames, graph=None, device="cpu"):
        """the INT8 engine's arithmetic (tests/int8_sim.py) on the group's ops from int8 buffer contents init {buffer: [N, C, H, W]}
        and u8 frames [N, H, W, 3] (the patches of an im2col op; the geometry of the others), with the graph's scale table `scales`
        -> ({buffer: int8 [N, C, H, W]} of every buffer the ops touch, conf, paf)"""
        init = {self.used.index(b): a for b, a in init.items() if b in self.used}
        conf, paf, bufs = int8_sim.run_graph(graph or self.graph, np.asarray(scales, np.float32)[self.used], frames_u8=frames, init=init,
                                             device=device)
        return {b: bufs[i] for i, b in enumerate(self.used)}, conf, paf


def launch_groups(g, kernels, dtype):
    """the graph's launch groups from the kernel names of its ops (Engine.debug_op_kernel).  The INT8 engine launches every op on
    its own (no fusion, no halo kernel, no PDL): its im2col op (im2col_i8) is a group, and so is the conv that reads the patches."""
    spans = []
    for i, (op, k) in enumerate(zip(g.ops, kernels)):
        if op.type == models.OP_CONV and op.im2col_input and dtype != "int8":
            assert spans and g.ops[spans[-1][0]].type == models.OP_IM2COL3 and spans[-1][1] == i - 1 and g.ops[i - 1].out_buf == op.in_buf, \
                f"op {i}: a conv on im2col patches that does not follow its im2col op"
            spans[-1][1] = i
        elif k == "none" and op.type != models.OP_IM2COL3:
            assert spans, f"op {i}: nothing launches it"
            spans[-1][1] = i
        else:
            spans.append([i, i])
    return [Group(g, a, b, dtype) for a, b in spans]


def _fusable_kernels(g):
    """kernel names as the fp16 engine's fusion rules would give them where they apply to this graph, without a GPU: "none" for the
    im2col op, a max-pool right after the conv that makes its input, a stride-1 1x1 depthwise op right after the conv that makes its
    input, and the second of two depthwise 3x3 ops on the same input range"""
    names = []
    for i, op in enumerate(g.ops):
        prev = g.ops[i - 1] if i else None
        fused = op.type == models.OP_IM2COL3
        if prev is not None and prev.type == models.OP_CONV and prev.out_mode == models.OUT_F16_NHWC and op.in_buf == prev.out_buf and \
                op.in_ch_off == prev.out_ch_off:
            fused |= op.type == models.OP_MAXPOOL2 or (op.type == models.OP_DWCONV and op.R == 1 and op.stride == 1)
        if prev is not None and prev.type == op.type == models.OP_DWCONV and names[-1] != "none" and op.R == prev.R == 3 and \
                op.stride == prev.stride == 1 and (op.in_buf, op.in_ch_off, op.cout_g) == (prev.in_buf, prev.in_ch_off, prev.cout_g):
            fused = True
        names.append("none" if fused else "op")
    return names


# ---- engine side ------------------------------------------------------------------------------------------------------------
def _clean_env(monkeypatch):
    for k in list(os.environ):
        if k.startswith("HPB_"):
            monkeypatch.delenv(k)


def _build(cid, monkeypatch):
    _, name, H, W, B, dtype = CFG[cid]
    _clean_env(monkeypatch)
    g = getattr(models, name)(seed=0)
    if dtype == "int8":   # as tools/bench_int8.py: one max_batch of calibration frames through a TF32 engine
        cal = capi.Engine(g.to_pack(), (W, H), max_batch_size=B, dtype="tf32")
        g.set_int8_scales(cal.calibrate(syn.make_frames_u8(CAL_SEED, B, H, W)))
        cal.close()
    eng = capi.Engine(g.to_pack(), (W, H), max_batch_size=B, dtype=dtype)
    return g, eng, syn.make_frames_u8(FRAME_SEED, B, H, W)


def _frame_hashes(a):
    return [hashlib.blake2b(np.ascontiguousarray(a[i]).tobytes(), digest_size=16).digest() for i in range(a.shape[0])]


def _read(eng, bi, n):
    """n frames of buffer bi's memory as it stands: also a buffer whose final content a fused epilogue never stores (MobilenetThin's
    ping-pong buffers after their last 1x1 depthwise op), which earlier ops still write and read"""
    return eng.debug_read_buffer(bi, n, raw=True)


def _state(eng, bufs, n):
    """{buffer | "conf" | "paf": per-frame hashes of n frames}"""
    st = {bi: _frame_hashes(_read(eng, bi, n)) for bi in bufs}
    conf, paf = eng.read_outputs(n)
    st["conf"], st["paf"] = _frame_hashes(conf), _frame_hashes(paf)
    return st


def _diff_state(a, b, frames=None):
    """[(buffer, frame)] where the hashes differ"""
    return [(k, i) for k in a for i in (frames if frames is not None else range(len(a[k]))) if a[k][i] != b[k][i]]


def _buf_hw(g, bi, H, W):
    d = g.buffers[bi][1]
    for _ in range(d):
        H, W = (H + 1) // 2, (W + 1) // 2
    return H, W


def _launch_info(eng, g, grp, B, H, W, sms):
    """printable kernels, epilogue and work items / CTAs of the group's launches"""
    parts = []
    for i in range(grp.first, grp.last + 1):
        k = eng.debug_op_kernel(i)
        if k == "none":
            continue
        s = k
        if k.startswith("conv<"):
            s += f"[{eng.debug_op_conv_epilogue(i)}]"
        elif k.startswith("halo<"):
            s += f"[{eng.debug_op_epilogue(i)}]"
        if k.startswith(("conv<", "halo<")):
            h, w = _buf_hw(g, g.ops[i].in_buf, H, W)
            items = work_items(k, g.ops[i], B, h, w)
            s += f" {items} items on {min(sms, items)} CTAs"
        parts.append(s)
    return ", ".join(parts)


def _nchw(a, sel):
    return a[sel].astype(np.float64).transpose(0, 3, 1, 2)


def _bound(grp, ref, mag, plane):
    b = (0.0 if plane else 2.0 ** -11) * np.abs(ref) + (grp.K + 2) * 2.0 ** -23 * mag + 2.0 ** -24
    return b + 2.0 ** -11 * mag if grp.dw1 else b


def _ratio(got, ref, bound):
    return np.abs(got - ref) / bound


def _tap_mutant(g, i):
    """g with the filter of conv op i missing taps: the centre tap of a 3 x 3 filter, the centre 3 x 3 taps of a larger one, the first
    8 input channels of a 1 x 1 filter (the network's pointwise convs pad their input channels with zero weights at the end).  One tap
    of a 7 x 7 filter over 185 channels (K = 9408) is too small a change for the accumulation term of the bound: it broke it on 46 % of
    the changed outputs of OpenPose's first refinement conv."""
    g = copy.deepcopy(g)
    w = g.ops[i].weight                      # [G, cout_g, cin_g, R, S]
    R, S = w.shape[-2:]
    if (R, S) == (1, 1):
        w[:, :, :8] = 0
    else:
        r, s = (1, 1) if R * S <= 9 else (3, 3)
        w[..., R // 2 - r // 2:R // 2 + r // 2 + 1, S // 2 - s // 2:S // 2 + s // 2 + 1] = 0
    return g


def _check_group(grp, eng, g, ins, got, planes, frames, sel, mutate, dev):
    """(a) and (c) for one group -> worst |got - ref| / bound"""
    H, W = frames.shape[1:3]
    fr = frames[sel]
    if grp.head:
        op = grp.ops[-1]
        if op.type == models.OP_PIFPAF_HEAD:
            ho, wo = eng.out_h, eng.out_w
            pairs = [(planes["conf"][sel].reshape(len(sel), 17, 5, ho, wo), _head_ref(ins[op.in_buf][sel], 17, 5, False)[0]),
                     (planes["paf"][sel].reshape(len(sel), 19, 9, ho, wo), _head_ref(ins[op.res_buf][sel], 19, 9, True)[0])]
        else:
            K, E = eng.c_conf // 6, eng.c_paf
            rbox, redge = ppn_head_ref(_nchw(ins[op.in_buf], sel), K, E, H, W)
            pairs = [(planes["conf"][sel], rbox), (planes["paf"][sel], redge)]
        worst = 0.0
        for gv, rv in pairs:
            r = _ratio(gv.astype(np.float64), rv, 2.0 ** -20 * np.abs(rv) + 2.0 ** -40)
            i = np.unravel_index(np.argmax(r), r.shape)
            assert r[i] <= 1.0, f"ops {grp.first}..{grp.last} (head): |got - ref| / bound {r[i]:.3f} at {i}: {gv[i]!r} vs {rv[i]!r}"
            worst = max(worst, float(r.max()))
        return worst
    init = {b: _nchw(a, sel) for b, a in ins.items()}
    ref, rconf, rpaf = grp.reference(init, fr, device=dev)
    if grp.pool:
        (b, off, c), = grp.outs
        want = ref[b][:, off:off + c].cpu().numpy().transpose(0, 2, 3, 1).astype(np.float16 if grp.dtype == "f16" else np.float32)
        assert got[b][sel][..., off:off + c].tobytes() == want.tobytes(), f"op {grp.first} (max-pool) differs from the reference"
        return 0.0
    mag, mconf, mpaf = grp.reference(init, fr, magnitude=True, device=dev)

    def pick(res, conf, paf, o):
        b, off, c = o
        if isinstance(b, str):
            return (conf if b == "conf" else paf).cpu().numpy()
        return res[b][:, off:off + c].cpu().numpy()

    def mine(o):
        b, off, c = o
        return planes[b][sel].astype(np.float64) if isinstance(b, str) else _nchw(got[b][..., off:off + c], sel)

    worst = 0.0
    bounds = []
    for o in grp.outs:
        r, m, gv = pick(ref, rconf, rpaf, o), pick(mag, mconf, mpaf, o), mine(o)
        bd = _bound(grp, r, m, isinstance(o[0], str))
        bounds.append(bd)
        assert np.isfinite(gv).all(), f"ops {grp.first}..{grp.last}: {o[0]}: non-finite output at {np.argwhere(~np.isfinite(gv))[0].tolist()}"
        q = _ratio(gv, r, bd)
        i = np.unravel_index(np.argmax(q), q.shape)
        assert q[i] <= 1.0, (f"ops {grp.first}..{grp.last} ({grp.ops[-1].name}): {o[0]}: |got - ref| = {abs(gv[i] - r[i]):.3e} > bound {bd[i]:.3e} "
                             f"at frame {sel[i[0]]}, channel {i[1]}, pixel {i[2:]} (got {gv[i]}, ref {r[i]})")
        worst = max(worst, float(q.max()))
    if mutate:   # (c) on frame 0
        mg = _tap_mutant(grp.graph, grp.conv)
        mref, mconf, mpaf = grp.reference({b: a[:1] for b, a in init.items()}, fr[:1], graph=mg, device=dev)
        changed = broken = 0
        for o, bd in zip(grp.outs, bounds):
            r, mr, gv = pick(ref, rconf, rpaf, o)[:1], pick(mref, mconf, mpaf, o), mine(o)[:1]
            ch = mr != r
            changed += int(ch.sum())
            broken += int((np.abs(gv - mr) > bd[:1])[ch].sum())
        assert changed > 0, f"ops {grp.first}..{grp.last}: the tap mutation changes nothing"
        assert broken > 0.5 * changed, f"ops {grp.first}..{grp.last}: the bound accepts the tap-mutated reference on {changed - broken} of {changed} changed outputs"
    return worst


def _check_group_int8(grp, g, ins, got, planes, frames, sel, mutate, dev):
    """(a) and (c) for one group of the INT8 engine -> (fewest distinct values in one of its outputs, fraction of its int8 outputs
    at +-127)"""
    fr = frames[sel]
    init = {b: np.ascontiguousarray(a[sel].transpose(0, 3, 1, 2)) for b, a in ins.items()}
    ref, rconf, rpaf = grp.reference_int8(g.act_scales, init, fr, device=dev)

    def pick(res, conf, paf, o):
        b, off, c = o
        if isinstance(b, str):
            return conf if b == "conf" else paf
        return res[b][:, off:None if c is None else off + c]

    def mine(o):
        b, off, c = o
        return planes[b][sel] if isinstance(b, str) else got[b][sel][..., off:None if c is None else off + c].transpose(0, 3, 1, 2)

    def bits(a):   # int8 bytes as they are, fp32 planes by their bit patterns
        return a.view(np.uint32) if a.dtype == np.float32 else a

    distinct, sat, n = [], 0, 0
    for o in grp.outs:
        r, gv = np.ascontiguousarray(pick(ref, rconf, rpaf, o)), np.ascontiguousarray(mine(o))
        bad = np.argwhere(bits(gv) != bits(r))
        assert bad.size == 0, (f"ops {grp.first}..{grp.last} ({grp.ops[-1].name}): {o[0]}: {len(bad)} of {r.size} values differ from the INT8 model, "
                               f"first at frame {sel[bad[0][0]]}, channel {bad[0][1]}, pixel {bad[0][2:].tolist()}: got {gv[tuple(bad[0])]}, "
                               f"want {r[tuple(bad[0])]}")
        distinct.append(len(np.unique(gv)))
        if gv.dtype == np.int8:
            sat += int(((gv == 127) | (gv == -127)).sum())
            n += gv.size
    assert min(distinct) >= 16, f"ops {grp.first}..{grp.last}: an output holds {min(distinct)} distinct values: the exact comparison says little"
    if mutate:   # (c) on frame 0: the reference depends on the taps
        mg = _tap_mutant(grp.graph, grp.conv)
        mref, mconf, mpaf = grp.reference_int8(g.act_scales, {b: a[:1] for b, a in init.items()}, fr[:1], graph=mg, device=dev)
        changed = total = 0
        for o in grp.outs:
            r, mr = pick(ref, rconf, rpaf, o)[:1], pick(mref, mconf, mpaf, o)
            changed += int((bits(np.ascontiguousarray(mr)) != bits(np.ascontiguousarray(r))).sum())
            total += r.size
        assert changed >= 0.01 * total, f"ops {grp.first}..{grp.last}: the tap mutation changes {changed} of {total} outputs of frame 0"
    return min(distinct), sat / n if n else 0.0


def _replay(g, eng, frames, groups, B, dev, cid):
    """steps 3 .. 5 of test 1 for every group, in order -> worst ratio of the network (0 on the INT8 engine: every group is exact)"""
    H, W = frames.shape[1:3]
    sel = sorted({0, 1, B - 1})
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    int8 = eng.dtype == "int8"
    # the sentinel: NaN, or on the INT8 engine -128, which no kernel stores (quantize_i8 clamps to +-127)
    nan = np.float16(np.nan) if eng.dtype == "f16" else np.int8(-128) if int8 else np.float32(np.nan)
    mutated, worst = set(), 0.0
    for grp in groups:
        ins = {b: _read(eng, b, B) for b in grp.in_bufs}
        before = {b: (ins[b] if b in ins else _read(eng, b, B)) for b in grp.out_bufs}
        written = {b: np.zeros(before[b].shape[-1], bool) for b in grp.out_bufs}
        for b, off, c in grp.outs:
            if not isinstance(b, str):
                written[b][off:None if c is None else off + c] = True
        for b in grp.out_bufs:
            s = before[b].copy()
            keep = ~written[b]
            for rb, off, c in grp.reads:   # channels the group also reads, up to its padded K chunks, keep their contents (an INT8
                if rb == b:                # k-step past the channels read meets zero weights: -128 there adds nothing)
                    c = c if c is not None else s.shape[-1]
                    keep[off:off + (c if int8 else _r(c, 64))] = True
            s[..., ~keep] = nan
            eng.debug_write_buffer(b, s)
        writes_planes = any(isinstance(o[0], str) for o in grp.outs)
        if writes_planes:   # the output conv or head writes every element of both planes
            conf, paf = eng.read_outputs(B)
            eng.debug_write_outputs(np.full_like(conf, np.nan), np.full_like(paf, np.nan))
        eng.debug_run_ops(grp.first, grp.last, B)
        got = {b: _read(eng, b, B) for b in grp.out_bufs}
        planes = dict(zip(("conf", "paf"), eng.read_outputs(B))) if writes_planes else None
        for b in grp.out_bufs:   # (b)
            keep = ~written[b]
            assert got[b][..., keep].tobytes() == before[b][..., keep].tobytes(), \
                f"{cid}: ops {grp.first}..{grp.last}: buffer {b}: channels outside the outputs were written"
        kernels = [eng.debug_op_kernel(i) for i in range(grp.first, grp.last + 1)]
        conv_k = next((k for k in kernels if k.startswith(("conv<", "halo<"))), None)
        mutate = conv_k is not None and conv_k not in mutated and grp.conv is not None
        if mutate:
            mutated.add(conv_k)
        info = _launch_info(eng, g, grp, B, H, W, sms) or kernels[0]
        if int8:
            distinct, sat = _check_group_int8(grp, g, ins, got, planes, frames, sel, mutate, dev)
            print(f"[network ops] {cid} ops {grp.first}..{grp.last} {grp.ops[-1].name}: {info}; byte-exact, {distinct} distinct values, "
                  f"{sat:.4f} at +-127" + (" (the tap mutation changes the reference)" if mutate else ""))
            continue
        w = _check_group(grp, eng, g, ins, got, planes, frames, sel, mutate, dev)
        worst = max(worst, w)
        print(f"[network ops] {cid} ops {grp.first}..{grp.last} {grp.ops[-1].name}: {info}; "
              f"worst |got - ref| / bound {w:.3f}" + (" (bound rejects the tap mutation)" if mutate else ""))
    return worst, mutated


def _ref_device():
    return "cuda" if torch.cuda.is_available() else "cpu"


@gpu
@pytest.mark.parametrize("cid", [c[0] for c in CONFIGS])
def test_network_ops_against_fp64_and_replay(cid, monkeypatch):
    """test 1: every launch group of the benchmark's engine against float64, and the op-by-op replay byte-identical to the whole run"""
    t0 = time.time()
    g, eng, frames = _build(cid, monkeypatch)
    B = frames.shape[0]
    kernels = [eng.debug_op_kernel(i) for i in range(len(g.ops))]
    bufs = range(len(g.buffers))
    eng.infer_u8(frames)
    whole = _state(eng, bufs, B)
    groups = launch_groups(g, kernels, eng.dtype)
    worst, mutated = _replay(g, eng, frames, groups, B, _ref_device(), cid)
    replay = _state(eng, bufs, B)
    bad = _diff_state(whole, replay)
    assert not bad, f"{cid}: the op-by-op replay differs from the whole run at (buffer, frame) {bad[:8]} ({len(bad)} in all)"
    assert mutated, f"{cid}: no conv kernel"
    print(f"[network ops] {cid}: {len(groups)} launch groups, PDL {eng.debug_uses_pdl()}, conv kernels {sorted(mutated)}; " +
          ("every group byte-exact" if eng.dtype == "int8" else f"worst |got - ref| / bound {worst:.3f}") + f"; {time.time() - t0:.1f} s")
    eng.close()


@gpu
def test_some_benchmark_network_runs_with_pdl(monkeypatch):
    """the replay test above sees a PDL chain only if some benchmark engine launches with programmatic dependent launch (cfg2 does
    today; which others do is a heuristic of the work per launch, not asserted)"""
    pdl = {}
    for cid, _, H, W, B, _ in sorted(CONFIGS, key=lambda c: c[2] * c[3] * c[4]):   # the least work per step first; stop at the first
        g, eng, _ = _build(cid, monkeypatch)
        pdl[cid] = eng.debug_uses_pdl()
        eng.close()
        if pdl[cid]:
            break
    print(f"[network ops] PDL: {pdl}")
    assert any(pdl.values()), pdl


@gpu
@pytest.mark.parametrize("cid", [c[0] for c in CONFIGS])
def test_short_batch_at_benchmark_plans(cid, monkeypatch):
    """test 2: infer_u8 on N' = B/2 + 1 frames of the benchmark engine: frames < N' as in the full run, frames >= N' untouched"""
    g, eng, frames = _build(cid, monkeypatch)
    B = frames.shape[0]
    n = B // 2 + 1
    bufs = range(len(g.buffers))
    eng.infer_u8(frames)
    full = _state(eng, bufs, B)
    sentinel = {}
    for bi in bufs:
        a = _read(eng, bi, B)
        a[n:] = -128 if eng.dtype == "int8" else np.nan
        eng.debug_write_buffer(bi, a)
        sentinel[bi] = _frame_hashes(a)
    eng.infer_u8(frames[:n])
    short = _state(eng, bufs, B)
    bad = _diff_state(full, short, range(n))
    assert not bad, f"{cid}: frames < {n} of the short batch differ from the full run at (buffer, frame) {bad[:8]}"
    past = [(bi, i) for bi in bufs for i in range(n, B) if short[bi][i] != sentinel[bi][i]]
    past += [(k, i) for k in ("conf", "paf") for i in range(n, B) if short[k][i] != full[k][i]]
    assert not past, f"{cid}: the {n}-frame batch wrote past frame {n} at (buffer, frame) {past[:8]}"
    eng.close()


@gpu
@pytest.mark.parametrize("cid", ["cfg3", "cfg5", "cfg3-int8"])
def test_pipelined_pose_call_matches_infer(cid, monkeypatch):
    """test 3: submit_pose / collect_pose (a captured CUDA graph for the PAF parser; for OpenPifPaf, conv grids narrowed by the SMs
    reserved for the decoder) compute every buffer and both outputs as infer_u8 does.  The parsers only read the outputs."""
    g, eng, frames = _build(cid, monkeypatch)
    B = frames.shape[0]
    bufs = range(len(g.buffers))
    eng.infer_u8(frames)
    direct = _state(eng, bufs, B)
    conf, paf = eng.read_outputs(B)
    if eng.head_type == 1:
        parser = capi.PifPafParser(eng.in_h, eng.in_w, 0.1)
    else:
        parser = capi.PafParser(float(np.quantile(conf[:, :18], 0.97)), float(np.quantile(paf, 0.5)))
        parser.set_capacity(peaks_per_part=1024, candidates_per_limb=1 << 15, humans=128)
    humans = eng.collect_pose(eng.submit_pose(parser, frames), cap=128)
    piped = _state(eng, bufs, B)
    bad = _diff_state(direct, piped)
    assert not bad, f"{cid}: the pipelined call differs from infer_u8 at (buffer, frame) {bad[:8]}"
    assert len(humans) == B
    if eng.head_type != 1:   # (random weights give OpenPifPaf fields without people: its decode is tested in test_pifpaf_stages.py)
        want = parser.process_batch(conf, paf, cap=128)
        assert all(a.tobytes() == b.tobytes() for a, b in zip(humans, want)), f"{cid}: pipelined humans differ from a parse of the outputs"
        assert eng.pose_stats()["graph_captures"] >= 1
    parser.close()
    eng.close()


# ---- frame resize at camera sizes -------------------------------------------------------------------------------------------
def _resize_src(i):
    sh, sw, _, _ = RESIZE_CASES[i]
    return np.random.default_rng(200 + i).integers(0, 256, (sh, sw, 3), dtype=np.uint8)


@gpu
def test_frame_resize_every_pinned_case(golden_dir):
    """test 4a: every RESIZE_CASES source into its network size, plain and letterboxed (keep_ratio), bit-exact against the oracle
    and the cv2 sha it is pinned to"""
    pin = np.load(os.path.join(golden_dir, "cv_pin.npz"))
    by_dst = {}
    for i, (_, _, dh, dw) in enumerate(RESIZE_CASES):
        by_dst.setdefault((dh, dw), []).append(i)
    for (dh, dw), idx in by_dst.items():
        eng = capi.Engine(models.tiny_test_net(0).to_pack(), (dw, dh), max_batch_size=2)
        for i in idx:
            img = _resize_src(i)
            for slot, keep in enumerate((False, True)):
                eng.stage_frame(slot, img, keep_ratio=keep)
            got = eng.debug_read_frames(2)
            for slot, keep in enumerate((False, True)):
                want = oracle.resize_linear_u8(img, dh, dw, letterbox=keep)
                assert np.array_equal(got[slot], want), f"case {i} {img.shape[:2]} -> {dh}x{dw} keep_ratio={keep}: max |diff| " \
                                                        f"{np.abs(got[slot].astype(int) - want.astype(int)).max()}"
                assert sha(got[slot]) == str(pin[f"{'lb' if keep else 'rz'}{i}_sha"])
        eng.close()


@gpu
def test_frame_resize_mixed_camera_batch():
    """test 4b: one batch of 720p, 1080p, identity, 736 x 1312 (the exact-2x area path) and 1080p frames into 368 x 656, keep_ratio
    alternating: the staging regions grow mid-batch and the tables are uploaded again between frames.  Every frame is bit-exact, and
    infer_staged computes what infer_u8 does on the read-back frames."""
    cases = {(sh, sw): i for i, (sh, sw, dh, dw) in enumerate(RESIZE_CASES) if (dh, dw) == (368, 656)}
    order = [((720, 1280), False), ((1080, 1920), True), ((368, 656), False), ((736, 1312), True), ((1080, 1920), False)]
    g = models.tiny_test_net(0)
    eng = capi.Engine(g.to_pack(), (656, 368), max_batch_size=len(order))
    imgs = [_resize_src(cases[hw]) for hw, _ in order]
    for slot, (img, (_, keep)) in enumerate(zip(imgs, order)):
        eng.stage_frame(slot, img, keep_ratio=keep)
    got = eng.debug_read_frames(len(order))
    for slot, (img, (hw, keep)) in enumerate(zip(imgs, order)):
        want = oracle.resize_linear_u8(img, 368, 656, letterbox=keep)
        assert np.array_equal(got[slot], want), f"slot {slot} {hw} keep_ratio={keep}"
    assert np.array_equal(got[2], imgs[2])
    bufs = range(len(g.buffers))
    eng.infer_staged(len(order))
    staged = _state(eng, bufs, len(order))
    eng.infer_u8(got)
    direct = _state(eng, bufs, len(order))
    assert not _diff_state(staged, direct)
    eng.close()


# ---- the harness on the CPU -------------------------------------------------------------------------------------------------
CPU_SIZES = {"resnet50_pifpaf": (97, 97), "ppn_resnet18": (64, 64), "ppn_resnet50": (64, 64)}


@pytest.mark.parametrize("name", sorted({c[1] for c in CONFIGS}))
def test_group_references_chain_to_the_whole_graph(name):
    """the per-group float64 references, chained over their own buffers, reproduce run_graph of the whole graph bit for bit (the
    sub-graph renumbering, the init of untouched channels and the im2col / stem handling of Group.reference), on the groups the fp16
    engine's fusions would form"""
    H, W = CPU_SIZES.get(name, (64, 96))
    g = getattr(models, name)(seed=0)
    frames = syn.make_frames_u8(3, 2, H, W)
    groups = launch_groups(g, _fusable_kernels(g), "f16")
    assert any(len(grp.ops) > 1 for grp in groups)
    conf, paf, whole = torch_backbone.run_graph(g, frames, device="cpu", dtype=torch.float64, rounding="fp16", round_stores=False)
    state = [torch.zeros_like(b) for b in whole]
    cc = pc = None
    for grp in groups:
        if grp.ops[-1].type == models.OP_PPN_HEAD:   # checked against ppn_head_ref on the GPU; run_graph has no PPN head
            continue
        bufs, c, p = grp.reference({b: state[b].numpy() for b in grp.used}, frames)
        for b, t in bufs.items():
            state[b] = t
        if c is not None:
            cc, pc = c, p
    for b, (x, y) in enumerate(zip(whole, state)):
        assert torch.equal(x, y), f"{name}: buffer {b} differs"
    if conf is not None:
        assert torch.equal(conf, cc) and torch.equal(paf, pc)


@pytest.mark.parametrize("name", sorted({CFG[c][1] for c in INT8}))
def test_int8_group_references_chain_to_the_whole_graph(name):
    """the same for the INT8 engine's groups (one per op, the im2col op on its own): the per-group int8_sim references, chained over
    their own buffers, reproduce int8_sim.run_graph of the whole graph byte for byte.  Scales: set_int8_scales on per-buffer max |x|
    of a float run of the graph."""
    H, W = CPU_SIZES.get(name, (64, 96))
    g = getattr(models, name)(seed=0)
    frames = syn.make_frames_u8(3, 2, H, W)
    g.set_int8_scales(int8_sim.float_absmax(g, frames))
    groups = launch_groups(g, ["op"] * len(g.ops), "int8")
    assert len(groups) == len(g.ops) and groups[0].ops[0].type == models.OP_IM2COL3 and groups[0].outs == [(g.ops[0].out_buf, 0, None)]
    conf, paf, whole = int8_sim.run_graph(g, g.act_scales, frames_u8=frames)
    state = [np.zeros_like(b) for b in whole]
    cc = pc = None
    for grp in groups:
        bufs, c, p = grp.reference_int8(g.act_scales, {b: state[b] for b in grp.used}, frames)
        for b, a in bufs.items():
            state[b] = a
        if c is not None:
            cc, pc = c, p
    for b, (x, y) in enumerate(zip(whole, state)):
        assert x.tobytes() == y.tobytes(), f"{name}: buffer {b} differs"
    assert all(len(np.unique(whole[b])) >= 16 for b in (g.ops[0].out_buf, g.ops[-1].in_buf))   # the patches and the last features
    assert conf.tobytes() == cc.tobytes() and paf.tobytes() == pc.tobytes()
