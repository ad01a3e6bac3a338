"""ctypes binding of the C ABI declared in include/hyperpose_b200.h.

This is the only way Python (tests, bench.py, smoke) reaches the product: through the same
`extern "C"` entry points the C++ `hyperpose::parser::paf` / `hyperpose::dnn::tensorrt`
wrappers call.  The shared library must have been built in-tree (hyperpose_b200/build.py);
there is no fallback of any kind -- a missing library or a missing CUDA device raises.
"""
from __future__ import annotations

import ctypes as C
import os
import struct

import numpy as np

PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(PKG, "libhyperpose_b200.so")

N_PARTS, N_PAIRS = 18, 19
HP_OK, HP_ERR_ARG, HP_ERR_CAPACITY, HP_ERR_UNSUPPORTED, HP_ERR_CUDA, HP_ERR_BATCH = 0, -1, -2, -3, -4, -5

PART_DT = np.dtype({"names": ["has_value", "x", "y", "score"], "formats": ["<i4", "<f4", "<f4", "<f4"]})
HUMAN_DT = np.dtype([("parts", PART_DT, (N_PARTS,)), ("score", "<f4")])
PEAK_DT = np.dtype([("part_id", "<i4"), ("x", "<i4"), ("y", "<i4"), ("score", "<f4"), ("id", "<i4")])
CONN_DT = np.dtype([("cid1", "<i4"), ("cid2", "<i4"), ("score", "<f4")])
assert HUMAN_DT.itemsize == 292

# every symbol include/hyperpose_b200.h declares (tests check the library exports all of them)
EXPORTS = [
    "hp_last_error", "hp_device_count", "hp_version",
    "hp_paf_create", "hp_paf_destroy", "hp_paf_set_conf_thresh", "hp_paf_set_paf_thresh", "hp_paf_set_capacity",
    "hp_paf_process_host", "hp_paf_process_host_batched", "hp_paf_process_device", "hp_paf_fetch",
    "hp_paf_debug_peaks", "hp_paf_debug_connections", "hp_paf_launch_count", "hp_paf_copy_results_device", "hp_paf_debug_timing",
    "hp_paf_debug_plan",
]


class HyperposeError(RuntimeError):
    def __init__(self, status, msg):
        super().__init__(f"hyperpose_b200 status {status}: {msg}")
        self.status = status


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise FileNotFoundError(f"{LIB_PATH} is missing: run `python -m hyperpose_b200.build` "
                                    "(there is no CPU / PyTorch fallback)")
        L = C.CDLL(LIB_PATH)
        fp, ip, vp = C.POINTER(C.c_float), C.POINTER(C.c_int), C.c_void_p
        L.hp_last_error.restype = C.c_char_p
        L.hp_version.restype = C.c_char_p
        L.hp_device_count.restype = C.c_int
        L.hp_paf_create.argtypes = [C.POINTER(vp), C.c_float, C.c_float, C.c_int, C.c_int, C.c_int]
        L.hp_paf_destroy.argtypes = [vp]
        L.hp_paf_destroy.restype = None
        L.hp_paf_set_conf_thresh.argtypes = [vp, C.c_float]
        L.hp_paf_set_paf_thresh.argtypes = [vp, C.c_float]
        L.hp_paf_set_capacity.argtypes = [vp, C.c_int, C.c_int, C.c_int]
        L.hp_paf_process_host.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, C.c_int, ip]
        L.hp_paf_process_host_batched.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, C.c_int, ip]
        L.hp_paf_process_device.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp]
        L.hp_paf_fetch.argtypes = [vp, vp, C.c_int, ip, C.c_int]
        L.hp_paf_debug_peaks.argtypes = [vp, C.c_int, vp, C.c_int, ip]
        L.hp_paf_debug_connections.argtypes = [vp, C.c_int, C.c_int, vp, C.c_int, ip]
        L.hp_paf_launch_count.argtypes = [vp]
        L.hp_paf_launch_count.restype = C.c_longlong
        L.hp_paf_copy_results_device.argtypes = [vp, vp, vp, C.c_int, C.c_int, vp]
        _lib = L
    return _lib


def check(rc):
    if rc != HP_OK:
        raise HyperposeError(rc, lib().hp_last_error().decode())


class PafParser:
    """Mirror of hyperpose::parser::paf (include/hyperpose/operator/parser/paf.hpp:17-93):
    same constructor arguments, process(conf, paf) -> humans, set_*_thresh."""

    def __init__(self, conf_thresh: float = 0.05, paf_thresh: float = 0.05, resolution_size=(-1, -1), device: int = 0):
        self._h = C.c_void_p()
        check(lib().hp_paf_create(C.byref(self._h), conf_thresh, paf_thresh, resolution_size[0], resolution_size[1], device))

    def close(self):
        if getattr(self, "_h", None) and _lib is not None:
            _lib.hp_paf_destroy(self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_conf_thresh(self, t):
        check(lib().hp_paf_set_conf_thresh(self._h, t))

    def set_paf_thresh(self, t):
        check(lib().hp_paf_set_paf_thresh(self._h, t))

    def set_capacity(self, peaks_per_part=0, candidates_per_limb=0, humans=0):
        check(lib().hp_paf_set_capacity(self._h, peaks_per_part, candidates_per_limb, humans))

    def process(self, conf: np.ndarray, paf: np.ndarray, cap: int = 128) -> np.ndarray:
        """One frame, host tensors conf[C,H,W], paf[2L,H,W] -> structured array of HUMAN_DT."""
        conf = np.ascontiguousarray(conf, np.float32)
        paf = np.ascontiguousarray(paf, np.float32)
        if conf.ndim != 3 or paf.ndim != 3:
            raise HyperposeError(HP_ERR_ARG, "Input of PAF::PROCESS didn't meet requirements: [conf, paf], tensor.dims() == 3")
        out = np.zeros(cap, HUMAN_DT)
        n = C.c_int(0)
        check(lib().hp_paf_process_host(self._h, conf.ctypes.data, paf.ctypes.data, conf.shape[0], paf.shape[0],
                                        conf.shape[1], conf.shape[2], out.ctypes.data, cap, C.byref(n)))
        return out[:n.value].copy()

    def process_batch(self, conf: np.ndarray, paf: np.ndarray, cap: int = 128):
        """N frames conf[N,C,H,W], paf[N,2L,H,W] -> list of N structured arrays."""
        conf = np.ascontiguousarray(conf, np.float32)
        paf = np.ascontiguousarray(paf, np.float32)
        N = conf.shape[0]
        out = np.zeros((N, cap), HUMAN_DT)
        n = (C.c_int * N)()
        check(lib().hp_paf_process_host_batched(self._h, conf.ctypes.data, paf.ctypes.data, N, conf.shape[1], paf.shape[1],
                                                conf.shape[2], conf.shape[3], out.ctypes.data, cap, n))
        return [out[i, :n[i]].copy() for i in range(N)]

    def process_device(self, d_conf_ptr: int, d_paf_ptr: int, N, c_conf, c_paf, H, W, stream: int = 0):
        check(lib().hp_paf_process_device(self._h, d_conf_ptr, d_paf_ptr, N, c_conf, c_paf, H, W, stream))

    def fetch(self, N: int, cap: int = 128):
        out = np.zeros((N, cap), HUMAN_DT)
        n = (C.c_int * N)()
        check(lib().hp_paf_fetch(self._h, out.ctypes.data, cap, n, N))
        return [out[i, :n[i]].copy() for i in range(N)]

    def debug_peaks(self, frame: int = 0, cap: int = 1 << 16) -> np.ndarray:
        out = np.zeros(cap, PEAK_DT)
        n = C.c_int(0)
        check(lib().hp_paf_debug_peaks(self._h, frame, out.ctypes.data, cap, C.byref(n)))
        return out[:n.value].copy()

    def debug_connections(self, frame: int, pair_id: int, cap: int = 4096) -> np.ndarray:
        out = np.zeros(cap, CONN_DT)
        n = C.c_int(0)
        check(lib().hp_paf_debug_connections(self._h, frame, pair_id, out.ctypes.data, cap, C.byref(n)))
        return out[:n.value].copy()

    @property
    def launch_count(self) -> int:
        return int(lib().hp_paf_launch_count(self._h))

    def debug_timing(self, N: int):
        """HPB_PAF_TIMING=1: (cta[N,19,4] ns stamps: start, ordered, candidates, matched; asm[N,6]: assembly start, end | path in the low
        two bits (2 component-parallel, 1 sequential), then -- component-parallel path only -- staged, labelled, grouped, lanes done)"""
        out = np.zeros(N * (N_PAIRS * 4 + 6), np.uint64)
        lib().hp_paf_debug_timing.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        check(lib().hp_paf_debug_timing(self._h, out.ctypes.data, N))
        return out[:N * N_PAIRS * 4].reshape(N, N_PAIRS, 4), out[N * N_PAIRS * 4:].reshape(N, 6)

    PLAN_FIELDS = ("generic", "rz_mode", "tab_staged", "stage_bytes", "limb_dyn_bytes", "fast_asm", "wide_tile_rows", "wide_tile_cols")

    def debug_plan(self) -> dict:
        """the code paths the last launch took (hp_paf_debug_plan): up-maps materialised (generic) and their resize regime, up-sampling
        tables (tab_staged) and PAF planes (stage_bytes > 0) in the limb kernel's shared memory, the limb kernel's dynamic shared
        memory, component-parallel assembly (fast_asm), the peak kernel's tile rows on the direct up-sampling path (wide_tile_rows)
        and tile columns on the generic staging loop (wide_tile_cols)"""
        out = np.zeros(len(self.PLAN_FIELDS), np.int32)
        lib().hp_paf_debug_plan.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        check(lib().hp_paf_debug_plan(self._h, out.ctypes.data, len(out)))
        return dict(zip(self.PLAN_FIELDS, (int(v) for v in out)))

    def copy_results_device(self, d_humans_ptr: int, d_counts_ptr: int, N: int, cap: int, stream: int = 0):
        check(lib().hp_paf_copy_results_device(self._h, d_humans_ptr, d_counts_ptr, N, cap, stream))


def handoff_stats() -> dict:
    """counters of the device-resident engine -> parser hand-off (csrc/handoff.h)"""
    L = lib()
    if not getattr(L, "_engine_bound", False):
        _bind_engine(L)
        L._engine_bound = True
    v = [C.c_longlong() for _ in range(4)]
    check(L.hp_handoff_stats(*[C.byref(x) for x in v]))
    return dict(zip(("published", "hits", "batch_parses", "misses"), [x.value for x in v]))


def handoff_enable(on: bool):
    L = lib()
    if not getattr(L, "_engine_bound", False):
        _bind_engine(L)
        L._engine_bound = True
    check(L.hp_handoff_enable(1 if on else 0))


# ---------------------------------------------------------------------------------------------
# DNN engine
# ---------------------------------------------------------------------------------------------
EXPORTS += [
    "hp_engine_create", "hp_engine_destroy", "hp_engine_info", "hp_engine_infer_u8_host", "hp_engine_infer_u8_device",
    "hp_engine_infer_f32_host", "hp_engine_outputs", "hp_engine_read_outputs_host", "hp_engine_copy_outputs_device", "hp_engine_sync",
    "hp_engine_launch_count", "hp_engine_debug_read_buffer", "hp_engine_debug_write_buffer", "hp_engine_debug_run_ops",
    "hp_pose_run_u8_host", "hp_engine_stage_frame_u8", "hp_engine_infer_staged", "hp_engine_debug_read_frames", "hp_engine_set_output_override", "hp_engine_set_profiling", "hp_engine_get_profile",
    "hp_engine_read_outputs_frames", "hp_engine_head_type", "hp_handoff_enable", "hp_handoff_stats",
    "hp_pose_submit_u8_host", "hp_pose_collect", "hp_pose_stats", "hp_paf_prepare", "hp_paf_state", "hp_paf_copy_results_host_async",
    "hp_paf_grow_capacity", "hp_pool_create", "hp_pool_destroy", "hp_pool_size", "hp_pool_set_capacity", "hp_pool_run_u8_host",
    "hp_pool_set_output_override", "hp_pool_launch_count", "hp_default_device", "hp_handoff_device_of",
    "hp_engine_create_ex", "hp_engine_dtype", "hp_pose_submit_u8_device", "hp_engine_debug_op_kernel",
    "hp_engine_debug_op_epilogue", "hp_engine_debug_op_conv_epilogue", "hp_engine_debug_uses_pdl",
    "hp_engine_debug_read_buffer_raw", "hp_engine_debug_write_outputs",
    "hp_engine_calibrate_u8", "hp_pack_int8_calibrated", "hp_pose_debug_read_slot_frames",
]   # (+ the frame calls of FRAME_CALLS, below)


class FrameU8(C.Structure):
    """hp_frame_u8: one HWC BGR frame of any size, rows packed"""
    _fields_ = [("data", C.c_void_p), ("height", C.c_int32), ("width", C.c_int32)]


class FrameYUV420(C.Structure):
    """hp_frame_yuv420: one YUV 4:2:0 frame (BT.601 limited range) of any even size, planes pitched.  uv_step 2: semi-planar
    (NV12: v = u + 1, NV21: u = v + 1); 1: planar (I420, YV12)"""
    _fields_ = [("y", C.c_void_p), ("u", C.c_void_p), ("v", C.c_void_p), ("height", C.c_int32), ("width", C.c_int32),
                ("pitch_y", C.c_int32), ("pitch_uv", C.c_int32), ("uv_step", C.c_int32)]


# cv2's packed (3H/2, W) layouts: byte offsets of the U and V planes after the H x W luma plane, chroma pitch, chroma step
YUV420_LAYOUTS = {"nv12": lambda H, W: (H * W, H * W + 1, W, 2), "nv21": lambda H, W: (H * W + 1, H * W, W, 2),
                  "i420": lambda H, W: (H * W, H * W + H * W // 4, W // 2, 1), "yv12": lambda H, W: (H * W + H * W // 4, H * W, W // 2, 1)}


def yuv420_record(frame: np.ndarray, layout: str) -> FrameYUV420:
    """the FrameYUV420 of a host frame in cv2's packed layout: uint8 (3H/2, W), C-contiguous"""
    H, W = frame.shape[0] * 2 // 3, frame.shape[1]
    u, v, pitch_uv, step = YUV420_LAYOUTS[layout](H, W)
    p = frame.ctypes.data
    return FrameYUV420(p, p + u, p + v, H, W, W, pitch_uv, step)


class FrameInterleaved(C.Structure):
    """hp_frame_interleaved: one interleaved frame of any size (width even for 4:2:2), rows `pitch` bytes apart; `format` is a
    PIXEL_FORMATS value"""
    _fields_ = [("data", C.c_void_p), ("height", C.c_int32), ("width", C.c_int32), ("pitch", C.c_int32), ("format", C.c_int32)]


# hp_pixel_format: the value and the trailing dimension of a uint8 frame array ((H, W) for gray)
PIXEL_FORMATS = {"bgr": 0, "rgb": 1, "bgra": 2, "rgba": 3, "gray": 4, "yuyv": 5, "uyvy": 6, "yvyu": 7}
PIXEL_CHANNELS = {"bgr": 3, "rgb": 3, "bgra": 4, "rgba": 4, "gray": None, "yuyv": 2, "uyvy": 2, "yvyu": 2}


def interleaved_record(frame: np.ndarray, fmt: str) -> FrameInterleaved:
    """the FrameInterleaved of a host frame: uint8 (H, W, C) or (H, W) for gray, each row's bytes contiguous; the pitch is strides[0]"""
    return FrameInterleaved(frame.ctypes.data, frame.shape[0], frame.shape[1], frame.strides[0], PIXEL_FORMATS[fmt])


class FrameYUV420_16(C.Structure):
    """hp_frame_yuv420_16: FrameYUV420 with 16-bit samples holding `bits` significant bits, LSB-aligned (9..16; 16 for P010 /
    P016).  Pitches in bytes, uv_step in samples: 2 semi-planar (P010 / P016: v = u + 1 sample; V first: u = v + 1), 1 planar"""
    _fields_ = [("y", C.c_void_p), ("u", C.c_void_p), ("v", C.c_void_p), ("height", C.c_int32), ("width", C.c_int32),
                ("pitch_y", C.c_int32), ("pitch_uv", C.c_int32), ("uv_step", C.c_int32), ("bits", C.c_int32)]


# the uint16 (3H/2, W) layouts of submit_pose_yuv420_16, as cv2's packed 8-bit layouts with 16-bit samples: P010 / P016 (U V, NV12's
# order), the same with V first (NV21's), planar U then V (I420's: yuv420p10le / p12le / p16le) and planar V then U (YV12's)
YUV420_16_LAYOUTS = {"p016": "nv12", "p016_vu": "nv21", "i420": "i420", "yv12": "yv12"}


def yuv420_16_record(frame: np.ndarray, layout: str, bits: int) -> FrameYUV420_16:
    """the FrameYUV420_16 of a host frame: uint16 (3H/2, W) in a YUV420_16_LAYOUTS layout, C-contiguous"""
    H, W = frame.shape[0] * 2 // 3, frame.shape[1]
    u, v, pitch_uv, step = YUV420_LAYOUTS[YUV420_16_LAYOUTS[layout]](H, W)   # in samples
    p = frame.ctypes.data
    return FrameYUV420_16(p, p + 2 * u, p + 2 * v, H, W, 2 * W, 2 * pitch_uv, step, bits)


class FrameInterleaved16(C.Structure):
    """hp_frame_interleaved16: FrameInterleaved with 16-bit samples holding `bits` significant bits, LSB-aligned (9..16); `format` is
    a PIXEL_FORMATS value of bgr, rgb, bgra, rgba or gray (INTERLEAVED16_FORMATS), rows `pitch` bytes apart"""
    _fields_ = [("data", C.c_void_p), ("height", C.c_int32), ("width", C.c_int32), ("pitch", C.c_int32), ("format", C.c_int32),
                ("bits", C.c_int32)]


# the formats of submit_pose_interleaved16: the 8-bit format each one is, with 16-bit samples
INTERLEAVED16_FORMATS = {"bgr48": "bgr", "rgb48": "rgb", "bgra64": "bgra", "rgba64": "rgba", "gray16": "gray"}


def interleaved16_record(frame: np.ndarray, fmt: str, bits: int) -> FrameInterleaved16:
    """the FrameInterleaved16 of a host frame: uint16 (H, W, C) or (H, W) for gray16, each row's samples contiguous; the pitch is
    strides[0]"""
    return FrameInterleaved16(frame.ctypes.data, frame.shape[0], frame.shape[1], frame.strides[0],
                              PIXEL_FORMATS[INTERLEAVED16_FORMATS[fmt]], bits)


# The frame calls hp_pose_submit{,_pifpaf,_ppn}_frames_<format>_{host,device}: each format's record type, and the form of its calls
# that takes a per-frame rotation table (int32[N], or NULL for upright): "_rotated" names a twin of each upright call, "" the call
# itself (16-bit frames), None none (BGR frames).
FRAME_CALLS = {"u8": (FrameU8, None), "yuv420": (FrameYUV420, "_rotated"), "interleaved": (FrameInterleaved, "_rotated"),
               "yuv420_16": (FrameYUV420_16, ""), "interleaved16": (FrameInterleaved16, "")}


def frame_call(head: str, fmt: str, device: bool, rotated: bool) -> str:
    """the symbol of a frame call: head "", "_pifpaf" or "_ppn"; rotated: the form that takes a rotation table"""
    return f"hp_pose_submit{head}_frames_{fmt}{FRAME_CALLS[fmt][1] if rotated else ''}_{'device' if device else 'host'}"


def frame_calls():
    """(symbol, record type, takes a rotation table) of every frame call"""
    for fmt, (rec, rot) in FRAME_CALLS.items():
        for head in ("", "_pifpaf", "_ppn"):
            for device in (False, True):
                for rotated in ((False,) if rot is None else (True,) if rot == "" else (False, True)):
                    yield frame_call(head, fmt, device, rotated), rec, rotated


EXPORTS += [name for name, _, _ in frame_calls()]


def bits_list(bits, n: int) -> list:
    """the per-frame significant bits of a 16-bit batch, from one int or one per frame, each 9..16; anything else is refused before
    the library is called"""
    bl = [bits] * n if isinstance(bits, (int, np.integer)) else list(bits) if isinstance(bits, (list, tuple, np.ndarray)) else None
    if bl is None or len(bl) != n:
        raise HyperposeError(HP_ERR_ARG, f"bits {bits!r}: expected an int in 9..16, or one per frame ({n})")
    for i, b in enumerate(bl):
        if isinstance(b, (bool, np.bool_)) or not isinstance(b, (int, np.integer)) or not 9 <= int(b) <= 16:
            raise HyperposeError(HP_ERR_ARG, f"frame {i}: bits {b!r} is not an int in 9..16")
    return [int(b) for b in bl]


# cv::rotate's clockwise rotations, in degrees: ROTATE_90_CLOCKWISE, ROTATE_180, ROTATE_90_COUNTERCLOCKWISE, and upright
ROTATIONS = (0, 90, 180, 270)


def rotation_table(rotation, n: int):
    """the int32[n] per-frame clockwise degrees of the _rotated_ calls, from one int for the whole batch or one per frame; anything else,
    or a value outside ROTATIONS, is refused before the library is called"""
    rots = None
    if isinstance(rotation, (int, np.integer)):
        rots = [rotation] * n
    elif isinstance(rotation, (list, tuple, np.ndarray)):
        rots = list(rotation)
    if rots is None or len(rots) != n:
        raise HyperposeError(HP_ERR_ARG, f"rotation {rotation!r}: expected one of {ROTATIONS} degrees, or one per frame ({n})")
    for i, r in enumerate(rots):
        if isinstance(r, (bool, np.bool_)) or not isinstance(r, (int, np.integer)) or int(r) not in ROTATIONS:
            raise HyperposeError(HP_ERR_ARG, f"frame {i}: rotation {r!r} is not one of {ROTATIONS} clockwise degrees")
    return (C.c_int32 * n)(*[int(r) for r in rots])


def _rotation_arg(rotation, n: int) -> dict:
    """the rotation= of _submit_frame_table: nothing for None (upright), else rotation_table's int32[n]"""
    return {} if rotation is None else {"rotation": rotation_table(rotation, n)}


def _per_frame(value, n: int, allowed, what: str) -> list:
    """a per-batch layout or format as one per frame: one name for the batch or a list of n names, each in `allowed`; anything else
    is refused before the library is called"""
    values = [value] * n if isinstance(value, str) else list(value)
    if len(values) != n or any(v not in allowed for v in values):
        raise HyperposeError(HP_ERR_ARG, f"{what} {value!r}: expected one of {sorted(allowed)}, or one per frame")
    return values


def _record_table(frames, rec):
    """the ctypes array of a device call's frame records, each of which must be a `rec`"""
    for i, f in enumerate(frames):
        if not isinstance(f, rec):
            raise HyperposeError(HP_ERR_ARG, f"frame {i}: expected a {rec.__name__}, got {type(f).__name__}")
    return (rec * len(frames))(*frames)


def _head(parser) -> str:
    """the infix of the pose calls for a parser's head: _pifpaf for OpenPifPaf packs, _ppn for Pose Proposal Network packs"""
    return "_pifpaf" if isinstance(parser, PifPafParser) else "_ppn" if isinstance(parser, PoseProposalParser) else ""


def _bind_engine(L):
    vp, ip = C.c_void_p, C.POINTER(C.c_int)
    L.hp_engine_create.argtypes = [C.POINTER(vp), vp, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, C.c_int]
    L.hp_engine_create_ex.argtypes = [C.POINTER(vp), vp, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, C.c_int, C.c_int]
    L.hp_engine_dtype.argtypes = [vp]
    L.hp_engine_destroy.argtypes = [vp]
    L.hp_engine_destroy.restype = None
    L.hp_engine_info.argtypes = [vp, ip, ip, ip, ip, ip, ip, ip, C.POINTER(C.c_double)]
    L.hp_engine_infer_u8_host.argtypes = [vp, vp, C.c_int]
    L.hp_engine_infer_u8_device.argtypes = [vp, vp, C.c_int, vp]
    L.hp_engine_infer_f32_host.argtypes = [vp, vp, C.c_int]
    L.hp_engine_outputs.argtypes = [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]
    L.hp_engine_read_outputs_host.argtypes = [vp, vp, vp, C.c_int]
    L.hp_engine_sync.argtypes = [vp]
    L.hp_engine_copy_outputs_device.argtypes = [vp, vp, vp, C.c_int, vp]
    L.hp_engine_launch_count.argtypes = [vp]
    L.hp_engine_launch_count.restype = C.c_longlong
    L.hp_engine_debug_read_buffer.argtypes = [vp, C.c_int, vp, C.c_int, ip, ip, ip]
    L.hp_engine_debug_write_buffer.argtypes = [vp, C.c_int, vp, C.c_int]
    L.hp_engine_debug_run_ops.argtypes = [vp, C.c_int, C.c_int, C.c_int]
    L.hp_engine_debug_op_kernel.argtypes = [vp, C.c_int, C.c_char_p, C.c_int]
    L.hp_engine_debug_op_epilogue.argtypes = [vp, C.c_int, ip]
    L.hp_engine_debug_op_conv_epilogue.argtypes = [vp, C.c_int, ip]
    L.hp_engine_debug_uses_pdl.argtypes = [vp, ip]
    L.hp_engine_debug_read_buffer_raw.argtypes = [vp, C.c_int, vp, C.c_int]
    L.hp_engine_debug_write_outputs.argtypes = [vp, vp, vp, C.c_int]
    L.hp_engine_calibrate_u8.argtypes = [vp, vp, C.c_int, vp, C.c_int]
    L.hp_pack_int8_calibrated.argtypes = [vp, C.c_size_t]
    L.hp_pose_run_u8_host.argtypes = [vp, vp, vp, C.c_int, vp, C.c_int, ip]
    L.hp_engine_stage_frame_u8.argtypes = [vp, C.c_int, vp, C.c_int, C.c_int, C.c_int]
    L.hp_engine_infer_staged.argtypes = [vp, C.c_int]
    L.hp_engine_debug_read_frames.argtypes = [vp, vp, C.c_int]
    L.hp_engine_set_output_override.argtypes = [vp, vp, vp]
    L.hp_engine_set_profiling.argtypes = [vp, C.c_int]
    L.hp_engine_get_profile.argtypes = [vp, vp, vp, vp, C.c_int, ip, C.POINTER(C.c_longlong)]
    L.hp_engine_read_outputs_frames.argtypes = [vp, C.POINTER(vp), C.POINTER(vp), C.c_int, C.c_int]
    L.hp_engine_head_type.argtypes = [vp]
    L.hp_handoff_enable.argtypes = [C.c_int]
    L.hp_handoff_stats.argtypes = [C.POINTER(C.c_longlong)] * 4
    L.hp_pose_submit_u8_host.argtypes = [vp, vp, vp, C.c_int, ip]
    L.hp_pose_submit_u8_device.argtypes = [vp, vp, vp, C.c_int, ip]
    L.hp_pose_collect.argtypes = [vp, C.c_int, vp, C.c_int, ip]
    L.hp_pose_submit_pifpaf_u8_host.argtypes = [vp, vp, vp, C.c_int, ip]
    L.hp_pose_submit_pifpaf_u8_device.argtypes = [vp, vp, vp, C.c_int, ip]
    for name, rec, rotated in frame_calls():
        getattr(L, name).argtypes = [vp, vp, C.POINTER(rec)] + [C.POINTER(C.c_int32)] * rotated + [C.c_int, C.c_int, ip]
    L.hp_pose_submit_ppn_u8_host.argtypes = [vp, vp, vp, C.c_int, ip]
    L.hp_pose_submit_ppn_u8_device.argtypes = [vp, vp, vp, C.c_int, ip]
    L.hp_pose_debug_read_slot_frames.argtypes = [vp, C.c_int, vp, C.c_int]
    L.hp_pose_stats.argtypes = [vp, C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)]
    L.hp_pool_create.argtypes = [C.POINTER(vp), ip, C.c_int, vp, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, C.c_float, C.c_float]
    L.hp_pool_destroy.argtypes = [vp]
    L.hp_pool_destroy.restype = None
    L.hp_pool_size.argtypes = [vp]
    L.hp_pool_set_capacity.argtypes = [vp, C.c_int, C.c_int, C.c_int]
    L.hp_pool_run_u8_host.argtypes = [vp, vp, C.c_int, vp, C.c_int, ip]
    L.hp_pool_set_output_override.argtypes = [vp, C.POINTER(vp), C.POINTER(vp)]
    L.hp_pool_launch_count.argtypes = [vp]
    L.hp_pool_launch_count.restype = C.c_longlong
    L.hp_default_device.restype = C.c_int
    L.hp_handoff_device_of.argtypes = [vp]


class Engine:
    """Mirror of hyperpose::dnn::tensorrt (include/hyperpose/operator/dnn/tensorrt.hpp:33-141):
    Engine(model_pack, input_size=(w, h), max_batch_size, factor=1/255, flip_rgb=True); inference(frames)."""

    def __init__(self, pack: bytes, input_size, max_batch_size: int = 8, factor: float = 1.0 / 255, flip_rgb: bool = True,
                 device: int = 0, dtype: str = "f16"):
        """dtype: "f16" (= data_type::kHALF), "tf32" (= data_type::kFLOAT of the reference ctor, tensorrt.hpp:14-22) or "int8"
        (= data_type::kINT8: needs a pack with a scale table, Graph.set_int8_scales)"""
        L = lib()
        if not getattr(L, "_engine_bound", False):
            _bind_engine(L)
            L._engine_bound = True
        self._h = C.c_void_p()
        self._pack = pack
        self.dtype = dtype
        check(L.hp_engine_create_ex(C.byref(self._h), pack, len(pack), int(input_size[0]), int(input_size[1]), max_batch_size,
                                    factor, 1 if flip_rgb else 0, device, {"f16": 0, "tf32": 1, "int8": 2}[dtype]))
        v = [C.c_int() for _ in range(7)]
        fl = C.c_double()
        check(L.hp_engine_info(self._h, *[C.byref(x) for x in v], C.byref(fl)))
        (self.in_w, self.in_h, self.max_batch, self.c_conf, self.c_paf, self.out_h, self.out_w) = [x.value for x in v]
        self.flops_per_frame = fl.value

    def close(self):
        if getattr(self, "_h", None) and _lib is not None:
            _lib.hp_engine_destroy(self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def max_batch_size(self):
        return self.max_batch

    def input_size(self):
        return (self.in_w, self.in_h)

    def infer_u8(self, frames: np.ndarray):
        """frames u8[N,in_h,in_w,3] (BGR, already network-sized).  Asynchronous; outputs stay on the device."""
        frames = np.ascontiguousarray(frames, np.uint8)
        assert frames.ndim == 4 and frames.shape[1:] == (self.in_h, self.in_w, 3), frames.shape
        check(lib().hp_engine_infer_u8_host(self._h, frames.ctypes.data, frames.shape[0]))
        self._last_n = frames.shape[0]

    def stage_frame(self, slot: int, frame: np.ndarray, keep_ratio: bool = False):
        """one u8 HWC3 frame of ANY size -> GPU resize (cv::resize / non_scaling_resize) into batch slot `slot`"""
        frame = np.ascontiguousarray(frame, np.uint8)
        assert frame.ndim == 3 and frame.shape[2] == 3
        check(lib().hp_engine_stage_frame_u8(self._h, slot, frame.ctypes.data, frame.shape[0], frame.shape[1], 1 if keep_ratio else 0))

    def infer_staged(self, n: int):
        check(lib().hp_engine_infer_staged(self._h, n))
        self._last_n = n

    def debug_read_frames(self, n: int) -> np.ndarray:
        out = np.empty((n, self.in_h, self.in_w, 3), np.uint8)
        check(lib().hp_engine_debug_read_frames(self._h, out.ctypes.data, n))
        return out

    def infer_u8_device(self, d_ptr: int, n: int, stream: int = 0):
        check(lib().hp_engine_infer_u8_device(self._h, d_ptr, n, stream))
        self._last_n = n

    def infer_f32(self, nchw: np.ndarray):
        nchw = np.ascontiguousarray(nchw, np.float32)
        check(lib().hp_engine_infer_f32_host(self._h, nchw.ctypes.data, nchw.shape[0]))
        self._last_n = nchw.shape[0]

    def inference(self, frames: np.ndarray):
        """tensorrt::inference(std::vector<cv::Mat>): returns per image [conf[C,h,w], paf[2L,h,w]] host tensors
        (ordered by name: conf < paf, src/tensorrt.cpp:405)."""
        self.infer_u8(frames)
        conf, paf = self.read_outputs(frames.shape[0])
        return [[conf[i], paf[i]] for i in range(frames.shape[0])]

    def read_outputs(self, n: int):
        conf = np.empty((n, self.c_conf, self.out_h, self.out_w), np.float32)
        paf = np.empty((n, self.c_paf, self.out_h, self.out_w), np.float32)
        check(lib().hp_engine_read_outputs_host(self._h, conf.ctypes.data, paf.ctypes.data, n))
        return conf, paf

    def read_outputs_frames(self, n: int, publish: bool = False):
        """tensorrt::inference's return value: per image its own host buffers [conf_i, paf_i] (the feature_map_t storage,
        src/tensorrt.cpp:398-431).  publish=True (what the C++ drop-in does, where feature_map_t is read-only) registers them
        for the device-resident hand-off (handoff.h); a look-up compares every byte, so editing the arrays afterwards is safe."""
        if self.head_type == 1:
            sa, sb = (17, 5, self.out_h, self.out_w), (19, 9, self.out_h, self.out_w)
        else:
            sa, sb = (self.c_conf, self.out_h, self.out_w), (self.c_paf, self.out_h, self.out_w)
        a = [np.empty(sa, np.float32) for _ in range(n)]
        b = [np.empty(sb, np.float32) for _ in range(n)]
        pa = (C.c_void_p * n)(*[x.ctypes.data for x in a])
        pb = (C.c_void_p * n)(*[x.ctypes.data for x in b])
        check(lib().hp_engine_read_outputs_frames(self._h, pa, pb, n, 1 if publish else 0))
        return [[a[i], b[i]] for i in range(n)]

    @property
    def head_type(self) -> int:
        return int(lib().hp_engine_head_type(self._h))

    def device_outputs(self):
        a, b, s = C.c_void_p(), C.c_void_p(), C.c_void_p()
        check(lib().hp_engine_outputs(self._h, C.byref(a), C.byref(b), C.byref(s)))
        return a.value, b.value, (s.value or 0)

    def sync(self):
        check(lib().hp_engine_sync(self._h))

    def copy_outputs_device(self, d_conf_ptr: int, d_paf_ptr: int, n: int, stream: int = 0):
        check(lib().hp_engine_copy_outputs_device(self._h, d_conf_ptr, d_paf_ptr, n, stream))

    @property
    def launch_count(self) -> int:
        return int(lib().hp_engine_launch_count(self._h))

    def debug_read_buffer(self, buf: int, n: int, raw: bool = False) -> np.ndarray:
        """n frames of buffer `buf` (NHWC).  raw=True reads its memory as it stands, also when its final content is never stored
        (a buffer whose last reader runs in its producer's epilogue) and the plain read refuses"""
        H, W, Cc = C.c_int(), C.c_int(), C.c_int()
        check(lib().hp_engine_debug_read_buffer(self._h, buf, None, n, C.byref(H), C.byref(W), C.byref(Cc)))
        out = np.empty((n, H.value, W.value, Cc.value), self._elem)
        if raw:
            check(lib().hp_engine_debug_read_buffer_raw(self._h, buf, out.ctypes.data, n))
        else:
            check(lib().hp_engine_debug_read_buffer(self._h, buf, out.ctypes.data, n, C.byref(H), C.byref(W), C.byref(Cc)))
        return out

    def debug_write_outputs(self, conf: np.ndarray, paf: np.ndarray):
        """write frames of the fp32 conf / paf outputs (the arrays read_outputs returns)"""
        conf, paf = np.ascontiguousarray(conf, np.float32), np.ascontiguousarray(paf, np.float32)
        assert conf.shape[0] == paf.shape[0]
        assert conf.shape[1:] == (self.c_conf, self.out_h, self.out_w) and paf.shape[1:] == (self.c_paf, self.out_h, self.out_w)
        check(lib().hp_engine_debug_write_outputs(self._h, conf.ctypes.data, paf.ctypes.data, conf.shape[0]))

    def debug_write_buffer(self, buf: int, arr: np.ndarray):
        arr = np.ascontiguousarray(arr, self._elem)
        check(lib().hp_engine_debug_write_buffer(self._h, buf, arr.ctypes.data, arr.shape[0]))

    @property
    def _elem(self):
        """element type of the activation buffers"""
        return {"f16": np.float16, "tf32": np.float32, "int8": np.int8}[self.dtype]

    def calibrate(self, frames: np.ndarray, absmax=None) -> np.ndarray:
        """INT8 calibration (TensorRT's min-max calibrator) on a "tf32" engine: u8 frames [N,in_h,in_w,3] (N may exceed max_batch)
        -> per-buffer max |x|, folded into `absmax` when given (a running maximum).  Graph.set_int8_scales turns it into scales."""
        frames = np.ascontiguousarray(frames, np.uint8)
        assert frames.ndim == 4 and frames.shape[1:] == (self.in_h, self.in_w, 3), frames.shape
        n_buf = struct.unpack_from("<I", self._pack, 12)[0]
        out = np.zeros(n_buf, np.float32) if absmax is None else np.array(absmax, np.float32).reshape(-1).copy()
        check(lib().hp_engine_calibrate_u8(self._h, frames.ctypes.data, frames.shape[0], out.ctypes.data, out.size))
        return out

    def debug_run_ops(self, first: int, last: int, n: int):
        check(lib().hp_engine_debug_run_ops(self._h, first, last, n))

    def debug_op_kernel(self, op: int) -> str:
        """the kernel op `op` launches on the next run over u8 frames, e.g. "conv<f16,48,res>", "halo<64,pool>", "none" """
        buf = C.create_string_buffer(64)
        check(lib().hp_engine_debug_op_kernel(self._h, op, buf, len(buf)))
        return buf.value.decode()

    def debug_op_epilogue(self, op: int) -> str:
        """"tma" when op `op` runs the halo kernel with its TMA-store epilogue, "reg" otherwise"""
        v = C.c_int(0)
        check(lib().hp_engine_debug_op_epilogue(self._h, op, C.byref(v)))
        return "tma" if v.value else "reg"

    def debug_op_conv_epilogue(self, op: int) -> str:
        """"tma" when op `op` runs the im2col conv kernel with its TMA-store epilogue, "reg" otherwise"""
        v = C.c_int(0)
        check(lib().hp_engine_debug_op_conv_epilogue(self._h, op, C.byref(v)))
        return "tma" if v.value else "reg"

    def debug_uses_pdl(self) -> bool:
        """True when the engine launches its conv and depthwise kernels with programmatic dependent launch"""
        v = C.c_int(0)
        check(lib().hp_engine_debug_uses_pdl(self._h, C.byref(v)))
        return bool(v.value)

    def set_output_override(self, d_conf_ptr: int, d_paf_ptr: int):
        check(lib().hp_engine_set_output_override(self._h, d_conf_ptr, d_paf_ptr))

    def set_profiling(self, enable: bool):
        check(lib().hp_engine_set_profiling(self._h, 1 if enable else 0))

    def get_profile(self):
        """-> (ms_per_op[n], op_type[n], flops_per_frame_per_op[n], runs)"""
        cap = 1024
        ms = np.zeros(cap, np.float64); ty = np.zeros(cap, np.int32); fl = np.zeros(cap, np.float64)
        n, runs = C.c_int(), C.c_longlong()
        check(lib().hp_engine_get_profile(self._h, ms.ctypes.data, ty.ctypes.data, fl.ctypes.data, cap, C.byref(n), C.byref(runs)))
        return ms[:n.value], ty[:n.value], fl[:n.value], runs.value

    def run_pose(self, parser: "PafParser", frames: np.ndarray, cap: int = 128):
        """hp_pose_run_u8_host: frames in, humans out (list of N structured arrays)."""
        frames = np.ascontiguousarray(frames, np.uint8)
        N = frames.shape[0]
        out = np.zeros((N, cap), HUMAN_DT)
        n = (C.c_int * N)()
        check(lib().hp_pose_run_u8_host(self._h, parser._h, frames.ctypes.data, N, out.ctypes.data, cap, n))
        return [out[i, :n[i]].copy() for i in range(N)]


    def _submit(self, name: str, parser, *args, n: int) -> int:
        """lib().<name>(engine, parser, *args, &ticket) for a batch of n frames; returns the ticket for collect_pose"""
        t = C.c_int(-1)
        check(getattr(lib(), name)(self._h, parser._h, *args, C.byref(t)))
        self._ticket_n = getattr(self, "_ticket_n", {})
        self._ticket_n[t.value] = n
        return t.value

    def _keep_until_collect(self, ticket: int, frames: list) -> int:
        """host frames stay referenced until their ticket is collected: page-locked ones are read by DMA after submit returns"""
        self._ticket_frames = getattr(self, "_ticket_frames", {})
        self._ticket_frames[ticket] = frames
        return ticket

    def submit_pose(self, parser: "PafParser", frames: np.ndarray) -> int:
        """hp_pose_submit_u8_host (the _pifpaf_ / _ppn_ form for a PifPafParser / PoseProposalParser): enqueue one batch (H2D on the
        copy stream, graph replay, record D2H); returns the ticket.  An OpenPifPaf pack decodes on the decoder's own stream underneath
        the next batch's convs; a PPN pack parses inside the captured graph on the engine stream.
        `frames` must stay alive until collect_pose when it is page-locked memory (DMA reads it directly)."""
        assert frames.dtype == np.uint8 and frames.flags["C_CONTIGUOUS"]
        return self._submit(f"hp_pose_submit{_head(parser)}_u8_host", parser, frames.ctypes.data, frames.shape[0], n=frames.shape[0])

    def submit_pose_device(self, parser: "PafParser", d_frames_ptr: int, n: int) -> int:
        """hp_pose_submit_u8_device: the frames are already in device memory"""
        return self._submit(f"hp_pose_submit{_head(parser)}_u8_device", parser, d_frames_ptr, n, n=n)

    def _submit_frame_table(self, parser, table, keep_ratio, device: bool, fmt: str = "u8", rotation=None) -> int:
        """hp_pose_submit{,_pifpaf,_ppn}_frames_{fmt}_{host,device}, chosen by the parser's type; with a rotation table (rotation_table)
        the form of FRAME_CALLS that takes one.  The 16-bit calls (yuv420_16, interleaved16) take the table, or NULL for None, themselves."""
        rotated = rotation is not None or FRAME_CALLS[fmt][1] == ""
        rot = (rotation,) if rotated else ()
        return self._submit(frame_call(_head(parser), fmt, device, rotated), parser, table, *rot, len(table), 1 if keep_ratio else 0,
                            n=len(table))

    def submit_pose_frames(self, parser, frames, keep_ratio: bool = False) -> int:
        """hp_pose_submit_frames_u8_host (hp_pose_submit_pifpaf_frames_u8_host for a PifPafParser, hp_pose_submit_ppn_frames_u8_host for a
        PoseProposalParser): a list of u8 HWC3 BGR frames of
        any sizes, resized on the GPU as cv::resize / non_scaling_resize (keep_ratio) do; returns the ticket for collect_pose.
        Page-locked frames are read by DMA after submit returns: they are kept referenced here until the ticket is collected."""
        for i, f in enumerate(frames):
            if not isinstance(f, np.ndarray) or f.dtype != np.uint8 or f.ndim != 3 or f.shape[2] != 3:
                raise HyperposeError(HP_ERR_ARG, f"frame {i}: expected a uint8 HWC array with 3 channels, got "
                                                 f"{getattr(f, 'dtype', type(f).__name__)} {getattr(f, 'shape', '')}")
        frames = [np.ascontiguousarray(f) for f in frames]
        table = (FrameU8 * len(frames))(*[FrameU8(f.ctypes.data, f.shape[0], f.shape[1]) for f in frames])
        return self._keep_until_collect(self._submit_frame_table(parser, table, keep_ratio, device=False), frames)

    def submit_pose_frames_device(self, parser, frames, keep_ratio: bool = False) -> int:
        """the same for frames in device memory, given as [(ptr, h, w), ...] (u8 HWC3, rows packed).  The resize kernel reads them in
        place: they must stay valid and unchanged until the ticket is collected."""
        table = (FrameU8 * len(frames))(*[FrameU8(int(p), int(h), int(w)) for p, h, w in frames])
        return self._submit_frame_table(parser, table, keep_ratio, device=True)

    def submit_pose_yuv420(self, parser, frames, layout, keep_ratio: bool = False, rotation=None) -> int:
        """hp_pose_submit{,_pifpaf,_ppn}_frames_yuv420_host, by the parser's type: a list of YUV 4:2:0 frames, each uint8 (3H/2, W) in
        cv2's packed layout for `layout` (nv12, nv21, i420 or yv12; or a list of those, one per frame), converted as cv::cvtColor does
        and resized on the GPU as submit_pose_frames resizes BGR frames; returns the ticket for collect_pose.  Page-locked frames are
        kept referenced until the ticket is collected.  rotation: clockwise degrees (0, 90, 180, 270), one for the batch or one per
        frame, applied as cv::rotate after the conversion (the _rotated_ call); None: upright."""
        rot = _rotation_arg(rotation, len(frames))
        layouts = _per_frame(layout, len(frames), YUV420_LAYOUTS, "layout")
        for i, f in enumerate(frames):
            if not isinstance(f, np.ndarray) or f.dtype != np.uint8 or f.ndim != 2 or f.shape[0] % 3 or f.shape[0] == 0:
                raise HyperposeError(HP_ERR_ARG, f"frame {i}: expected a uint8 (3H/2, W) YUV 4:2:0 array, got "
                                                 f"{getattr(f, 'dtype', type(f).__name__)} {getattr(f, 'shape', '')}")
        frames = [np.ascontiguousarray(f) for f in frames]
        table = (FrameYUV420 * len(frames))(*[yuv420_record(f, lay) for f, lay in zip(frames, layouts)])
        return self._keep_until_collect(self._submit_frame_table(parser, table, keep_ratio, device=False, fmt="yuv420", **rot), frames)

    def submit_pose_yuv420_device(self, parser, frames, keep_ratio: bool = False, rotation=None) -> int:
        """the same for YUV 4:2:0 frames in device memory, given as FrameYUV420 records (device plane pointers and pitches, e.g. an
        NVDEC surface).  The resize kernel reads them in place: they must stay valid and unchanged until the ticket is collected."""
        rot = _rotation_arg(rotation, len(frames))
        return self._submit_frame_table(parser, _record_table(frames, FrameYUV420), keep_ratio, device=True, fmt="yuv420", **rot)

    def submit_pose_interleaved(self, parser, frames, format, keep_ratio: bool = False, rotation=None) -> int:
        """hp_pose_submit{,_pifpaf,_ppn}_frames_interleaved_host, by the parser's type: a list of uint8 frames, (H, W, 3) for bgr / rgb,
        (H, W, 4) for bgra / rgba, (H, W) for gray, (H, W, 2) for yuyv / uyvy / yvyu; `format` is one of those names or a list of them,
        one per frame.  Each frame is converted as cv::cvtColor(..., COLOR_<format>2BGR) does and resized on the GPU as
        submit_pose_frames resizes BGR frames; returns the ticket for collect_pose.  A frame whose rows are contiguous but strided (a
        crop view of a larger frame) is passed with strides[0] as its pitch, not copied.  Page-locked frames are kept referenced until
        the ticket is collected.  rotation as for submit_pose_yuv420."""
        rot = _rotation_arg(rotation, len(frames))
        formats = _per_frame(format, len(frames), PIXEL_FORMATS, "format")
        for i, (f, fmt) in enumerate(zip(frames, formats)):
            ch = PIXEL_CHANNELS[fmt]
            shape = "(H, W)" if ch is None else f"(H, W, {ch})"
            if not isinstance(f, np.ndarray) or f.dtype != np.uint8 or f.ndim != (2 if ch is None else 3) or (ch and f.shape[2] != ch):
                raise HyperposeError(HP_ERR_ARG, f"frame {i}: expected a uint8 {shape} {fmt} array, got "
                                                 f"{getattr(f, 'dtype', type(f).__name__)} {getattr(f, 'shape', '')}")
            row = f.shape[1] * (ch or 1)
            if f.strides[-1] != 1 or (ch and f.strides[1] != ch) or f.strides[0] < row or f.strides[0] >= 1 << 31:
                raise HyperposeError(HP_ERR_ARG, f"frame {i}: the bytes of each row must be contiguous, rows at least {row} bytes apart "
                                                 f"(strides {f.strides})")
        table = (FrameInterleaved * len(frames))(*[interleaved_record(f, fmt) for f, fmt in zip(frames, formats)])
        return self._keep_until_collect(self._submit_frame_table(parser, table, keep_ratio, device=False, fmt="interleaved", **rot),
                                        list(frames))

    def submit_pose_interleaved_device(self, parser, frames, keep_ratio: bool = False, rotation=None) -> int:
        """the same for interleaved frames in device memory, given as FrameInterleaved records (device pointer, size, pitch, format:
        a cudaMallocPitch allocation, an NvBufSurface, a crop of either).  The resize kernel reads them in place: they must stay valid
        and unchanged until the ticket is collected."""
        rot = _rotation_arg(rotation, len(frames))
        return self._submit_frame_table(parser, _record_table(frames, FrameInterleaved), keep_ratio, device=True, fmt="interleaved", **rot)

    def submit_pose_yuv420_16(self, parser, frames, layout, bits, keep_ratio: bool = False, rotation=None) -> int:
        """hp_pose_submit{,_pifpaf,_ppn}_frames_yuv420_16_host, by the parser's type: submit_pose_yuv420 for YUV 4:2:0 frames of 16-bit
        samples, each uint16 (3H/2, W) in a YUV420_16_LAYOUTS layout (p016, p016_vu, i420 or yv12; or one per frame).  bits: the
        significant bits of the samples, LSB-aligned, 9..16, one for the batch or one per frame (16 for P010 / P016, 10 for
        yuv420p10le).  Each sample is reduced as src.convertTo(CV_8U, 2^-(bits-8)) does, then converted, rotated and resized as by
        submit_pose_yuv420."""
        rot = _rotation_arg(rotation, len(frames))
        bl = bits_list(bits, len(frames))
        layouts = _per_frame(layout, len(frames), YUV420_16_LAYOUTS, "layout")
        for i, f in enumerate(frames):
            if not isinstance(f, np.ndarray) or f.dtype != np.uint16 or f.ndim != 2 or f.shape[0] % 3 or f.shape[0] == 0:
                raise HyperposeError(HP_ERR_ARG, f"frame {i}: expected a uint16 (3H/2, W) YUV 4:2:0 array, got "
                                                 f"{getattr(f, 'dtype', type(f).__name__)} {getattr(f, 'shape', '')}")
        frames = [np.ascontiguousarray(f) for f in frames]
        table = (FrameYUV420_16 * len(frames))(*[yuv420_16_record(f, lay, b) for f, lay, b in zip(frames, layouts, bl)])
        return self._keep_until_collect(self._submit_frame_table(parser, table, keep_ratio, device=False, fmt="yuv420_16", **rot), frames)

    def submit_pose_yuv420_16_device(self, parser, frames, keep_ratio: bool = False, rotation=None) -> int:
        """the same for 16-bit YUV 4:2:0 frames in device memory, given as FrameYUV420_16 records, each with its bits (a P010 / P016
        NVDEC surface).  The resize kernel reads them in place: they must stay valid and unchanged until the ticket is collected."""
        rot = _rotation_arg(rotation, len(frames))
        return self._submit_frame_table(parser, _record_table(frames, FrameYUV420_16), keep_ratio, device=True, fmt="yuv420_16", **rot)

    def submit_pose_interleaved16(self, parser, frames, format, bits, keep_ratio: bool = False, rotation=None) -> int:
        """hp_pose_submit{,_pifpaf,_ppn}_frames_interleaved16_host, by the parser's type: submit_pose_interleaved for frames of 16-bit
        samples, uint16 (H, W, 3) for bgr48 / rgb48, (H, W, 4) for bgra64 / rgba64, (H, W) for gray16; `format` is one of those names
        or one per frame.  bits as for submit_pose_yuv420_16.  A frame whose rows are contiguous but strided is passed with
        strides[0] as its pitch, not copied."""
        rot = _rotation_arg(rotation, len(frames))
        bl = bits_list(bits, len(frames))
        formats = _per_frame(format, len(frames), INTERLEAVED16_FORMATS, "format")
        for i, (f, fmt) in enumerate(zip(frames, formats)):
            ch = PIXEL_CHANNELS[INTERLEAVED16_FORMATS[fmt]]
            shape = "(H, W)" if ch is None else f"(H, W, {ch})"
            if not isinstance(f, np.ndarray) or f.dtype != np.uint16 or f.ndim != (2 if ch is None else 3) or (ch and f.shape[2] != ch):
                raise HyperposeError(HP_ERR_ARG, f"frame {i}: expected a uint16 {shape} {fmt} array, got "
                                                 f"{getattr(f, 'dtype', type(f).__name__)} {getattr(f, 'shape', '')}")
            row = 2 * f.shape[1] * (ch or 1)
            if f.strides[-1] != 2 or (ch and f.strides[1] != 2 * ch) or f.strides[0] < row or f.strides[0] % 2 or f.strides[0] >= 1 << 31:
                raise HyperposeError(HP_ERR_ARG, f"frame {i}: the samples of each row must be contiguous, rows at least {row} bytes "
                                                 f"apart (strides {f.strides})")
        table = (FrameInterleaved16 * len(frames))(*[interleaved16_record(f, fmt, b) for f, fmt, b in zip(frames, formats, bl)])
        return self._keep_until_collect(self._submit_frame_table(parser, table, keep_ratio, device=False, fmt="interleaved16", **rot),
                                        list(frames))

    def submit_pose_interleaved16_device(self, parser, frames, keep_ratio: bool = False, rotation=None) -> int:
        """the same for 16-bit interleaved frames in device memory, given as FrameInterleaved16 records, each with its bits.  The
        resize kernel reads them in place: they must stay valid and unchanged until the ticket is collected."""
        rot = _rotation_arg(rotation, len(frames))
        return self._submit_frame_table(parser, _record_table(frames, FrameInterleaved16), keep_ratio, device=True, fmt="interleaved16",
                                        **rot)

    def debug_read_slot_frames(self, ticket: int, n: int) -> np.ndarray:
        """the first n resized network-size frames u8[n,in_h,in_w,3] of a ticket in flight or collected"""
        out = np.empty((n, self.in_h, self.in_w, 3), np.uint8)
        check(lib().hp_pose_debug_read_slot_frames(self._h, ticket, out.ctypes.data, n))
        return out

    def collect_pose(self, ticket: int, cap: int = 128):
        N = self._ticket_n[ticket]
        out = np.zeros((N, cap), HUMAN_DT)
        n = (C.c_int * N)()
        try:
            check(lib().hp_pose_collect(self._h, ticket, out.ctypes.data, cap, n))
        finally:   # (the batch has been waited for: its source frames may go)
            getattr(self, "_ticket_frames", {}).pop(ticket, None)
        return [out[i, :n[i]].copy() for i in range(N)]

    def pose_stats(self):
        a, b = C.c_longlong(), C.c_longlong()
        check(lib().hp_pose_stats(self._h, C.byref(a), C.byref(b)))
        return {"graph_captures": a.value, "graph_launches": b.value}


class Pool:
    """hp_pool_*: one engine + parser + host thread per GPU inside this process; frames shard in blocks of max_batch
    (SURVEY 8e), humans come back in frame order."""

    def __init__(self, pack: bytes, input_size, max_batch_size: int, devices=None, factor: float = 1.0 / 255, flip_rgb: bool = True,
                 conf_thresh: float = 0.05, paf_thresh: float = 0.05):
        L = lib()
        if not getattr(L, "_engine_bound", False):
            _bind_engine(L)
            L._engine_bound = True
        n = len(devices) if devices is not None else L.hp_device_count()
        devs = (C.c_int * n)(*(devices if devices is not None else range(n)))
        self._h = C.c_void_p()
        check(L.hp_pool_create(C.byref(self._h), devs, n, pack, len(pack), int(input_size[0]), int(input_size[1]), max_batch_size,
                               factor, 1 if flip_rgb else 0, conf_thresh, paf_thresh))
        self.n_gpus, self.in_w, self.in_h, self.max_batch = n, int(input_size[0]), int(input_size[1]), max_batch_size

    def close(self):
        if getattr(self, "_h", None) and _lib is not None:
            _lib.hp_pool_destroy(self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_capacity(self, peaks_per_part=0, candidates_per_limb=0, humans=0):
        check(lib().hp_pool_set_capacity(self._h, peaks_per_part, candidates_per_limb, humans))

    def set_output_override(self, d_conf_ptrs, d_paf_ptrs):
        n = self.n_gpus
        a = (C.c_void_p * n)(*d_conf_ptrs)
        b = (C.c_void_p * n)(*d_paf_ptrs)
        check(lib().hp_pool_set_output_override(self._h, a, b))

    def run(self, frames: np.ndarray, cap: int = 128):
        """frames u8[N_total, in_h, in_w, 3] (any N_total) -> list of N_total HUMAN_DT arrays, frame order"""
        assert frames.dtype == np.uint8 and frames.flags["C_CONTIGUOUS"] and frames.shape[1:] == (self.in_h, self.in_w, 3)
        N = frames.shape[0]
        out = np.zeros((N, cap), HUMAN_DT)
        n = (C.c_int * N)()
        check(lib().hp_pool_run_u8_host(self._h, frames.ctypes.data, N, out.ctypes.data, cap, n))
        return [out[i, :n[i]].copy() for i in range(N)]

    @property
    def launch_count(self) -> int:
        return int(lib().hp_pool_launch_count(self._h))


# ---------------------------------------------------------------------------------------------
# OpenPifPaf decoder
# ---------------------------------------------------------------------------------------------
EXPORTS += ["hp_pifpaf_create", "hp_pifpaf_destroy", "hp_pifpaf_process_host", "hp_pifpaf_process_device", "hp_pifpaf_fetch",
            "hp_pifpaf_launch_count", "hp_pifpaf_debug_counts", "hp_pifpaf_debug_hr",
            "hp_pifpaf_pipeline_info", "hp_pifpaf_copy_results_host_async", "hp_pifpaf_grow_capacity",
            "hp_pose_submit_pifpaf_u8_host", "hp_pose_submit_pifpaf_u8_device"]


class PifPafParser:
    """Mirror of hyperpose::parser::pifpaf (include/hyperpose/operator/parser/pifpaf.hpp:8-26): PifPafParser(h, w, thresh)."""

    def __init__(self, net_h: int, net_w: int, thresh: float = 0.1, device: int = 0):
        L = lib()
        vp, ip = C.c_void_p, C.POINTER(C.c_int)
        L.hp_pifpaf_create.argtypes = [C.POINTER(vp), C.c_int, C.c_int, C.c_float, C.c_int]
        L.hp_pifpaf_destroy.argtypes = [vp]
        L.hp_pifpaf_destroy.restype = None
        L.hp_pifpaf_process_host.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int, vp, C.c_int, ip]
        L.hp_pifpaf_process_device.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int, vp]
        L.hp_pifpaf_fetch.argtypes = [vp, vp, C.c_int, ip, C.c_int]
        self._h = C.c_void_p()
        check(L.hp_pifpaf_create(C.byref(self._h), net_h, net_w, thresh, device))

    def close(self):
        if getattr(self, "_h", None) and _lib is not None:
            _lib.hp_pifpaf_destroy(self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def process_batch(self, pif: np.ndarray, paf: np.ndarray, cap: int = 128):
        """pif[N,17,5,h,w], paf[N,19,9,h,w] host tensors -> list of N HUMAN_DT arrays"""
        pif = np.ascontiguousarray(pif, np.float32)
        paf = np.ascontiguousarray(paf, np.float32)
        N, _, _, h, w = pif.shape
        out = np.zeros((N, cap), HUMAN_DT)
        n = (C.c_int * N)()
        check(lib().hp_pifpaf_process_host(self._h, pif.ctypes.data, paf.ctypes.data, N, h, w, out.ctypes.data, cap, n))
        return [out[i, :n[i]].copy() for i in range(N)]

    def process(self, pif: np.ndarray, paf: np.ndarray, cap: int = 128):
        return self.process_batch(pif[None], paf[None], cap)[0]

    def process_device(self, d_pif_ptr: int, d_paf_ptr: int, N: int, h: int, w: int, stream: int = 0):
        check(lib().hp_pifpaf_process_device(self._h, d_pif_ptr, d_paf_ptr, N, h, w, stream))

    def fetch(self, N: int, cap: int = 128):
        out = np.zeros((N, cap), HUMAN_DT)
        n = (C.c_int * N)()
        check(lib().hp_pifpaf_fetch(self._h, out.ctypes.data, cap, n, N))
        return [out[i, :n[i]].copy() for i in range(N)]

    @property
    def launch_count(self) -> int:
        lib().hp_pifpaf_launch_count.argtypes = [C.c_void_p]
        lib().hp_pifpaf_launch_count.restype = C.c_longlong
        return int(lib().hp_pifpaf_launch_count(self._h))

    def debug_hr(self, frame: int, field: int, h: int, w: int) -> np.ndarray:
        out = np.zeros(((h - 1) * 8 + 1, (w - 1) * 8 + 1), np.float32)
        lib().hp_pifpaf_debug_hr.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        check(lib().hp_pifpaf_debug_hr(self._h, frame, field, out.ctypes.data))
        return out

    def debug_counts(self, frame: int = 0):
        out = (C.c_int * 7)()
        lib().hp_pifpaf_debug_counts.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int)]
        check(lib().hp_pifpaf_debug_counts(self._h, frame, out))
        return dict(zip(["seeds", "anns", "kept", "flags", "nms_h", "nms_w", "caf_entries"], list(out)))


EXPORTS += ["hp_ppn_create", "hp_ppn_destroy", "hp_ppn_set_point_thresh", "hp_ppn_set_limb_thresh", "hp_ppn_set_nms_thresh",
            "hp_ppn_process_host", "hp_ppn_process_device", "hp_ppn_process_device_strided", "hp_ppn_fetch", "hp_ppn_launch_count",
            "hp_ppn_prepare", "hp_ppn_state", "hp_ppn_copy_results_host_async", "hp_ppn_grow_capacity",
            "hp_pose_submit_ppn_u8_host", "hp_pose_submit_ppn_u8_device"]


class PoseProposalParser:
    """Mirror of hyperpose::parser::pose_proposal (include/hyperpose/operator/parser/proposal_network.hpp:18-80):
    PoseProposalParser((net_w, net_h), point_thresh=0.10, limb_thresh=0.05, nms_thresh=0.3)."""

    def __init__(self, net_resolution, point_thresh: float = 0.10, limb_thresh: float = 0.05, nms_thresh: float = 0.3, device: int = 0):
        L = lib()
        vp, ip, ci, cf = C.c_void_p, C.POINTER(C.c_int), C.c_int, C.c_float
        L.hp_ppn_create.argtypes = [C.POINTER(vp), ci, ci, cf, cf, cf, ci]
        L.hp_ppn_destroy.argtypes = [vp]
        L.hp_ppn_destroy.restype = None
        for f in (L.hp_ppn_set_point_thresh, L.hp_ppn_set_limb_thresh, L.hp_ppn_set_nms_thresh):
            f.argtypes = [vp, cf]
        L.hp_ppn_process_host.argtypes = [vp] + [vp] * 6 + [ci] * 7 + [vp, ci, ip]
        L.hp_ppn_process_device.argtypes = [vp] + [vp] * 6 + [ci] * 7 + [vp]
        L.hp_ppn_process_device_strided.argtypes = [vp] + [vp] * 6 + [ci] * 7 + [C.c_size_t] * 2 + [vp]
        L.hp_ppn_fetch.argtypes = [vp, vp, ci, ip, ci]
        L.hp_ppn_launch_count.argtypes = [vp]
        L.hp_ppn_launch_count.restype = C.c_longlong
        self._h = C.c_void_p()
        check(L.hp_ppn_create(C.byref(self._h), int(net_resolution[0]), int(net_resolution[1]), point_thresh, limb_thresh, nms_thresh, device))

    def close(self):
        if getattr(self, "_h", None) and _lib is not None:
            _lib.hp_ppn_destroy(self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_point_thresh(self, t: float):
        check(lib().hp_ppn_set_point_thresh(self._h, t))

    def set_limb_thresh(self, t: float):
        check(lib().hp_ppn_set_limb_thresh(self._h, t))

    def set_nms_thresh(self, t: float):
        check(lib().hp_ppn_set_nms_thresh(self._h, t))

    def process_batch(self, conf_point, x, y, w, h, edge, cap: int = 256):
        """host tensors [N,K,gh,gw] x5 and edge [N,E,nh,nw,gh,gw] -> list of N HUMAN_DT arrays"""
        a = [np.ascontiguousarray(t, np.float32) for t in (conf_point, x, y, w, h, edge)]
        N, K, gh, gw = a[0].shape
        E, nh, nw = a[5].shape[1:4]
        out = np.zeros((N, cap), HUMAN_DT)
        n = (C.c_int * N)()
        check(lib().hp_ppn_process_host(self._h, *[t.ctypes.data for t in a], N, K, gh, gw, E, nh, nw, out.ctypes.data, cap, n))
        return [out[i, :n[i]].copy() for i in range(N)]

    def process(self, conf_point, conf_iou, x, y, w, h, edge, cap: int = 256):
        """pose_proposal::process(conf_point, conf_iou, x, y, w, h, edge): one frame; conf_iou is ignored like in the
        reference (src/pose_proposal.cpp:74) apart from its leading dimension"""
        K = np.asarray(conf_iou).shape[0]
        return self.process_batch(*[np.asarray(t)[None, :K] for t in (conf_point, x, y, w, h)], np.asarray(edge)[None], cap=cap)[0]

    def process_device(self, d_conf_point: int, d_x: int, d_y: int, d_w: int, d_h: int, d_edge: int, N: int, K: int, gh: int, gw: int,
                       E: int, nh: int, nw: int, stream: int = 0, box_frame_stride: int | None = None, edge_frame_stride: int | None = None):
        """device tensors (pointers), asynchronous; results by fetch(N).  The frame strides are in floats (default: dense,
        K*gh*gw and E*nh*nw*gh*gw).  A PPN engine's outputs parse in place: see ppn_engine_pointers."""
        check(lib().hp_ppn_process_device_strided(
            self._h, d_conf_point, d_x, d_y, d_w, d_h, d_edge, N, K, gh, gw, E, nh, nw,
            K * gh * gw if box_frame_stride is None else box_frame_stride,
            E * nh * nw * gh * gw if edge_frame_stride is None else edge_frame_stride, stream))

    def fetch(self, N: int, cap: int = 256):
        out = np.zeros((N, cap), HUMAN_DT)
        n = (C.c_int * N)()
        check(lib().hp_ppn_fetch(self._h, out.ctypes.data, cap, n, N))
        return [out[i, :n[i]].copy() for i in range(N)]

    @property
    def launch_count(self) -> int:
        return int(lib().hp_ppn_launch_count(self._h))


def ppn_engine_pointers(engine: "Engine") -> dict:
    """PoseProposalParser.process_device arguments for a PPN engine's (head_type 2) device outputs, parsed in place: conf slot
    [N,6,K,gh,gw] -> conf_point + 0, x + 2KG, y + 3KG, w + 4KG, h + 5KG floats (G = gh*gw), box_frame_stride 6KG; the paf slot
    [N,E,nh,nw,gh,gw] is the edge tensor, edge_frame_stride E*nh*nw*G"""
    d_conf, d_paf, _ = engine.device_outputs()
    K, G = engine.c_conf // 6, engine.out_h * engine.out_w
    ptrs = [d_conf + t * K * G * 4 for t in (0, 2, 3, 4, 5)] + [d_paf]
    return dict(ptrs=ptrs, K=K, gh=engine.out_h, gw=engine.out_w, box_frame_stride=6 * K * G, edge_frame_stride=engine.c_paf * G)
