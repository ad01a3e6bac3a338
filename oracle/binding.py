"""ctypes binding of oracle/liborc_paf.so (C restatement) and oracle/_ref/libref_paf.so
(the reference's own src/paf.cpp compiled verbatim over oracle/shim).

TEST INFRASTRUCTURE ONLY -- see oracle/__init__.py.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
N_PARTS, N_PAIRS = 18, 19


class OrcPart(C.Structure):
    _fields_ = [("has_value", C.c_int32), ("x", C.c_float), ("y", C.c_float), ("score", C.c_float)]


class OrcHuman(C.Structure):
    _fields_ = [("parts", OrcPart * N_PARTS), ("score", C.c_float)]


class OrcPeak(C.Structure):
    _fields_ = [("part_id", C.c_int32), ("x", C.c_int32), ("y", C.c_int32), ("score", C.c_float), ("id", C.c_int32)]


class OrcConn(C.Structure):
    _fields_ = [("cid1", C.c_int32), ("cid2", C.c_int32), ("score", C.c_float)]


HUMAN_DT = np.dtype({"names": ["has_value", "x", "y", "score"], "formats": ["<i4", "<f4", "<f4", "<f4"]})
HUMAN_REC = np.dtype([("parts", HUMAN_DT, (N_PARTS,)), ("score", "<f4")])
PEAK_REC = np.dtype([("part_id", "<i4"), ("x", "<i4"), ("y", "<i4"), ("score", "<f4"), ("id", "<i4")])
CONN_REC = np.dtype([("cid1", "<i4"), ("cid2", "<i4"), ("score", "<f4")])
assert HUMAN_REC.itemsize == C.sizeof(OrcHuman) == 292


def build(force: bool = False) -> None:
    """make -C oracle (compiles the restatement; and _ref when /root/reference exists)."""
    so = os.path.join(HERE, "liborc_paf.so")
    ref = os.path.join(HERE, "_ref", "libref_paf.so")
    need = force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(os.path.join(HERE, "paf_oracle.c"))
    if os.path.isdir("/root/reference/src") and not os.path.exists(ref):
        need = True
    if need:
        subprocess.check_call(["make", "-C", HERE, "-s"], stdout=subprocess.DEVNULL)


_orc = None
_ref = None


def load_oracle():
    global _orc
    if _orc is None:
        build()
        lib = C.CDLL(os.path.join(HERE, "liborc_paf.so"))
        fp = C.POINTER(C.c_float)
        lib.orc_paf_process.restype = C.c_int
        lib.orc_paf_process.argtypes = [fp, fp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float,
                                        C.c_void_p, C.c_int, C.POINTER(C.c_int),
                                        C.c_void_p, C.c_int, C.POINTER(C.c_int),
                                        C.c_void_p, C.c_int, C.POINTER(C.c_int)]
        for fn in (lib.orc_resize_area_up, lib.orc_resize_area):
            fn.restype = C.c_int
            fn.argtypes = [fp, C.c_int, C.c_int, fp, C.c_int, C.c_int]
        lib.orc_gaussian17.restype = None
        lib.orc_gaussian17.argtypes = [fp, fp, C.c_int, C.c_int]
        lib.orc_gauss17_kernel.restype = fp
        lib.orc_area_up_tab.restype = None
        lib.orc_area_up_tab.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_int32), fp]
        u8p = C.POINTER(C.c_uint8)
        for fn in (lib.orc_resize_linear_u8c3, lib.orc_letterbox_u8c3):
            fn.restype = C.c_int
            fn.argtypes = [u8p, C.c_int, C.c_int, u8p, C.c_int, C.c_int]
        _orc = lib
    return _orc


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def resize_area_up(img: np.ndarray, dh: int, dw: int) -> np.ndarray:
    img = np.ascontiguousarray(img, np.float32)
    out = np.empty((dh, dw), np.float32)
    rc = load_oracle().orc_resize_area_up(_fp(img), img.shape[0], img.shape[1], _fp(out), dh, dw)
    if rc:
        raise ValueError(f"orc_resize_area_up rc={rc}")
    return out


def resize_area(img: np.ndarray, dh: int, dw: int) -> np.ndarray:
    """cv::resize(INTER_AREA) on one fp32 plane, any sizes (true area averaging when both axes shrink)"""
    img = np.ascontiguousarray(img, np.float32)
    out = np.empty((dh, dw), np.float32)
    rc = load_oracle().orc_resize_area(_fp(img), img.shape[0], img.shape[1], _fp(out), dh, dw)
    if rc:
        raise ValueError(f"orc_resize_area rc={rc}")
    return out


def area_up_tab(src: int, dst: int):
    idx = np.empty(dst, np.int32)
    fr = np.empty(dst, np.float32)
    load_oracle().orc_area_up_tab(src, dst, idx.ctypes.data_as(C.POINTER(C.c_int32)), _fp(fr))
    return idx, fr


def resize_linear_u8(img: np.ndarray, dh: int, dw: int, letterbox: bool = False) -> np.ndarray:
    """cv::resize(INTER_LINEAR) on u8 HWC3 (letterbox=True: non_scaling_resize, src/data.cpp:53-69)"""
    img = np.ascontiguousarray(img, np.uint8)
    assert img.ndim == 3 and img.shape[2] == 3
    out = np.empty((dh, dw, 3), np.uint8)
    u8p = C.POINTER(C.c_uint8)
    fn = load_oracle().orc_letterbox_u8c3 if letterbox else load_oracle().orc_resize_linear_u8c3
    rc = fn(img.ctypes.data_as(u8p), img.shape[0], img.shape[1], out.ctypes.data_as(u8p), dh, dw)
    if rc:
        raise ValueError(f"resize rc={rc}")
    return out


def gaussian17(img: np.ndarray) -> np.ndarray:
    img = np.ascontiguousarray(img, np.float32)
    out = np.empty_like(img)
    load_oracle().orc_gaussian17(_fp(img), _fp(out), img.shape[0], img.shape[1])
    return out


def gauss_kernel() -> np.ndarray:
    p = load_oracle().orc_gauss17_kernel()
    return np.ctypeslib.as_array(p, shape=(17,)).copy()


def oracle_process(conf: np.ndarray, paf: np.ndarray, conf_thresh: float = 0.05, paf_thresh: float = 0.05,
                   res_w: int = -1, res_h: int = -1, human_cap: int = 512, peak_cap: int = 65536, conn_cap: int = 4096,
                   feat_height: int = -1):
    """Run the restatement on one frame.  Returns dict(humans, peaks, conns[19 lists]).  res_w / res_h / feat_height: what a
    paf handle fixed at its first call (the resolution, and the W of that call's maps for the length penalty); -1 = this frame's."""
    conf = np.ascontiguousarray(conf, np.float32)
    paf = np.ascontiguousarray(paf, np.float32)
    assert conf.ndim == 3 and paf.ndim == 3 and conf.shape[1:] == paf.shape[1:]
    humans = np.zeros(human_cap, HUMAN_REC)
    peaks = np.zeros(peak_cap, PEAK_REC)
    conns = np.zeros((N_PAIRS, conn_cap), CONN_REC)
    nh, npk = C.c_int(0), C.c_int(0)
    ncn = (C.c_int * N_PAIRS)()
    rc = load_oracle().orc_paf_process(_fp(conf), _fp(paf), conf.shape[0], paf.shape[0], conf.shape[1], conf.shape[2],
                                       res_w, res_h, feat_height, conf_thresh, paf_thresh,
                                       humans.ctypes.data, human_cap, C.byref(nh),
                                       peaks.ctypes.data, peak_cap, C.byref(npk),
                                       conns.ctypes.data, conn_cap, ncn)
    if rc:
        raise RuntimeError(f"orc_paf_process rc={rc}")
    return {"humans": humans[:nh.value].copy(), "peaks": peaks[:npk.value].copy(),
            "conns": [conns[p, :ncn[p]].copy() for p in range(N_PAIRS)]}


def ref_available() -> bool:
    if os.path.isdir("/root/reference/src"):
        build()
    return os.path.exists(os.path.join(HERE, "_ref", "libref_paf.so"))


def load_ref():
    global _ref
    if _ref is None:
        if not ref_available():
            raise FileNotFoundError("oracle/_ref/libref_paf.so not built (needs /root/reference)")
        lib = C.CDLL(os.path.join(HERE, "_ref", "libref_paf.so"))
        fp = C.POINTER(C.c_float)
        lib.ref_paf_create.restype = C.c_void_p
        lib.ref_paf_create.argtypes = [C.c_float, C.c_float, C.c_int, C.c_int]
        lib.ref_paf_destroy.argtypes = [C.c_void_p]
        lib.ref_paf_process.restype = C.c_int
        lib.ref_paf_process.argtypes = [C.c_void_p, fp, fp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int]
        _ref = lib
    return _ref


class RefParser:
    """The reference's own hyperpose::parser::paf (stateful, like the original)."""

    def __init__(self, conf_thresh=0.05, paf_thresh=0.05, res_w=-1, res_h=-1):
        self.lib = load_ref()
        self.h = self.lib.ref_paf_create(conf_thresh, paf_thresh, res_w, res_h)

    def process(self, conf, paf, cap=512):
        conf = np.ascontiguousarray(conf, np.float32)
        paf = np.ascontiguousarray(paf, np.float32)
        out = np.zeros(cap, HUMAN_REC)
        n = self.lib.ref_paf_process(self.h, _fp(conf), _fp(paf), conf.shape[0], paf.shape[0], conf.shape[1], conf.shape[2],
                                     out.ctypes.data, cap)
        if n < 0:
            raise RuntimeError(f"ref_paf_process rc={n}")
        return out[:n].copy()

    def close(self):
        if self.h:
            self.lib.ref_paf_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_refpp = None


def pifpaf_ref_available() -> bool:
    if os.path.isdir("/root/reference/src"):
        build()
    return os.path.exists(os.path.join(HERE, "_ref", "libref_pifpaf.so"))


def ref_pifpaf_process(pif: np.ndarray, paf: np.ndarray, net_h: int, net_w: int, thresh: float = 0.1, cap: int = 256) -> np.ndarray:
    """The reference's own hyperpose::parser::pifpaf (src/pifpaf.cpp + src/pifpaf_decoder compiled verbatim) on one frame."""
    global _refpp
    if _refpp is None:
        if not pifpaf_ref_available():
            raise FileNotFoundError("oracle/_ref/libref_pifpaf.so not built (needs /root/reference)")
        lib = C.CDLL(os.path.join(HERE, "_ref", "libref_pifpaf.so"))
        fp = C.POINTER(C.c_float)
        lib.ref_pifpaf_process.restype = C.c_int
        lib.ref_pifpaf_process.argtypes = [fp, fp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_int]
        _refpp = lib
    pif = np.ascontiguousarray(pif, np.float32)
    paf = np.ascontiguousarray(paf, np.float32)
    out = np.zeros(cap, HUMAN_REC)
    n = _refpp.ref_pifpaf_process(_fp(pif), _fp(paf), pif.shape[2], pif.shape[3], net_h, net_w, thresh, out.ctypes.data, cap)
    if n < 0:
        raise RuntimeError(f"ref_pifpaf_process rc={n}")
    return out[:n].copy()


_refppn = None


def ppn_ref_available() -> bool:
    if os.path.isdir("/root/reference/src"):
        build()
    return os.path.exists(os.path.join(HERE, "_ref", "libref_ppn.so"))


def ref_ppn_process(conf_point, conf_iou, x, y, w, h, edge, net_w: int, net_h: int, point_thresh: float = 0.10,
                    limb_thresh: float = 0.05, nms_thresh: float = 0.3, cap: int = 1024) -> np.ndarray:
    """The reference's own hyperpose::parser::pose_proposal (src/pose_proposal.cpp compiled verbatim) on one frame."""
    global _refppn
    if _refppn is None:
        if not ppn_ref_available():
            raise FileNotFoundError("oracle/_ref/libref_ppn.so not built (needs /root/reference)")
        lib = C.CDLL(os.path.join(HERE, "_ref", "libref_ppn.so"))
        fp = C.POINTER(C.c_float)
        lib.ref_ppn_process.restype = C.c_int
        lib.ref_ppn_process.argtypes = [fp] * 7 + [C.c_int] * 8 + [C.c_float] * 3 + [C.c_void_p, C.c_int]
        _refppn = lib
    arrs = [np.ascontiguousarray(a, np.float32) for a in (conf_point, conf_iou, x, y, w, h, edge)]
    K, gh, gw = arrs[0].shape
    E, nh, nw = arrs[6].shape[:3]
    out = np.zeros(cap, HUMAN_REC)
    n = _refppn.ref_ppn_process(*[_fp(a) for a in arrs], K, gh, gw, E, nh, nw, net_w, net_h, point_thresh, limb_thresh, nms_thresh,
                                out.ctypes.data, cap)
    if n < 0:
        raise RuntimeError(f"ref_ppn_process rc={n}")
    return out[:n].copy()
