"""The frame calls' mappings without a GPU: which C entry point each Python submit_pose* call reaches, with how many arguments, and
the status and message each of the 48 hp_pose_submit* entry points gives for a NULL engine (which also shows that a frame list is
validated before the submit core runs)."""
import ctypes

import numpy as np
import pytest

from hyperpose_b200 import capi

HEADS = {capi.PafParser: "", capi.PifPafParser: "_pifpaf", capi.PoseProposalParser: "_ppn"}


def _recording(monkeypatch):
    """an Engine and a library that records (symbol, arguments) of every call"""
    calls = []

    class FakeLib:
        def __getattr__(self, name):
            def fn(*a):
                calls.append((name, a))
                return capi.HP_OK
            return fn

    monkeypatch.setattr(capi, "lib", lambda: FakeLib())
    eng = object.__new__(capi.Engine)
    eng._h = None
    return eng, calls


def _parser(cls):
    p = cls.__new__(cls)
    p._h = None
    return p


def _submits(eng, parser, rotation):
    """(format, device, submit()) of every submit_pose* method; the u8 network-size and BGR frame calls take no rotation"""
    u8 = np.zeros((2, 4, 6, 3), np.uint8)
    nv12, p016 = np.zeros((9, 8), np.uint8), np.zeros((9, 8), np.uint16)
    bgra, bgra64 = np.zeros((6, 8, 4), np.uint8), np.zeros((6, 8, 4), np.uint16)
    rot = {"rotation": rotation}
    calls = [("yuv420", False, lambda: eng.submit_pose_yuv420(parser, [nv12, nv12], "nv12", **rot)),
             ("yuv420", True, lambda: eng.submit_pose_yuv420_device(parser, [capi.FrameYUV420()] * 2, **rot)),
             ("interleaved", False, lambda: eng.submit_pose_interleaved(parser, [bgra, bgra], "bgra", **rot)),
             ("interleaved", True, lambda: eng.submit_pose_interleaved_device(parser, [capi.FrameInterleaved()] * 2, **rot)),
             ("yuv420_16", False, lambda: eng.submit_pose_yuv420_16(parser, [p016, p016], "p016", 10, **rot)),
             ("yuv420_16", True, lambda: eng.submit_pose_yuv420_16_device(parser, [capi.FrameYUV420_16()] * 2, **rot)),
             ("interleaved16", False, lambda: eng.submit_pose_interleaved16(parser, [bgra64, bgra64], "bgra64", 12, **rot)),
             ("interleaved16", True, lambda: eng.submit_pose_interleaved16_device(parser, [capi.FrameInterleaved16()] * 2, **rot))]
    if rotation is None:
        calls += [("u8_net", False, lambda: eng.submit_pose(parser, u8)),
                  ("u8_net", True, lambda: eng.submit_pose_device(parser, 1, 2)),
                  ("u8", False, lambda: eng.submit_pose_frames(parser, [u8[0], u8[1]])),
                  ("u8", True, lambda: eng.submit_pose_frames_device(parser, [(1, 4, 6), (2, 4, 6)]))]
    return calls


@pytest.mark.parametrize("parser_cls", list(HEADS), ids=lambda c: c.__name__)
@pytest.mark.parametrize("rotation", [None, 90])
def test_python_calls_reach_their_entry_points(monkeypatch, parser_cls, rotation):
    eng, calls = _recording(monkeypatch)
    head = HEADS[parser_cls]
    for fmt, device, submit in _submits(eng, _parser(parser_cls), rotation):
        calls.clear()
        submit()
        where = "device" if device else "host"
        if fmt == "u8_net":
            want, nargs = f"hp_pose_submit{head}_u8_{where}", 5
        elif fmt in ("yuv420_16", "interleaved16"):   # one entry point, the rotation table or NULL
            want, nargs = f"hp_pose_submit{head}_frames_{fmt}_{where}", 7
        elif rotation is None:   # upright 8-bit frames: the entry points without a rotation
            want, nargs = f"hp_pose_submit{head}_frames_{fmt}_{where}", 6
        else:
            want, nargs = f"hp_pose_submit{head}_frames_{fmt}_rotated_{where}", 7
        assert [(name, len(a)) for name, a in calls] == [(want, nargs)], (fmt, device)
        if nargs == 7:
            table = calls[0][1][3]
            assert (table is None) if rotation is None else (list(table) == [rotation] * 2), (fmt, device)
        assert eng._ticket_n[-1] == 2
        eng._ticket_frames = {}


def _entry_points():
    """(symbol, argument count, hp_last_error text for a NULL engine) of every hp_pose_submit* entry point.  A frame call reports its
    format's validator whatever its head; a network-size call reports its head's submit."""
    validator = {"u8": "hp_pose_submit_frames", "yuv420": "hp_pose_submit_frames_yuv420",
                 "interleaved": "hp_pose_submit_frames_interleaved", "yuv420_16": "hp_pose_submit_frames_yuv420_16",
                 "interleaved16": "hp_pose_submit_frames_interleaved16"}
    out = []
    for head in ("", "_pifpaf", "_ppn"):
        for where in ("host", "device"):
            out.append((f"hp_pose_submit{head}_u8_{where}", 5, f"hp_pose_submit{head}: null argument"))
            out.append((f"hp_pose_submit{head}_frames_u8_{where}", 6, f"{validator['u8']}: null argument"))
            for fmt in ("yuv420", "interleaved"):
                out.append((f"hp_pose_submit{head}_frames_{fmt}_{where}", 6, f"{validator[fmt]}: null argument"))
                out.append((f"hp_pose_submit{head}_frames_{fmt}_rotated_{where}", 7, f"{validator[fmt]}: null argument"))
            for fmt in ("yuv420_16", "interleaved16"):
                out.append((f"hp_pose_submit{head}_frames_{fmt}_{where}", 7, f"{validator[fmt]}: null argument"))
    return out


def test_every_entry_point_refuses_a_null_engine():
    points = _entry_points()
    assert len(points) == 48
    assert {name for name, _, _ in points} == {s for s in capi.EXPORTS if s.startswith("hp_pose_submit")}
    L = ctypes.CDLL(capi.LIB_PATH)
    L.hp_last_error.restype = ctypes.c_char_p
    for name, nargs, msg in points:
        assert getattr(L, name)(*([None] * nargs)) == capi.HP_ERR_ARG, name
        assert L.hp_last_error().decode() == msg, name
