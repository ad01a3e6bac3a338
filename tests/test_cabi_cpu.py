"""CPU-side checks of the drop-in boundary: the C-ABI library loads, exports every symbol the
header declares, and fails loudly (no fallback) when no CUDA device exists."""
import ctypes
import os
import re

import numpy as np
import pytest

from hyperpose_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def test_library_is_built_in_tree():
    assert os.path.exists(capi.LIB_PATH), "run python -m hyperpose_b200.build"


def test_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "hyperpose_b200.h")).read()
    declared = set(re.findall(r"\b(hp_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    L = ctypes.CDLL(capi.LIB_PATH)
    for sym in sorted(declared):
        assert hasattr(L, sym), f"{sym} declared in include/hyperpose_b200.h but not exported"
    assert declared == set(capi.EXPORTS), (declared ^ set(capi.EXPORTS))


def test_pod_layout_matches_human_t():
    # human.hpp:14-27: 18 x {bool,float,float,float} + float; the POD mirror is 18*16+4
    assert capi.HUMAN_DT.itemsize == 292 and capi.PART_DT.itemsize == 16


@pytest.mark.skipif(_has_gpu(), reason="CPU-only behaviour")
def test_no_cpu_fallback():
    assert capi.lib().hp_device_count() == 0
    with pytest.raises(capi.HyperposeError) as e:
        capi.PafParser()
    assert e.value.status == capi.HP_ERR_CUDA


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "hyperpose_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cpp", ".h", ".cuh", ".hpp")):
                src = open(os.path.join(dp, f), errors="ignore").read()
                assert not re.search(r"^\s*(from|import)\s+oracle|#include\s+[\"<].*oracle", src, re.M), f


def test_docs_have_no_unfilled_number_placeholders():
    """DESIGN.md / README.md quote measured numbers; a placeholder left in the text means the docs were not refreshed after the
    last measurement."""
    import re
    for name in ("DESIGN.md", "README.md", "INTEGRATION.md"):
        text = open(os.path.join(ROOT, name)).read()
        assert not re.findall(r"\{[A-Z][A-Z0-9]{2,}\}", text), name
