"""Every launcher of include/iggt_b200.h that takes a 16-bit `dtype` (and iggt_layernorm, whose `out_kind` picks the
output type) refuses an unknown code with -3 before it does anything else: the other arguments are all 0 / NULL here,
so a launcher that checked anything first would return another status, and one that went on to CUDA would return a
CUDA error.  The calls pass placeholder arguments, so the test runs only where there is no device."""
import ctypes
import os
import re

import pytest
import torch

from iggt_official_b200 import _lib

pytestmark = pytest.mark.skipif(torch.cuda.is_available(),
                                reason="placeholder arguments: run only where no CUDA device can be reached")

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "iggt_b200.h")
INVALID = {"dtype": (2, -1), "out_kind": (3, -1)}       # dtype: 0 fp16, 1 bf16; out_kind: 0 fp16, 1 bf16, 2 fp32


def _launchers():
    """{name: (parameter names, name of the type-code parameter)} from the header's declarations"""
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    found = {}
    for name, params in re.findall(r"\bint\s+(iggt_\w+)\s*\(([^;]*?)\)\s*;", text, flags=re.S):
        names = [re.findall(r"\w+", p)[-1] for p in params.split(",")]
        code = "out_kind" if name == "iggt_layernorm" else "dtype"
        if code in names:
            found[name] = (names, code)
    return found


LAUNCHERS = _launchers()
CASES = [(name, bad) for name in sorted(LAUNCHERS) for bad in INVALID[LAUNCHERS[name][1]]]


def test_header_declares_the_launchers():
    assert len(LAUNCHERS) >= 25
    assert {"iggt_gemm_store16", "iggt_conv_nhwc", "iggt_attention_fwd_ws", "iggt_camera_head", "iggt_kv_gather_maps",
            "iggt_channel_mean", "iggt_layernorm", "iggt_layernorm_rows"} <= LAUNCHERS.keys()


@pytest.mark.parametrize("name,bad", CASES)
def test_invalid_type_code_returns_minus_3(name, bad):
    names, code = LAUNCHERS[name]
    argtypes = _lib.SIGNATURES[name]
    assert len(argtypes) == len(names), (name, names)
    args = [0 if t in (ctypes.c_int, ctypes.c_int64, ctypes.c_float) else None for t in argtypes]
    args[names.index(code)] = bad
    assert getattr(_lib.load(), name)(*args) == -3
