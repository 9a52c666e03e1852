"""CPU: where the tensor-core prompt pass reads its 16-bit layer matrices (gridllm_b200/csrc/prefill_weights.h through
tests/hostcheck/prefill_weights_shim.cpp): the resident copy when it fits beside a 4 GB margin, the streamed staging buffer
otherwise, GL_PREFILL_WEIGHTS forcing either, and prefill_mode 1 building neither."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GB = 1 << 30
NONE, RESIDENT, STREAMED = 0, 1, 2
# (n_layer, n_embd, n_head, n_kv, head_dim, n_ff)
LLAMA3_8B = (32, 4096, 32, 8, 128, 14336)
LLAMA3_70B = (80, 8192, 64, 8, 128, 28672)


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    """CPU build of prefill_weights.h -- test infrastructure only"""
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    out = str(tmp_path_factory.mktemp("pw") / "libprefill_weights_shim.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-shared", "-fPIC", "-o", out,
                           os.path.join(ROOT, "tests", "hostcheck", "prefill_weights_shim.cpp")])
    lib = ctypes.CDLL(out)
    lib.pw_copy_bytes.restype = ctypes.c_uint64
    lib.pw_stage_bytes.restype = ctypes.c_uint64
    lib.pw_margin.restype = ctypes.c_uint64
    lib.pw_source.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_uint64, ctypes.c_uint64]
    return lib


def _layer_elems(n_embd, n_head, n_kv, hd, n_ff):
    return (n_head + 2 * n_kv) * hd * n_embd + n_embd * n_head * hd + 2 * n_ff * n_embd + n_embd * n_ff


@pytest.mark.parametrize("shape,gb", [(LLAMA3_8B, 13.96), (LLAMA3_70B, 136.9)])
def test_copy_bytes(shim, shape, gb):
    n_layer, *rest = shape
    got = shim.pw_copy_bytes(*shape)
    assert got == 2 * n_layer * _layer_elems(*rest)
    assert round(got / 1e9, 2 if gb < 100 else 1) == gb


def test_stage_is_the_gate_up_operand(shim):
    assert shim.pw_stage_bytes(*LLAMA3_70B[1:]) == 2 * 2 * 28672 * 8192            # 940 MB
    assert round(shim.pw_stage_bytes(*LLAMA3_70B[1:]) / 1e6) == 940
    assert shim.pw_stage_bytes(*LLAMA3_8B[1:]) == 2 * 2 * 14336 * 4096
    # an unusual shape whose Q | K | V operand is the largest: the buffer still holds every operand
    assert shim.pw_stage_bytes(256, 4, 4, 64, 8) == 2 * 3 * 256 * 256


def test_margin_at_the_boundary(shim):
    assert shim.pw_margin() == 4 * GB
    copy = shim.pw_copy_bytes(*LLAMA3_8B)
    assert shim.pw_source(0, 0, copy, copy + 4 * GB) == RESIDENT
    assert shim.pw_source(0, 0, copy, copy + 4 * GB - 1) == STREAMED
    assert shim.pw_source(0, 1, copy, copy + 4 * GB) == RESIDENT
    assert shim.pw_source(0, 1, copy, copy + 4 * GB - 1) == -1


def test_h100_cases(shim):
    """80 GB card: the 8B q4_K_M (4.9 GB of weights) keeps its copy; the 70B q4_K_M (42.5 GB) streams"""
    free_8b = 80 * GB - int(4.9e9) - int(1.1e9)
    free_70b = 80 * GB - int(42.5e9) - int(2.7e9)
    assert shim.pw_source(0, 0, shim.pw_copy_bytes(*LLAMA3_8B), free_8b) == RESIDENT
    assert shim.pw_source(0, 0, shim.pw_copy_bytes(*LLAMA3_70B), free_70b) == STREAMED
    assert shim.pw_source(0, 1, shim.pw_copy_bytes(*LLAMA3_70B), free_70b) == -1


@pytest.mark.parametrize("request_", [0, 1, 2, 3, -1])
def test_each_request(shim, request_):
    copy = 10 * GB
    for free in (0, 14 * GB - 1, 14 * GB, 100 * GB):
        fits = copy + 4 * GB <= free
        got = shim.pw_source(0, request_, copy, free)
        if request_ == 2:
            want = STREAMED
        elif request_ == 1:
            want = RESIDENT if fits else -1
        else:                                           # 0 and anything else: auto
            want = RESIDENT if fits else STREAMED
        assert got == want, (request_, free)
        # prefill_mode 1: sequential decode steps, no copy and no staging buffer, whatever is asked
        assert shim.pw_source(1, request_, copy, free) == NONE


def test_documented():
    text = open(os.path.join(ROOT, "include", "gridllm_native.h")).read()
    assert "GL_PREFILL_WEIGHTS" in text
    assert re.search(r"resident", text) and re.search(r"streamed", text)
