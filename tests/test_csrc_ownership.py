"""CPU: every CUDA allocation, stream and event of libb200match has an owner, and every CUDA error one path.  The raw
allocate / free / create / destroy calls live in pycolmap_b200/csrc/cuda_owned.cuh only (DeviceArray, PinnedArray,
Stream, Event), and B2M_CUDA_TRY there is the only error macro: a hand-kept release list or a module's own copy of
the error macro is how buffers leaked and the same out-of-memory condition came to raise different exceptions."""
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "pycolmap_b200", "csrc")
OWNER = "cuda_owned.cuh"

RAW_CALL = re.compile(r"\b(cudaMalloc|cudaMallocHost|cudaHostAlloc|cudaFree|cudaFreeHost|cudaStreamCreate\w*|"
                      r"cudaEventCreate\w*|cudaStreamDestroy|cudaEventDestroy)\s*\(")
TRY_MACRO = re.compile(r"#\s*define\s+(\w*_TRY)\b")


def _sources():
    files = [f for ext in ("cu", "cuh", "h") for f in glob.glob(os.path.join(CSRC, "*." + ext))]
    assert any(os.path.basename(f) == OWNER for f in files)
    return sorted(files)


def _code(path):
    """The file without its comments, so that prose may name the calls."""
    text = open(path).read()
    return re.sub(r"//[^\n]*|/\*.*?\*/", "", text, flags=re.S)


def test_raw_cuda_resource_calls_only_in_the_ownership_header():
    found = []
    for path in _sources():
        if os.path.basename(path) == OWNER:
            continue
        for n, line in enumerate(_code(path).splitlines(), 1):
            for m in RAW_CALL.finditer(line):
                found.append(f"{os.path.basename(path)}:{n}: {m.group(1)}")
    assert not found, "\n".join(found)


def test_one_cuda_error_macro():
    found = []
    for path in _sources():
        for m in TRY_MACRO.finditer(_code(path)):
            if os.path.basename(path) != OWNER or m.group(1) != "B2M_CUDA_TRY":
                found.append(f"{os.path.basename(path)}: {m.group(1)}")
    assert not found, found
