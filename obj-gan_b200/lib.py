"""ctypes binding of libobjgan_b200.so -- the only way the Python host code reaches the kernels.

The prototypes are parsed from ``include/objgan_b200.h`` so the header is the single source of truth
for the C ABI.  There is NO fallback: if the shared object is missing or a symbol cannot be resolved
the import fails loudly (the product never routes around the CUDA library).
"""
from __future__ import annotations

import ctypes
import os
import re

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
HEADER = os.path.join(ROOT, "include", "objgan_b200.h")
LIB_PATH = os.path.join(HERE, "libobjgan_b200.so")

_CT = {
    "int": ctypes.c_int, "long long": ctypes.c_longlong, "float": ctypes.c_float, "double": ctypes.c_double,
    "cudaStream_t": ctypes.c_void_p,
}

# constants mirrored from the header enums
ACT_NONE, ACT_LRELU, ACT_TANH, ACT_SIGMOID = 0, 1, 2, 3
NA_NONE, NA_LRELU, NA_GLU = 0, 1, 2
PAD_ZERO, PAD_REFLECT, UPSAMPLE2X, TRANSPOSED = 0, 1, 2, 3


def parse_header(path: str = HEADER):
    """Returns {function name: [ctypes argtypes]} for every prototype in the header."""
    text = open(path).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    protos = {}
    for m in re.finditer(r"\bint\s+(\w+)\s*\(([^;{]*?)\)\s*;", text, flags=re.S):
        name, args = m.group(1), m.group(2)
        types = []
        for a in args.split(","):
            a = " ".join(a.split())
            if "*" in a:
                types.append(ctypes.c_void_p)
                continue
            a = re.sub(r"\bconst\b", "", a).strip()
            base = a.rsplit(" ", 1)[0].strip()
            types.append(_CT[base])
        protos[name] = types
    return protos


class _Lib:
    def __init__(self):
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'`. "
                "objgan_b200 has no CPU or library fallback.")
        self.cdll = ctypes.CDLL(LIB_PATH)
        self.protos = parse_header()
        self.fn = {}
        for name, argtypes in self.protos.items():
            f = getattr(self.cdll, name)  # AttributeError if the .so does not export a declared symbol
            f.argtypes = argtypes
            f.restype = ctypes.c_int
            self.fn[name] = f
        self.launches = 0  # number of library calls issued (each launches >= 1 kernel)

    def call(self, name: str, *args):
        rc = self.fn[name](*args)
        self.launches += 1
        ok = (rc == 1) if name.startswith("ROIAlign") else (rc == 0)
        if not ok:
            raise RuntimeError(f"{name} failed with code {rc}")


_lib = None
# Dry run, for the CPU unit tests: the host code takes the same dispatch as on the GPU, ops._chk accepts host
# tensors, and ops._call checks each call's argument count against the header and counts it instead of launching
# (outputs stay uninitialised).  Nothing else reads it, so shapes / autograd wiring / call sequences / state_dict
# plumbing are those of a device run, exercised on a machine without a GPU.  It is not a compute path.
DRY_RUN = False


def get() -> _Lib:
    global _lib
    if _lib is None:
        _lib = _Lib()
    return _lib


def stream() -> int:
    """Raw cudaStream_t of torch's current stream on the current device (the C-level query: torch.cuda.current_stream()
    builds a Stream object through several Python layers, ~10 us per kernel launch)."""
    import torch
    return torch._C._cuda_getCurrentRawStream(torch._C._cuda_getDevice())
