"""ctypes binding of the aqlm_b200 C-ABI (include/aqlm_b200.h) + the in-tree nvcc build.

PyTorch is plumbing here (device memory, streams); the product is `csrc/libaqlm_b200.so`.  There is no
CPU fallback: if the library is missing or the device is not sm_90, every op raises.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
# AQLM_B200_LIB overrides the library file (used by tools/ to compare two builds side by side)
LIB_PATH = os.environ.get("AQLM_B200_LIB") or os.path.join(CSRC, "libaqlm_b200.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "aqlm_b200.h")
SOURCES = ["capi.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC", "-shared",
]

OK, ERR_DTYPE, ERR_UNSUPPORTED, ERR_SHAPE, ERR_CUDA, ERR_ARCH = range(6)
F16, BF16 = 0, 1
FLAG_PARTIAL_F32 = 1


class Weight(ctypes.Structure):
    """aqlm_b200_weight_t"""
    _fields_ = [
        ("codes", ctypes.c_void_p), ("codebooks", ctypes.c_void_p), ("scales", ctypes.c_void_p),
        ("bias", ctypes.c_void_p), ("in_features", ctypes.c_int64), ("out_features", ctypes.c_int64),
        ("num_codebooks", ctypes.c_int32), ("nbits_per_codebook", ctypes.c_int32), ("in_group_size", ctypes.c_int32),
        ("out_group_size", ctypes.c_int32), ("dtype", ctypes.c_int32), ("reserved", ctypes.c_int32),
    ]


_lib = None
_lock = threading.Lock()


def _stale() -> bool:
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh"))]
    if os.path.exists(HEADER_PATH):  # absent in a pip-installed copy (the sources include it by relative path)
        deps.append(HEADER_PATH)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile csrc/*.cu for sm_90a into csrc/libaqlm_b200.so (nvcc cross-compiles without a GPU)."""
    if force or _stale():
        cmd = ["nvcc", *NVCC_FLAGS, "-o", LIB_PATH, *[os.path.join(CSRC, s) for s in SOURCES]]
        if verbose:
            print(" ".join(cmd), flush=True)
        subprocess.check_call(cmd, cwd=CSRC)
    return LIB_PATH


def lib():
    """Load the C-ABI library.  Raises (never falls back) when it has not been built."""
    global _lib
    if _lib is None:
        with _lock:
            if _lib is None:
                if not os.path.exists(LIB_PATH):
                    raise RuntimeError(
                        f"aqlm_b200: CUDA extension {LIB_PATH} is missing. Build it with "
                        "`python -c 'import __graft_entry__ as g; g.build()'` (needs nvcc); there is no CPU fallback.")
                L = ctypes.CDLL(LIB_PATH)
                vp, i64, i32, u32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32, ctypes.c_uint32
                wp = ctypes.POINTER(Weight)
                L.aqlm_b200_version.restype = ctypes.c_int
                L.aqlm_b200_last_error.restype = ctypes.c_char_p
                L.aqlm_b200_launch_count.restype = ctypes.c_uint64
                L.aqlm_b200_reload_tunables.restype = None
                L.aqlm_b200_matmat.argtypes = [wp, vp, vp, i64, vp]
                L.aqlm_b200_matmat_ex.argtypes = [wp, vp, vp, i64, u32, vp]
                L.aqlm_b200_matmat_dequant.argtypes = [wp, vp, vp, i64, vp]
                L.aqlm_b200_matmat_grouped.argtypes = [wp, ctypes.POINTER(i64), ctypes.c_int, vp, vp, i64, u32, vp]
                L.aqlm_b200_matmat_workspace_bytes.argtypes = [wp, i64]
                L.aqlm_b200_matmat_workspace_bytes.restype = ctypes.c_size_t
                L.aqlm_b200_matmat_ws.argtypes = [wp, vp, vp, i64, u32, vp, ctypes.c_size_t, vp]
                L.aqlm_b200_matmat_dequant_workspace_bytes.argtypes = [wp, i64]
                L.aqlm_b200_matmat_dequant_workspace_bytes.restype = ctypes.c_size_t
                L.aqlm_b200_matmat_dequant_ws.argtypes = [wp, vp, vp, i64, vp, ctypes.c_size_t, vp]
                L.aqlm_b200_matmat_dequant_ex.argtypes = [wp, vp, vp, i64, u32, vp, ctypes.c_size_t, vp]
                L.aqlm_b200_dequant.argtypes = [wp, vp, ctypes.c_int, vp]
                L.aqlm_b200_matmat_dequant_transposed.argtypes = [wp, vp, vp, i64, vp, ctypes.c_size_t, vp]
                L.aqlm_b200_matmat_dequant_transposed_workspace_bytes.argtypes = [wp, i64]
                L.aqlm_b200_matmat_dequant_transposed_workspace_bytes.restype = ctypes.c_size_t
                L.aqlm_b200_matmat_dequant_grouped.argtypes = [wp, ctypes.POINTER(i64), ctypes.c_int, vp, vp, i64, u32, vp,
                                                              ctypes.c_size_t, vp]
                L.aqlm_b200_matmat_dequant_transposed_grouped.argtypes = [wp, ctypes.POINTER(i64), ctypes.c_int, vp, vp, i64,
                                                                         vp, ctypes.c_size_t, vp]
                L.aqlm_b200_matmat_dequant_routed_workspace_bytes.argtypes = [wp, ctypes.c_int, i64, ctypes.c_int]
                L.aqlm_b200_matmat_dequant_routed_workspace_bytes.restype = ctypes.c_size_t
                L.aqlm_b200_matmat_dequant_routed.argtypes = [wp, ctypes.POINTER(i64), ctypes.c_int, ctypes.c_int, vp, vp,
                                                             vp, i64, vp, ctypes.c_size_t, vp]
                L.aqlm_b200_matmat_dequant_transposed_routed.argtypes = [wp, ctypes.POINTER(i64), ctypes.c_int,
                                                                        ctypes.c_int, vp, vp, vp, i64, vp,
                                                                        ctypes.c_size_t, vp]
                L.aqlm_b200_matmat_weight_grad_workspace_bytes.argtypes = [wp, i64]
                L.aqlm_b200_matmat_weight_grad_workspace_bytes.restype = ctypes.c_size_t
                L.aqlm_b200_matmat_weight_grad.argtypes = [wp, vp, vp, i64, vp, vp, vp, ctypes.c_size_t, vp]
                L.aqlm_b200_scale_bias.argtypes = [vp, vp, vp, vp, i64, i64, i32, vp]
                L.aqlm_b200_matmat_host.argtypes = [wp, vp, vp, vp, vp, i64, vp]
                L.aqlm_b200_comm_shared_bytes.argtypes = [ctypes.c_int, i64]
                L.aqlm_b200_comm_shared_bytes.restype = ctypes.c_size_t
                L.aqlm_b200_shared_alloc.argtypes = [ctypes.c_size_t, ctypes.POINTER(vp), vp]
                L.aqlm_b200_shared_open.argtypes = [vp, ctypes.POINTER(vp)]
                L.aqlm_b200_comm_create.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.POINTER(vp), i64, ctypes.POINTER(vp)]
                L.aqlm_b200_comm_partials.argtypes = [vp]
                L.aqlm_b200_comm_partials.restype = vp
                L.aqlm_b200_comm_destroy.argtypes = [vp]
                L.aqlm_b200_allreduce_scale_bias.argtypes = [vp, vp, vp, vp, vp, i64, i64, i32, vp]
                L.aqlm_b200_matmat_allreduce.argtypes = [vp, wp, ctypes.POINTER(i64), ctypes.c_int, vp, vp, i64, vp]
                flat_mm_g = [vp, vp, vp, vp, vp, vp, i64, i64, i64, i32, i32, vp]
                flat_mm = [vp, vp, vp, vp, vp, vp, i64, i64, i64, i32, vp]
                L.aqlm_b200_code1x16_matmat.argtypes = flat_mm_g
                L.aqlm_b200_code1x16_matmat_dequant.argtypes = flat_mm_g
                for n in ("code2x8_matmat", "code1x8_matmat", "code2x8_matmat_dequant", "code1x8_matmat_dequant"):
                    getattr(L, "aqlm_b200_" + n).argtypes = flat_mm
                L.aqlm_b200_code1x16_dequant.argtypes = [vp, vp, vp, vp, i64, i64, i32, i32, vp]
                L.aqlm_b200_code2x8_dequant.argtypes = [vp, vp, vp, vp, i64, i64, i32, vp]
                L.aqlm_b200_code1x8_dequant.argtypes = [vp, vp, vp, vp, i64, i64, i32, vp]
                _lib = L
    return _lib


def header_symbols() -> list[str]:
    """Every function name declared in include/aqlm_b200.h (used by the symbol-export test)."""
    import re

    with open(HEADER_PATH) as f:
        text = f.read()
    return sorted(set(re.findall(r"\b(aqlm_b200_[a-z0-9_]+)\s*\(", text)))


def check(status: int) -> None:
    """Map a C status to the exception type the reference raises (SURVEY §8b 'Errors')."""
    if status == OK:
        return
    msg = lib().aqlm_b200_last_error().decode("utf-8", "replace")
    if status in (ERR_DTYPE, ERR_UNSUPPORTED):
        raise NotImplementedError(msg)
    if status == ERR_SHAPE:
        raise ValueError(msg)
    raise RuntimeError(f"aqlm_b200: {msg}")


def reload_tunables() -> None:
    """Re-read the AQLM_B200_* experiment switches after changing os.environ (they are cached per process)."""
    lib().aqlm_b200_reload_tunables()


def launch_count() -> int:
    return int(lib().aqlm_b200_launch_count())
