"""ctypes loader for the C ABI (include/scannet_b200.h).

There is deliberately NO fallback: if libscannet_b200.so is missing the import fails loudly
with build instructions, and every compute entry point fails with SCN_ERR_CUDA when no CUDA
device is visible.  The test oracles are never loaded from this package."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# SCN_B200_LIB: A/B runs of another build of the same library (bench scripts only)
LIB_PATH = os.environ.get("SCN_B200_LIB") or os.path.join(_HERE, "lib", "libscannet_b200.so")


class ScnError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"scannet_b200 error {code}: {msg}")
        self.code = code


class TsdfParams(C.Structure):
    _fields_ = [("voxel_size", C.c_float), ("trunc_base", C.c_float), ("trunc_scale", C.c_float),
                ("depth_min", C.c_float), ("depth_max", C.c_float), ("max_integration_distance", C.c_float),
                ("weight_sample", C.c_uint32), ("weight_max", C.c_uint32),
                ("width", C.c_uint32), ("height", C.c_uint32), ("depth_shift", C.c_float),
                ("hash_slots", C.c_uint64), ("max_blocks", C.c_uint64),
                ("batch_frames", C.c_uint32), ("flags", C.c_uint32),
                ("depth_filter", C.c_uint32), ("depth_sigma_d", C.c_float), ("depth_sigma_r", C.c_float)]


class TsdfStats(C.Structure):
    _fields_ = [("frames_integrated", C.c_uint64), ("frames_skipped", C.c_uint64),
                ("blocks_allocated", C.c_uint64), ("voxels_updated", C.c_uint64),
                ("blocks_visited", C.c_uint64), ("algorithmic_bytes", C.c_uint64),
                ("kernel_launches", C.c_uint64), ("error_flags", C.c_uint32)]


class SensInfo(C.Structure):
    _fields_ = [("version", C.c_uint32),
                ("color_width", C.c_uint32), ("color_height", C.c_uint32),
                ("depth_width", C.c_uint32), ("depth_height", C.c_uint32),
                ("color_compression", C.c_int32), ("depth_compression", C.c_int32),
                ("depth_shift", C.c_float), ("n_frames", C.c_uint64), ("n_imu_frames", C.c_uint64),
                ("color_intrinsic", C.c_float * 16), ("color_extrinsic", C.c_float * 16),
                ("depth_intrinsic", C.c_float * 16), ("depth_extrinsic", C.c_float * 16),
                ("sensor_name", C.c_char * 256)]


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} not found — the CUDA extension is required (no CPU fallback). "
                "Build it with `make lib` or `python -c 'import __graft_entry__ as g; g.build()'`.")
        _lib = C.CDLL(LIB_PATH)
        _lib.scn_last_error.restype = C.c_char_p
        _lib.scn_host_alloc.restype = C.c_void_p
        _lib.scn_host_alloc.argtypes = [C.c_size_t]
        _lib.scn_host_free.argtypes = [C.c_void_p]
        _lib.scn_free.argtypes = [C.c_void_p]
        _lib.scn_device_alloc.restype = C.c_void_p
        _lib.scn_device_alloc.argtypes = [C.c_size_t]
        _lib.scn_device_free.argtypes = [C.c_void_p]
        _lib.scn_memcpy_h2d.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    return _lib


def check(rc: int) -> int:
    if rc < 0:
        raise ScnError(rc, (lib().scn_last_error() or b"").decode("utf-8", "replace"))
    return rc
