"""Host-side handle for the TSDF fusion path: thin ctypes mirror of ``scn_tsdf_*``.

Mirrors the contract of the reference's external reconstruction stage
(/root/reference/Server/scan_processor.py:123-138): frames of a ``.sens`` stream plus their
camera-to-world poses in, fused voxel blocks (and later a mesh) out."""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._lib import TsdfParams, TsdfStats, check, lib

VOXEL_DTYPE = np.dtype([("sdf", "<f4"), ("r", "u1"), ("g", "u1"), ("b", "u1"), ("w", "u1")])
NO_STATS = 1
KERNEL_TMA = 4
KERNEL_COLUMN = 8


def default_params(**over) -> TsdfParams:
    p = TsdfParams()
    lib().scn_tsdf_default_params(C.byref(p))
    for k, v in over.items():
        if not hasattr(p, k):
            raise AttributeError(k)
        setattr(p, k, v)
    return p


def params_from_file(path: str, base: TsdfParams | None = None) -> TsdfParams:
    p = base or default_params()
    check(lib().scn_tsdf_params_from_file(path.encode(), C.byref(p)))
    return p


class TsdfVolume:
    def __init__(self, params: TsdfParams | None = None, device: int = 0, stream: int | None = None):
        self.params = params or default_params()
        self._h = C.c_void_p()
        check(lib().scn_tsdf_create(C.byref(self.params), device, C.byref(self._h)))
        if stream is not None:
            check(lib().scn_tsdf_set_stream(self._h, C.c_void_p(stream)))

    def close(self):
        if self._h:
            lib().scn_tsdf_destroy(self._h)
            self._h = C.c_void_p()

    __del__ = close

    def integrate(self, depth: np.ndarray, rgb, cam2world: np.ndarray, K: np.ndarray):
        depth = np.ascontiguousarray(depth, np.uint16)
        T = np.ascontiguousarray(cam2world, np.float32); Kc = np.ascontiguousarray(K, np.float32)
        rp = None
        if rgb is not None:
            rgb = np.ascontiguousarray(rgb, np.uint8); rp = rgb.ctypes.data_as(C.c_void_p)
        check(lib().scn_tsdf_integrate(self._h, depth.ctypes.data_as(C.c_void_p), rp,
                                       T.ctypes.data_as(C.c_void_p), Kc.ctypes.data_as(C.c_void_p)))

    def integrate_batch(self, depth: np.ndarray, rgb, poses: np.ndarray, K: np.ndarray):
        """depth [N,H,W] u16 host, rgb [N,H,W,3] or None, poses [N,4,4]."""
        depth = np.ascontiguousarray(depth, np.uint16)
        P = np.ascontiguousarray(poses, np.float32); Kc = np.ascontiguousarray(K, np.float32)
        rp = None
        if rgb is not None:
            rgb = np.ascontiguousarray(rgb, np.uint8); rp = rgb.ctypes.data_as(C.c_void_p)
        check(lib().scn_tsdf_integrate_batch(self._h, C.c_uint32(len(depth)), depth.ctypes.data_as(C.c_void_p), rp,
                                             P.ctypes.data_as(C.c_void_p), Kc.ctypes.data_as(C.c_void_p)))

    def integrate_batch_ptr(self, n: int, depth_host_ptr: int, rgb_host_ptr: int | None, poses: np.ndarray, K: np.ndarray):
        """Host pointers (e.g. pinned torch tensors' data_ptr())."""
        P = np.ascontiguousarray(poses, np.float32); Kc = np.ascontiguousarray(K, np.float32)
        check(lib().scn_tsdf_integrate_batch(self._h, C.c_uint32(n), C.c_void_p(depth_host_ptr),
                                             C.c_void_p(rgb_host_ptr) if rgb_host_ptr else None,
                                             P.ctypes.data_as(C.c_void_p), Kc.ctypes.data_as(C.c_void_p)))

    def integrate_device(self, n: int, d_depth_ptr: int, d_rgb_ptr: int | None, poses: np.ndarray, K: np.ndarray):
        P = np.ascontiguousarray(poses, np.float32); Kc = np.ascontiguousarray(K, np.float32)
        check(lib().scn_tsdf_integrate_device(self._h, C.c_uint32(n), C.c_void_p(d_depth_ptr),
                                              C.c_void_p(d_rgb_ptr) if d_rgb_ptr else None,
                                              P.ctypes.data_as(C.c_void_p), Kc.ctypes.data_as(C.c_void_p)))

    def profile(self, enable: bool = True):
        check(lib().scn_tsdf_profile(self._h, 1 if enable else 0))

    def kernel_times(self):
        """(alloc_ms, integrate_ms, n_batches, union_blocks) summed since profile(True)."""
        a = C.c_double(); b = C.c_double(); n = C.c_uint64(); u = C.c_uint64()
        check(lib().scn_tsdf_kernel_times(self._h, C.byref(a), C.byref(b), C.byref(n), C.byref(u)))
        return a.value, b.value, n.value, u.value

    def sync(self):
        check(lib().scn_tsdf_sync(self._h))

    def reset(self):
        check(lib().scn_tsdf_reset(self._h))

    def stats(self) -> TsdfStats:
        s = TsdfStats()
        check(lib().scn_tsdf_stats(self._h, C.byref(s)))
        return s

    def extract_mesh(self):
        """Marching cubes: returns (xyz float32 [V,3], rgb uint8 [V,3], tri uint32 [F,3])."""
        xyz = C.POINTER(C.c_float)(); rgb = C.POINTER(C.c_uint8)(); tri = C.POINTER(C.c_uint32)()
        nv = C.c_uint64(); nf = C.c_uint64()
        check(lib().scn_tsdf_extract_mesh(self._h, C.byref(xyz), C.byref(rgb), C.byref(tri), C.byref(nv), C.byref(nf)))
        V, F = nv.value, nf.value
        a = np.ctypeslib.as_array(xyz, (max(V * 3, 1),))[: V * 3].copy().reshape(-1, 3)
        c = np.ctypeslib.as_array(rgb, (max(V * 3, 1),))[: V * 3].copy().reshape(-1, 3)
        t = np.ctypeslib.as_array(tri, (max(F * 3, 1),))[: F * 3].copy().reshape(-1, 3)
        for p in (xyz, rgb, tri):
            lib().scn_free(p)
        return a, c, t

    def download_blocks(self, sort: bool = True):
        """Returns (block_xyz int32 [n,3], voxels VOXEL_DTYPE [n,512]) sorted by packed key."""
        n = C.c_uint64()
        check(lib().scn_tsdf_download_blocks(self._h, None, None, C.c_uint64(0), C.byref(n)))
        nb = n.value
        xyz = np.zeros((nb, 3), np.int32); vox = np.zeros((nb, 512), VOXEL_DTYPE)
        if nb:
            check(lib().scn_tsdf_download_blocks(self._h, xyz.ctypes.data_as(C.c_void_p), vox.ctypes.data_as(C.c_void_p),
                                                 C.c_uint64(nb), C.byref(n)))
        if sort and nb:
            B = 1 << 20
            key = (xyz[:, 0].astype(np.int64) + B) | ((xyz[:, 1].astype(np.int64) + B) << 21) | ((xyz[:, 2].astype(np.int64) + B) << 42)
            o = np.argsort(key, kind="stable")
            xyz, vox = xyz[o], vox[o]
        return xyz, vox

    def upload_blocks(self, block_xyz: np.ndarray, voxels: np.ndarray):
        """Adds blocks (int32 [n,3], VOXEL_DTYPE [n,512], as download_blocks returns them) to the volume."""
        xyz = np.ascontiguousarray(block_xyz, np.int32).reshape(-1, 3)
        vox = np.ascontiguousarray(voxels, VOXEL_DTYPE).reshape(-1, 512)
        if len(xyz) != len(vox):
            raise ValueError(f"{len(xyz)} block coordinates for {len(vox)} voxel blocks")
        check(lib().scn_tsdf_upload_blocks(self._h, xyz.ctypes.data_as(C.c_void_p), vox.ctypes.data_as(C.c_void_p),
                                           C.c_uint64(len(xyz))))


def bilateral_filter(depth: np.ndarray, depth_shift: float = 1000.0, sigma_d: float = 2.0, sigma_r: float = 0.05) -> np.ndarray:
    """Depth bilateral pre-filter (scn_depth_bilateral_filter): uint16 [H,W] -> float32 metres, -inf = invalid."""
    depth = np.ascontiguousarray(depth, np.uint16)
    out = np.zeros(depth.shape, np.float32)
    check(lib().scn_depth_bilateral_filter(depth.ctypes.data_as(C.c_void_p), C.c_uint32(depth.shape[1]), C.c_uint32(depth.shape[0]),
                                           C.c_float(depth_shift), C.c_float(sigma_d), C.c_float(sigma_r), out.ctypes.data_as(C.c_void_p)))
    return out
