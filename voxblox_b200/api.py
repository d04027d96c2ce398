"""Host-side mirror of the reference's operator interface for the TSDF / ESDF hot path.

Same names, argument meaning and error behaviour as the reference's C++ API
(voxblox/include/voxblox/integrator/tsdf_integrator.h:51-209,
 voxblox/include/voxblox/integrator/esdf_integrator.h:25-178,
 voxblox/include/voxblox/core/layer.h:24-296), bound to the C-ABI of
include/voxblox_b200.h through ctypes.  There is NO CPU fallback: if
libvoxblox_b200.so is missing or no CUDA device is present, constructing an
integrator raises.  (The reference aborts through glog CHECK / LOG(FATAL); here the
same conditions raise VoxbloxError with the C-ABI's message.)
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, Iterable, Optional, Sequence, Tuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libvoxblox_b200.so")

# TsdfVoxel / EsdfVoxel exactly as the reference lays them out (core/voxel.h:12-37)
TSDF_DTYPE = np.dtype([("distance", "<f4"), ("weight", "<f4"), ("color", "u1", (4,))])
ESDF_DTYPE = np.dtype([("distance", "<f4"), ("observed", "u1"), ("hallucinated", "u1"),
                       ("in_queue", "u1"), ("fixed", "u1"), ("parent", "<i4", (3,))])
assert TSDF_DTYPE.itemsize == 12 and ESDF_DTYPE.itemsize == 20

LAYER_TSDF, LAYER_ESDF = 0, 1
UPDATED_MAP, UPDATED_MESH, UPDATED_ESDF = 1, 2, 4  # Update::Status, core/block.h:15-18
UPDATED_MIRROR = 8  # the engine's own "changed since it was last mirrored" mark (VBX_UPDATED_MIRROR)


class TsdfIntegratorType:  # tsdf_integrator.h:30-41
    kSimple, kMerged, kFast = 1, 2, 3


kTsdfIntegratorTypeNames = ("simple", "merged", "fast")


class VoxbloxError(RuntimeError):
    pass


class TsdfIntegratorConfig(C.Structure):
    """TsdfIntegratorBase::Config (tsdf_integrator.h:56-89), same field names and defaults.

    integration_order_mode accepts "mixed"/"sorted" or 0/1."""
    _fields_ = [("default_truncation_distance", C.c_float), ("max_weight", C.c_float),
                ("voxel_carving_enabled", C.c_int32), ("min_ray_length_m", C.c_float),
                ("max_ray_length_m", C.c_float), ("use_const_weight", C.c_int32),
                ("allow_clear", C.c_int32), ("use_weight_dropoff", C.c_int32),
                ("use_sparsity_compensation_factor", C.c_int32),
                ("sparsity_compensation_factor", C.c_float), ("integrator_threads", C.c_int32),
                ("integration_order_mode", C.c_int32), ("enable_anti_grazing", C.c_int32),
                ("start_voxel_subsampling_factor", C.c_float),
                ("max_consecutive_ray_collisions", C.c_int32),
                ("clear_checks_every_n_frames", C.c_int32), ("max_integration_time_s", C.c_float)]

    def __init__(self, **kw):
        d = dict(default_truncation_distance=0.1, max_weight=10000.0, voxel_carving_enabled=1,
                 min_ray_length_m=0.1, max_ray_length_m=5.0, use_const_weight=0, allow_clear=1,
                 use_weight_dropoff=1, use_sparsity_compensation_factor=0,
                 sparsity_compensation_factor=1.0, integrator_threads=os.cpu_count() or 1,
                 integration_order_mode=0, enable_anti_grazing=0,
                 start_voxel_subsampling_factor=2.0, max_consecutive_ray_collisions=2,
                 clear_checks_every_n_frames=1, max_integration_time_s=3.4028234663852886e38)
        d.update(kw)
        mode = d["integration_order_mode"]
        if isinstance(mode, str):
            if mode not in ("mixed", "sorted"):  # LOG(FATAL), integrator_utils.cc:12
                raise VoxbloxError(f"Unknown integration order mode: '{mode}'!")
            d["integration_order_mode"] = 0 if mode == "mixed" else 1
        super().__init__(**d)

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class EsdfIntegratorConfig(C.Structure):
    """EsdfIntegrator::Config (esdf_integrator.h:29-78)."""
    _fields_ = [("full_euclidean_distance", C.c_int32), ("max_distance_m", C.c_float),
                ("min_distance_m", C.c_float), ("default_distance_m", C.c_float),
                ("min_diff_m", C.c_float), ("min_weight", C.c_float), ("num_buckets", C.c_int32),
                ("multi_queue", C.c_int32), ("add_occupied_crust", C.c_int32),
                ("clear_sphere_radius", C.c_float), ("occupied_sphere_radius", C.c_float)]

    def __init__(self, **kw):
        d = dict(full_euclidean_distance=0, max_distance_m=2.0, min_distance_m=0.2,
                 default_distance_m=2.0, min_diff_m=0.001, min_weight=1e-6, num_buckets=20,
                 multi_queue=0, add_occupied_crust=0, clear_sphere_radius=1.5,
                 occupied_sphere_radius=5.0)
        d.update(kw)
        super().__init__(**d)


class MeshIntegratorConfig(C.Structure):
    """MeshIntegratorConfig (mesh/mesh_integrator.h:46-66); integrator_threads has no meaning here."""
    _fields_ = [("use_color", C.c_int32), ("min_weight", C.c_float)]

    def __init__(self, use_color: bool = True, min_weight: float = 1e-4):
        super().__init__(use_color=int(bool(use_color)), min_weight=float(min_weight))


class ICPConfig(C.Structure):
    """ICP::Config (alignment/icp.h:76-108), field names as spelled there.  num_threads defaults to 1 (the
    reference default, hardware_concurrency(), makes its result depend on thread timing); 1..32 here."""
    _fields_ = [("refine_roll_pitch", C.c_int32), ("mini_batch_size", C.c_int32), ("min_match_ratio", C.c_float),
                ("subsample_keep_ratio", C.c_float), ("inital_translation_weighting", C.c_float),
                ("inital_rotation_weighting", C.c_float), ("num_threads", C.c_int32), ("reserved", C.c_int32)]

    def __init__(self, **kw):
        d = dict(refine_roll_pitch=0, mini_batch_size=20, min_match_ratio=0.8, subsample_keep_ratio=0.5,
                 inital_translation_weighting=100.0, inital_rotation_weighting=100.0, num_threads=1, reserved=0)
        d.update(kw)
        super().__init__(**d)


class EngineOptions(C.Structure):
    """vbx_engine_options: device-side sizing (no reference counterpart)."""
    _fields_ = [("device", C.c_int32), ("max_blocks", C.c_uint32),
                ("max_points_per_scan", C.c_uint32), ("max_updates_per_pass", C.c_uint64),
                ("rank", C.c_int32), ("world_size", C.c_int32)]

    def __init__(self, **kw):
        d = dict(device=-1, max_blocks=0, max_points_per_scan=0, max_updates_per_pass=0, rank=0,
                 world_size=1)
        d.update(kw)
        super().__init__(**d)


EXPORTS = ["vbx_create", "vbx_destroy", "vbx_last_error", "vbx_version", "vbx_get_tsdf_config",
           "vbx_tsdf_integrate", "vbx_tsdf_integrate_device", "vbx_get_counters",
           "vbx_last_device_ms", "vbx_num_blocks", "vbx_list_blocks", "vbx_download_blocks",
           "vbx_upload_blocks", "vbx_remove_blocks", "vbx_clear", "vbx_clear_updated",
           "vbx_esdf_create", "vbx_esdf_update", "vbx_esdf_get_counters", "vbx_sync",
           "vbx_timer_start", "vbx_timer_stop_ms", "vbx_set_stage_profiling", "vbx_get_stage_ms",
           "vbx_host_alloc", "vbx_host_free", "vbx_host_copy_ms", "vbx_block_owner",
           "vbx_debug_sort", "vbx_debug_scan", "vbx_debug_bundle_order", "vbx_debug_apply", "vbx_debug_apply_paths", "vbx_debug_count_apply_paths", "vbx_debug_serial_fast", "vbx_debug_async_timeline", "vbx_tsdf_integrate_async", "vbx_esdf_update_blocks", "vbx_esdf_set_max_distance",
           "vbx_esdf_set_full_euclidean", "vbx_esdf_get_config", "vbx_esdf_add_robot_position", "vbx_esdf_clear", "vbx_mesh_generate", "vbx_mesh_download", "vbx_icp_run", "vbx_icp_run_device", "vbx_mirror_updated", "vbx_serialize_updated", "vbx_deserialize_blocks", "vbx_save_layer", "vbx_load_layer",
           "vbx_proto_encode_layer", "vbx_proto_encode_block", "vbx_proto_decode_block",
           "vbx_gather_updated_device", "vbx_upload_blocks_device", "vbx_debug_staging_bytes",
           "vbx_debug_icp_solve"]

_lib = None


def load_library():
    """dlopen the engine; raises (never falls back) when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    # more hardware work queues for the pipelined path's streams (effective only if CUDA is not initialised yet
    # in this process; see bench.py / INTEGRATION.md)
    os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
    if not os.path.exists(LIB_PATH):
        raise VoxbloxError(f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ "
                           "as g; g.build()'` (there is no CPU fallback)")
    lib = C.CDLL(LIB_PATH)
    vp, i32, u64 = C.c_void_p, C.c_int, C.c_uint64
    lib.vbx_create.restype = i32
    lib.vbx_create.argtypes = [C.POINTER(TsdfIntegratorConfig), C.c_float, i32,
                               C.POINTER(EngineOptions), C.POINTER(vp)]
    lib.vbx_destroy.restype = None
    lib.vbx_destroy.argtypes = [vp]
    lib.vbx_last_error.restype = C.c_char_p
    lib.vbx_last_error.argtypes = [vp]
    lib.vbx_version.restype = C.c_char_p
    lib.vbx_get_tsdf_config.restype = i32
    lib.vbx_get_tsdf_config.argtypes = [vp, C.POINTER(TsdfIntegratorConfig)]
    for name in ("vbx_tsdf_integrate", "vbx_tsdf_integrate_device"):
        f = getattr(lib, name)
        f.restype = i32
        f.argtypes = [vp, i32, vp, vp, vp, vp, u64, i32]
    lib.vbx_tsdf_integrate_async.restype = i32
    lib.vbx_tsdf_integrate_async.argtypes = [vp, i32, vp, vp, vp, vp, u64, i32, i32]
    lib.vbx_get_counters.restype = i32
    lib.vbx_get_counters.argtypes = [vp, vp]
    lib.vbx_debug_apply.restype = i32
    lib.vbx_debug_apply.argtypes = [vp, vp, C.c_uint32, u64, vp, vp, vp, vp, vp, vp]
    lib.vbx_debug_apply_paths.restype = i32
    lib.vbx_debug_apply_paths.argtypes = [vp, vp]
    lib.vbx_debug_count_apply_paths.restype = i32
    lib.vbx_debug_count_apply_paths.argtypes = [vp, i32]
    lib.vbx_debug_serial_fast.restype = i32
    lib.vbx_debug_serial_fast.argtypes = [vp, i32]
    lib.vbx_esdf_get_counters.restype = i32
    lib.vbx_esdf_get_counters.argtypes = [vp, vp]
    lib.vbx_last_device_ms.restype = i32
    lib.vbx_last_device_ms.argtypes = [vp, C.POINTER(C.c_float)]
    lib.vbx_num_blocks.restype = i32
    lib.vbx_num_blocks.argtypes = [vp, i32, C.POINTER(u64)]
    lib.vbx_list_blocks.restype = i32
    lib.vbx_list_blocks.argtypes = [vp, i32, i32, vp, u64, C.POINTER(u64)]
    lib.vbx_download_blocks.restype = i32
    lib.vbx_download_blocks.argtypes = [vp, i32, vp, u64, vp, vp]
    lib.vbx_upload_blocks.restype = i32
    lib.vbx_upload_blocks.argtypes = [vp, i32, vp, u64, vp, vp]
    lib.vbx_remove_blocks.restype = i32
    lib.vbx_remove_blocks.argtypes = [vp, i32, vp, u64]
    lib.vbx_clear.restype = i32
    lib.vbx_clear.argtypes = [vp, i32]
    lib.vbx_clear_updated.restype = i32
    lib.vbx_clear_updated.argtypes = [vp, i32, i32]
    lib.vbx_esdf_create.restype = i32
    lib.vbx_esdf_create.argtypes = [vp, C.POINTER(EsdfIntegratorConfig)]
    lib.vbx_mirror_updated.restype = i32
    lib.vbx_mirror_updated.argtypes = [vp, i32, i32, i32, vp, vp, vp, u64, C.POINTER(u64)]
    lib.vbx_serialize_updated.restype = i32
    lib.vbx_serialize_updated.argtypes = [vp, i32, i32, i32, vp, vp, vp, u64, C.POINTER(u64)]
    lib.vbx_deserialize_blocks.restype = i32
    lib.vbx_deserialize_blocks.argtypes = [vp, i32, vp, u64, vp, vp]
    lib.vbx_gather_updated_device.argtypes = [vp, i32, i32, i32, i32, vp, vp, u64, C.POINTER(u64)]
    lib.vbx_gather_updated_device.restype = i32
    lib.vbx_upload_blocks_device.argtypes = [vp, i32, vp, u64, vp, C.c_uint8]
    lib.vbx_upload_blocks_device.restype = i32
    lib.vbx_debug_staging_bytes.restype = i32
    lib.vbx_debug_staging_bytes.argtypes = [vp, C.POINTER(u64)]
    lib.vbx_debug_icp_solve.restype = i32
    lib.vbx_debug_icp_solve.argtypes = [vp, C.c_uint32, i32] + [vp] * 9
    lib.vbx_save_layer.restype = i32
    lib.vbx_save_layer.argtypes = [vp, i32, C.c_char_p, i32]
    lib.vbx_load_layer.restype = i32
    lib.vbx_load_layer.argtypes = [vp, i32, C.c_char_p, C.POINTER(u64)]
    lib.vbx_proto_encode_layer.restype = i32
    lib.vbx_proto_encode_layer.argtypes = [C.c_double, C.c_uint32, C.c_char_p, vp, u64, C.POINTER(u64)]
    lib.vbx_proto_encode_block.restype = i32
    lib.vbx_proto_encode_block.argtypes = [i32, C.c_double, vp, i32, vp, u64, vp, u64, C.POINTER(u64)]
    lib.vbx_proto_decode_block.restype = i32
    lib.vbx_proto_decode_block.argtypes = [vp, u64, vp, vp, vp, vp, vp, u64, C.POINTER(u64)]
    lib.vbx_esdf_update_blocks.restype = i32
    lib.vbx_esdf_update_blocks.argtypes = [vp, vp, u64, i32]
    lib.vbx_esdf_set_max_distance.restype = i32
    lib.vbx_esdf_set_max_distance.argtypes = [vp, C.c_float]
    lib.vbx_esdf_set_full_euclidean.restype = i32
    lib.vbx_esdf_set_full_euclidean.argtypes = [vp, i32]
    lib.vbx_esdf_get_config.restype = i32
    lib.vbx_esdf_get_config.argtypes = [vp, C.POINTER(EsdfIntegratorConfig)]
    lib.vbx_esdf_update.restype = i32
    lib.vbx_esdf_update.argtypes = [vp, i32, i32]
    lib.vbx_esdf_add_robot_position.restype = i32
    lib.vbx_esdf_add_robot_position.argtypes = [vp, vp]
    lib.vbx_esdf_clear.restype = i32
    lib.vbx_esdf_clear.argtypes = [vp]
    for name in ("vbx_icp_run", "vbx_icp_run_device"):
        f = getattr(lib, name)
        f.restype = i32
        f.argtypes = [vp, C.POINTER(ICPConfig), vp, u64, vp, vp, C.c_uint32, vp, vp, C.POINTER(u64)]
    lib.vbx_mesh_generate.restype = i32
    lib.vbx_mesh_generate.argtypes = [vp, C.POINTER(MeshIntegratorConfig), i32, i32, C.POINTER(u64), C.POINTER(u64)]
    lib.vbx_mesh_download.restype = i32
    lib.vbx_mesh_download.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.vbx_sync.restype = i32
    lib.vbx_sync.argtypes = [vp]
    lib.vbx_block_owner.restype = i32
    lib.vbx_block_owner.argtypes = [vp, vp, C.POINTER(C.c_int32)]
    lib.vbx_host_alloc.restype = i32
    lib.vbx_host_alloc.argtypes = [vp, C.c_size_t, C.POINTER(vp)]
    lib.vbx_host_free.restype = i32
    lib.vbx_host_free.argtypes = [vp, vp]
    lib.vbx_host_copy_ms.restype = i32
    lib.vbx_host_copy_ms.argtypes = [vp, vp, C.c_size_t, C.POINTER(C.c_float)]
    lib.vbx_timer_start.restype = i32
    lib.vbx_timer_start.argtypes = [vp]
    lib.vbx_timer_stop_ms.restype = i32
    lib.vbx_timer_stop_ms.argtypes = [vp, C.POINTER(C.c_float)]
    lib.vbx_set_stage_profiling.restype = i32
    lib.vbx_set_stage_profiling.argtypes = [vp, i32]
    lib.vbx_get_stage_ms.restype = i32
    lib.vbx_get_stage_ms.argtypes = [vp, vp, vp]
    _lib = lib
    return lib


class _Context:
    """One vbx_ctx: the device-resident map shared by a TSDF layer, its ESDF layer and
    the integrators attached to them."""

    def __init__(self, config: TsdfIntegratorConfig, voxel_size: float, voxels_per_side: int,
                 options: Optional[EngineOptions]):
        self.lib = load_library()
        self.handle = C.c_void_p()
        self.config = config
        self.vps = voxels_per_side
        opt = options if options is not None else EngineOptions()
        rc = self.lib.vbx_create(C.byref(config), voxel_size, voxels_per_side, C.byref(opt),
                                 C.byref(self.handle))
        if rc != 0:
            msg = self.lib.vbx_last_error(self.handle).decode() if self.handle else "invalid arguments"
            if self.handle:
                self.lib.vbx_destroy(self.handle)
                self.handle = C.c_void_p()
            raise VoxbloxError(f"vbx_create failed ({rc}): {msg}")

    def check(self, rc: int, what: str):
        if rc != 0:
            raise VoxbloxError(f"{what} failed ({rc}): {self.lib.vbx_last_error(self.handle).decode()}")

    def close(self):
        if self.handle:
            self.lib.vbx_destroy(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Layer:
    """Layer<VoxelType> (core/layer.h:24-296) whose blocks live in HBM.

    Construct it like the reference's (voxel_size, voxels_per_side); it binds to the
    device map when the first integrator is created on it.  Read access downloads
    blocks on demand (the lazy host mirror, SURVEY.md section 8f N1)."""

    def __init__(self, voxel_size: float, voxels_per_side: int = 16, voxel_type: str = "tsdf",
                 engine_options: Optional[EngineOptions] = None):
        if not voxel_size > 0.0:  # CHECK_GT(voxel_size_, 0.0f), core/layer.h:38
            raise VoxbloxError("Check failed: voxel_size_ > 0.0f")
        if voxels_per_side <= 0:
            raise VoxbloxError("Check failed: voxels_per_side_ > 0u")
        self._voxel_size = float(np.float32(voxel_size))
        self._vps = int(voxels_per_side)
        self.voxel_type = voxel_type
        self.engine_options = engine_options
        self._ctx: Optional[_Context] = None
        self._layer_id = LAYER_TSDF if voxel_type == "tsdf" else LAYER_ESDF

    # -- reference accessors (core/layer.h:241-246)
    def voxel_size(self) -> float:
        return self._voxel_size

    def voxels_per_side(self) -> int:
        return self._vps

    def block_size(self) -> float:
        return float(np.float32(self._voxel_size) * np.float32(self._vps))

    def _bound(self) -> _Context:
        if self._ctx is None:
            raise VoxbloxError("layer is not attached to an integrator yet")
        return self._ctx

    def getNumberOfAllocatedBlocks(self) -> int:  # core/layer.h:205
        if self._ctx is None:
            return 0
        n = C.c_uint64(0)
        self._ctx.check(self._ctx.lib.vbx_num_blocks(self._ctx.handle, self._layer_id, C.byref(n)),
                        "vbx_num_blocks")
        return int(n.value)

    def _list(self, mask: int) -> np.ndarray:
        if self._ctx is None:
            return np.zeros((0, 3), dtype=np.int32)
        ctx = self._ctx
        n = C.c_uint64(0)
        ctx.check(ctx.lib.vbx_list_blocks(ctx.handle, self._layer_id, mask, None, 0, C.byref(n)),
                  "vbx_list_blocks")
        out = np.zeros((int(n.value), 3), dtype=np.int32)
        if n.value:
            ctx.check(ctx.lib.vbx_list_blocks(ctx.handle, self._layer_id, mask, out.ctypes.data,
                                              n.value, C.byref(n)), "vbx_list_blocks")
        return out

    def getAllAllocatedBlocks(self) -> np.ndarray:  # core/layer.h:184-192 (sorted here)
        return self._list(0)

    def getAllUpdatedBlocks(self, bit: int) -> np.ndarray:  # core/layer.h:194-203
        return self._list(1 << bit if bit < 3 else bit)

    def hasBlock(self, index: Sequence[int]) -> bool:  # core/layer.h:207-209
        idx = self.getAllAllocatedBlocks()
        return bool(len(idx)) and bool((idx == np.asarray(index, dtype=np.int32)).all(axis=1).any())

    def getBlocks(self, indices: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
        """Download blocks: (voxels [m, vps^3] structured, updated bits [m] u8)."""
        ctx = self._bound()
        idx = np.ascontiguousarray(indices, dtype=np.int32).reshape(-1, 3)
        dt = TSDF_DTYPE if self._layer_id == LAYER_TSDF else ESDF_DTYPE
        vox = np.zeros((idx.shape[0], self._vps ** 3), dtype=dt)
        upd = np.zeros(idx.shape[0], dtype=np.uint8)
        if idx.shape[0]:
            ctx.check(ctx.lib.vbx_download_blocks(ctx.handle, self._layer_id, idx.ctypes.data,
                                                  idx.shape[0], vox.ctypes.data, upd.ctypes.data),
                      "vbx_download_blocks")
        return vox, upd

    def mirrorUpdated(self, bit_mask: int = 0, clear_mask: int = 0, voxels_out: Optional[np.ndarray] = None):
        """getAllUpdatedBlocks(bit) + block payloads + updated().reset(bit) in one call
        (vbx_mirror_updated).  Returns (indices [m,3], voxels [m, vps^3], updated bits [m]);
        voxels_out may be a page-locked buffer from hostBuffer() (filled in place, no staging)."""
        ctx = self._bound()
        dt = TSDF_DTYPE if self._layer_id == LAYER_TSDF else ESDF_DTYPE
        n = C.c_uint64(0)
        cap = 0 if voxels_out is None else int(voxels_out.shape[0])
        while True:
            idx = np.zeros((max(cap, 1), 3), dtype=np.int32)
            upd = np.zeros(max(cap, 1), dtype=np.uint8)
            vox = voxels_out if (voxels_out is not None and cap <= voxels_out.shape[0]) else \
                np.zeros((max(cap, 1), self._vps ** 3), dtype=dt)
            ctx.check(ctx.lib.vbx_mirror_updated(ctx.handle, self._layer_id, int(bit_mask), int(clear_mask),
                                                 idx.ctypes.data, vox.ctypes.data, upd.ctypes.data, cap, C.byref(n)),
                      "vbx_mirror_updated")
            if n.value <= cap:
                m = int(n.value)
                return idx[:m], vox[:m], upd[:m]
            cap = int(n.value)
            voxels_out = None if (voxels_out is not None and cap > voxels_out.shape[0]) else voxels_out

    def serializeUpdated(self, bit_mask: int = 0, clear_mask: int = 0):
        """Block::serializeToIntegers (src/core/block.cc:159-183 / :203-234) of every block whose
        updated bits match, packed on the device.  Returns (indices [m,3], words [m, vps^3 * (3|2)] u32,
        updated bits [m])."""
        ctx = self._bound()
        wpv = 3 if self._layer_id == LAYER_TSDF else 2
        n = C.c_uint64(0)
        cap = 0
        while True:
            idx = np.zeros((max(cap, 1), 3), dtype=np.int32)
            upd = np.zeros(max(cap, 1), dtype=np.uint8)
            words = np.zeros((max(cap, 1), self._vps ** 3 * wpv), dtype=np.uint32)
            ctx.check(ctx.lib.vbx_serialize_updated(ctx.handle, self._layer_id, int(bit_mask), int(clear_mask),
                                                    idx.ctypes.data, words.ctypes.data, upd.ctypes.data, cap, C.byref(n)),
                      "vbx_serialize_updated")
            if n.value <= cap:
                m = int(n.value)
                return idx[:m], words[:m], upd[:m]
            cap = int(n.value)

    def insertSerializedBlocks(self, indices: np.ndarray, words: np.ndarray, updated_bits: Optional[np.ndarray] = None):
        """Block(BlockProto): deserializeFromIntegers into (new) blocks (core/block_inl.h:73-109)."""
        ctx = self._bound()
        idx = np.ascontiguousarray(indices, dtype=np.int32).reshape(-1, 3)
        w = np.ascontiguousarray(words, dtype=np.uint32).reshape(idx.shape[0], -1)
        upd = None if updated_bits is None else np.ascontiguousarray(updated_bits, dtype=np.uint8)
        ctx.check(ctx.lib.vbx_deserialize_blocks(ctx.handle, self._layer_id, idx.ctypes.data, idx.shape[0], w.ctypes.data,
                                                 None if upd is None else upd.ctypes.data), "vbx_deserialize_blocks")

    def saveToFile(self, file_path: str, clear_file: bool = True) -> bool:  # core/layer_inl.h:81-86
        ctx = self._bound()
        ctx.check(ctx.lib.vbx_save_layer(ctx.handle, self._layer_id, str(file_path).encode(), int(bool(clear_file))),
                  "saveToFile")
        return True

    def loadBlocksFromFile(self, file_path: str) -> int:
        """io::LoadBlocksFromFile(file_path, kReplace, multiple_layer_support=true, this)
        (io/layer_io_inl.h:13-90); returns the number of blocks loaded."""
        ctx = self._bound()
        n = C.c_uint64(0)
        ctx.check(ctx.lib.vbx_load_layer(ctx.handle, self._layer_id, str(file_path).encode(), C.byref(n)),
                  "LoadBlocksFromFile")
        return int(n.value)

    def getBlockByIndex(self, index: Sequence[int]) -> np.ndarray:
        """core/layer.h:55-62: LOG(FATAL) "Accessed unallocated block" -> VoxbloxError."""
        vox, _ = self.getBlocks(np.asarray([index], dtype=np.int32))
        return vox[0]

    def blocks(self) -> Dict[Tuple[int, int, int], np.ndarray]:
        idx = self.getAllAllocatedBlocks()
        vox, _ = self.getBlocks(idx)
        return {tuple(int(v) for v in i): vox[k] for k, i in enumerate(idx)}

    # -- measurement aids (reference: timing::Timer, utils/timing.h:132-199)
    def timerStart(self):
        ctx = self._bound()
        ctx.check(ctx.lib.vbx_timer_start(ctx.handle), "vbx_timer_start")

    def timerStopMs(self) -> float:
        ctx = self._bound()
        ms = C.c_float(0)
        ctx.check(ctx.lib.vbx_timer_stop_ms(ctx.handle, C.byref(ms)), "vbx_timer_stop_ms")
        return float(ms.value)

    def hostBuffer(self, shape, dtype) -> np.ndarray:
        """A page-locked numpy array (cudaHostAlloc) for clouds handed to integratePointCloud."""
        ctx = self._bound()
        dt = np.dtype(dtype)
        nbytes = int(np.prod(shape)) * dt.itemsize
        ptr = C.c_void_p()
        ctx.check(ctx.lib.vbx_host_alloc(ctx.handle, max(nbytes, 1), C.byref(ptr)), "vbx_host_alloc")
        buf = (C.c_char * max(nbytes, 1)).from_address(ptr.value)
        arr = np.frombuffer(buf, dtype=dt, count=int(np.prod(shape))).reshape(shape)
        ctx._host_allocs = getattr(ctx, "_host_allocs", [])
        ctx._host_allocs.append(ptr)
        return arr

    def hostCopyMs(self, arr: np.ndarray) -> float:
        ctx = self._bound()
        ms = C.c_float(0)
        a = np.ascontiguousarray(arr)
        ctx.check(ctx.lib.vbx_host_copy_ms(ctx.handle, a.ctypes.data, a.nbytes, C.byref(ms)), "vbx_host_copy_ms")
        return float(ms.value)

    def setStageProfiling(self, enabled: bool):
        ctx = self._bound()
        ctx.check(ctx.lib.vbx_set_stage_profiling(ctx.handle, int(enabled)), "vbx_set_stage_profiling")

    STAGE_NAMES = ("point_keys", "point_sort", "ray_count", "scan", "assign", "ray_emit",
                   "update_sort", "apply", "bundle_merge", "esdf_propagate", "esdf_raise", "esdf_lower", "bundle_order")

    def stageMs(self):
        ctx = self._bound()
        ms = np.zeros(16, dtype=np.float64)
        calls = np.zeros(16, dtype=np.uint64)
        ctx.check(ctx.lib.vbx_get_stage_ms(ctx.handle, ms.ctypes.data, calls.ctypes.data), "vbx_get_stage_ms")
        return {n: (float(ms[i]), int(calls[i])) for i, n in enumerate(self.STAGE_NAMES)}

    def sync(self):
        ctx = self._bound()
        ctx.check(ctx.lib.vbx_sync(ctx.handle), "vbx_sync")

    def insertBlocks(self, indices: np.ndarray, voxels: np.ndarray, updated_bits: Optional[np.ndarray] = None):
        """Layer::insertBlock / allocateBlockPtrByIndex + voxel copy (core/layer.h:103-111,152-161)."""
        ctx = self._bound()
        idx = np.ascontiguousarray(indices, dtype=np.int32).reshape(-1, 3)
        dt = TSDF_DTYPE if self._layer_id == LAYER_TSDF else ESDF_DTYPE
        vox = np.ascontiguousarray(voxels, dtype=dt).reshape(idx.shape[0], self._vps ** 3)
        upd = None if updated_bits is None else np.ascontiguousarray(updated_bits, dtype=np.uint8)
        ctx.check(ctx.lib.vbx_upload_blocks(ctx.handle, self._layer_id, idx.ctypes.data, idx.shape[0], vox.ctypes.data,
                                            None if upd is None else upd.ctypes.data), "vbx_upload_blocks")

    def _block_bytes(self) -> int:
        return (TSDF_DTYPE if self._layer_id == LAYER_TSDF else ESDF_DTYPE).itemsize * self._vps ** 3

    def gatherUpdatedDevice(self, bit_mask: int = 0, clear_mask: int = 0, owned_only: bool = False,
                            d_idx3=None, d_voxels=None, cap: Optional[int] = None) -> int:
        """vbx_gather_updated_device: the blocks whose updated bits match `bit_mask` (0 = all; with owned_only
        only the blocks this rank owns), ascending (x, y, z), gathered on the device into `d_idx3` (3 int32 per
        block) and `d_voxels` (raw voxel payloads) -- CUDA tensors, or raw device pointers with `cap` -- and
        `clear_mask` reset on them.  Returns the number of matching blocks; when it exceeds the capacity
        (default: what both tensors hold, 0 without buffers) nothing is copied or cleared."""
        ctx = self._bound()
        if cap is None:
            cap = 0 if d_idx3 is None else min(_nbytes(d_idx3) // 12, _nbytes(d_voxels) // self._block_bytes())
        n = C.c_uint64(0)
        ctx.check(ctx.lib.vbx_gather_updated_device(ctx.handle, self._layer_id, int(bit_mask), int(clear_mask),
                                                    int(bool(owned_only)), _device_ptr(d_idx3), _device_ptr(d_voxels),
                                                    int(cap), C.byref(n)), "vbx_gather_updated_device")
        return int(n.value)

    def insertBlocksDevice(self, d_idx3, d_voxels, m: Optional[int] = None,
                           updated_bits: int = UPDATED_MAP | UPDATED_MESH | UPDATED_ESDF):
        """vbx_upload_blocks_device: insertBlocks with the indices (m x 3 int32) and raw voxel payloads already on
        the device (CUDA tensors, or raw device pointers with `m`); every written block's updated() bits become
        `updated_bits` -- by default what Block::updated().set() gives a block a scan touched.  A sharded engine
        refuses blocks its own rank owns."""
        ctx = self._bound()
        if m is None:
            m = _nbytes(d_idx3) // 12
        ctx.check(ctx.lib.vbx_upload_blocks_device(ctx.handle, self._layer_id, _device_ptr(d_idx3), int(m),
                                                   _device_ptr(d_voxels), int(updated_bits)), "vbx_upload_blocks_device")

    def stagingBytes(self) -> int:
        """Bytes of the engine's page-locked staging buffer (0: never allocated; vbx_debug_staging_bytes)."""
        ctx = self._bound()
        n = C.c_uint64(0)
        ctx.check(ctx.lib.vbx_debug_staging_bytes(ctx.handle, C.byref(n)), "vbx_debug_staging_bytes")
        return int(n.value)

    def removeBlock(self, index: Sequence[int]):  # core/layer.h:163
        self.removeBlocks(np.asarray([index], dtype=np.int32))

    def removeBlocks(self, indices: np.ndarray):
        ctx = self._bound()
        idx = np.ascontiguousarray(indices, dtype=np.int32).reshape(-1, 3)
        ctx.check(ctx.lib.vbx_remove_blocks(ctx.handle, self._layer_id, idx.ctypes.data, idx.shape[0]),
                  "vbx_remove_blocks")

    def removeAllBlocks(self):  # core/layer.h:164
        ctx = self._bound()
        ctx.check(ctx.lib.vbx_clear(ctx.handle, self._layer_id), "vbx_clear")

    def clearUpdated(self, bit: int):
        """block.updated().reset(bit) on every block (esdf_integrator.cc:113-121)."""
        ctx = self._bound()
        ctx.check(ctx.lib.vbx_clear_updated(ctx.handle, self._layer_id, 1 << bit), "vbx_clear_updated")


def _device_ptr(x) -> Optional[int]:
    """A CUDA tensor's (contiguous) data pointer, or a raw pointer as given."""
    if x is None or isinstance(x, int):
        return x
    if not (x.is_cuda and x.is_contiguous()):
        raise VoxbloxError("expected a contiguous CUDA tensor")
    return x.data_ptr()


def _nbytes(x) -> int:
    if x is None or isinstance(x, int):
        raise VoxbloxError("raw device pointers need an explicit size")
    return x.numel() * x.element_size()


def _as_pose(T_G_C) -> Tuple[np.ndarray, np.ndarray]:
    q, t = T_G_C
    q = np.ascontiguousarray(q, dtype=np.float32).reshape(4)
    t = np.ascontiguousarray(t, dtype=np.float32).reshape(3)
    return q, t


class TsdfIntegratorBase:
    """TsdfIntegratorBase (tsdf_integrator.h:51-198) dispatching to the device."""

    kind = 0

    def __init__(self, config: TsdfIntegratorConfig, layer: Layer):
        if layer is None:  # CHECK_NOTNULL(layer), tsdf_integrator.cc:69
            raise VoxbloxError("Check failed: 'layer' Must be non NULL")
        if layer.voxel_type != "tsdf":
            raise VoxbloxError("TSDF integrators need a Layer<TsdfVoxel>")
        if layer._ctx is None:
            layer._ctx = _Context(config, layer.voxel_size(), layer.voxels_per_side(),
                                  layer.engine_options)
        elif bytes(layer._ctx.config) != bytes(config):
            raise VoxbloxError("integrators sharing one device layer must share one Config")
        self.layer_ = layer
        self._ctx = layer._ctx
        cfg = TsdfIntegratorConfig()
        self._ctx.check(self._ctx.lib.vbx_get_tsdf_config(self._ctx.handle, C.byref(cfg)),
                        "vbx_get_tsdf_config")
        self.config_ = cfg

    def getConfig(self) -> TsdfIntegratorConfig:  # tsdf_integrator.h:106
        return self.config_

    def integratePointCloud(self, T_G_C, points_C: np.ndarray, colors: np.ndarray,
                            freespace_points: bool = False) -> None:
        """tsdf_integrator.h:100-103.  points_C [N,3] f32 (Pointcloud), colors [N,4] u8
        (Colors) in HOST memory; CHECK_EQ(points_C.size(), colors.size()) (cc:247)."""
        q, t = _as_pose(T_G_C)
        pts = np.ascontiguousarray(points_C, dtype=np.float32).reshape(-1, 3)
        cols = np.ascontiguousarray(colors, dtype=np.uint8).reshape(-1, 4)
        if pts.shape[0] != cols.shape[0]:
            raise VoxbloxError("Check failed: points_C.size() == colors.size()")
        ctx = self._ctx
        ctx.check(ctx.lib.vbx_tsdf_integrate(ctx.handle, self.kind, q.ctypes.data, t.ctypes.data,
                                             pts.ctypes.data, cols.ctypes.data, pts.shape[0],
                                             int(bool(freespace_points))), "integratePointCloud")

    def integratePointCloudDevice(self, T_G_C, d_xyz: int, d_rgba: int, n: int,
                                  freespace_points: bool = False) -> None:
        """Same call with the cloud already resident in HBM (raw device pointers)."""
        q, t = _as_pose(T_G_C)
        ctx = self._ctx
        ctx.check(ctx.lib.vbx_tsdf_integrate_device(ctx.handle, self.kind, q.ctypes.data,
                                                    t.ctypes.data, d_xyz, d_rgba, n,
                                                    int(bool(freespace_points))),
                  "integratePointCloudDevice")

    def integratePointCloudAsync(self, T_G_C, points, colors, n: Optional[int] = None,
                                 freespace_points: bool = False) -> None:
        """Enqueue a scan and return (vbx_tsdf_integrate_async).  points / colors are either
        page-locked host numpy arrays (kept alive and untouched by the caller until Layer.sync())
        or raw device pointers (ints) with n given."""
        q, t = _as_pose(T_G_C)
        ctx = self._ctx
        if isinstance(points, (int, np.integer)):
            px, pc, cnt, on_dev = int(points), int(colors), int(n), 1
        else:
            assert points.dtype == np.float32 and points.flags.c_contiguous
            assert colors.dtype == np.uint8 and colors.flags.c_contiguous
            if points.shape[0] != colors.shape[0]:
                raise VoxbloxError("Check failed: points_C.size() == colors.size()")
            px, pc, cnt, on_dev = points.ctypes.data, colors.ctypes.data, points.shape[0], 0
        ctx.check(ctx.lib.vbx_tsdf_integrate_async(ctx.handle, self.kind, q.ctypes.data, t.ctypes.data, px, pc, cnt,
                                                   int(bool(freespace_points)), on_dev), "integratePointCloudAsync")

    def counters(self) -> Dict[str, int]:
        out = np.zeros(16, dtype=np.uint64)
        self._ctx.check(self._ctx.lib.vbx_get_counters(self._ctx.handle, out.ctypes.data),
                        "vbx_get_counters")
        names = ["rays", "clear_rays", "updates", "voxels_touched", "blocks_touched",
                 "blocks_allocated", "valid_points", "kernel_launches", "kernel_launches_total", "refolded_bundles",
                 "refolded_points", "passes", "bundle_key_bits", "async_redone_total", "async_wait_ns_total", "async_submit_ns_total"]
        return {k: int(v) for k, v in zip(names, out)}

    APPLY_PATHS = ["long_runs", "long_rested", "step_saturated", "step_int_scan", "step_prefix", "chunk_saturated",
                   "chunk_const", "chunk_prefix", "chunk_sequential", "chunk_exact", "short_runs", "short_crossed"]

    def countApplyPaths(self, enabled: bool = True) -> None:
        """Make later integrate calls count the apply's paths (vbx_debug_count_apply_paths; off by default)."""
        self._ctx.check(self._ctx.lib.vbx_debug_count_apply_paths(self._ctx.handle, int(bool(enabled))),
                        "vbx_debug_count_apply_paths")

    def serialFast(self, enabled: bool = True) -> None:
        """Make later Fast calls walk their rays on one thread in point order, the reference's one-thread
        schedule (vbx_debug_serial_fast; off by default, for tests)."""
        self._ctx.check(self._ctx.lib.vbx_debug_serial_fast(self._ctx.handle, int(bool(enabled))),
                        "vbx_debug_serial_fast")

    def applyPaths(self) -> Dict[str, int]:
        """How often each arithmetic path of the apply ran in the last call (vbx_debug_apply_paths)."""
        out = np.zeros(16, dtype=np.uint64)
        self._ctx.check(self._ctx.lib.vbx_debug_apply_paths(self._ctx.handle, out.ctypes.data), "vbx_debug_apply_paths")
        return {k: int(v) for k, v in zip(self.APPLY_PATHS, out)}

    def lastDeviceMs(self) -> float:
        ms = C.c_float(0)
        self._ctx.check(self._ctx.lib.vbx_last_device_ms(self._ctx.handle, C.byref(ms)),
                        "vbx_last_device_ms")
        return float(ms.value)


class SimpleTsdfIntegrator(TsdfIntegratorBase):  # tsdf_integrator.h:211-230
    kind = TsdfIntegratorType.kSimple


class MergedTsdfIntegrator(TsdfIntegratorBase):  # tsdf_integrator.h:232-271
    kind = TsdfIntegratorType.kMerged


class FastTsdfIntegrator(TsdfIntegratorBase):  # tsdf_integrator.h:273-341
    kind = TsdfIntegratorType.kFast


class TsdfIntegratorFactory:
    """TsdfIntegratorFactory::create (tsdf_integrator.cc:8-46)."""

    @staticmethod
    def create(integrator_type, config: TsdfIntegratorConfig, layer: Layer) -> TsdfIntegratorBase:
        if isinstance(integrator_type, str):
            if not integrator_type:
                raise VoxbloxError("Check failed: !integrator_type_name.empty()")
            if integrator_type not in kTsdfIntegratorTypeNames:
                raise VoxbloxError(f"Unknown TSDF integrator type: {integrator_type}")
            integrator_type = kTsdfIntegratorTypeNames.index(integrator_type) + 1
        if layer is None:
            raise VoxbloxError("Check failed: 'layer' Must be non NULL")
        cls = {1: SimpleTsdfIntegrator, 2: MergedTsdfIntegrator, 3: FastTsdfIntegrator}.get(
            int(integrator_type))
        if cls is None:
            raise VoxbloxError(f"Unknown TSDF integrator type: {int(integrator_type)}")
        return cls(config, layer)


class EsdfIntegrator:
    """EsdfIntegrator (esdf_integrator.h:25-178) over the device map."""

    def __init__(self, config: EsdfIntegratorConfig, tsdf_layer: Layer, esdf_layer: Layer):
        if tsdf_layer is None or esdf_layer is None:  # CHECK(tsdf_layer_), esdf_integrator.cc:11-12
            raise VoxbloxError("Check failed: tsdf_layer_ / esdf_layer_")
        if esdf_layer.voxels_per_side() != tsdf_layer.voxels_per_side():  # cc:17
            raise VoxbloxError("Check failed: esdf_layer_->voxels_per_side() == tsdf_layer_->voxels_per_side()")
        if abs(esdf_layer.voxel_size() - tsdf_layer.voxel_size()) > 1e-6:  # cc:18
            raise VoxbloxError("Check failed: voxel sizes differ")
        ctx = tsdf_layer._bound()
        self._ctx = ctx
        self.config_ = config
        esdf_layer._ctx = ctx
        esdf_layer._layer_id = LAYER_ESDF
        self.tsdf_layer_, self.esdf_layer_ = tsdf_layer, esdf_layer
        ctx.check(ctx.lib.vbx_esdf_create(ctx.handle, C.byref(config)), "vbx_esdf_create")

    def updateFromTsdfLayer(self, clear_updated_flag: bool) -> None:  # esdf_integrator.cc:104-122
        self._ctx.check(self._ctx.lib.vbx_esdf_update(self._ctx.handle, 0, int(bool(clear_updated_flag))),
                        "updateFromTsdfLayer")

    def updateFromTsdfBlocks(self, tsdf_blocks, incremental: bool = False) -> None:  # esdf_integrator.cc:124-302
        idx = np.ascontiguousarray(tsdf_blocks, dtype=np.int32).reshape(-1, 3)
        self._ctx.check(self._ctx.lib.vbx_esdf_update_blocks(self._ctx.handle, idx.ctypes.data, idx.shape[0],
                                                             int(bool(incremental))), "updateFromTsdfBlocks")

    def _config(self) -> EsdfIntegratorConfig:
        out = EsdfIntegratorConfig()
        self._ctx.check(self._ctx.lib.vbx_esdf_get_config(self._ctx.handle, C.byref(out)), "vbx_esdf_get_config")
        return out

    def getEsdfMaxDistance(self) -> float:  # esdf_integrator.h:139
        return float(self._config().max_distance_m)

    def setEsdfMaxDistance(self, max_distance: float) -> None:  # esdf_integrator.h:140-145
        self._ctx.check(self._ctx.lib.vbx_esdf_set_max_distance(self._ctx.handle, float(max_distance)),
                        "setEsdfMaxDistance")

    def getFullEuclidean(self) -> bool:  # esdf_integrator.h:146
        return bool(self._config().full_euclidean_distance)

    def setFullEuclidean(self, full_euclidean: bool) -> None:  # esdf_integrator.h:147-149
        self._ctx.check(self._ctx.lib.vbx_esdf_set_full_euclidean(self._ctx.handle, int(bool(full_euclidean))),
                        "setFullEuclidean")

    def addNewRobotPosition(self, position) -> None:  # esdf_integrator.cc:25-92
        p = np.ascontiguousarray(position, dtype=np.float32).reshape(3)
        self._ctx.check(self._ctx.lib.vbx_esdf_add_robot_position(self._ctx.handle, p.ctypes.data),
                        "addNewRobotPosition")

    def clear(self) -> None:  # esdf_integrator.h:135-140
        self._ctx.check(self._ctx.lib.vbx_esdf_clear(self._ctx.handle), "EsdfIntegrator::clear")

    def updateFromTsdfLayerBatch(self) -> None:  # esdf_integrator.cc:94-102
        self._ctx.check(self._ctx.lib.vbx_esdf_update(self._ctx.handle, 1, 0), "updateFromTsdfLayerBatch")

    def counters(self) -> Dict[str, int]:
        out = np.zeros(16, dtype=np.uint64)
        self._ctx.check(self._ctx.lib.vbx_esdf_get_counters(self._ctx.handle, out.ctypes.data),
                        "vbx_esdf_get_counters")
        names = ["blocks", "lower", "raise", "new", "raised_voxels", "relaxations", "sweeps",
                 "kernel_launches"]
        return {k: int(v) for k, v in zip(names, out)}

    def lastDeviceMs(self) -> float:
        ms = C.c_float(0)
        self._ctx.check(self._ctx.lib.vbx_last_device_ms(self._ctx.handle, C.byref(ms)),
                        "vbx_last_device_ms")
        return float(ms.value)


class Mesh:
    """Mesh (mesh/mesh.h:36-164): the triangles of one block, three consecutive vertices each."""

    def __init__(self, block_size: float, origin):
        self.block_size = block_size
        self.origin = np.asarray(origin, dtype=np.float32)
        self.vertices = np.zeros((0, 3), np.float32)
        self.normals = np.zeros((0, 3), np.float32)
        self.colors = np.zeros((0, 4), np.uint8)
        self.indices = np.zeros(0, np.uint64)
        self.updated = False

    def size(self) -> int:
        return int(self.vertices.shape[0])


class MeshLayer:
    """MeshLayer (mesh/mesh_layer.h:22-310): block index -> Mesh, kept on the host like the
    reference's (its consumers -- ROS publishing, PLY output -- read it there)."""

    def __init__(self, block_size: float):
        self._block_size = float(np.float32(block_size))
        self._meshes: Dict[Tuple[int, int, int], Mesh] = {}

    def block_size(self) -> float:
        return self._block_size

    def allocateMeshPtrByIndex(self, index) -> Mesh:  # mesh_layer.h:79-87, :108-121
        key = tuple(int(v) for v in index)
        m = self._meshes.get(key)
        if m is None:
            origin = np.asarray(key, dtype=np.float32) * np.float32(self._block_size)
            m = self._meshes[key] = Mesh(self._block_size, origin)
        return m

    def getMeshPtrByIndex(self, index) -> Optional[Mesh]:
        return self._meshes.get(tuple(int(v) for v in index))

    def getAllAllocatedMeshes(self) -> np.ndarray:  # sorted by (x, y, z)
        return np.array(sorted(self._meshes), dtype=np.int32).reshape(-1, 3)

    def getAllUpdatedMeshes(self) -> np.ndarray:
        return np.array(sorted(k for k, m in self._meshes.items() if m.updated), dtype=np.int32).reshape(-1, 3)

    def getNumberOfAllocatedMeshes(self) -> int:
        return len(self._meshes)


class ICP:
    """voxblox::ICP (alignment/icp.h:72-233): point-to-TSDF pose refinement against the device map."""

    def __init__(self, config: ICPConfig):
        self.config_ = config

    def refiningRollPitch(self) -> bool:  # icp.h:125
        return bool(self.config_.refine_roll_pitch)

    def runICP(self, tsdf_layer: "Layer", points, inital_T_tsdf_sensor, seed: int):
        """runICP(tsdf_layer, points, inital_T_tsdf_sensor, &refined_T_tsdf_sensor, seed) (icp.h:118-123):
        returns (number of successful mini batches, (q_wxyz, t) refined)."""
        return self._run(tsdf_layer, np.ascontiguousarray(points, dtype=np.float32).ctypes.data, int(len(points)),
                         inital_T_tsdf_sensor, seed, device=False)

    def runICPDevice(self, tsdf_layer: "Layer", d_points_ptr: int, n: int, inital_T_tsdf_sensor, seed: int):
        """The same with the cloud (3n floats) already in device memory."""
        return self._run(tsdf_layer, d_points_ptr, n, inital_T_tsdf_sensor, seed, device=True)

    def _run(self, tsdf_layer, ptr, n, T, seed, device):
        ctx = tsdf_layer._bound()
        q = np.ascontiguousarray(T[0], dtype=np.float32)
        t = np.ascontiguousarray(T[1], dtype=np.float32)
        oq, ot, nu = np.zeros(4, np.float32), np.zeros(3, np.float32), C.c_uint64(0)
        f = ctx.lib.vbx_icp_run_device if device else ctx.lib.vbx_icp_run
        ctx.check(f(ctx.handle, C.byref(self.config_), ptr, n, q.ctypes.data, t.ctypes.data, int(seed) & 0xffffffff,
                    oq.ctypes.data, ot.ctypes.data, C.byref(nu)), "runICP")
        return int(nu.value), (oq, ot)


class MeshIntegrator:
    """MeshIntegrator<TsdfVoxel> (mesh/mesh_integrator.h:72-412) over the device map."""

    def __init__(self, config: MeshIntegratorConfig, sdf_layer: Layer, mesh_layer: MeshLayer):
        if sdf_layer is None or mesh_layer is None:  # CHECK_NOTNULL, mesh_integrator.h:89-91
            raise VoxbloxError("Check failed: 'sdf_layer' / 'mesh_layer' Must be non NULL")
        self.config_ = config
        self.sdf_layer_ = sdf_layer
        self.mesh_layer_ = mesh_layer

    def generateMesh(self, only_mesh_updated_blocks: bool, clear_updated_flag: bool) -> None:  # :132-160
        ctx = self.sdf_layer_._bound()
        nb, nv = C.c_uint64(0), C.c_uint64(0)
        ctx.check(ctx.lib.vbx_mesh_generate(ctx.handle, C.byref(self.config_), int(bool(only_mesh_updated_blocks)),
                                            int(bool(clear_updated_flag)), C.byref(nb), C.byref(nv)), "generateMesh")
        nb, nv = int(nb.value), int(nv.value)
        self.last_blocks, self.last_vertices = nb, nv
        if nb == 0:
            return
        idx = np.zeros((nb, 3), np.int32)
        first = np.zeros(nb + 1, np.uint64)
        vertices = np.zeros((nv, 3), np.float32)
        normals = np.zeros((nv, 3), np.float32)
        use_color = bool(self.config_.use_color)
        colors = np.zeros((nv, 4), np.uint8)
        ctx.check(ctx.lib.vbx_mesh_download(ctx.handle, idx.ctypes.data, first.ctypes.data, vertices.ctypes.data,
                                            normals.ctypes.data, colors.ctypes.data if use_color and nv else None),
                  "vbx_mesh_download")
        for b in range(nb):
            lo, hi = int(first[b]), int(first[b + 1])
            m = self.mesh_layer_.allocateMeshPtrByIndex(idx[b])  # :146-149
            m.vertices = vertices[lo:hi].copy()                   # updateMeshForBlock: clear + refill, :238-260
            m.normals = normals[lo:hi].copy()
            m.colors = colors[lo:hi].copy() if use_color else np.zeros((0, 4), np.uint8)
            m.indices = np.arange(hi - lo, dtype=np.uint64)       # marching_cubes.h:97-99
            m.updated = True

    def lastDeviceMs(self) -> float:
        ctx = self.sdf_layer_._bound()
        ms = C.c_float(0)
        ctx.check(ctx.lib.vbx_last_device_ms(ctx.handle, C.byref(ms)), "vbx_last_device_ms")
        return float(ms.value)
