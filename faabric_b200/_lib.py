"""ctypes binding to the in-tree native library ``lib/libfaabric_b200.so``.

The library is built by :mod:`faabric_b200.build` (nvcc sm_90a + g++).  Import
fails loudly if it is missing on a GPU box: there is no Python/eager fallback
for the device ops.
"""

from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

_LIB_PATH = Path(__file__).resolve().parent / "lib" / "libfaabric_b200.so"
_lib = None


class FbConfig(C.Structure):
    _fields_ = [
        ("heapBytes", C.c_uint64),
        ("stageBytes", C.c_uint64),
        ("slotBytes", C.c_uint64),
        ("timeoutMs", C.c_uint64),
        ("useVmm", C.c_int32),
        ("useMulticast", C.c_int32),
        ("maxBlocks", C.c_int32),
        ("threads", C.c_int32),
        ("channels", C.c_int32),
        ("reserved", C.c_int32),
        ("llMaxBytes", C.c_uint64),
        ("oneShotMaxBytes", C.c_uint64),
        ("nvlsMinBytes", C.c_uint64),
        ("bcast2StepMinBytes", C.c_uint64),
        ("p2pBounceBytes", C.c_uint64),
        ("groupBlocks", C.c_int32),
        ("streamSync", C.c_int32),
    ]


class FbMergeRegion(C.Structure):
    _fields_ = [
        ("offset", C.c_uint64),
        ("length", C.c_uint64),
        ("dataType", C.c_int32),
        ("op", C.c_int32),
    ]


class FbDiffDesc(C.Structure):
    _fields_ = [
        ("offset", C.c_uint64),
        ("length", C.c_uint64),
        ("dataType", C.c_int32),
        ("op", C.c_int32),
    ]


def _sig(lib, name, restype, argtypes):
    fn = getattr(lib, name)
    fn.restype = restype
    fn.argtypes = argtypes
    return fn


def load():
    """Load (building first if necessary) and return the ctypes library."""
    global _lib
    if _lib is not None:
        return _lib
    if not _LIB_PATH.exists() or os.environ.get("FAABRIC_B200_REBUILD"):
        from . import build as _build

        _build.build(verbose=False, bins=False)
    lib = C.CDLL(str(_LIB_PATH), mode=C.RTLD_GLOBAL)
    vp, u64, i32, u32 = C.c_void_p, C.c_uint64, C.c_int, C.c_uint32
    cfgp = C.POINTER(FbConfig)

    _sig(lib, "fb_last_error", C.c_char_p, [])
    _sig(lib, "fb_error_string", C.c_char_p, [i32])
    _sig(lib, "fb_cuda_device_count", i32, [])
    _sig(lib, "fb_default_config", None, [cfgp])
    _sig(lib, "fb_group_create_local", vp, [i32, C.POINTER(C.c_int), cfgp])
    _sig(lib, "fb_group_comm", vp, [vp, i32])
    _sig(lib, "fb_group_destroy", None, [vp])
    _sig(lib, "fb_comm_create_ipc", vp, [i32, i32, i32, C.c_char_p, cfgp])
    _sig(lib, "fb_comm_destroy", None, [vp])
    for n in ("rank", "size", "device", "has_multicast", "last_algo"):
        _sig(lib, f"fb_comm_{n}", i32, [vp])
    _sig(lib, "fb_comm_backing", C.c_char_p, [vp])
    _sig(lib, "fb_comm_configure", i32, [vp, i32, u64])
    _sig(lib, "fb_comm_set_allreduce_table", i32, [vp, i32, C.POINTER(C.c_uint64), C.POINTER(C.c_int)])
    _sig(lib, "fb_comm_load_tuning", i32, [vp, C.c_char_p])
    _sig(lib, "fb_tuning_normalise", i32, [C.c_char_p, C.c_char_p, i32])
    _sig(lib, "fb_comm_stats", None, [vp, C.POINTER(C.c_uint64), i32])
    _sig(lib, "fb_comm_alloc", C.c_int64, [vp, u64])
    _sig(lib, "fb_comm_free", None, [vp, u64])
    _sig(lib, "fb_comm_heap_ptr", vp, [vp, u64, i32])
    _sig(lib, "fb_comm_in_heap", i32, [vp, vp, u64])
    _sig(lib, "fb_comm_check_error", u32, [vp, vp])
    _sig(lib, "fb_comm_host_barrier", None, [vp])
    _sig(lib, "fb_comm_subset", vp, [vp, C.POINTER(C.c_int), i32, i32])
    _sig(lib, "fb_comm_free_subset_slots", u32, [vp])
    _sig(lib, "fb_comm_is_subset", i32, [vp])

    _sig(lib, "fb_allreduce", i32, [vp, vp, vp, u64, i32, i32, i32, i32, vp])
    _sig(lib, "fb_reduce", i32, [vp, vp, vp, u64, i32, i32, i32, i32, vp])
    _sig(lib, "fb_reduce_scatter", i32, [vp, vp, vp, u64, i32, i32, i32, vp])
    _sig(lib, "fb_scan", i32, [vp, vp, vp, u64, i32, i32, i32, vp])
    _sig(lib, "fb_broadcast", i32, [vp, vp, u64, i32, i32, vp])
    _sig(lib, "fb_allgather", i32, [vp, vp, vp, u64, i32, vp])
    _sig(lib, "fb_gather", i32, [vp, vp, vp, u64, i32, i32, vp])
    _sig(lib, "fb_scatter", i32, [vp, vp, vp, u64, i32, i32, vp])
    _sig(lib, "fb_alltoall", i32, [vp, vp, vp, u64, i32, vp])
    _sig(lib, "fb_barrier", i32, [vp, vp])
    _sig(lib, "fb_send", i32, [vp, vp, u64, i32, vp])
    _sig(lib, "fb_recv", i32, [vp, vp, u64, i32, vp])
    _sig(lib, "fb_sendrecv", i32, [vp, vp, u64, i32, vp, u64, i32, vp])
    _sig(lib, "fb_comm_stream_sync", i32, [vp])
    _sig(lib, "fb_comm_stream_wait_supported", i32, [vp])
    _sig(lib, "fb_comm_sync_bounded", i32, [vp, vp, u64])
    vpp = C.POINTER(C.c_void_p)
    u64p = C.POINTER(C.c_uint64)
    _sig(lib, "fb_group_prepare", vp, [vp, i32, i32, vpp, vpp, u64p, i32])
    _sig(lib, "fb_group_launch", i32, [vp, i32, vp, i32, i32, i32, vp])
    _sig(lib, "fb_group_many", i32, [vp, i32, i32, vpp, vpp, u64p, i32, i32, i32, i32, vp])
    _sig(lib, "fb_group_plan_launches", i32, [vp])
    _sig(lib, "fb_group_plan_free", None, [vp])
    _sig(lib, "fb_comm_set_neighbors", i32, [vp, i32, C.POINTER(C.c_int), C.POINTER(C.c_int), i32, i32, i32])
    _nv = [vp, i32, i32, vpp, vpp, u64p, u64p, i32, u64p, u64p, i32, i32]
    _sig(lib, "fb_neighbor_v_streams", i32, _nv + [u64p, i32])
    _sig(lib, "fb_group_prepare_v", vp, _nv + [u64p, i32])
    _sig(lib, "fb_group_many_v", i32, _nv + [u64p, i32, i32, vp])
    _sig(lib, "fb_put_signal", i32, [vp, vp, u64, u64, i32, i32, i32, vp])
    _sig(lib, "fb_wait_signal", i32, [vp, i32, u32, vp])
    _sig(lib, "fb_accumulate", i32, [vp, vp, u64, u64, i32, i32, i32, vp, vp])
    _sig(lib, "fb_compare_and_swap", i32, [vp, vp, vp, vp, u64, i32, i32, vp])
    i32p = C.POINTER(C.c_int32)
    _sig(lib, "fb_put_get_many", i32, [vp, i32, vpp, u64p, u64p, i32p, i32p, vp])
    _sig(lib, "fb_accumulate_many", i32, [vp, i32, vpp, vpp, u64p, u64p, i32p, i32, i32, vp])

    regp = C.POINTER(FbMergeRegion)
    _sig(
        lib,
        "fb_snapshot_prepare_regions",
        i32,
        [regp, i32, i32, u64, regp, i32, C.POINTER(C.c_int32), C.POINTER(C.c_int)],
    )
    _sig(
        lib,
        "fb_snapshot_diff_push",
        i32,
        [vp, vp, vp, u64, vp, i32, vp, i32, vp, vp, vp, vp, i32, i32, vp],
    )
    _sig(lib, "fb_dirty_scan", i32, [vp, vp, u64, vp, vp, i32, vp])
    _sig(lib, "fb_flags_or", i32, [vp, vp, u64, vp])
    _sig(lib, "fb_state_push_dirty", i32, [vp, vp, vp, u64, vp, i32, vp])
    _sig(lib, "fb_state_flag_range", i32, [vp, u64, u64, vp])
    _sig(lib, "fb_state_block_bytes", i32, [])
    _sig(lib, "fb_chunk_runs", i32, [vp, u64, u32, u64, vp, u32, vp, vp])
    _sig(lib, "fb_snapshot_apply", i32, [vp, u64, vp, vp, vp, u32, vp])
    _lib = lib
    return lib


def lib_path() -> Path:
    return _LIB_PATH


def last_error() -> str:
    return load().fb_last_error().decode()
