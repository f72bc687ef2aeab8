"""ctypes binding of libmzgpu.so — the C ABI declared in include/mzgpu.h.

This is the same binding surface a Rust timely worker would use through
``extern "C"`` (see INTEGRATION.md).  There is no CPU fallback: if the CUDA
library is missing this module raises at import time, and every call fails
loudly (``MzGpuError``) when there is no usable CUDA device.
"""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libmzgpu.so")

if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
        "(nvcc, sm_90a). materialize_b200 has no CPU fallback."
    )

lib = C.CDLL(LIB_PATH)

# ---------------------------------------------------------------- row dtypes
R16 = np.dtype([("key", "<u8"), ("diff", "<i8")])
R32 = np.dtype([("key", "<u8"), ("val", "<u8"), ("time", "<u8"), ("diff", "<i8")])
R40 = np.dtype([("key", "<u8"), ("val1", "<u8"), ("val2", "<u8"), ("time", "<u8"), ("diff", "<i8")])
RACC = np.dtype(
    [
        ("key", "<u8"),
        ("time", "<u8"),
        ("total", "<i8"),
        ("non_nulls", "<i8"),
        ("acc_lo", "<u8"),
        ("acc_hi", "<i8"),
        ("pos_infs", "<i8"),
        ("neg_infs", "<i8"),
        ("nans", "<i8"),
        ("_pad", "<i8"),
    ]
)
ROUT = np.dtype(
    [
        ("key", "<u8"),
        ("count", "<i8"),
        ("sum_lo", "<u8"),
        ("sum_hi", "<i8"),
        ("flags", "<u8"),
        ("time", "<u8"),
        ("diff", "<i8"),
        ("_pad", "<i8"),
    ]
)
# The lanes operator (mzgpu_reduce_lanes_new): the lane count rounds up to a class C in
# {1, 2, 4, 8}; rows hold C lanes (unused ones zero).  Class 1 has the RACC / ROUT bytes.  The pad
# words are fields, so that copies of these arrays keep every byte.
ACCUM_LANE = np.dtype(
    [("non_nulls", "<i8"), ("acc_lo", "<u8"), ("acc_hi", "<i8"), ("pos_infs", "<i8"), ("neg_infs", "<i8"), ("nans", "<i8")]
)
OUT_LANE = np.dtype([("count", "<i8"), ("sum_lo", "<u8"), ("sum_hi", "<i8")])
LANE_CLASSES = (1, 2, 4, 8)
# class -> (arrangement row bytes, output row bytes), as in include/mzgpu.h
LANE_ROW_BYTES = {1: (80, 64), 2: (128, 96), 4: (224, 144), 8: (416, 240)}


def lane_class(n_lanes):
    return next(c for c in LANE_CLASSES if c >= n_lanes)


RACC_LANES = {
    c: np.dtype(
        {
            "names": ["key", "time", "total", "lanes", "_pad"],
            "formats": ["<u8", "<u8", "<i8", (ACCUM_LANE, (c,)), "<i8"],
            "offsets": [0, 8, 16, 24, 24 + 48 * c],
            "itemsize": LANE_ROW_BYTES[c][0],
        }
    )
    for c in LANE_CLASSES
}
ROUT_LANES = {
    c: np.dtype(
        {
            "names": ["key", "lanes", "flags", "time", "diff", "_pad"],
            "formats": ["<u8", (OUT_LANE, (c,)), "<u8", "<u8", "<i8", ("<i8", (LANE_ROW_BYTES[c][1] - 32 - 24 * c) // 8)],
            "offsets": [0, 8, 8 + 24 * c, 16 + 24 * c, 24 + 24 * c, 32 + 24 * c],
            "itemsize": LANE_ROW_BYTES[c][1],
        }
    )
    for c in LANE_CLASSES
}
DTYPES = {16: R16, 32: R32, 40: R40, 80: RACC, 64: ROUT}
DTYPES.update({LANE_ROW_BYTES[c][0]: RACC_LANES[c] for c in LANE_CLASSES[1:]})
DTYPES.update({LANE_ROW_BYTES[c][1]: ROUT_LANES[c] for c in LANE_CLASSES[1:]})

MEM_HOST, MEM_DEVICE = 0, 1
FRONTIER_EMPTY = 2**64 - 1
OK, E_INVALID, E_CUDA, E_CAPACITY, E_UNSUPPORTED, E_NCCL, E_FRONTIER = 0, -1, -2, -3, -4, -5, -6
HALFJOIN_LE, HALFJOIN_LT = 0, 1
AGG_COUNT_SUM_I64, AGG_COUNT_SUM_F64, AGG_DISTINCT, AGG_THRESHOLD, AGG_MIN, AGG_MAX, AGG_TOPK = 0, 1, 2, 3, 4, 5, 6
MAX_ACCUM_LANES = 8
ACCUM_DISTINCT = 0x100  # OR'd into a lane's kind: COUNT(DISTINCT col) / SUM(DISTINCT col)
COMM_ID_BYTES = 128
P2P_HANDLE_BYTES = 64


class Field(C.Structure):
    _fields_ = [("src", C.c_uint8), ("shift", C.c_uint8), ("bits", C.c_uint8), ("dst_shift", C.c_uint8)]


class AccumLane(C.Structure):
    _fields_ = [("kind", C.c_int32), ("sign_extend", C.c_uint32), ("field", Field)]


class Filter(C.Structure):
    _fields_ = [("field", Field), ("op", C.c_uint32), ("rhs", C.c_uint64)]


class Closure(C.Structure):
    _fields_ = [
        ("n_key_fields", C.c_uint32),
        ("n_val_fields", C.c_uint32),
        ("n_filters", C.c_uint32),
        ("expr_kind", C.c_uint32),
        ("key_fields", Field * 6),
        ("val_fields", Field * 6),
        ("filters", Filter * 4),
        ("expr_a", Field),
        ("expr_b", Field),
        ("expr_c", C.c_uint64),
    ]


LINEAR_MAX_STAGES = 6


class LinearStagePlan(C.Structure):
    _fields_ = [("stream_key", Closure), ("closure", Closure)]


class LinearJoinPlan(C.Structure):
    _fields_ = [
        ("has_initial_closure", C.c_int32),
        ("has_final_closure", C.c_int32),
        ("n_stages", C.c_uint32),
        ("_pad", C.c_uint32),
        ("initial_closure", Closure),
        ("final_closure", Closure),
        ("stages", LinearStagePlan * LINEAR_MAX_STAGES),
    ]


class Desc(C.Structure):
    _fields_ = [("lower", C.c_uint64), ("upper", C.c_uint64), ("since", C.c_uint64)]


class Stats(C.Structure):
    _fields_ = [
        ("kernel_launches", C.c_uint64),
        ("device_bytes_in_use", C.c_uint64),
        ("device_bytes_peak", C.c_uint64),
        ("rows_in", C.c_uint64),
        ("rows_out", C.c_uint64),
        ("h2d_bytes", C.c_uint64),
        ("d2h_bytes", C.c_uint64),
        ("host_syncs", C.c_uint64),
    ]


vp, u64, u32, i32 = C.c_void_p, C.c_uint64, C.c_uint32, C.c_int32
PV, PU64, PU32, PI32 = C.POINTER(vp), C.POINTER(u64), C.POINTER(u32), C.POINTER(i32)

# name -> (restype, argtypes); one entry per function declared in include/mzgpu.h
SIGNATURES = {
    "mzgpu_ctx_create": (i32, [i32, i32, i32, PV]),
    "mzgpu_ctx_destroy": (None, [vp]),
    "mzgpu_last_error": (C.c_char_p, [vp]),
    "mzgpu_ctx_sync": (i32, [vp]),
    "mzgpu_ctx_stats": (i32, [vp, C.POINTER(Stats)]),
    "mzgpu_ctx_stream": (vp, [vp]),
    "mzgpu_profile_enable": (i32, [vp, i32]),
    "mzgpu_profile_report": (i32, [vp, C.c_char_p, u64]),
    "mzgpu_profile_fused_phases": (i32, [vp, PU64, u32, PU32]),
    "mzgpu_buf_new": (i32, [vp, u32, PV]),
    "mzgpu_buf_free": (None, [vp]),
    "mzgpu_buf_len": (u64, [vp]),
    "mzgpu_buf_row_bytes": (u32, [vp]),
    "mzgpu_buf_device_ptr": (vp, [vp]),
    "mzgpu_buf_upload": (i32, [vp, vp, u64, i32]),
    "mzgpu_buf_append": (i32, [vp, vp, u64, i32]),
    "mzgpu_buf_append_buf": (i32, [vp, vp]),
    "mzgpu_buf_append_buf_at_most": (i32, [vp, vp, u64]),
    "mzgpu_batcher_push_buf": (i32, [vp, vp]),
    "mzgpu_half_join_buf": (i32, [vp, vp, vp, i32, C.POINTER(Closure), i32, vp]),
    "mzgpu_half_join_many": (i32, [vp, u32, vp, vp, vp, vp, vp]),
    "mzgpu_delta_first_stage_many": (i32, [vp, u32, vp, vp, vp, vp, vp, vp, vp]),
    "mzgpu_reduce_accumulable_buf": (i32, [vp, vp, u64, vp]),
    "mzgpu_buf_download": (i32, [vp, vp, u64, i32, PU64]),
    "mzgpu_buf_clear": (i32, [vp]),
    "mzgpu_consolidate_r16": (i32, [vp, vp, u64, i32, PU64]),
    "mzgpu_consolidate_r32": (i32, [vp, vp, u64, i32, PU64]),
    "mzgpu_buf_consolidate": (i32, [vp]),
    "mzgpu_batcher_new": (i32, [vp, u32, PV]),
    "mzgpu_batcher_free": (None, [vp]),
    "mzgpu_batcher_push": (i32, [vp, vp, u64, i32]),
    "mzgpu_batcher_seal": (i32, [vp, u64, PV, PU64]),
    "mzgpu_batcher_seal_many": (i32, [u32, vp, u64, vp]),
    "mzgpu_batcher_frontier": (u64, [vp]),
    "mzgpu_batcher_len": (u64, [vp]),
    "mzgpu_batch_build": (i32, [vp, u32, vp, u64, i32, Desc, PV]),
    "mzgpu_batch_len": (u64, [vp]),
    "mzgpu_batch_keys": (u64, [vp]),
    "mzgpu_batch_desc": (Desc, [vp]),
    "mzgpu_batch_retain": (None, [vp]),
    "mzgpu_batch_release": (None, [vp]),
    "mzgpu_batch_export": (i32, [vp, vp, u64, i32, PU64]),
    "mzgpu_batch_merge": (i32, [vp, vp, u64, PV]),
    "mzgpu_spine_new": (i32, [vp, u32, u32, PV]),
    "mzgpu_spine_free": (None, [vp]),
    "mzgpu_spine_insert": (i32, [vp, vp]),
    "mzgpu_spine_exert": (i32, [vp, u64, PI32]),
    "mzgpu_spine_exert_logic": (u64, [vp, u32]),
    "mzgpu_spine_set_logical_compaction": (i32, [vp, u64]),
    "mzgpu_spine_set_physical_compaction": (i32, [vp, u64]),
    "mzgpu_spine_get_logical_compaction": (u64, [vp]),
    "mzgpu_spine_get_physical_compaction": (u64, [vp]),
    "mzgpu_spine_read_upper": (u64, [vp]),
    "mzgpu_spine_batches_through": (i32, [vp, u64, PV, u32, PU32]),
    "mzgpu_spine_layers": (i32, [vp, PU64, u32, PU32]),
    "mzgpu_spine_export": (i32, [vp, vp]),
    "mzgpu_join_new": (i32, [vp, vp, vp, C.POINTER(Closure), PV]),
    "mzgpu_join_free": (None, [vp]),
    "mzgpu_join_core_push": (i32, [vp, i32, vp, u64]),
    "mzgpu_join_core_work": (i32, [vp, u64, vp, PI32]),
    "mzgpu_half_join": (i32, [vp, vp, u64, i32, vp, i32, C.POINTER(Closure), i32, vp]),
    "mzgpu_update_stream": (i32, [vp, vp, C.POINTER(Closure), u64, vp]),
    "mzgpu_map_rows": (i32, [vp, vp, u64, i32, C.POINTER(Closure), vp]),
    "mzgpu_reduce_new": (i32, [vp, i32, PV]),
    "mzgpu_topk_new": (i32, [vp, C.c_int64, u64, i32, PV]),
    "mzgpu_reduce_free": (None, [vp]),
    "mzgpu_reduce_accumulable": (i32, [vp, vp, u64, i32, u64, vp]),
    "mzgpu_reduce_input_trace": (vp, [vp]),
    "mzgpu_reduce_lanes_row_bytes": (i32, [u32, PU32, PU32]),
    "mzgpu_reduce_lanes_new": (i32, [vp, u32, vp, u32, PV]),
    "mzgpu_reduce_lanes": (i32, [vp, vp, u64, i32, u64, vp]),
    "mzgpu_reduce_lanes_buf": (i32, [vp, vp, u64, vp]),
    "mzgpu_reduce_lanes_distinct_trace": (vp, [vp, u32]),
    "mzgpu_comm_unique_id": (i32, [C.POINTER(C.c_uint8)]),
    "mzgpu_comm_init": (i32, [vp, C.POINTER(C.c_uint8)]),
    "mzgpu_exchange": (i32, [vp, vp, vp]),
    "mzgpu_exchange_many": (i32, [vp, u32, PV, PV]),
    "mzgpu_route": (u32, [u64, u32]),
    "mzgpu_partition_many": (i32, [vp, u32, PV, u32, PV, PU64]),
    "mzgpu_rowkey_pack": (i32, [C.POINTER(C.c_uint8), u64, PU64]),
    "mzgpu_rowkeys_pack": (i32, [C.POINTER(C.c_uint8), PU64, u64, PU64, PU64]),
    "mzgpu_rowkey_unpack": (i32, [u64, C.POINTER(C.c_uint8), PU64]),
    "mzgpu_correction_new": (i32, [vp, PV]),
    "mzgpu_correction_free": (None, [vp]),
    "mzgpu_correction_insert": (i32, [vp, vp, u64, i32, i32]),
    "mzgpu_correction_insert_buf": (i32, [vp, vp, i32]),
    "mzgpu_correction_updates_before": (i32, [vp, u64, vp]),
    "mzgpu_correction_advance_since": (i32, [vp, u64]),
    "mzgpu_correction_consolidate_at_since": (i32, [vp]),
    "mzgpu_correction_len": (u64, [vp]),
    "mzgpu_comm_p2p_export": (i32, [vp, u64, u32, C.POINTER(C.c_uint8)]),
    "mzgpu_comm_p2p_import": (i32, [vp, C.POINTER(C.c_uint8)]),
    "mzgpu_comm_p2p_zone": (vp, [vp]),
    "mzgpu_comm_p2p_import_local": (i32, [vp, PV]),
    "mzgpu_exchange_p2p": (i32, [vp, u32, PV, PV, PU64]),
    "mzgpu_exchange_p2p_send": (i32, [vp, u32, PV]),
    "mzgpu_exchange_p2p_recv": (i32, [vp, u32, PV, PU64]),
    "mzgpu_batch_seek_keys": (i32, [vp, vp, u64, i32, vp]),
    "mzgpu_batch_key_page": (i32, [vp, u64, u64, i32, vp, PU64]),
    "mzgpu_batch_rows": (i32, [vp, u64, u64, vp, i32]),
    "mzgpu_batch_index_export": (i32, [vp, vp, u64, i32, PU64, PU64, PU64]),
    "mzgpu_builder_new": (i32, [vp, u32, u64, PV]),
    "mzgpu_builder_free": (None, [vp]),
    "mzgpu_builder_push": (i32, [vp, vp, u64, i32]),
    "mzgpu_builder_push_buf": (i32, [vp, vp]),
    "mzgpu_builder_done": (i32, [vp, Desc, PV]),
    "mzgpu_spine_size": (i32, [vp, vp]),
    "mzgpu_join_core_work_until": (i32, [vp, u64, u64, vp, PI32]),
    "mzgpu_ctx_host_times": (i32, [vp, PU64]),
    "mzgpu_linear_join_new": (i32, [vp, C.POINTER(LinearJoinPlan), PV, PV]),
    "mzgpu_linear_join_free": (None, [vp]),
    "mzgpu_linear_join_step": (i32, [vp, vp, PV, u64, vp]),
    "mzgpu_linear_join_stage_trace": (vp, [vp, u32]),
    "mzgpu_column_length_in_words": (u64, [i32, u64, u64, u64]),
    "mzgpu_column_at_capacity": (i32, [u64]),
    "mzgpu_column_ship_rows": (u64, [i32]),
    "mzgpu_column_decode": (i32, [vp, i32, vp, u64, i32, vp]),
    "mzgpu_column_encode": (i32, [vp, i32, u64, u64, vp, u64, i32, PU64]),
    "mzgpu_column_build": (i32, [vp, i32, vp, u64, i32, PU64, PU64, u32, PU32]),
    "mzgpu_batch_walk_column": (i32, [vp, PU64, u64, u64, i32, vp, u64, i32, PU64, PU64]),
}
COLUMN_U64X4, COLUMN_U64X2, COLUMN_ROWROW = 0, 1, 2

KEY_RUN = np.dtype([("key", "<u8"), ("first", "<u8"), ("len", "<u8")])
HASH_SLOT = np.dtype([("key", "<u8"), ("meta", "<u8")])
ARRANGEMENT_SIZE = np.dtype([("size_bytes", "<u8"), ("capacity_bytes", "<u8"), ("allocations", "<u8"), ("batches", "<u8"), ("updates", "<u8")])

for _name, (_res, _args) in SIGNATURES.items():
    _fn = getattr(lib, _name)  # AttributeError here = the .so does not export a declared symbol
    _fn.restype = _res
    _fn.argtypes = _args


class MzGpuError(RuntimeError):
    def __init__(self, status, message):
        super().__init__(f"mzgpu status {status}: {message}")
        self.status = status
