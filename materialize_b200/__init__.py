"""materialize_b200 — an H100-native differential-dataflow operator core.

The hot path of Materialize's compute layer (update consolidation, arrangement
build/merge, delta/linear join, accumulable reduce) as hand-written sm_90a CUDA
behind the C ABI of include/mzgpu.h.  See DESIGN.md and INTEGRATION.md.

Importing this package loads libmzgpu.so and raises if it is missing: there is
no CPU fallback.
"""
from . import _ffi  # noqa: F401  (loads the CUDA library; raises if absent)
from .api import (  # noqa: F401
    ACCUM_DISTINCT,
    AGG_COUNT_SUM_F64,
    AGG_DISTINCT,
    AGG_THRESHOLD,
    AGG_MIN,
    AGG_MAX,
    AGG_COUNT_SUM_I64,
    FRONTIER_EMPTY,
    HALFJOIN_LE,
    HALFJOIN_LT,
    R16,
    R32,
    R40,
    RACC,
    ROUT,
    Batch,
    Batcher,
    Builder,
    Closure,
    Context,
    Correction,
    DeviceRows,
    JoinCore,
    LinearJoin,
    MzGpuError,
    ReduceAccumulable,
    ReduceLanes,
    accum_lane,
    Spine,
    TopK,
    half_join,
    seal_many,
    half_join_dev,
    half_join_many,
    delta_first_stage_many,
    make_closure,
    map_rows,
    partition_many,
    p2p_export,
    p2p_import,
    p2p_connect_local,
    exchange_p2p_send,
    exchange_p2p_recv,
    route,
    update_stream,
    update_stream_dev,
    column_decode,
    column_encode,
    column_build,
    batch_walk_column,
)
from ._ffi import COLUMN_ROWROW, COLUMN_U64X2, COLUMN_U64X4  # noqa: F401
