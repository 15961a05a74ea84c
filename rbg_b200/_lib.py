"""ctypes binding of include/rbgtopo.h.  The shared library is built in-tree by
``__graft_entry__.build()`` (nvcc, sm_90a).  A missing library is a hard error:
this package has no CPU or PyTorch fallback."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# RBGTOPO_LIB selects another build of the library (profiling builds such as -DRBGTOPO_PHASE_CLOCKS)
LIB_PATH = os.environ.get("RBGTOPO_LIB") or os.path.join(_HERE, "csrc", "librbgtopo.so")

i32p = C.POINTER(C.c_int32)
u64p = C.POINTER(C.c_uint64)
f32p = C.POINTER(C.c_float)


class Config(C.Structure):
    _fields_ = [("device", C.c_int32), ("rank", C.c_int32), ("world", C.c_int32),
                ("slots", C.c_int32), ("emit_matrix", C.c_int32), ("chunk_nodes", C.c_int32),
                ("flags", C.c_int32), ("reserved", C.c_int32)]


CFG_LEVEL_PLACEMENT = 1  # RBGTOPO_CFG_LEVEL_PLACEMENT: place groups / steps at exclusive levels >= 1
CFG_COMMIT_LEVELS = 2    # RBGTOPO_CFG_COMMIT_LEVELS: committed batches at levels >= 1 too (with the flag above)
CFG_LW_COMMIT_LEVELS = 4  # RBGTOPO_CFG_LW_COMMIT_LEVELS: committed leader-worker batches at levels >= 1 (with both above)
CFG_LW_SHARDS = 8  # RBGTOPO_CFG_LW_SHARDS: place_groups_lw[_committed] at world > 1, the world = 1 results on every rank


class Timing(C.Structure):
    _fields_ = [("h2d_ms", C.c_float), ("base_ms", C.c_float), ("score_ms", C.c_float),
                ("select_ms", C.c_float), ("d2h_ms", C.c_float), ("total_ms", C.c_float),
                ("launches", C.c_int32), ("h2d_words", C.c_int32), ("scores", C.c_int64),
                ("algo_bytes", C.c_int64)]


# name -> (restype, argtypes): exactly the symbols include/rbgtopo.h declares
SIGNATURES = {
    "rbgtopo_create": (C.c_int32, [C.POINTER(Config), C.POINTER(C.c_void_p)]),
    "rbgtopo_destroy": (C.c_int32, [C.c_void_p]),
    "rbgtopo_abi_version": (C.c_int32, []),
    "rbgtopo_last_error": (C.c_int32, [C.c_void_p, C.c_char_p, C.c_int32]),
    "rbgtopo_set_topology": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int64, i32p, i32p, i32p, i32p,
                                         i32p, C.c_int32, i32p, C.c_uint64]),
    "rbgtopo_update_nodes": (C.c_int32, [C.c_void_p, i32p, i32p, C.c_uint64]),
    "rbgtopo_update_nodes_delta": (C.c_int32, [C.c_void_p, C.c_int32, i32p, i32p, C.c_uint64]),
    "rbgtopo_set_exclusive_levels": (C.c_int32, [C.c_void_p, C.c_int32, i32p, i32p, C.c_int32, i32p, C.c_uint64]),
    "rbgtopo_set_node_classes": (C.c_int32, [C.c_void_p, C.c_int32, i32p, C.c_uint64]),
    "rbgtopo_score_assign": (C.c_int32, [C.c_void_p, i32p, C.c_int64, i32p, i32p, i32p]),
    "rbgtopo_place_groups": (C.c_int32, [C.c_void_p, i32p, C.c_int64, i32p, i32p, i32p]),
    "rbgtopo_place_groups_committed": (C.c_int32, [C.c_void_p, i32p, C.c_int64, i32p, i32p, i32p, i32p]),
    "rbgtopo_place_groups_ranked": (C.c_int32, [C.c_void_p, i32p, C.c_int64, C.c_int32, i32p, i32p, i32p, f32p, i32p,
                                                f32p]),
    "rbgtopo_place_groups_committed_ranked": (C.c_int32, [C.c_void_p, i32p, C.c_int64, C.c_int32, i32p, i32p, i32p,
                                                          i32p, f32p, i32p, f32p]),
    "rbgtopo_place_groups_lw": (C.c_int32, [C.c_void_p, i32p, C.c_int64, i32p, C.c_int64, i32p, i32p, i32p]),
    "rbgtopo_place_groups_lw_committed": (C.c_int32, [C.c_void_p, i32p, C.c_int64, i32p, C.c_int64, i32p, i32p, i32p,
                                                      i32p]),
    "rbgtopo_place_groups_lw_committed_ranked": (C.c_int32, [C.c_void_p, i32p, C.c_int64, i32p, C.c_int64, C.c_int32,
                                                             i32p, i32p, i32p, i32p, f32p, i32p, f32p]),
    "rbgtopo_place_groups_lw_ranked": (C.c_int32, [C.c_void_p, i32p, C.c_int64, i32p, C.c_int64, C.c_int32, i32p, i32p,
                                                   i32p, f32p, i32p, f32p]),
    "rbgtopo_place_groups_eligible": (C.c_int32, [C.c_void_p, i32p, C.c_int64, i32p, C.c_int64, u64p, C.c_int64, i32p,
                                                  i32p, i32p]),
    "rbgtopo_place_groups_eligible_ranked": (C.c_int32, [C.c_void_p, i32p, C.c_int64, i32p, C.c_int64, u64p, C.c_int64,
                                                         C.c_int32, i32p, i32p, i32p, f32p, i32p, f32p]),
    "rbgtopo_place_groups_eligible_committed": (C.c_int32, [C.c_void_p, i32p, C.c_int64, i32p, C.c_int64, u64p,
                                                            C.c_int64, i32p, i32p, i32p, i32p]),
    "rbgtopo_place_groups_eligible_committed_ranked": (C.c_int32, [C.c_void_p, i32p, C.c_int64, i32p, C.c_int64, u64p,
                                                                   C.c_int64, C.c_int32, i32p, i32p, i32p, i32p, f32p,
                                                                   i32p, f32p]),
    "rbgtopo_shard_place_groups_ranked": (C.c_int32, [C.c_void_p, i32p, C.c_int64, C.c_int32, i32p, i32p, i32p, i32p,
                                                      C.POINTER(C.c_void_p), C.POINTER(C.c_int64)]),
    "rbgtopo_shard_place_groups_committed_ranked": (C.c_int32, [C.c_void_p, i32p, C.c_int64, C.c_int32, i32p, i32p,
                                                                i32p, i32p, i32p, C.POINTER(C.c_void_p),
                                                                C.POINTER(C.c_int64)]),
    "rbgtopo_shard_place_groups_lw_ranked": (C.c_int32, [C.c_void_p, i32p, C.c_int64, i32p, C.c_int64, C.c_int32, i32p,
                                                         i32p, i32p, i32p, C.POINTER(C.c_void_p),
                                                         C.POINTER(C.c_int64)]),
    "rbgtopo_shard_place_groups_lw_committed_ranked": (C.c_int32, [C.c_void_p, i32p, C.c_int64, i32p, C.c_int64,
                                                                   C.c_int32, i32p, i32p, i32p, i32p, i32p,
                                                                   C.POINTER(C.c_void_p), C.POINTER(C.c_int64)]),
    "rbgtopo_shard_alternates_merge": (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p, f32p, i32p, f32p]),
    "rbgtopo_stage_groups": (C.c_int32, [C.c_void_p, i32p, C.c_int64, i32p]),
    "rbgtopo_stage": (C.c_int32, [C.c_void_p, i32p, C.c_int64, i32p]),
    "rbgtopo_run_staged": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int32]),
    "rbgtopo_fetch": (C.c_int32, [C.c_void_p, C.c_int32, i32p, i32p, i32p]),
    "rbgtopo_release": (C.c_int32, [C.c_void_p, C.c_int32]),
    "rbgtopo_read_scores": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int32, f32p, C.c_int32]),
    "rbgtopo_read_topk": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int32, u64p, C.c_int32]),
    "rbgtopo_read_snapshot": (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.POINTER(C.c_int64)]),
    "rbgtopo_shard_waves": (C.c_int32, [C.c_void_p, C.c_int32, i32p]),
    "rbgtopo_shard_wave_score": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_void_p), C.POINTER(C.c_int64)]),
    "rbgtopo_shard_wave_merge": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, i32p, C.POINTER(C.c_void_p),
                                             C.POINTER(C.c_int64)]),
    "rbgtopo_shard_wave_assign": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]),
    "rbgtopo_shard_score": (C.c_int32, [C.c_void_p, C.c_int32, C.POINTER(C.c_void_p), C.POINTER(C.c_int64)]),
    "rbgtopo_shard_merge": (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p, i32p, C.POINTER(C.c_void_p),
                                        C.POINTER(C.c_int64)]),
    "rbgtopo_shard_assign": (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p]),
    "rbgtopo_p2p_export": (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.POINTER(C.c_void_p)]),
    "rbgtopo_p2p_import": (C.c_int32, [C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]),
    "rbgtopo_run_staged_p2p": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int32]),
    "rbgtopo_p2p_stats": (C.c_int32, [C.c_void_p, C.POINTER(C.c_int64), i32p]),
    "rbgtopo_slab": (C.c_int32, [C.c_void_p, i32p, i32p]),
    "rbgtopo_set_stream": (C.c_int32, [C.c_void_p, C.c_void_p]),
    "rbgtopo_set_kernel_timing": (C.c_int32, [C.c_void_p, C.c_int32]),
    "rbgtopo_run_staged_chain": (C.c_int32, [C.c_void_p, i32p, C.c_int32, C.c_int32]),
    "rbgtopo_place_describe": (C.c_int32, [i32p, C.c_int64, C.c_int32, C.c_int32, i32p, C.c_int64, i32p, C.c_int64, i32p]),
    "rbgtopo_last_timing": (C.c_int32, [C.c_void_p, C.POINTER(Timing)]),
    "rbgtopo_last_pass_times": (C.c_int32, [C.c_void_p, f32p, f32p, C.c_int32, i32p]),
    "rbgtopo_stats": (C.c_int32, [C.c_void_p, u64p, C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                                  C.POINTER(C.c_int64)]),
    "rbgtopo_plan_occupancy": (C.c_int32, [C.c_void_p, i32p, i32p, i32p]),
    "rbgtopo_group_size": (C.c_int32, [C.c_int32, i32p, i32p]),
    "rbgtopo_dependency_levels": (C.c_int32, [C.c_int32, C.POINTER(C.c_char_p), i32p, i32p, i32p, i32p]),
    "rbgtopo_parse_percentage": (C.c_int32, [C.c_char_p, C.POINTER(C.c_double)]),
    "rbgtopo_calculate_target_replicas": (C.c_int32, [C.c_double, C.c_int32, C.c_int32, i32p, i32p, i32p,
                                                      i32p, i32p]),
    "rbgtopo_scaled_value": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "rbgtopo_updated_replicas_bound": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, i32p, i32p]),
    "rbgtopo_next_rolling_target": (C.c_int32, [C.c_int32, C.c_int32, i32p, i32p, i32p, i32p]),
    "rbgtopo_partition_replicas": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, i32p]),
    "rbgtopo_intstr_non_zero": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, i32p]),
    "rbgtopo_merge_rolling_update": (C.c_int32, [i32p, i32p, i32p]),
    "rbgtopo_workload_name": (C.c_int32, [C.c_char_p, C.c_char_p, C.c_char_p, C.c_int32]),
    "rbgtopo_group_unique_key": (C.c_int32, [C.c_char_p, C.c_char_p, C.c_char_p, C.c_int32]),
    "rbgtopo_inherits_annotation": (C.c_int32, [C.c_char_p, C.c_int32, C.POINTER(C.c_char_p)]),
    "rbgtopo_plan_describe": (C.c_int32, [i32p, C.c_int64, C.c_int32, C.c_int32, i32p, C.c_int64, i32p, C.c_int64,
                                          i32p, i32p, C.POINTER(C.c_int64)]),
}

_lib = None


def load() -> C.CDLL:
    """Load librbgtopo.so and bind every declared symbol (missing symbol = error)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc -gencode arch=compute_90a,code=sm_90a). rbg_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib
