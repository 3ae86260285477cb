"""ctypes binding of include/b2rl.h.  Fails loudly: there is no CPU fallback."""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libb2rl.so")
MAX_FIELDS = 8

c_i64, c_i32, c_u64, c_u32 = C.c_int64, C.c_int32, C.c_uint64, C.c_uint32
c_f32, c_f64, c_vp = C.c_float, C.c_double, C.c_void_p


class ReplayDesc(C.Structure):
    _fields_ = [("capacity", c_i64), ("n_fields", c_i32), ("device", c_i32),
                ("field_bytes", c_i64 * MAX_FIELDS)]


IPC_HANDLE_BYTES = 64


class ServeLayout(C.Structure):
    """b2rl_serve_layout: byte offsets of the device serve ring (include/b2rl.h)."""
    _fields_ = [("batch", c_i64), ("slots", c_i64), ("n_fields", c_i64), ("field_bytes", c_i64 * MAX_FIELDS),
                ("field_off", c_i64 * MAX_FIELDS), ("idx_off", c_i64), ("w_off", c_i64), ("slot_bytes", c_i64),
                ("upd_idx_off", c_i64), ("upd_prio_off", c_i64), ("upd_slot_bytes", c_i64), ("upd_base", c_i64),
                ("total_bytes", c_i64)]


class Frames(C.Structure):
    """b2rl_frames: where conv_1 reads frame row r (include/b2rl.h); exactly one of base, table and pool + planes.
    plane_stride 0 means 8 (the Ape-X plane table).  offsets (with pool_units, pool_frames) makes the pool a coded
    one, whose frames conv_1 decodes on chip."""
    _fields_ = [("base", c_vp), ("table", c_vp), ("pool", c_vp), ("planes", c_vp), ("row_stride", c_i64),
                ("rows", c_i64), ("plane_base", c_i32), ("plane_stride", c_i32), ("offsets", c_vp),
                ("pool_units", c_i64), ("pool_frames", c_i64)]


# name -> (restype, argtypes); must list every symbol include/b2rl.h declares.
SIGNATURES = {
    "b2rl_last_error": (C.c_char_p, []),
    "b2rl_version": (C.c_int, []),
    "b2rl_replay_create": (C.c_int, [C.POINTER(ReplayDesc), C.POINTER(c_vp)]),
    "b2rl_replay_destroy": (C.c_int, [c_vp]),
    "b2rl_replay_create_placed": (C.c_int, [C.POINTER(ReplayDesc), C.POINTER(c_i32), C.POINTER(c_vp)]),
    "b2rl_replay_field_placement": (C.c_int, [c_vp, c_i32, C.POINTER(c_i32)]),
    "b2rl_replay_size": (C.c_int, [c_vp, C.POINTER(c_i64), C.POINTER(c_i64), C.POINTER(c_i64)]),
    "b2rl_replay_field_ptr": (C.c_int, [c_vp, c_i32, C.POINTER(c_vp)]),
    "b2rl_replay_push": (C.c_int, [c_vp, C.POINTER(c_vp), c_vp, c_i64, c_vp]),
    "b2rl_replay_reserve": (C.c_int, [c_vp, c_i64, C.POINTER(c_i64), c_vp]),
    "b2rl_replay_copy_payload": (C.c_int, [c_vp, C.POINTER(c_vp), c_i64, c_i64, c_vp]),
    "b2rl_replay_commit": (C.c_int, [c_vp, c_vp, c_i64, c_vp]),
    "b2rl_replay_ingest_pipelined": (C.c_int, [c_vp, C.POINTER(c_vp), c_vp, c_i64, c_vp]),
    "b2rl_replay_evict": (C.c_int, [c_vp, c_i64, c_vp]),
    "b2rl_replay_fill_hash": (C.c_int, [c_vp, c_i64, c_u32, c_vp]),
    "b2rl_tree_build": (C.c_int, [c_vp, c_vp, c_i64, c_vp]),
    "b2rl_tree_sample": (C.c_int, [c_vp, c_vp, c_u64, c_u64, c_i64, c_f32, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b2rl_replay_seed": (C.c_int, [c_vp, c_u64, c_u64, c_vp]),
    "b2rl_tree_sample_stream": (C.c_int, [c_vp, c_i64, c_f32, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b2rl_tree_sample_fetch": (C.c_int, [c_vp, c_i64, c_f32, c_vp, c_vp, c_vp, c_vp, C.POINTER(c_vp), c_vp]),
    "b2rl_philox_uniforms": (C.c_int, [c_u64, c_u64, c_i64, c_vp, c_vp]),
    "b2rl_tree_update": (C.c_int, [c_vp, c_vp, c_vp, c_i64, c_vp]),
    "b2rl_tree_stats": (C.c_int, [c_vp, c_f32, c_vp, c_vp, c_vp]),
    "b2rl_tree_leaves": (C.c_int, [c_vp, c_i64, c_i64, c_vp, c_vp]),
    "b2rl_tree_level": (C.c_int, [c_vp, c_i32, C.POINTER(c_i64), C.POINTER(c_i32), C.POINTER(c_i32), c_vp, c_vp,
                                  c_vp]),
    "b2rl_replay_gather": (C.c_int, [c_vp, c_vp, c_i64, C.POINTER(c_vp), c_vp]),
    "b2rl_uniform_fetch": (C.c_int, [c_vp, c_i64, c_i32, c_vp, C.POINTER(c_vp), c_vp, c_vp]),
    "b2rl_apex_target": (C.c_int, [c_vp] * 7 + [c_i32, c_i32, c_f32, c_f32] + [c_vp] * 6),
    "b2rl_r2d2_target": (C.c_int, [c_vp] * 6 + [c_i32, c_i32, c_i32, c_i32, c_f64, c_f32, c_i32]
                         + [c_vp] * 6),
    "b2rl_vtrace": (C.c_int, [c_vp] * 5 + [c_i32, c_i32, c_f32, c_f32, c_f32, c_f32] + [c_vp] * 3),
    "b2rl_conv1_pack": (C.c_int, [c_vp, c_i32, c_i32, c_i32, c_vp, c_vp, c_vp]),
    "b2rl_conv1_pack_jobs": (C.c_int, [C.POINTER(c_vp), C.POINTER(c_i32), C.POINTER(c_i32), C.POINTER(c_vp),
                                       C.POINTER(c_vp), c_i32, c_i32, c_vp]),
    "b2rl_conv1_fused": (C.c_int, [C.POINTER(Frames), c_vp, c_i64, c_vp, c_vp, c_i32, c_i32, c_vp, c_i32, c_vp]),
    "b2rl_conv1_wgrad_workspace_floats": (c_i64, [c_i32]),
    "b2rl_conv1_wgrad": (C.c_int, [C.POINTER(Frames), c_vp, c_i64, c_vp, c_vp, c_i32, c_vp, c_vp, c_i32, c_vp]),
    "b2rl_stem_pack": (C.c_int, [c_vp, c_vp, c_vp, c_vp]),
    "b2rl_stem_fused": (C.c_int, [C.POINTER(Frames), c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b2rl_stem_fused_pair": (C.c_int, [C.POINTER(Frames), c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b2rl_stem_wgrad_workspace_doubles": (c_i64, []),
    "b2rl_stem_wgrad": (C.c_int, [C.POINTER(Frames), c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_i32, c_vp]),
    "b2rl_dedup_attach": (C.c_int, [c_vp, c_i32, c_i64, c_i64, c_u64]),
    "b2rl_dedup_push": (C.c_int, [c_vp, c_vp, c_vp, C.POINTER(c_vp), c_vp, c_i64, c_vp]),
    "b2rl_dedup_attach_strips": (C.c_int, [c_vp, c_i32, c_i32, c_i64, c_i64, c_u64]),
    "b2rl_dedup_push_strips": (C.c_int, [c_vp, c_vp, C.POINTER(c_vp), c_vp, c_i64, c_vp]),
    "b2rl_dedup_info": (C.c_int, [c_vp, C.POINTER(c_vp), C.POINTER(c_i64), C.POINTER(c_i64)]),
    "b2rl_dedup_attach_strips_placed": (C.c_int, [c_vp, c_i32, c_i32, c_i64, c_i64, c_u64, c_i32]),
    "b2rl_dedup_attach_rollouts": (C.c_int, [c_vp, c_i32, c_i32, c_i64, c_i64, c_u64]),
    "b2rl_dedup_pool_placement": (C.c_int, [c_vp, C.POINTER(c_i32), C.POINTER(c_vp)]),
    "b2rl_dedup_attach_strips_coded": (C.c_int, [c_vp, c_i32, c_i32, c_i64, c_i64, c_u64, c_i64]),
    "b2rl_dedup_attach_coded": (C.c_int, [c_vp, c_i32, c_i64, c_i64, c_u64, c_i64]),
    "b2rl_dedup_coded_offsets": (C.c_int, [c_vp, C.POINTER(c_vp)]),
    "b2rl_dedup_attach_rollouts_coded": (C.c_int, [c_vp, c_i32, c_i32, c_i64, c_i64, c_u64, c_i64]),
    "b2rl_dedup_stage_rollouts": (C.c_int, [c_vp, c_vp, c_i64, c_vp, c_vp, c_vp]),
    "b2rl_dedup_codec_stats": (C.c_int, [c_vp, C.POINTER(c_i64), C.POINTER(c_i64), C.POINTER(c_i64)]),
    "b2rl_frame_encode": (C.c_int, [c_vp, c_i64, c_vp, c_vp, c_vp]),
    "b2rl_frame_decode": (C.c_int, [c_vp, c_i64, c_vp, c_vp]),
    "b2rl_replay_gather_planes": (C.c_int, [c_vp, c_vp, c_i64, C.POINTER(c_vp), C.POINTER(c_vp), c_vp]),
    "b2rl_rmsprop_step": (C.c_int, [C.POINTER(c_vp), C.POINTER(c_vp), C.POINTER(c_vp), C.POINTER(c_vp),
                                    C.POINTER(c_i64), c_i32, c_f64, c_f64, c_f64, c_i32, C.POINTER(c_i64), c_vp, c_vp,
                                    c_vp]),
    "b2rl_rmsprop_norm_finish": (C.c_int, [c_vp, c_i32, c_vp, c_vp]),
    "b2rl_peer_allreduce_max_ctas": (c_i32, []),
    "b2rl_peer_allreduce_mean": (C.c_int, [c_vp, c_vp, c_i32, c_i32, c_i64, c_vp, c_i64, c_vp, c_vp, c_vp]),
    "b2rl_peer_allreduce_mean_big": (C.c_int, [c_vp, c_vp, c_vp, c_i32, c_i32, c_i64, c_i64, c_i32, c_vp, c_vp, c_vp]),
    "b2rl_gemm_packed_floats": (c_i64, [c_i64, c_i64, c_i32]),
    "b2rl_gemm_split_pack": (C.c_int, [c_vp, c_i64, c_i64, c_i64, c_i32, c_i32, c_vp, c_vp]),
    "b2rl_gemm_split_pack_into": (C.c_int, [c_vp, c_i64, c_i64, c_i64, c_i32, c_i32, c_vp, c_i64, c_i64, c_i64, c_i64, c_vp]),
    "b2rl_gemm_pack_act_nhwc": (C.c_int, [c_vp, c_i64, c_i64, c_i64, c_i32, c_i32, c_vp, c_vp]),
    "b2rl_unflatten_relu_mask": (C.c_int, [c_vp, c_i64, c_i32, c_i64, c_vp, c_i64, c_i64, c_i64, c_vp, c_vp]),
    "b2rl_gemm_workspace_floats": (c_i64, [c_i64, c_i64, c_i64, c_i64]),
    "b2rl_gemm_tf32x3": (C.c_int, [c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_i64, c_vp, c_vp]),
    "b2rl_gemm_tf32x3_partials": (C.c_int, [c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_i64, c_vp]),
    "b2rl_dueling_forward": (C.c_int, [c_vp, c_i32, c_i64, c_i64, c_i64, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp]),
    "b2rl_dueling_backward": (C.c_int, [c_vp, c_vp, c_i64, c_i64, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b2rl_dueling_backward_w": (C.c_int, [c_vp, c_vp, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp]),
    "b2rl_launch_count": (c_i64, []),
    "b2rl_wire_decode": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_vp, c_i32, c_vp, c_i32, c_vp, c_i32, c_vp,
                                   C.POINTER(c_vp), C.POINTER(c_i64), c_i32, c_vp, c_i64, c_vp]),
    "b2rl_wire_gather": (C.c_int, [C.POINTER(C.c_char_p), C.POINTER(c_i64), c_i64, c_vp, c_i64, c_vp]),
    "b2rl_serve_layout_init": (C.c_int, [c_i64, c_i32, c_i32, C.POINTER(c_i64), C.POINTER(ServeLayout)]),
    "b2rl_serve_ring_create": (C.c_int, [c_vp, c_i64, c_i32, C.POINTER(c_vp)]),
    "b2rl_serve_ring_layout": (C.c_int, [c_vp, C.POINTER(ServeLayout)]),
    "b2rl_serve_ring_export": (C.c_int, [c_vp, c_vp]),
    "b2rl_serve_ring_open": (C.c_int, [c_vp, C.POINTER(ServeLayout), c_i32, C.POINTER(c_vp)]),
    "b2rl_serve_ring_close": (C.c_int, [c_vp]),
    "b2rl_serve_ring_destroy": (C.c_int, [c_vp]),
    "b2rl_serve_slot_ptrs": (C.c_int, [c_vp, c_i32, C.POINTER(c_vp), C.POINTER(c_vp)]),
    "b2rl_serve_fill": (C.c_int, [c_vp, c_vp, c_i32, c_u64, c_f32, c_vp, c_vp]),
    "b2rl_serve_fill_uniform": (C.c_int, [c_vp, c_vp, c_i32, c_u64, c_i32, c_vp]),
    "b2rl_serve_take": (C.c_int, [c_vp, c_i32, c_vp, c_vp]),
    "b2rl_serve_bind": (C.c_int, [c_vp, C.POINTER(ServeLayout), c_i64, c_vp, c_vp, c_vp, C.POINTER(c_vp),
                                  C.POINTER(c_vp), c_vp]),
    "b2rl_serve_put_update": (C.c_int, [c_vp, c_i32, c_u64, c_vp, c_vp, c_i64, c_vp]),
}

_lib = None


class B2RLError(RuntimeError):
    pass


def load() -> C.CDLL:
    """Load libb2rl.so.  No fallback: a missing library is a hard error."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise B2RLError(
            f"{LIB_PATH} is missing — build it with `python -m distributed_rl_b200.build` "
            "(nvcc, sm_90a).  There is deliberately no CPU fallback for the product path.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            raise B2RLError(f"libb2rl.so does not export {name}")
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc != 0:
        raise B2RLError(f"libb2rl error {rc}: {load().b2rl_last_error().decode()}")
