"""ctypes binding of libdspgn.so (C ABI declared in include/dspgn.h).

The product path has no CPU fallback: if the CUDA library is missing or no sm_90 GPU is present,
loading / creating handles raises.  Nothing here imports oracle/.
"""
import ctypes as C
import os

MAX_CODE = 64
MAX_LINEAR = 12
RESULT_FLOATS = 88

ENGINE_AUTO, ENGINE_SIMT, ENGINE_TC, ENGINE_TC_WIDE = 0, 1, 2, 3
SCHED_AUTO, SCHED_LAUNCHES, SCHED_PERSISTENT = 0, 1, 2
MODE_JOINT, MODE_POSE = 0, 1
GATE_OFF, GATE_KEPT, GATE_REJECTED = 0, 1, 2
MESH_OFF, MESH_DONE, MESH_FAILED, MESH_LOST = 0, 1, 2, 3
INFO_OK, INFO_NONE = 0, 1
ST_OK, ST_SDF_NAN, ST_RENDER_FEW, ST_RENDER_NAN, ST_SOLVE, ST_BAD_INPUT, ST_STOPPED = 0, 1, 2, 3, 4, 5, 6
E_ARG, E_CUDA, E_NOGPU, E_ALLOC, E_PEER, E_BUSY = -1, -2, -3, -4, -5, -6
IPC_HANDLE_BYTES = 64
FRAME_RESERVE_SMS = 4      # DSPGN_FRAME_RESERVE_SMS: SMs the solvers leave free while a frame handle is alive

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdspgn.so")


class DecoderSpec(C.Structure):
    _fields_ = [("latent_size", C.c_int32), ("num_linear", C.c_int32),
                ("in_dim", C.c_int32 * MAX_LINEAR), ("out_dim", C.c_int32 * MAX_LINEAR),
                ("latent_in_layer", C.c_int32),
                ("cat_kind", C.c_int32 * MAX_LINEAR), ("layer_norm", C.c_int32 * MAX_LINEAR),
                ("use_tanh", C.c_int32), ("reserved_", C.c_int32)]


class Config(C.Structure):
    _fields_ = [("k1", C.c_float), ("k2", C.c_float), ("k3", C.c_float), ("k4", C.c_float),
                ("b1", C.c_float), ("b2", C.c_float), ("lr", C.c_float), ("s_damp", C.c_float),
                ("num_iterations", C.c_int32), ("code_len", C.c_int32),
                ("num_depth_samples", C.c_int32), ("cut_off", C.c_float),
                ("pose_only_iterations", C.c_int32), ("sdf_only", C.c_int32), ("engine", C.c_int32),
                ("schedule", C.c_int32)]


_FP = C.POINTER(C.c_float)


class ObjectIn(C.Structure):
    _fields_ = [("t_cam_obj", _FP), ("t_rs", C.c_int32), ("t_cs", C.c_int32),
                ("pts", _FP), ("n_pts", C.c_int32), ("pts_rs", C.c_int32), ("pts_cs", C.c_int32),
                ("rays", _FP), ("n_rays", C.c_int32), ("rays_rs", C.c_int32), ("rays_cs", C.c_int32),
                ("depth", _FP), ("n_depth", C.c_int32),
                ("code", _FP), ("scale", C.c_float), ("class_id", C.c_int32),
                ("pixels", _FP), ("pix_rs", C.c_int32), ("pix_cs", C.c_int32),
                ("inv_k", _FP), ("t_cam_world", _FP)]


class ObjectOut(C.Structure):
    _fields_ = [("t_cam_obj", C.c_float * 16), ("code", C.c_float * MAX_CODE), ("loss", C.c_float),
                ("status", C.c_int32), ("n_valid", C.c_int32), ("n_band", C.c_int32),
                ("iters_done", C.c_int32), ("gate", C.c_int32), ("pad_", C.c_int32 * 2)]

    @property
    def mesh(self):
        """DSPGN_MESH_* of dspgn_keyframe_batch_meshed (the header's `mesh`, the first word of pad_); 0 elsewhere."""
        return self.pad_[0]


class GateIn(C.Structure):
    _fields_ = [("t_cam_obj_map", _FP), ("map_rs", C.c_int32), ("map_cs", C.c_int32),
                ("t_cam_obj_sim3", _FP), ("sim3_rs", C.c_int32), ("sim3_cs", C.c_int32),
                ("gate", C.c_int32)]


class MeshSpec(C.Structure):
    _fields_ = [("voxels_dim", C.c_int32), ("pair", C.POINTER(C.c_int32))]


class Counters(C.Structure):
    _fields_ = [("rows_fwd_bwd", C.c_int64), ("rows_fwd_only", C.c_int64),
                ("kernel_launches", C.c_int64), ("decoder_ms", C.c_float), ("total_ms", C.c_float),
                ("solve_ms", C.c_float), ("pad_", C.c_float)]


class IpcHandle(C.Structure):
    _fields_ = [("bytes", C.c_ubyte * IPC_HANDLE_BYTES)]


class LidarSpec(C.Structure):
    _fields_ = [("k", C.c_float * 9), ("inv_k", C.c_float * 9), ("t_cam_velo", C.c_float * 16),
                ("img_h", C.c_int32), ("img_w", C.c_int32), ("num_lidar_max", C.c_int32),
                ("min_mask_area", C.c_int32), ("downsample_ratio", C.c_int32), ("reserved_", C.c_int32)]


class LidarBox(C.Structure):
    _fields_ = [("t_obj_velo", C.c_float * 12), ("trans", C.c_float * 3), ("size", C.c_float * 3),
                ("front", C.c_int32)]


class LidarBoxOut(C.Structure):
    _fields_ = [("n_pts", C.c_int32), ("n_rays", C.c_int32), ("mask", C.c_int32), ("n_selected", C.c_int32)]


class MonoSpec(C.Structure):
    _fields_ = [("k", C.c_double * 9), ("inv_k", C.c_double * 9), ("k1", C.c_double), ("k2", C.c_double),
                ("img_h", C.c_int32), ("img_w", C.c_int32), ("downsample_ratio", C.c_int32), ("mask_erosion", C.c_int32)]


class MonoOut(C.Structure):
    _fields_ = [("mask", C.c_int32), ("n_nonsurface", C.c_int32), ("n_rays", C.c_int32), ("n_feature", C.c_int32)]


assert C.sizeof(ObjectOut) == 4 * RESULT_FLOATS

# every symbol include/dspgn.h declares: (name, restype, argtypes)
_VP = C.c_void_p
SYMBOLS = [
    ("dspgn_last_error", C.c_char_p, []),
    ("dspgn_version", C.c_int, []),
    ("dspgn_decoder_create", C.c_int, [C.POINTER(DecoderSpec), C.POINTER(_FP), C.POINTER(_FP), C.c_int, C.POINTER(_VP)]),
    ("dspgn_decoder_create_ex", C.c_int, [C.POINTER(DecoderSpec), C.POINTER(_FP), C.POINTER(_FP), C.POINTER(_FP), C.POINTER(_FP),
                                          C.c_int, C.POINTER(_VP)]),
    ("dspgn_decoder_destroy", None, [_VP]),
    ("dspgn_solver_create", C.c_int, [C.POINTER(Config), C.POINTER(_VP), C.c_int, C.c_int, C.POINTER(_VP)]),
    ("dspgn_solver_destroy", None, [_VP]),
    ("dspgn_solver_set_stream", C.c_int, [_VP, _VP]),
    ("dspgn_solver_engine", C.c_int, [_VP]),
    ("dspgn_solver_sync", C.c_int, [_VP]),
    ("dspgn_reconstruct_batch", C.c_int, [_VP, C.c_int, C.POINTER(ObjectIn), C.POINTER(ObjectOut)]),
    ("dspgn_estimate_pose_batch", C.c_int, [_VP, C.c_int, C.POINTER(ObjectIn), C.POINTER(ObjectOut)]),
    ("dspgn_upload_batch", C.c_int, [_VP, C.c_int, C.POINTER(ObjectIn)]),
    ("dspgn_run_batch", C.c_int, [_VP, C.c_int]),
    ("dspgn_results", C.c_int, [_VP, C.POINTER(ObjectOut)]),
    ("dspgn_results_device", _VP, [_VP]),
    ("dspgn_run_batch_modes", C.c_int, [_VP, C.POINTER(C.c_int32)]),
    ("dspgn_keyframe_batch", C.c_int, [_VP, C.c_int, C.POINTER(ObjectIn), C.POINTER(C.c_int32), C.POINTER(ObjectOut)]),
    ("dspgn_keyframe_batch_gated", C.c_int, [_VP, C.c_int, C.POINTER(ObjectIn), C.POINTER(C.c_int32), C.POINTER(GateIn),
                                             C.POINTER(ObjectOut)]),
    ("dspgn_keyframe_batch_meshed", C.c_int, [_VP, C.c_int, C.POINTER(ObjectIn), C.POINTER(C.c_int32), C.POINTER(GateIn),
                                              C.POINTER(MeshSpec), C.POINTER(ObjectOut), C.POINTER(C.c_int32),
                                              C.POINTER(C.c_int32)]),
    ("dspgn_keyframe_submit", C.c_int, [_VP, C.c_int, C.POINTER(ObjectIn), C.POINTER(C.c_int32), C.POINTER(GateIn),
                                        C.POINTER(MeshSpec)]),
    ("dspgn_keyframe_query", C.c_int, [_VP]),
    ("dspgn_keyframe_wait", C.c_int, [_VP, C.POINTER(ObjectOut), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    ("dspgn_pose_information", C.c_int, [_VP, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_int32)]),
    ("dspgn_debug_host_syncs", C.c_int, [_VP, C.POINTER(C.c_int64)]),
    ("dspgn_keyframe_stop", C.c_int, [_VP]),
    ("dspgn_solver_set_stop_flag", C.c_int, [_VP, _VP]),
    ("dspgn_debug_stop_at", C.c_int, [_VP, C.c_int, C.c_int]),
    ("dspgn_debug_mesh_arena", C.c_int, [_VP, C.c_int64, C.c_int64]),
    ("dspgn_debug_sm_budget", C.c_int, [_VP, C.c_int, C.POINTER(C.c_int32)]),
    ("dspgn_decode_sdf", C.c_int, [_VP, C.c_int, _FP, _FP, C.c_int, C.c_int, C.c_int, _FP]),
    ("dspgn_mesh_batch", C.c_int, [_VP, C.c_int, _FP, C.c_int, C.POINTER(C.c_int32), C.c_int, C.POINTER(C.c_int32),
                                   C.POINTER(C.c_int32)]),
    ("dspgn_mesh_results", C.c_int, [_VP, _FP, C.POINTER(C.c_int32), _FP]),
    ("dspgn_debug_mesh_grid", C.c_int, [_VP, C.c_int, C.c_int, _FP, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    ("dspgn_counters", C.c_int, [_VP, C.POINTER(Counters)]),
    ("dspgn_enable_timing", C.c_int, [_VP, C.c_int]),
    ("dspgn_gather_create", C.c_int, [_VP, C.c_int, C.c_int, C.POINTER(IpcHandle)]),
    ("dspgn_gather_open", C.c_int, [_VP, C.POINTER(IpcHandle), C.c_int, C.c_int, C.c_int]),
    ("dspgn_gather_bind", C.c_int, [_VP, C.POINTER(C.c_int32), C.c_int]),
    ("dspgn_run_batch_gather", C.c_int, [_VP, C.c_int, C.c_int]),
    ("dspgn_gather_results", C.c_int, [_VP, C.c_int, C.c_int, C.POINTER(ObjectOut)]),
    ("dspgn_gather_device", _VP, [_VP, C.c_int]),
    ("dspgn_gather_wait_ns", C.c_longlong, [_VP]),
    ("dspgn_gather_close", None, [_VP]),
    ("dspgn_debug_exp", C.c_int, [C.c_int, C.c_int, _FP, C.c_int, _FP]),
    ("dspgn_debug_system", C.c_int, [_VP, C.c_int, C.c_int, _FP, _FP, _FP, _FP, _FP, _FP]),
    ("dspgn_debug_system_iter", C.c_int, [_VP, C.c_int, C.c_int, C.c_int, _FP, _FP, _FP, _FP, _FP, _FP]),
    ("dspgn_debug_inputs", C.c_int, [_VP, C.c_int, _FP, _FP, _FP]),
    ("dspgn_debug_events", C.c_int, [_VP, C.POINTER(C.c_longlong), C.c_int]),
    ("dspgn_tc_selftest", C.c_int, [C.c_int, C.c_int, C.c_int, _FP, _FP, _FP]),
    ("dspgn_lidar_frame_create", C.c_int, [C.POINTER(LidarSpec), C.c_int, C.POINTER(_VP)]),
    ("dspgn_lidar_frame_destroy", None, [_VP]),
    ("dspgn_lidar_frame_set_stream", C.c_int, [_VP, _VP]),
    ("dspgn_lidar_frame_run", C.c_int, [_VP, _FP, C.c_int, C.POINTER(LidarBox), C.c_int, C.POINTER(C.c_uint8),
                                        C.POINTER(C.c_int32), C.c_int, C.POINTER(LidarBoxOut)]),
    ("dspgn_lidar_frame_results", C.c_int, [_VP, _FP, _FP, _FP]),
    ("dspgn_mono_frame_create", C.c_int, [C.POINTER(MonoSpec), C.c_int, C.POINTER(_VP)]),
    ("dspgn_mono_frame_destroy", None, [_VP]),
    ("dspgn_mono_frame_set_stream", C.c_int, [_VP, _VP]),
    ("dspgn_mono_frame_run", C.c_int, [_VP, C.POINTER(C.c_uint8), C.POINTER(C.c_int32), C.c_int, _FP, C.c_int,
                                       C.POINTER(MonoOut)]),
    ("dspgn_mono_frame_results", C.c_int, [_VP, _FP, C.POINTER(C.c_int32)]),
]

_lib = None


class DspgnError(RuntimeError):
    pass


def load():
    """Load libdspgn.so and bind every declared symbol.  Raises if the library is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise DspgnError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, res, args in SYMBOLS:
        fn = getattr(lib, name)          # AttributeError if the export is missing
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        msg = load().dspgn_last_error()
        err = DspgnError(f"libdspgn error {rc}: {msg.decode() if msg else ''}")
        err.code = rc
        raise err
