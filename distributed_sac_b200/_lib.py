"""ctypes binding of libb200sac.so (include/b200sac.h).  No fallback: if the CUDA
library is missing or fails to load, importing the product path raises."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libb200sac.so")
MAX_HIDDEN = 8

PARAMS, ADAM_M, ADAM_V, GRADS = 0, 1, 2, 3


class Cfg(C.Structure):
    _fields_ = [
        ("state_dim", C.c_int32), ("act_dim", C.c_int32), ("num_tasks", C.c_int32),
        ("n_actor_hidden", C.c_int32), ("n_critic_hidden", C.c_int32),
        ("actor_hidden", C.c_int32 * MAX_HIDDEN), ("critic_hidden", C.c_int32 * MAX_HIDDEN),
        ("batch", C.c_int32), ("weighted_loss", C.c_int32), ("replicas", C.c_int32),
        ("precision", C.c_int32), ("care", C.c_int32),
        ("gamma", C.c_double), ("tau", C.c_double), ("reward_scale", C.c_double),
        ("lr_actor", C.c_double), ("lr_critic", C.c_double), ("lr_alpha", C.c_double),
        ("action_scale", C.c_double),
        ("beta1", C.c_double), ("beta2", C.c_double), ("adam_eps", C.c_double),
        ("log_alpha_init", C.c_double),
        ("num_encoders", C.c_int32), ("n_mix_hidden", C.c_int32), ("mix_hidden", C.c_int32 * MAX_HIDDEN),
        ("mix_out", C.c_int32), ("ctx_in", C.c_int32), ("n_ctx_hidden", C.c_int32),
        ("ctx_hidden", C.c_int32 * MAX_HIDDEN), ("ctx_out", C.c_int32), ("emb_dim", C.c_int32),
        ("tau_se", C.c_double), ("lr_ctx", C.c_double),
        ("grad_clip", C.c_int32), ("pcgrad", C.c_int32), ("critic_ensemble", C.c_int32), ("critic_ln", C.c_int32),
        ("critic_dropout", C.c_int32),
    ]


class Hparams(C.Structure):
    _fields_ = [
        ("gamma", C.c_double), ("reward_scale", C.c_double), ("tau", C.c_double),
        ("lr_critic", C.c_double), ("lr_actor", C.c_double), ("lr_alpha", C.c_double),
        ("tau_se", C.c_double), ("lr_ctx", C.c_double),
    ]


class TensorDesc(C.Structure):
    _fields_ = [("name", C.c_char * 48), ("offset", C.c_int64), ("rows", C.c_int32), ("cols", C.c_int32),
                ("trainable", C.c_int32), ("opt", C.c_int32), ("pitch", C.c_int32), ("reserved", C.c_int32)]


RESET_ACTOR, RESET_CRITIC, RESET_ALPHA, RESET_ENCODER, RESET_CONTEXT, RESET_PARTS = 0, 1, 2, 3, 4, 5


class ResetPart(C.Structure):
    _fields_ = [("layers", C.c_int32), ("reserved", C.c_int32), ("shrink", C.c_double)]


class ResetSpec(C.Structure):
    _fields_ = [("part", ResetPart * RESET_PARTS)]


_F = C.POINTER(C.c_float)
_VP = C.c_void_p

# name -> (restype, argtypes); every symbol include/b200sac.h declares
SYMBOLS = {
    "b200sac_last_error": (C.c_char_p, []),
    "b200sac_version": (C.c_char_p, []),
    "b200sac_layout": (C.c_int, [C.POINTER(Cfg), C.POINTER(TensorDesc), C.c_int32, C.POINTER(C.c_int32),
                                 C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "b200sac_create": (C.c_int, [C.POINTER(Cfg), C.c_int32, C.c_uint64, C.POINTER(_VP)]),
    "b200sac_destroy": (C.c_int, [_VP]),
    "b200sac_export": (C.c_int, [_VP, C.c_int32, C.c_int32, _VP, C.c_int64, _VP]),
    "b200sac_import": (C.c_int, [_VP, C.c_int32, C.c_int32, _VP, C.c_int64, _VP]),
    "b200sac_read_range": (C.c_int, [_VP, C.c_int32, C.c_int32, C.c_int64, C.c_int64, _VP, _VP]),
    "b200sac_arena_ptr": (C.c_int, [_VP, C.c_int32, C.POINTER(_VP), C.POINTER(C.c_int64)]),
    "b200sac_get_steps": (C.c_int, [_VP, C.c_int32, C.POINTER(C.c_int64)]),
    "b200sac_set_steps": (C.c_int, [_VP, C.c_int32, C.POINTER(C.c_int64)]),
    "b200sac_get_hparams": (C.c_int, [_VP, C.c_int32, C.POINTER(Hparams)]),
    "b200sac_set_hparams": (C.c_int, [_VP, C.c_int32, C.POINTER(Hparams), _VP]),
    "b200sac_copy_replica": (C.c_int, [_VP, C.c_int32, C.c_int32, _VP]),
    "b200sac_reset": (C.c_int, [_VP, C.c_int32, C.POINTER(ResetSpec), C.c_uint64, _VP]),
    "b200sac_redo": (C.c_int, [_VP, C.c_int32, C.c_int32, _VP, _VP, C.c_double, C.c_double, C.c_uint64, _VP]),
    "b200sac_read_redo": (C.c_int, [_VP, C.c_int32, _VP, _VP, C.c_int64, C.POINTER(C.c_int64), _VP]),
    "b200sac_set_update_intervals": (C.c_int, [_VP, C.c_int32, C.c_int32, C.c_int32, _VP]),
    "b200sac_get_update_intervals": (C.c_int, [_VP, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "b200sac_set_grad_clip": (C.c_int, [_VP, C.c_int32, C.c_double, C.c_double, C.c_double, _VP]),
    "b200sac_get_grad_clip": (C.c_int, [_VP, C.c_int32] + [C.POINTER(C.c_double)] * 3),
    "b200sac_read_grad_norms": (C.c_int, [_VP, C.c_int32, _VP, _VP]),
    "b200sac_set_critic_dropout": (C.c_int, [_VP, C.c_int32, C.c_double, _VP]),
    "b200sac_get_critic_dropout": (C.c_int, [_VP, C.c_int32, C.POINTER(C.c_double)]),
    "b200sac_set_ensemble": (C.c_int, [_VP, C.c_int32, C.c_int32, C.c_int32, _VP]),
    "b200sac_get_ensemble": (C.c_int, [_VP, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "b200sac_set_pcgrad": (C.c_int, [_VP, C.c_int32, C.c_int32, C.c_int32, _VP]),
    "b200sac_get_pcgrad": (C.c_int, [_VP, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "b200sac_read_pcgrad": (C.c_int, [_VP, C.c_int32, _VP, _VP, _VP, _VP, C.POINTER(C.c_int32), _VP]),
    "b200sac_export_task_grad": (C.c_int, [_VP, C.c_int32, C.c_int32, _VP, C.c_int64, _VP]),
    "b200sac_set_cagrad": (C.c_int, [_VP, C.c_int32, C.c_double, C.c_double, _VP]),
    "b200sac_get_cagrad": (C.c_int, [_VP, C.c_int32, C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "b200sac_read_cagrad": (C.c_int, [_VP, C.c_int32] + [_VP] * 6 + [_VP]),
    "b200sac_cagrad_solve_test": (C.c_int, [C.c_int32, _VP, C.c_double] + [_VP] * 7),
    "b200sac_step": (C.c_int, [_VP] + [_VP] * 7 + [_VP]),
    "b200sac_step_host": (C.c_int, [_VP] + [_VP] * 7 + [_VP, _VP]),
    "b200sac_step_sampled": (C.c_int, [_VP, _VP, C.c_int32, _VP]),
    "b200sac_update": (C.c_int, [_VP, _VP, _VP, _VP]),
    "b200sac_prepare": (C.c_int, [_VP, _VP, _VP]),
    "b200sac_read_losses": (C.c_int, [_VP, C.c_int32, _VP, _VP]),
    "b200sac_soft_update": (C.c_int, [_VP, C.c_double, _VP]),
    "b200sac_soft_update_critic": (C.c_int, [_VP, C.c_int32, C.c_double, _VP]),
    "b200sac_act": (C.c_int, [_VP, C.c_int32, C.c_int32, _VP, _VP, C.c_int32, _VP, _VP]),
    "b200sac_critic_values": (C.c_int, [_VP, C.c_int32, C.c_int64, _VP, _VP, C.c_int32, _VP, _VP]),
    "b200sac_critic_values_chunk": (C.c_int, [_VP, C.POINTER(C.c_int64)]),
    "b200sac_blob_template": (C.c_int, [_VP, C.c_int32, _VP, C.c_int64, C.c_int64, _VP, _VP]),
    "b200sac_blob_begin": (C.c_int, [_VP, _VP]),
    "b200sac_blob_wait": (C.c_int, [_VP, C.POINTER(_VP), C.POINTER(C.c_int64)]),
    "b200sac_debug_read": (C.c_int, [_VP, C.c_char_p, C.c_int32, _VP, C.c_int64, C.POINTER(C.c_int64), _VP]),
    "b200sac_profile_step": (C.c_int, [_VP, _VP, C.c_int32, _VP, C.c_int32, C.POINTER(C.c_int32), C.c_char_p, C.c_int32, _VP]),
    "b200sac_graph_timeline": (C.c_int, [_VP, _VP, C.c_int32, _VP, C.c_int32, C.POINTER(C.c_int32), _VP]),
    "b200sac_tc_gemm_test": (C.c_int, [C.c_int32] * 4 + [_VP, C.c_int32, _VP, C.c_int32, _VP, _VP, C.c_int32, _VP, C.c_int32, _VP, C.c_int32, _VP]),
    "b200sac_gemm_test": (C.c_int, [C.c_int32] * 5 + [_VP, C.c_int32, _VP, C.c_int32, _VP, _VP, C.c_int32, _VP, C.c_int32, _VP, C.c_int32, _VP]),
    "b200sac_launches_per_step": (C.c_int, [_VP, C.POINTER(C.c_int32)]),
    "b200sac_replay_create": (C.c_int, [_VP, C.c_int64, C.c_int32, C.c_uint64, C.POINTER(_VP)]),
    "b200sac_replay_destroy": (C.c_int, [_VP]),
    "b200sac_replay_push": (C.c_int, [_VP, C.c_int32, C.c_int64] + [_VP] * 5),
    "b200sac_replay_fill_synthetic": (C.c_int, [_VP, C.c_int64, C.c_uint64, _VP]),
    "b200sac_replay_size": (C.c_int, [_VP, C.c_int32, C.POINTER(C.c_int64)]),
    "b200sac_replay_sample": (C.c_int, [_VP, C.c_int32] + [_VP] * 5 + [_VP]),
    "b200sac_replay_create_prioritized": (C.c_int, [_VP, C.c_int64, C.c_uint64, C.c_double, C.c_double, C.c_double, C.POINTER(_VP)]),
    "b200sac_replay_set_beta": (C.c_int, [_VP, C.c_int32, C.c_double, _VP]),
    "b200sac_replay_set_priorities": (C.c_int, [_VP, C.c_int32, C.c_int64, _VP, _VP]),
    "b200sac_replay_get_priorities": (C.c_int, [_VP, C.c_int32, C.c_int64, _VP, _VP]),
    "b200sac_replay_get_tree": (C.c_int, [_VP, C.c_int32, C.c_int32, C.c_int64, _VP]),
    "b200sac_replay_sample_prioritized": (C.c_int, [_VP, C.c_int32] + [_VP] * 5 + [_VP, _VP]),
    "b200sac_replay_enable_trajectories": (C.c_int, [_VP]),
    "b200sac_replay_push_traj": (C.c_int, [_VP, C.c_int32, C.c_int64] + [_VP] * 5 + [_VP, _VP]),
    "b200sac_replay_close_streams": (C.c_int, [_VP, C.c_int32, C.c_int64, _VP]),
    "b200sac_replay_set_nstep": (C.c_int, [_VP, C.c_int32, C.c_int32, _VP]),
    "b200sac_replay_get_nstep": (C.c_int, [_VP, C.c_int32, C.POINTER(C.c_int32)]),
    "b200sac_replay_get_links": (C.c_int, [_VP, C.c_int32, C.c_int32, C.c_int64, _VP]),
    "b200sac_replay_fold": (C.c_int, [_VP, C.c_int32, C.c_int64] + [_VP] * 8),
    "b200sac_replay_refresh_priorities": (C.c_int, [_VP, C.c_int32, C.c_int64, _VP, C.c_uint64, C.c_int32, _VP]),
    "b200sac_replay_attach_prior": (C.c_int, [_VP, _VP]),
    "b200sac_replay_set_prior_rows": (C.c_int, [_VP, C.c_int32, C.c_int32, _VP]),
    "b200sac_replay_get_prior_rows": (C.c_int, [_VP, C.c_int32, C.POINTER(C.c_int32)]),
}

_lib = None


def load():
    """dlopen the library and type every entry point.  Raises if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a).  There is no CPU or PyTorch fallback for the learner hot path.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)      # AttributeError if the header and the .so disagree
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        raise RuntimeError(f"b200sac error {rc}: {load().b200sac_last_error().decode()}")
