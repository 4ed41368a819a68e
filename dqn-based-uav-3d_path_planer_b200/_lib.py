"""ctypes binding of libuavrl_b200.so (include/uavrl.h).

There is no CPU fallback: if the CUDA library is missing or cannot be built, importing callers get
an ImportError here, and without a CUDA device `uavrl_env_create` / `uavrl_learner_create` fail with
UAVRL_ERR_CUDA (surfaced as UavrlError).
"""
import ctypes as C
import os

from . import _build

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = _build.LIB
OBS_DIM = 100
MAX_HIDDEN = 4

ACT_CONT_F32, ACT_CONT_F64, ACT_DISCRETE27, ACT_CONT_F32X2 = 0, 1, 2, 3
ALGO_DQN, ALGO_DDQN, ALGO_DUELING = 0, 1, 2
INFO_NAMES = ("normal", "success", "lose")
SAC_COMM_HANDLE_BYTES = 128         # UAVRL_SAC_COMM_HANDLE_BYTES: CUDA IPC handle + PCI bus id


class UavrlError(RuntimeError):
    pass


class EnvConfig(C.Structure):
    _fields_ = [("n_envs", C.c_int32), ("max_subgoals", C.c_int32),
                ("len", C.c_double), ("width", C.c_double), ("h", C.c_double),
                ("max_v", C.c_double), ("min_v", C.c_double), ("steering_angle", C.c_double),
                ("max_step", C.c_int32), ("climb_rate", C.c_double),
                ("n_buildings", C.c_int32), ("buildings_host", C.POINTER(C.c_double)),
                ("device", C.c_int32), ("auto_reset", C.c_int32)]


class EnvStateHost(C.Structure):
    _fields_ = [(k, C.POINTER(C.c_double)) for k in
                ("px", "py", "pz", "vx", "vy", "V", "score", "total_score", "path_len", "reward64")] + \
               [(k, C.POINTER(C.c_int32)) for k in ("step", "cursor", "scenario")] + \
               [("done", C.POINTER(C.c_uint8))]


class EnvExtras(C.Structure):
    _fields_ = [("energy_enabled", C.c_int32)] + [(k, C.c_double) for k in ("P_i", "v_0", "d_0", "rho", "s", "A", "P_b", "F_b", "xi")] + \
               [("apf_enabled", C.c_int32), ("obstacle_v_host", C.POINTER(C.c_double)), ("track_envs", C.c_int32),
                ("track_capacity", C.c_int32)]


class EpisodeRecord(C.Structure):
    _fields_ = [(k, C.c_int32) for k in ("scenario", "env", "ordinal", "outcome", "steps", "subgoals", "collisions", "reserved")] + \
               [(k, C.c_double) for k in ("total_score", "path_len", "start2goal", "planner_len", "final_dist", "energy")]


class EvalStats(C.Structure):
    _fields_ = [("iterations", C.c_int64), ("records", C.c_int64), ("unfinished", C.c_int64)]


class LearnerConfig(C.Structure):
    _fields_ = [("in_dim", C.c_int32), ("n_hidden", C.c_int32), ("hidden", C.c_int32 * MAX_HIDDEN),
                ("n_actions", C.c_int32), ("dueling", C.c_int32), ("algo", C.c_int32),
                ("lr", C.c_float), ("gamma", C.c_float), ("batch_size", C.c_int32),
                ("update_loop", C.c_int32), ("replay_capacity", C.c_int64),
                ("lockstep_envs", C.c_int32), ("seed", C.c_uint64), ("device", C.c_int32), ("loss_kind", C.c_int32)]


class SacConfig(C.Structure):
    _fields_ = [("obs_dim", C.c_int32), ("hidden", C.c_int32), ("act_dim", C.c_int32), ("action_bound", C.c_float),
                ("actor_lr", C.c_float), ("critic_lr", C.c_float), ("alpha_lr", C.c_float), ("target_entropy", C.c_float),
                ("gamma", C.c_float), ("tau", C.c_float), ("batch_size", C.c_int32), ("replay_capacity", C.c_int64),
                ("lockstep_envs", C.c_int32), ("seed", C.c_uint64), ("device", C.c_int32), ("loss_kind", C.c_int32)]


class TrainStats(C.Structure):
    _fields_ = [("env_steps", C.c_int64), ("updates", C.c_int64), ("episodes_ended", C.c_int64),
                ("collisions", C.c_int64), ("n_success", C.c_int64), ("n_lose", C.c_int64),
                ("sum_reward", C.c_double), ("last_loss", C.c_float)]


_lib = None
VP = C.c_void_p

# name -> (restype, argtypes); every symbol include/uavrl.h declares
SIGNATURES = {
    "uavrl_env_create": (C.c_int, [C.POINTER(EnvConfig), C.POINTER(VP)]),
    "uavrl_env_destroy": (C.c_int, [VP]),
    "uavrl_env_set_pool": (C.c_int, [VP, C.c_int32, VP, VP, VP, VP, VP, VP]),
    "uavrl_env_reset": (C.c_int, [VP, C.c_int32, VP]),
    "uavrl_env_set_reset_stride": (C.c_int, [VP, C.c_int32]),
    "uavrl_make_scenarios": (C.c_int, [C.POINTER(EnvConfig), C.c_uint64, C.c_int32, C.c_int32, VP, VP, VP, VP, VP]),
    "uavrl_set_pdl": (C.c_int, [C.c_int32]),
    "uavrl_test_fail_alloc": (C.c_int, [C.c_int32]),
    "uavrl_set_fuse_act_env": (C.c_int, [C.c_int32]),
    "uavrl_set_fuse_dw_adam": (C.c_int, [C.c_int32]),
    "uavrl_set_fuse_td": (C.c_int, [C.c_int32]),
    "uavrl_learner_td_fused": (C.c_int, [C.c_void_p, C.c_int32]),
    "uavrl_learner_tc_route": (C.c_int, [VP, C.c_int32, VP]),
    "uavrl_env_set_extras": (C.c_int, [VP, VP]),
    "uavrl_env_get_energy": (C.c_int, [VP, VP]),
    "uavrl_env_get_energy_total": (C.c_int, [VP, C.POINTER(C.c_double)]),
    "uavrl_env_get_path": (C.c_int, [VP, C.c_int32, C.c_int32, C.c_int32, VP, VP]),
    "uavrl_env_get_subgoals": (C.c_int, [VP, VP]),
    "uavrl_env_set_records": (C.c_int, [VP, C.c_int64]),
    "uavrl_env_get_records": (C.c_int, [VP, C.c_int64, VP, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_int32]),
    "uavrl_env_clear_records": (C.c_int, [VP]),
    "uavrl_eval_run": (C.c_int, [VP, VP, C.c_int32, C.c_int32, C.c_int64, VP, C.POINTER(EvalStats), VP]),
    "uavrl_sac_eval_run": (C.c_int, [VP, VP, C.c_int32, C.c_int32, C.c_int32, C.c_int64, VP, C.POINTER(EvalStats), VP]),
    "uavrl_sac_act_mean": (C.c_int, [VP, VP, C.c_int32, VP, VP]),
    "uavrl_per_enable": (C.c_int, [VP, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double]),
    "uavrl_per_enable_trainers": (C.c_int, [VP, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double]),
    "uavrl_per_sample": (C.c_int, [VP, C.c_int32, VP, VP, VP, VP]),
    "uavrl_per_set_errors": (C.c_int, [VP, C.c_int32, VP, VP, C.c_int32, VP]),
    "uavrl_per_set_priorities": (C.c_int, [VP, C.c_int32, VP, VP, VP]),
    "uavrl_per_get": (C.c_int, [VP, VP, C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "uavrl_learner_update_batch_per": (C.c_int, [VP, C.c_int32, VP, VP, VP, VP, VP, VP, VP, VP, VP]),
    "uavrl_env_generate_pool": (C.c_int, [VP, C.c_int32, C.c_uint64, C.c_int32, VP]),
    "uavrl_env_get_pool": (C.c_int, [VP, VP, VP, VP, VP, VP]),
    "uavrl_env_observe": (C.c_int, [VP, VP, VP]),
    "uavrl_env_step": (C.c_int, [VP, C.c_int32, VP, VP, VP, VP, VP, VP, VP, VP]),
    "uavrl_env_step_host": (C.c_int, [VP, C.c_int32, VP, VP, VP, VP, VP, VP, VP]),
    "uavrl_env_get_state": (C.c_int, [VP, C.POINTER(EnvStateHost)]),
    "uavrl_env_set_state": (C.c_int, [VP, C.POINTER(EnvStateHost)]),
    "uavrl_env_threaten_rate": (C.c_int, [VP, C.c_int32, VP, VP]),
    "uavrl_env_set_motion": (C.c_int, [VP, VP, VP]),
    "uavrl_env_get_obstacles": (C.c_int, [VP, VP, VP, VP]),
    "uavrl_learner_create": (C.c_int, [C.POINTER(LearnerConfig), C.POINTER(VP)]),
    "uavrl_learner_create_trainers": (C.c_int, [C.POINTER(LearnerConfig), C.c_int32, C.POINTER(VP)]),
    "uavrl_learner_trainer_count": (C.c_int32, [VP]),
    "uavrl_learner_federate": (C.c_int, [VP, VP, VP, VP, VP, VP, VP]),
    "uavrl_learner_fed_shard": (C.c_int, [VP, C.c_int32, C.c_int32]),
    "uavrl_learner_fed_exchange_ptr": (VP, [VP, C.c_int32, C.POINTER(C.c_int64)]),
    "uavrl_learner_fed_local": (C.c_int, [VP, VP, VP, VP, VP]),
    "uavrl_learner_fed_columns": (C.c_int, [VP, VP]),
    "uavrl_learner_fed_rounds": (C.c_int, [VP, VP, VP, VP]),
    "uavrl_learner_destroy": (C.c_int, [VP]),
    "uavrl_learner_param_count": (C.c_int64, [VP]),
    "uavrl_learner_set_params": (C.c_int, [VP, C.c_int32, VP]),
    "uavrl_learner_get_params": (C.c_int, [VP, C.c_int32, VP]),
    "uavrl_learner_set_counters": (C.c_int, [VP, C.c_int64, C.c_int64]),
    "uavrl_learner_get_counters": (C.c_int, [VP, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "uavrl_learner_act": (C.c_int, [VP, VP, C.c_int32, C.c_float, C.c_int32, VP, VP, VP, VP, VP]),
    "uavrl_replay_push": (C.c_int, [VP, C.c_int32, VP, VP, VP, VP, VP, VP]),
    "uavrl_replay_size": (C.c_int64, [VP]),
    "uavrl_replay_gather": (C.c_int, [VP, C.c_int32, VP, VP, VP, VP, VP, VP]),
    "uavrl_learner_update": (C.c_int, [VP, VP, VP, VP]),
    "uavrl_learner_update_batch": (C.c_int, [VP, C.c_int32, VP, VP, VP, VP, VP, VP, VP]),
    "uavrl_learner_compute_grads": (C.c_int, [VP, VP, C.c_int32, VP, VP]),
    "uavrl_learner_grad_ptr": (VP, [VP]),
    "uavrl_learner_apply_grads": (C.c_int, [VP, VP]),
    "uavrl_learner_hard_update": (C.c_int, [VP, VP]),
    "uavrl_learner_lockstep_restart": (C.c_int, [VP]),
    "uavrl_learner_set_is_train": (C.c_int, [VP, C.c_int32]),
    "uavrl_learner_set_tensor_cores": (C.c_int, [VP, C.c_int32]),
    "uavrl_learner_comm_init": (C.c_int, [VP, C.c_int32, C.c_int32, VP, VP]),
    "uavrl_learner_comm_connect": (C.c_int, [VP, VP, VP]),
    "uavrl_learner_update_dp": (C.c_int, [VP, VP, C.c_int32, VP, VP]),
    "uavrl_train_run": (C.c_int, [VP, VP, C.c_int32, C.c_float, C.c_int32, C.c_int32, C.POINTER(TrainStats), VP]),
    "uavrl_sac_create": (C.c_int, [C.POINTER(SacConfig), C.POINTER(VP)]),
    "uavrl_sac_create_trainers": (C.c_int, [C.POINTER(SacConfig), C.c_int32, C.POINTER(VP)]),
    "uavrl_sac_trainer_count": (C.c_int32, [VP]),
    "uavrl_sac_set_alpha": (C.c_int, [VP, VP]),
    "uavrl_sac_get_alpha": (C.c_int, [VP, VP]),
    "uavrl_sac_federate_actors": (C.c_int, [VP, VP]),
    "uavrl_sac_fed_shard": (C.c_int, [VP, C.c_int32, C.c_int32]),
    "uavrl_sac_fed_exchange_ptr": (VP, [VP, C.POINTER(C.c_int64)]),
    "uavrl_sac_fed_local": (C.c_int, [VP, VP]),
    "uavrl_sac_federate_actors_sharded": (C.c_int, [VP, VP]),
    "uavrl_sac_destroy": (C.c_int, [VP]),
    "uavrl_sac_param_count": (C.c_int64, [VP, C.c_int32]),
    "uavrl_sac_set_params": (C.c_int, [VP, C.c_int32, VP]),
    "uavrl_sac_get_params": (C.c_int, [VP, C.c_int32, VP]),
    "uavrl_sac_set_scalars": (C.c_int, [VP, C.c_float, C.c_float, C.c_float, C.c_int64, C.c_int64]),
    "uavrl_sac_get_scalars": (C.c_int, [VP, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "uavrl_sac_act": (C.c_int, [VP, VP, C.c_int32, VP, VP, VP]),
    "uavrl_sac_update_batch": (C.c_int, [VP, C.c_int32, VP, VP, VP, VP, VP, VP, VP, VP, VP]),
    "uavrl_sac_train_run": (C.c_int, [VP, VP, C.c_int32, C.c_int32, C.POINTER(TrainStats), VP]),
    "uavrl_sac_smem_bytes": (C.c_int, [C.POINTER(SacConfig), VP]),
    "uavrl_sac_replay_size": (C.c_int64, [VP]),
    "uavrl_sac_replay_gather": (C.c_int, [VP, C.c_int32, VP, VP, VP, VP, VP, VP]),
    "uavrl_sac_update_replay": (C.c_int, [VP, VP, VP, VP, VP, VP]),
    "uavrl_sac_per_enable": (C.c_int, [VP, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double]),
    "uavrl_sac_per_sample": (C.c_int, [VP, C.c_int32, VP, VP, VP, VP]),
    "uavrl_sac_per_set_errors": (C.c_int, [VP, C.c_int32, VP, VP, C.c_int32, VP]),
    "uavrl_sac_per_set_priorities": (C.c_int, [VP, C.c_int32, VP, VP, VP]),
    "uavrl_sac_per_get": (C.c_int, [VP, VP, C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "uavrl_sac_update_batch_per": (C.c_int, [VP, C.c_int32, VP, VP, VP, VP, VP, VP, VP, VP, VP, VP, VP]),
    "uavrl_sac_comm_init": (C.c_int, [VP, C.c_int32, C.c_int32, VP]),
    "uavrl_sac_comm_connect": (C.c_int, [VP, VP]),
    "uavrl_sac_update_replay_dp": (C.c_int, [VP, VP, VP, VP, C.c_int32, VP, VP]),
    "uavrl_sac_critic_grads_replay": (C.c_int, [VP, VP, VP, C.c_int32, VP]),
    "uavrl_sac_critic_grads_batch": (C.c_int, [VP, C.c_int32, VP, VP, VP, VP, VP, VP, C.c_int32, VP]),
    "uavrl_sac_apply_critic_grads": (C.c_int, [VP, VP]),
    "uavrl_sac_actor_grads": (C.c_int, [VP, VP, VP]),
    "uavrl_sac_apply_actor_grads": (C.c_int, [VP, VP, VP]),
    "uavrl_sac_exchange_ptr": (VP, [VP, C.c_int32, C.POINTER(C.c_int64)]),
    "uavrl_sac_train_run_dp": (C.c_int, [VP, VP, C.c_int32, C.c_int32, VP]),
    "uavrl_train_run_dp": (C.c_int, [VP, VP, C.c_int32, C.c_float, C.c_int32, VP]),
    "uavrl_train_profile": (C.c_int, [VP, VP, C.c_int32, C.c_float, VP, VP]),
    "uavrl_last_error": (C.c_char_p, []),
    "uavrl_version": (C.c_char_p, []),
    "uavrl_launch_count": (C.c_int64, []),
}


def lib():
    """Load (building first if sources are newer) the CUDA library.  Fails loudly."""
    global _lib
    if _lib is not None:
        return _lib
    if _build.needs_build():
        _build.build()
    if not os.path.exists(LIB_PATH):
        raise ImportError("libuavrl_b200.so is missing and could not be built; there is no CPU fallback")
    try:
        import torch  # noqa: F401  (brings libcudart.so.12 into the process)
    except Exception:  # pragma: no cover
        pass
    L = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(L, name)       # AttributeError here = header/library mismatch: fail loudly
        fn.restype, fn.argtypes = res, args
    _lib = L
    return L


def check(rc):
    if rc != 0:
        raise UavrlError("uavrl error %d: %s" % (rc, lib().uavrl_last_error().decode()))


def launch_count():
    return int(lib().uavrl_launch_count())
