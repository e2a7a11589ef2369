"""ctypes binding of ``libb200pets.so`` (the C ABI in ``include/b200pets.h``).

The library is built in-tree by ``build.py`` (nvcc, sm_90a).  There is no CPU fallback: if the shared
object is missing or a call fails, a ``RuntimeError`` carrying ``b200pets_last_error()`` is raised.
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libb200pets.so")

# constants mirrored from include/b200pets.h
ACT = {"relu": 0, "silu": 1, "leaky_relu": 2}
PROC = {None: 0, "halfcheetah": 1, "cartpole": 2}
REWARD = {None: 0, "learned": 0, "cartpole": 1, "cartpole_pets": 2, "inverted_pendulum": 3, "halfcheetah": 4,
          "pusher": 5, "external": 255}
TERM = {"no_termination": 0, "cartpole": 1, "inverted_pendulum": 2, "hopper": 3, "walker2d": 4, "ant": 5,
        "humanoid": 6, "external": 255}
PROP = {"random_model": 0, "fixed_model": 1, "expectation": 2}
PREC = {"f32": 0, "bf16_tc": 1}
DTYPE = {"float32": 0, "float64": 1}
TS1_PERMS, TS1_TILE_SHUFFLE = 0, 1


class ModelDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("ensemble_size", "num_members", "obs_dim", "act_dim", "in_size", "out_size",
                                         "hid_size", "num_hidden", "activation")] + [("leaky_slope", C.c_float)] + \
               [(n, C.c_int32) for n in ("obs_process", "learned_rewards", "target_is_delta", "deterministic",
                                         "reward_fn", "term_fn", "norm_mode")]


class RolloutCfg(C.Structure):
    _fields_ = [("population", C.c_int32), ("horizon", C.c_int32), ("particles", C.c_int32), ("precision", C.c_int32),
                ("propagation", C.c_int32), ("ts1_mode", C.c_int32), ("seed", C.c_uint64), ("offset", C.c_uint64),
                ("first_sequence", C.c_int32), ("global_population", C.c_int32)]


class CemCfg(C.Structure):
    _fields_ = [("num_iterations", C.c_int32), ("elite_num", C.c_int32), ("alpha", C.c_float),
                ("return_mean_elites", C.c_int32), ("clipped_normal", C.c_int32)]


class MppiCfg(C.Structure):
    _fields_ = [("num_iterations", C.c_int32), ("gamma", C.c_float), ("beta", C.c_float), ("sample_seed", C.c_uint64),
                ("sample_counter", C.c_uint64)]


class LatentDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("action_size", "latent_size", "belief_size", "hidden_size")] + \
               [("min_std", C.c_float)]


LATENT_NUM_PARAMS = 16


class LatentTrainDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("action_size", "latent_size", "belief_size", "hidden_size", "encoding_size")] + \
               [("min_std", C.c_float)]


class LatentTape(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("e", "gates", "q1", "p1", "pre_std", "eps", "de", "dgi", "dghn", "dq", "dv", "dp")]


LATENT_TRAIN_NUM_PARAMS = 13


class PrepDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("obs_dim", "act_dim", "obs_process", "norm_mode", "target_is_delta",
                                         "learned_rewards", "dtype")]


class TrainDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("ensemble_size", "in_size", "out_size", "hid_size", "num_hidden", "activation")] + \
               [("leaky_slope", C.c_float), ("deterministic", C.c_int32), ("learn_logvar_bounds", C.c_int32)] + \
               [(n, C.c_double) for n in ("lr", "beta1", "beta2", "eps", "weight_decay")]


SAC_MAX_ACTIONS = 32
SAC_NUM_PARAMS, SAC_NUM_CRITIC_PARAMS = 20, 12


class SacDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("obs_dim", "act_dim", "hidden")] + \
               [("action_scale", C.c_float * SAC_MAX_ACTIONS), ("action_bias", C.c_float * SAC_MAX_ACTIONS)] + \
               [(n, C.c_double) for n in ("gamma", "tau", "lr", "beta1", "beta2", "eps")] + \
               [("automatic_entropy_tuning", C.c_int32), ("target_entropy", C.c_float),
                ("target_update_interval", C.c_int32)]


_P = C.c_void_p
_SIGNATURES = {
    "b200pets_version": (C.c_int, []),
    "b200pets_last_error": (C.c_char_p, []),
    "b200pets_device_info": (C.c_int, [C.POINTER(C.c_int32)] * 3),
    "b200pets_model_create": (C.c_int, [C.POINTER(ModelDesc), C.POINTER(_P), C.POINTER(_P), C.POINTER(C.c_int32),
                                        C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_float),
                                        C.POINTER(C.c_float), C.POINTER(C.c_int32), C.c_int32, _P, C.POINTER(_P)]),
    "b200pets_model_refresh": (C.c_int, [_P, C.POINTER(_P), C.POINTER(_P), C.POINTER(C.c_int32), C.POINTER(C.c_double),
                                         C.POINTER(C.c_double), C.POINTER(C.c_float), C.POINTER(C.c_float), _P]),
    "b200pets_model_destroy": (None, [_P]),
    "b200pets_model_supports_tc": (C.c_int, [_P]),
    "b200pets_model_plan_info": (C.c_int, [_P, C.c_int32, C.POINTER(C.c_int32)]),
    "b200pets_eval_workspace_bytes": (C.c_size_t, [_P, C.POINTER(RolloutCfg)]),
    "b200pets_eval_sequences": (C.c_int, [_P, C.POINTER(RolloutCfg), _P, _P, _P, _P, _P, _P, _P, C.c_size_t, _P]),
    "b200pets_trajectory_workspace_bytes": (C.c_size_t, [_P, C.POINTER(RolloutCfg)]),
    "b200pets_eval_trajectory": (C.c_int, [_P, C.POINTER(RolloutCfg), C.c_int32, C.c_int32, _P, _P, _P, _P, _P, _P, _P, _P,
                                           C.c_size_t, _P]),
    "b200pets_trajectory_returns": (C.c_int, [C.POINTER(RolloutCfg), C.c_int32, C.c_int32, _P, _P, _P, _P, _P, C.c_size_t,
                                              _P]),
    "b200pets_step": (C.c_int, [_P, C.c_int32, C.c_int32, C.c_int64, _P, _P, _P, _P, C.c_uint64, C.c_uint64, C.c_int32,
                                _P, _P, _P, _P]),
    "b200pets_mbpo_mask": (C.c_int, [C.c_int64, _P, _P, _P, _P]),
    "b200pets_mbpo_compact_workspace_bytes": (C.c_size_t, [C.c_int32, C.c_int64]),
    "b200pets_mbpo_compact": (C.c_int, [C.c_int32, C.c_int64, C.c_int32, C.c_int32] + [_P] * 12 + [_P, C.c_size_t, _P]),
    "b200pets_cem_sample": (C.c_int, [C.c_int32, C.c_int32, _P, _P, _P, _P, _P, C.c_uint64, C.c_uint64, C.c_int32, _P, _P]),
    "b200pets_cem_sample_shard": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, _P, _P, _P, _P, _P, C.c_uint64, C.c_uint64, C.c_int32,
                                            _P, _P]),
    "b200pets_shuffle_num_groups": (C.c_int64, [C.POINTER(RolloutCfg)]),
    "b200pets_shuffle_member_map": (C.c_int, [C.POINTER(RolloutCfg), C.c_int32, _P, _P]),
    "b200pets_cem_update_workspace_bytes": (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32]),
    "b200pets_cem_update": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_int32, C.c_int32, _P, _P, _P, _P,
                                      _P, _P, _P, _P, _P, C.c_size_t, _P]),
    "b200pets_cem_local_topk": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, _P, _P, _P, _P, C.c_size_t, _P]),
    "b200pets_cem_update_from_records": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_int32, C.c_int32, _P,
                                                   _P, _P, _P, _P, _P, _P, C.c_size_t, _P]),
    "b200pets_icem_sample": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.c_float, _P, _P, _P, _P, _P, _P, C.c_uint64,
                                       C.c_uint64, _P, _P]),
    "b200pets_icem_append_elites": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, _P, _P, C.c_int32, _P, _P, _P, C.c_uint64,
                                              C.c_uint64, _P, _P]),
    "b200pets_mppi_sample": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.c_float, _P, _P, _P, _P, _P, C.c_uint64, C.c_uint64,
                                       _P, _P]),
    "b200pets_mppi_update_workspace_bytes": (C.c_size_t, [C.c_int32, C.c_int32]),
    "b200pets_mppi_update": (C.c_int, [C.c_int32, C.c_int32, C.c_float, _P, _P, _P, _P, C.c_size_t, _P]),
    "b200pets_shift_solution": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, _P, _P, _P, _P]),
    "b200pets_cem_plan_workspace_bytes": (C.c_size_t, [_P, C.POINTER(RolloutCfg), C.POINTER(CemCfg)]),
    "b200pets_cem_plan": (C.c_int, [_P, C.POINTER(RolloutCfg), C.POINTER(CemCfg), _P, _P, _P, _P, _P, _P, _P, _P, _P, _P,
                                    C.c_size_t, _P]),
    "b200pets_eval_batch_workspace_bytes": (C.c_size_t, [_P, C.POINTER(RolloutCfg), C.c_int32]),
    "b200pets_eval_sequences_batch": (C.c_int, [_P, C.POINTER(RolloutCfg), C.c_int32, _P, _P, _P, _P, _P, _P, _P, C.c_size_t,
                                                _P]),
    "b200pets_cem_plan_batch_workspace_bytes": (C.c_size_t, [_P, C.POINTER(RolloutCfg), C.POINTER(CemCfg), C.c_int32]),
    "b200pets_cem_plan_batch": (C.c_int, [_P, C.POINTER(RolloutCfg), C.POINTER(CemCfg), C.c_int32, _P, _P, _P, _P, _P, _P, _P,
                                          _P, _P, _P, C.c_size_t, _P]),
    "b200pets_mppi_plan_batch_workspace_bytes": (C.c_size_t, [_P, C.POINTER(RolloutCfg), C.POINTER(MppiCfg), C.c_int32]),
    "b200pets_mppi_plan_batch": (C.c_int, [_P, C.POINTER(RolloutCfg), C.POINTER(MppiCfg), C.c_int32, _P, _P, _P, _P, _P, _P, _P,
                                           _P, _P, C.c_size_t, _P]),
    "b200pets_peer_buffer_bytes": (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "b200pets_peer_alloc": (C.c_int, [C.c_size_t, C.POINTER(C.c_void_p), C.c_char_p]),
    "b200pets_peer_open": (C.c_int, [C.c_char_p, C.POINTER(C.c_void_p)]),
    "b200pets_peer_close": (C.c_int, [_P, C.c_int32]),
    "b200pets_cem_values_push": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, _P, C.c_int32, C.c_int32, C.c_uint32,
                                           C.POINTER(C.c_void_p), _P]),
    "b200pets_cem_elites_refit": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_int32, C.c_int32,
                                            C.c_int32, C.c_uint32, C.POINTER(C.c_void_p), _P, _P, _P, _P, _P, C.c_int32, _P, _P,
                                            C.c_uint64, C.c_uint64, C.c_int32, _P, _P, _P]),
    "b200pets_selftest_wgmma": (C.c_int, [C.c_int32, C.c_int32, _P, _P, _P, _P]),
    "b200pets_latent_model_create": (C.c_int, [C.POINTER(LatentDesc), C.POINTER(_P), _P, C.POINTER(_P)]),
    "b200pets_latent_model_refresh": (C.c_int, [_P, C.POINTER(_P), _P]),
    "b200pets_latent_model_destroy": (None, [_P]),
    "b200pets_latent_plan_info": (C.c_int, [_P, C.c_int64, C.POINTER(C.c_int32)]),
    "b200pets_latent_step": (C.c_int, [_P, C.c_int64, _P, _P, _P, _P, C.c_uint64, C.c_uint64, C.c_int32, _P, _P, _P, _P]),
    "b200pets_latent_eval_workspace_bytes": (C.c_size_t, [_P, C.POINTER(RolloutCfg)]),
    "b200pets_latent_eval_sequences": (C.c_int, [_P, C.POINTER(RolloutCfg), _P, _P, _P, _P, _P, _P, _P, C.c_size_t, _P]),
    "b200pets_latent_cem_plan_workspace_bytes": (C.c_size_t, [_P, C.POINTER(RolloutCfg), C.POINTER(CemCfg)]),
    "b200pets_latent_cem_plan": (C.c_int, [_P, C.POINTER(RolloutCfg), C.POINTER(CemCfg), _P, _P, _P, _P, _P, _P, _P, _P, _P,
                                           _P, C.c_size_t, _P]),
    "b200pets_latent_train_supported": (C.c_int, [C.POINTER(LatentTrainDesc)]),
    "b200pets_latent_train_workspace_bytes": (C.c_size_t, [C.POINTER(LatentTrainDesc), C.c_int32, C.c_int32]),
    "b200pets_latent_seq_forward": (C.c_int, [C.POINTER(LatentTrainDesc), C.POINTER(_P), C.c_int32, C.c_int32, _P, _P, _P, _P,
                                              C.c_uint64, C.c_uint64, _P, _P, _P, _P, _P, C.POINTER(LatentTape), _P,
                                              C.c_size_t, _P]),
    "b200pets_latent_seq_backward": (C.c_int, [C.POINTER(LatentTrainDesc), C.POINTER(_P), C.c_int32, C.c_int32, _P, _P, _P,
                                               _P, _P, _P, C.POINTER(LatentTape), _P, _P]),
    "b200pets_train_preprocess": (C.c_int, [C.POINTER(PrepDesc), C.c_int64, _P, _P, _P, _P, _P, _P, C.POINTER(C.c_int32),
                                            C.c_int32, _P, _P, _P]),
    "b200pets_trainer_create": (C.c_int, [C.POINTER(TrainDesc), C.POINTER(_P), C.POINTER(_P), C.POINTER(_P), C.POINTER(_P)]),
    "b200pets_trainer_destroy": (None, [_P]),
    "b200pets_trainer_supported": (C.c_int, [C.POINTER(TrainDesc)]),
    "b200pets_train_workspace_bytes": (C.c_size_t, [_P, C.c_int32]),
    "b200pets_train_epoch": (C.c_int, [_P, C.c_int64, _P, _P, _P, C.c_int32, C.c_int32, C.c_int32, C.c_int64, _P, _P,
                                       C.c_size_t, _P]),
    "b200pets_eval_score_workspace_bytes": (C.c_size_t, [_P, C.c_int64]),
    "b200pets_eval_score": (C.c_int, [_P, C.c_int64, _P, _P, _P, _P, C.c_size_t, _P]),
    "b200pets_sac_supported": (C.c_int, [C.POINTER(SacDesc)]),
    "b200pets_sac_create": (C.c_int, [C.POINTER(SacDesc), C.POINTER(_P), C.POINTER(_P), C.POINTER(_P), C.POINTER(_P), _P, _P,
                                      _P, C.POINTER(_P)]),
    "b200pets_sac_destroy": (None, [_P]),
    "b200pets_sac_workspace_bytes": (C.c_size_t, [_P, C.c_int32]),
    "b200pets_sac_update": (C.c_int, [_P, C.c_int32, C.c_int64, C.c_int32, C.POINTER(C.c_int64), _P, _P, C.c_uint64,
                                      C.c_uint64, _P, _P, _P, C.c_size_t, _P]),
}

_lib = None


def exported_symbols():
    """Names ``include/b200pets.h`` declares (used by the CPU test that the library exports all of them)."""
    return list(_SIGNATURES)


def load():
    """Load (once) and return the ctypes handle; raises if the CUDA library has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` (needs nvcc). "
            "b200pets has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = load().b200pets_last_error().decode()
        if rc == -1:
            raise ValueError(msg)
        if rc == -2:
            raise NotImplementedError(msg)
        raise RuntimeError(f"{what}: {msg} (code {rc})")


def ptr(t):
    """Device pointer of a torch tensor (or None)."""
    return None if t is None else C.c_void_p(t.data_ptr())


def stream_ptr():
    import torch

    return C.c_void_p(torch.cuda.current_stream().cuda_stream)
