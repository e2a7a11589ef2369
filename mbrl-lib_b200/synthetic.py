"""Seeded synthetic inputs for the PETS planning hot path.

Everything is drawn from ``numpy.random.default_rng`` streams so that the same case name yields the
same arrays in the build container (where golden vectors are generated from the imported reference)
and on the GPU box (where only this repo exists).  Shapes follow the reference's conventions:

* ensemble weights ``W_l[E, K, N]``, biases ``b_l[E, 1, N]``     (mbrl/models/util.py:41-45)
* rows ``r = n * P + p`` (sequence-major, particle-minor)         (mbrl/models/model_env.py:170-182)
* one permutation of ``B = N * P`` rows per step (TS1) or one at reset (TSinf)
                                                                  (mbrl/models/gaussian_mlp.py:202-212)
"""
from __future__ import annotations

import dataclasses
import hashlib
import itertools
from typing import Dict, List, Optional, Sequence

import numpy as np


@dataclasses.dataclass
class CaseSpec:
    name: str
    obs_dim: int
    act_dim: int
    hid_size: int = 200
    num_layers: int = 4  # hidden layers
    ensemble_size: int = 7
    elites: Optional[Sequence[int]] = (0, 2, 3, 5, 6)
    activation: str = "silu"  # "relu" | "silu" | "leaky_relu"
    propagation: str = "random_model"  # "random_model" | "fixed_model" | "expectation"
    normalize: Optional[str] = "float64"  # "float64" | "float32" | None
    obs_process: Optional[str] = None  # None | "halfcheetah" | "cartpole"
    learned_rewards: bool = False
    target_is_delta: bool = True
    no_delta_list: Sequence[int] = ()
    reward_fn: Optional[str] = "halfcheetah"
    term_fn: str = "no_termination"
    deterministic: bool = False
    population: int = 500
    horizon: int = 30
    particles: int = 20
    action_lb: float = -1.0
    action_ub: float = 1.0
    obs0_first: Optional[float] = None  # e.g. 1.4 for humanoid height
    seed: int = 0
    # added to the output bias of every other logvar column (columns 0, 2, 4, ... take the offsets in turn), after
    # all draws: pushes raw logvars far outside [min_logvar, max_logvar]
    logvar_offsets: Sequence[float] = ()

    @property
    def proc_obs_dim(self) -> int:
        return self.obs_dim + (1 if self.obs_process == "cartpole" else 0)

    @property
    def in_size(self) -> int:
        return self.proc_obs_dim + self.act_dim

    @property
    def out_size(self) -> int:
        return self.obs_dim + (1 if self.learned_rewards else 0)

    @property
    def num_models(self) -> int:
        return len(self.elites) if self.elites is not None else self.ensemble_size

    @property
    def batch(self) -> int:
        return self.population * self.particles


# The configurations BASELINE.json names (SURVEY.md section 8d), plus reduced copies used as parity cases.
CASES: Dict[str, CaseSpec] = {}


def _register(c: CaseSpec) -> CaseSpec:
    CASES[c.name] = c
    return c


# config 1: cartpole tutorial (pets_example.ipynb), TSinf, LeakyReLU, fp32 normaliser, all members elite
_register(CaseSpec("cartpole", obs_dim=4, act_dim=1, num_layers=3, ensemble_size=5, elites=None,
                   activation="leaky_relu", propagation="fixed_model", normalize="float32",
                   reward_fn="cartpole", term_fn="cartpole", population=100, horizon=15, particles=20))
# config 2: headline, HalfCheetah-v4 dims, TS1
_register(CaseSpec("halfcheetah", obs_dim=17, act_dim=6))
_register(CaseSpec("halfcheetah_small", obs_dim=17, act_dim=6, population=40, horizon=12, particles=5))
# shipped pets_halfcheetah.yaml variant: obs 18 with preprocess_fn, no_delta_list=[0], pop 400
_register(CaseSpec("pets_halfcheetah", obs_dim=18, act_dim=6, obs_process="halfcheetah",
                   no_delta_list=(0,), population=400, horizon=30, particles=20))
_register(CaseSpec("pets_halfcheetah_small", obs_dim=18, act_dim=6, obs_process="halfcheetah",
                   no_delta_list=(0,), population=30, horizon=8, particles=10))
# config 3 (truncated-obs humanoid dims; learned reward, humanoid termination)
_register(CaseSpec("humanoid_trunc", obs_dim=45, act_dim=17, learned_rewards=True, reward_fn=None,
                   term_fn="humanoid", population=70, horizon=10, particles=5,
                   action_lb=-0.4, action_ub=0.4, obs0_first=1.4))
# config 3 at the real Humanoid-v4 dims (obs 376, act 17, learned reward): in 393 -> out 754; outside the tensor-core plan
_register(CaseSpec("humanoid_v4", obs_dim=376, act_dim=17, learned_rewards=True, reward_fn=None,
                   term_fn="humanoid", population=20, horizon=6, particles=5,
                   action_lb=-0.4, action_ub=0.4, obs0_first=1.4))
# config 4: MBPO step, learned rewards
_register(CaseSpec("mbpo_halfcheetah", obs_dim=17, act_dim=6, learned_rewards=True, reward_fn=None,
                   population=100000, horizon=1, particles=1))
_register(CaseSpec("mbpo_halfcheetah_small", obs_dim=17, act_dim=6, learned_rewards=True, reward_fn=None,
                   population=1000, horizon=1, particles=1))
# tensor-core plan edge cases: hid % 16 == 0 (bias columns spill into an extra K step), wide output layer that cannot
# start under the last hidden epilogue (2 * round16(out) > first N half), large input (8 K steps)
_register(CaseSpec("tc_hid64", obs_dim=9, act_dim=2, hid_size=64, num_layers=3, ensemble_size=3, elites=None,
                   activation="silu", propagation="random_model", normalize="float32", learned_rewards=True, reward_fn=None,
                   term_fn="no_termination", population=48, horizon=6, particles=4))
_register(CaseSpec("tc_shallow", obs_dim=6, act_dim=2, hid_size=32, num_layers=1, ensemble_size=4, elites=(2, 0),
                   activation="leaky_relu", propagation="random_model", normalize=None, reward_fn="halfcheetah",
                   term_fn="no_termination", population=33, horizon=9, particles=4))
_register(CaseSpec("tc_wide", obs_dim=100, act_dim=20, hid_size=240, num_layers=2, ensemble_size=2, elites=None,
                   activation="relu", propagation="fixed_model", normalize="float64", learned_rewards=True, reward_fn=None,
                   term_fn="humanoid", population=40, horizon=5, particles=4, obs0_first=1.4))
# coverage cases: relu + expectation / deterministic / cartpole_pets preprocess / hopper termination
_register(CaseSpec("relu_expectation", obs_dim=11, act_dim=3, hid_size=64, num_layers=2, ensemble_size=3,
                   elites=None, activation="relu", propagation="expectation", normalize=None,
                   reward_fn="inverted_pendulum", term_fn="inverted_pendulum",
                   population=24, horizon=6, particles=4))
# expectation propagation at the headline model shape (7 members / 5 elites, 4 x 200 SiLU, fp64 normaliser), continuous reward:
# the tensor-core kernel's member-pass path is pinned to the reference at the exact bars
_register(CaseSpec("silu_expectation", obs_dim=17, act_dim=6, propagation="expectation",
                   population=25, horizon=6, particles=4))
_register(CaseSpec("hopper_tsinf", obs_dim=11, act_dim=3, hid_size=96, num_layers=3, ensemble_size=4,
                   elites=(3, 1), activation="silu", propagation="fixed_model", normalize="float64",
                   learned_rewards=True, reward_fn=None, term_fn="hopper",
                   population=32, horizon=9, particles=6, obs0_first=1.2))
_register(CaseSpec("cartpole_pets", obs_dim=4, act_dim=1, hid_size=48, num_layers=2, ensemble_size=5,
                   elites=(4, 0, 2), activation="silu", propagation="random_model", normalize="float64",
                   obs_process="cartpole", reward_fn="cartpole_pets", term_fn="no_termination",
                   population=27, horizon=7, particles=3))
_register(CaseSpec("pusher_det", obs_dim=20, act_dim=7, hid_size=80, num_layers=2, ensemble_size=2,
                   elites=None, activation="silu", propagation="random_model", normalize="float32",
                   deterministic=True, reward_fn="pusher", term_fn="no_termination",
                   population=16, horizon=5, particles=2, action_lb=-2.0, action_ub=2.0))
_register(CaseSpec("walker_ant", obs_dim=17, act_dim=6, hid_size=72, num_layers=2, ensemble_size=2,
                   elites=None, activation="silu", propagation="random_model", normalize="float64",
                   learned_rewards=True, reward_fn=None, term_fn="walker2d",
                   population=20, horizon=8, particles=4, obs0_first=1.2))


# MBPO rollouts with terminations (hopper rule): the accum_dones mask of mbpo.py:44-62 is exercised
_register(CaseSpec("mbpo_hopper_small", obs_dim=11, act_dim=3, hid_size=64, num_layers=2, ensemble_size=4, elites=None,
                   activation="silu", propagation="random_model", normalize="float64", learned_rewards=True,
                   reward_fn=None, term_fn="hopper", population=1024, horizon=1, particles=1, obs0_first=1.0))
# learned reward column AND a named reward_fn (the explicit fn wins, model_env.py:124-128), ant termination
_register(CaseSpec("ant_learned_fn", obs_dim=27, act_dim=8, hid_size=64, num_layers=2, ensemble_size=3,
                   elites=None, activation="silu", propagation="random_model", normalize="float64",
                   learned_rewards=True, reward_fn="halfcheetah", term_fn="ant",
                   population=24, horizon=7, particles=5, obs0_first=0.6))



# Launch-plan cases: shapes that put the kernels on the launch plans the cases above never reach (the plan each one
# lands on is read back from b200pets_model_plan_info by tests/test_gpu_parity.py::test_launch_plans_are_covered).
# Tensor-core kernel: K steps per weight-ring slot 1 / 2 / 3, a two-slot ring, hidden widths of 16, 128, 144 and 256
# accumulator columns (hid % 16 of 14, 15 and 0: where the two bias-one columns sit against the accumulator's end),
# 256-column input and output layers, seven hidden layers, expectation at a shortened slice.  fp32 kernel: 32- and
# 16-row tiles.  Plus a model whose raw logvars sit far outside [min_logvar, max_logvar].
_register(CaseSpec("plan_hid14_deep", obs_dim=5, act_dim=2, hid_size=14, num_layers=7, ensemble_size=3, elites=None,
                   activation="relu", normalize="float32", population=37, horizon=5, particles=3))
_register(CaseSpec("plan_hid143", obs_dim=17, act_dim=6, hid_size=143, num_layers=3, ensemble_size=4, elites=(1, 3),
                   population=45, horizon=6, particles=4))
_register(CaseSpec("plan_hid128_det", obs_dim=20, act_dim=7, hid_size=128, num_layers=2, ensemble_size=2, elites=None,
                   normalize="float32", deterministic=True, reward_fn="pusher", population=30, horizon=5, particles=2,
                   action_lb=-2.0, action_ub=2.0))
_register(CaseSpec("plan_k3", obs_dim=90, act_dim=6, population=21, horizon=4, particles=5))
_register(CaseSpec("plan_k2_hid254", obs_dim=90, act_dim=17, hid_size=254, num_layers=3, ensemble_size=2, elites=None,
                   activation="relu", propagation="fixed_model", population=26, horizon=4, particles=4))
_register(CaseSpec("plan_k1_out256", obs_dim=127, act_dim=8, hid_size=254, num_layers=2, ensemble_size=2, elites=None,
                   activation="leaky_relu", learned_rewards=True, reward_fn=None, population=19, horizon=3, particles=4))
_register(CaseSpec("plan_in254", obs_dim=11, act_dim=243, num_layers=2, ensemble_size=2, elites=None,
                   population=17, horizon=3, particles=4))
_register(CaseSpec("plan_ring2", obs_dim=120, act_dim=17, num_layers=2, ensemble_size=2, elites=None,
                   learned_rewards=True, reward_fn=None, population=23, horizon=3, particles=4))
_register(CaseSpec("plan_k4_hid254", obs_dim=60, act_dim=20, hid_size=254, num_layers=2, ensemble_size=2, elites=None,
                   learned_rewards=True, reward_fn=None, population=22, horizon=3, particles=4))
_register(CaseSpec("plan_exp_k2", obs_dim=57, act_dim=8, hid_size=254, num_layers=2, ensemble_size=3, elites=None,
                   propagation="expectation", population=13, horizon=3, particles=3))
_register(CaseSpec("plan_f32_hid512", obs_dim=17, act_dim=6, hid_size=512, num_layers=2, ensemble_size=2, elites=None,
                   population=100, horizon=4, particles=4))
_register(CaseSpec("plan_f32_hid512_exp", obs_dim=17, act_dim=6, hid_size=512, num_layers=2, ensemble_size=2,
                   elites=None, propagation="expectation", population=25, horizon=4, particles=4))
_register(CaseSpec("plan_f32_humanoid_exp", obs_dim=376, act_dim=17, learned_rewards=True, reward_fn=None,
                   term_fn="humanoid", propagation="expectation", population=10, horizon=3, particles=4,
                   action_lb=-0.4, action_ub=0.4, obs0_first=1.4))
_register(CaseSpec("plan_logvar_extreme", obs_dim=17, act_dim=6, hid_size=64, num_layers=2, ensemble_size=3,
                   elites=None, population=30, horizon=5, particles=4, logvar_offsets=(10.0, -30.0, -100.0)))
PLAN_CASES = [n for n in CASES if n.startswith("plan_")]


def _rng(spec: CaseSpec, stream: int) -> np.random.Generator:
    return np.random.default_rng([spec.seed, stream, int(hashlib.sha1(spec.name.encode()).hexdigest()[:8], 16)])


def layer_dims(spec: CaseSpec) -> List[tuple]:
    dims = [(spec.in_size, spec.hid_size)]
    dims += [(spec.hid_size, spec.hid_size)] * (spec.num_layers - 1)
    dims += [(spec.hid_size, spec.out_size * (1 if spec.deterministic else 2))]
    return dims


def make_model_arrays(spec: CaseSpec) -> Dict[str, object]:
    """Weights / logvar bounds / normaliser statistics for ``spec`` as float32 (fp64 stats when asked)."""
    g = _rng(spec, 1)
    E = spec.ensemble_size
    weights, biases = [], []
    dims = layer_dims(spec)
    for li, (k, n) in enumerate(dims):
        std = 1.0 / (2.0 * np.sqrt(k))
        w = np.clip(g.standard_normal((E, k, n)), -2.0, 2.0) * std
        b = 0.05 * g.standard_normal((E, 1, n))
        if li == len(dims) - 1 and not spec.deterministic:
            # moderately confident model: raw logvar around -5 (sigma ~ 0.08)
            b[:, :, spec.out_size:] += -5.0
        if li == len(dims) - 1 and not spec.deterministic and spec.logvar_offsets:
            for j, off in zip(range(0, spec.out_size, 2), itertools.cycle(spec.logvar_offsets)):
                b[:, :, spec.out_size + j] += off
        weights.append(w.astype(np.float32))
        biases.append(b.astype(np.float32))
    out = {
        "weights": weights,
        "biases": biases,
        "min_logvar": (-10.0 + 0.5 * g.standard_normal((1, spec.out_size))).astype(np.float32),
        "max_logvar": (0.5 + 0.1 * g.standard_normal((1, spec.out_size))).astype(np.float32),
    }
    if spec.normalize is not None:
        dt = np.float64 if spec.normalize == "float64" else np.float32
        data = g.standard_normal((1000, spec.in_size))
        out["norm_mean"] = data.mean(0, keepdims=True).astype(dt)
        out["norm_std"] = data.std(0, ddof=1, keepdims=True).astype(dt)
    return out


def make_rollout_inputs(spec: CaseSpec, population: Optional[int] = None, horizon: Optional[int] = None,
                        particles: Optional[int] = None, with_noise: bool = True) -> Dict[str, np.ndarray]:
    """obs0, action sequences and the injected noise (eps, permutations) of one evaluation."""
    N = population or spec.population
    H = horizon or spec.horizon
    P = particles or spec.particles
    B = N * P
    g = _rng(spec, 2)
    obs0 = g.standard_normal(spec.obs_dim)
    if spec.obs0_first is not None:
        obs0[0] = spec.obs0_first
    if spec.term_fn in ("cartpole", "inverted_pendulum", "hopper", "walker2d", "ant"):
        obs0[1:] *= 0.05  # start inside the "alive" region
    out = {
        "obs0": obs0.astype(np.float64),  # envs hand fp64 observations to the agent
        "actions": g.uniform(spec.action_lb, spec.action_ub, (N, H, spec.act_dim)).astype(np.float32),
    }
    if with_noise:
        out["eps"] = g.standard_normal((H, B, spec.out_size), dtype=np.float32)
        nperm = 1 if spec.propagation == "fixed_model" else H
        out["perms"] = np.stack([g.permutation(B) for _ in range(nperm)]).astype(np.int64)
    return out


def make_step_inputs(spec: CaseSpec, batch: int) -> Dict[str, np.ndarray]:
    """A batch of start states / actions for ``ModelEnv.step`` (config 4)."""
    g = _rng(spec, 3)
    obs = g.standard_normal((batch, spec.obs_dim)).astype(np.float32)
    if spec.obs0_first is not None:
        obs[:, 0] = spec.obs0_first
    return {
        "obs": obs,
        "act": g.uniform(spec.action_lb, spec.action_ub, (batch, spec.act_dim)).astype(np.float32),
        "eps": g.standard_normal((batch, spec.out_size), dtype=np.float32),
        "perm": g.permutation(batch).astype(np.int64),
    }


def checksum(arrays) -> str:
    """Stable digest of a list/dict of arrays (used to pin that regenerated inputs equal the golden run's)."""
    h = hashlib.sha256()
    items = arrays.items() if isinstance(arrays, dict) else enumerate(arrays)
    for k, a in items:
        if isinstance(a, (list, tuple)):
            for x in a:
                h.update(np.ascontiguousarray(x).tobytes())
        else:
            h.update(np.ascontiguousarray(a).tobytes())
        h.update(str(k).encode())
    return h.hexdigest()[:16]


def make_cem_noise(spec: CaseSpec, iters: int, seed: int = 4321) -> Dict[str, np.ndarray]:
    """Injected draws for ``iters`` CEM iterations over the model rollout: truncated population noise
    z[i, N, H, A], model noise eps[i, H, B, out] and TS1 permutations perms[i, H, B]."""
    g = np.random.default_rng(seed)
    N, H, A, P = spec.population, spec.horizon, spec.act_dim, spec.particles
    B = N * P
    z = np.clip(g.standard_normal((iters, N, H, A)), -2, 2).astype(np.float32)
    eps = g.standard_normal((iters, H, B, spec.out_size), dtype=np.float32)
    perms = np.stack([[g.permutation(B) for _ in range(H)] for _ in range(iters)]).astype(np.int64)
    return {"z": z, "eps": eps, "perms": perms}


def counter_world(hid_size: int = 32):
    """A hand-built deterministic ReLU ensemble that IS the reference's known-answer model
    (tests/core/test_models.py:337-385): next_obs = obs + a, reward = next_obs, exact in fp32 and in bf16 for the
    small integers involved, so ``evaluate_action_sequences`` must return exactly H(H+1)/2 * a from obs0 = 0, a > 0.
    """
    spec = CaseSpec("counter_world", obs_dim=1, act_dim=1, hid_size=hid_size, num_layers=1, ensemble_size=2, elites=None,
                    activation="relu", propagation="random_model", normalize=None, learned_rewards=True,
                    reward_fn=None, deterministic=True, population=4, horizon=9, particles=9, action_lb=0.0, action_ub=2.0)
    w0 = np.zeros((2, 2, hid_size), np.float32)
    w0[:, 1, 0] = 1.0                   # h0 = relu(a)
    w0[:, 0, 1] = w0[:, 1, 1] = 1.0     # h1 = relu(obs + a)
    w1 = np.zeros((2, hid_size, 2), np.float32)
    w1[:, 0, 0] = 1.0                   # delta  = a
    w1[:, 1, 1] = 1.0                   # reward = obs + a
    arrays = {"weights": [w0, w1], "biases": [np.zeros((2, 1, hid_size), np.float32), np.zeros((2, 1, 2), np.float32)],
              "min_logvar": np.full((1, 2), -10.0, np.float32), "max_logvar": np.full((1, 2), 0.5, np.float32)}
    return spec, arrays
