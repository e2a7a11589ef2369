"""Trajectory optimisers and the MPC agent with the reference's plugin interface
(mbrl/planning/core.py:18-49, mbrl/planning/trajectory_opt.py) over the CUDA CEM / rollout kernels.

* ``CEMOptimizer`` / ``ICEMOptimizer``: same constructor kwargs as the YAML configs pass
  (conf/action_optimizer/cem.yaml, icem.yaml), same ``optimize(obj_fun, x0, callback)`` protocol.  With an
  opaque ``obj_fun`` each iteration is  sample kernel -> obj_fun(population) -> select/refit kernel  and no
  host synchronisation of ours (the reference syncs on ``.item()`` / ``best_values[0] > best_value``).
* When ``obj_fun`` is the ``evaluate_action_sequences`` closure built by
  :func:`create_trajectory_optim_agent_for_model`, ``CEMOptimizer`` runs the whole optimisation as one
  C call (``b200pets_cem_plan``): every iteration's sample -> rollout -> refit is enqueued back to back.
* ``TrajectoryOptimizer`` / ``TrajectoryOptimizerAgent`` / ``create_trajectory_optim_agent_for_model``:
  reference semantics (warm-start shift, action cache, RuntimeError when the eval fn is unset).
"""
from __future__ import annotations

import ctypes as C
import importlib
import time
from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib


# When mbrl-lib itself is importable (the drop-in case: a user's PETS script with mbrl installed), the classes below
# derive from ITS plugin bases, so `isinstance(x, mbrl.planning.Agent)` / `issubclass(cls, Optimizer)` checks in user
# code hold (SURVEY.md 8b row 1: "class X(mbrl.planning.Optimizer)").  Without it they stand alone.
try:  # pragma: no cover - depends on the host environment
    from mbrl.planning.core import Agent as _RefAgent
    from mbrl.planning.trajectory_opt import Optimizer as _RefOptimizer
except Exception:  # mbrl (or one of its own dependencies) is not installed
    _RefAgent = _RefOptimizer = object


class Agent(_RefAgent):  # mbrl/planning/core.py:18-49
    def act(self, obs: np.ndarray, **_kwargs) -> np.ndarray:
        raise NotImplementedError

    def plan(self, obs: np.ndarray, **_kwargs) -> np.ndarray:
        return self.act(obs, **_kwargs)

    def reset(self):
        pass


class Optimizer(_RefOptimizer):  # mbrl/planning/trajectory_opt.py:21-40
    def __init__(self):
        pass

    def optimize(self, obj_fun, x0=None, **kwargs):
        raise NotImplementedError


class _FusedObjective:
    """Callable handed to the optimiser when the objective is ModelEnv.evaluate_action_sequences."""

    def __init__(self, model_env, obs: np.ndarray, num_particles: int):
        self.model_env, self.obs, self.num_particles = model_env, obs, num_particles

    def __call__(self, action_sequences: torch.Tensor) -> torch.Tensor:
        return self.model_env.evaluate_action_sequences(action_sequences, initial_state=self.obs,
                                                        num_particles=self.num_particles)


def _next_seed_offset(obj) -> int:
    obj._offset = getattr(obj, "_offset", 0) + 1
    return obj._offset


class CEMOptimizer(Optimizer):
    """Cross-entropy method, trajectory_opt.py:43-188."""

    def __init__(self, num_iterations: int, elite_ratio: float, population_size: int,
                 lower_bound: Sequence[Sequence[float]], upper_bound: Sequence[Sequence[float]], alpha: float,
                 device, return_mean_elites: bool = False, clipped_normal: bool = False):
        super().__init__()
        self.num_iterations = num_iterations
        self.elite_ratio = elite_ratio
        self.population_size = population_size
        self.elite_num = int(np.ceil(self.population_size * self.elite_ratio).astype(np.int32))
        self.device = torch.device(device)
        self.lower_bound = torch.tensor(lower_bound, device=self.device, dtype=torch.float32).contiguous()
        self.upper_bound = torch.tensor(upper_bound, device=self.device, dtype=torch.float32).contiguous()
        self.alpha = alpha
        self.return_mean_elites = return_mean_elites
        self._clipped_normal = clipped_normal
        self.lib = _lib.load()
        self._seed = int(torch.initial_seed()) & 0xFFFFFFFFFFFFFFFF
        self._ws = None
        self._plan_ws = None
        self.record_values = False
        self.last_values = None

    def _buffers(self, shape):
        dims = int(np.prod(shape))
        key = (self.population_size, dims)
        if self._ws is None or self._ws["key"] != key:
            dev = self.device
            nbytes = self.lib.b200pets_cem_update_workspace_bytes(self.population_size, dims, self.elite_num)
            self._ws = {
                "key": key,
                "mu": torch.empty(dims, device=dev), "disp": torch.empty(dims, device=dev),
                "best_val": torch.empty(1, device=dev), "best_sol": torch.empty(dims, device=dev),
                "pop": torch.empty((self.population_size,) + tuple(shape), device=dev),
                "ws": torch.empty(nbytes, dtype=torch.uint8, device=dev),
            }
        return self._ws

    def optimize(self, obj_fun: Callable[[torch.Tensor], torch.Tensor], x0: Optional[torch.Tensor] = None,
                 callback: Optional[Callable[[torch.Tensor, torch.Tensor, int], None]] = None, *,
                 _noise: Optional[torch.Tensor] = None, _model_noise=None, **kwargs) -> torch.Tensor:
        x0 = x0.to(self.device, torch.float32).contiguous()
        if isinstance(obj_fun, _FusedObjective) and callback is None:
            return self._optimize_fused(obj_fun, x0, _noise, _model_noise)
        shape = tuple(x0.shape)
        dims = int(np.prod(shape))
        b = self._buffers(shape)
        mu, disp, pop = b["mu"], b["disp"], b["pop"]
        mu.copy_(x0.reshape(-1))
        if self._clipped_normal:
            disp.fill_(1.0)
        else:
            disp.copy_((((self.upper_bound - self.lower_bound) ** 2) / 16).reshape(-1))
        b["best_val"].fill_(float("-inf"))
        base = _next_seed_offset(self) * 1024
        with torch.cuda.device(self.device):
            stream = _lib.stream_ptr()
            for i in range(self.num_iterations):
                z = None if _noise is None else _noise[i].to(self.device, torch.float32).contiguous()
                _lib.check(self.lib.b200pets_cem_sample(
                    self.population_size, dims, _lib.ptr(mu), _lib.ptr(disp), _lib.ptr(self.lower_bound),
                    _lib.ptr(self.upper_bound), _lib.ptr(z), self._seed, base + i, int(self._clipped_normal), _lib.ptr(pop),
                    stream), "cem_sample")
                values = obj_fun(pop)
                if callback is not None:
                    callback(pop, values, i)
                values = values.to(self.device, torch.float32).contiguous()
                _lib.check(self.lib.b200pets_cem_update(
                    self.population_size, dims, self.elite_num, float(self.alpha), 1, int(self._clipped_normal),
                    _lib.ptr(pop), _lib.ptr(values), _lib.ptr(mu), _lib.ptr(disp), _lib.ptr(b["best_val"]),
                    _lib.ptr(b["best_sol"]), None, None, _lib.ptr(b["ws"]), b["ws"].numel(), stream), "cem_update")
        out = mu if self.return_mean_elites else b["best_sol"]
        return out.view(shape).clone()

    def _optimize_fused(self, obj: _FusedObjective, x0, noise, model_noise) -> torch.Tensor:
        env = obj.model_env
        env._fresh()
        H, A = x0.shape
        prop = env._propagation()
        perms = eps = None
        if model_noise is not None:
            perms, eps = model_noise
        if perms is None and prop in ("random_model", "fixed_model") and (
                env.ts1 == "perms" or env._few_groups(self.population_size, obj.num_particles)):
            B = self.population_size * obj.num_particles
            n = H if prop == "random_model" else 1
            perms = torch.stack([torch.stack([torch.randperm(B, device=self.device) for _ in range(n)])
                                 for _ in range(self.num_iterations)])
        rcfg = _lib.RolloutCfg(self.population_size, H, obj.num_particles, _lib.PREC[env.precision], _lib.PROP[prop],
                               _lib.TS1_PERMS if perms is not None else _lib.TS1_TILE_SHUFFLE, env._seed,
                               env._next_offset())
        ccfg = _lib.CemCfg(self.num_iterations, self.elite_num, float(self.alpha), int(self.return_mean_elites),
                           int(self._clipped_normal))
        need = self.lib.b200pets_cem_plan_workspace_bytes(env.staged.handle, C.byref(rcfg), C.byref(ccfg))
        if self._plan_ws is None or self._plan_ws.numel() < need:
            self._plan_ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        obs0 = env._obs_to_device(obj.obs)
        sol = torch.empty(H * A, dtype=torch.float32, device=self.device)
        z = None if noise is None else noise.to(self.device, torch.float32).contiguous()
        if perms is not None:
            perms = perms.to(torch.int64).contiguous()
        self.last_values = None
        if self.record_values:  # per-iteration objective values of the fused plan (diagnostics / tests)
            self.last_values = torch.empty(self.num_iterations, self.population_size, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.b200pets_cem_plan(
                env.staged.handle, C.byref(rcfg), C.byref(ccfg), _lib.ptr(obs0), _lib.ptr(x0), _lib.ptr(self.lower_bound),
                _lib.ptr(self.upper_bound), _lib.ptr(z), _lib.ptr(eps), _lib.ptr(perms), _lib.ptr(sol),
                _lib.ptr(self.last_values), _lib.ptr(self._plan_ws), self._plan_ws.numel(), _lib.stream_ptr()), "cem_plan")
        return sol.view(H, A)


class ICEMOptimizer(Optimizer):
    """Improved CEM, trajectory_opt.py:314-487."""

    def __init__(self, num_iterations: int, elite_ratio: float, population_size: int, population_decay_factor: float,
                 colored_noise_exponent: float, lower_bound: Sequence[Sequence[float]],
                 upper_bound: Sequence[Sequence[float]], keep_elite_frac: float, alpha: float, device,
                 return_mean_elites: bool = False, population_size_module: Optional[int] = None):
        super().__init__()
        self.num_iterations = num_iterations
        self.elite_ratio = elite_ratio
        self.population_size = population_size
        self.population_decay_factor = population_decay_factor
        self.elite_num = int(np.ceil(self.population_size * self.elite_ratio).astype(np.int32))
        self.colored_noise_exponent = colored_noise_exponent
        self.device = torch.device(device)
        self.lower_bound = torch.tensor(lower_bound, device=self.device, dtype=torch.float32).contiguous()
        self.upper_bound = torch.tensor(upper_bound, device=self.device, dtype=torch.float32).contiguous()
        self.initial_var = (((self.upper_bound - self.lower_bound) ** 2) / 16).contiguous()
        self.keep_elite_frac = keep_elite_frac
        self.keep_elite_size = int(np.ceil(keep_elite_frac * self.elite_num).astype(np.int32))
        self.elite: Optional[torch.Tensor] = None
        self.alpha = alpha
        self.return_mean_elites = return_mean_elites
        self.population_size_module = population_size_module
        if self.population_size_module:
            self.keep_elite_size = self._round_up_to_module(self.keep_elite_size, self.population_size_module)
        self.lib = _lib.load()
        self._seed = int(torch.initial_seed()) & 0xFFFFFFFFFFFFFFFF

    @staticmethod
    def _round_up_to_module(value: int, module: int) -> int:
        return value if value % module == 0 else value + (module - value % module)

    def population_sizes(self) -> List[int]:
        sizes = []
        for i in range(self.num_iterations):
            n = int(np.ceil(np.max((self.population_size * self.population_decay_factor ** -i, 2 * self.elite_num))).astype(np.int32))
            if self.population_size_module:
                n = self._round_up_to_module(n, self.population_size_module)
            sizes.append(n)
        return sizes

    def optimize(self, obj_fun, x0: Optional[torch.Tensor] = None, callback=None, *, _noise=None, **kwargs) -> torch.Tensor:
        x0 = x0.to(self.device, torch.float32).contiguous()
        H, A = x0.shape
        dims = H * A
        dev = self.device
        mu = x0.reshape(-1).clone()
        var = self.initial_var.reshape(-1).clone()
        best_val = torch.full((1,), float("-inf"), device=dev)
        best_sol = torch.empty(dims, device=dev)
        base = _next_seed_offset(self) * 1024
        sizes = self.population_sizes()
        elites_new = torch.empty(self.elite_num, H, A, device=dev)
        with torch.cuda.device(dev):
            stream = _lib.stream_ptr()
            for i in range(self.num_iterations):
                n = sizes[i]
                extra = 0
                # the reference indexes `randperm(elite_num)[:keep_elite_size]`: when population_size_module rounds
                # keep_elite_size above elite_num only elite_num rows exist (trajectory_opt.py:443-447)
                keep = min(self.keep_elite_size, self.elite_num)
                if self.elite is not None:
                    extra = 1 if (i == self.num_iterations - 1 and i != 0) else keep
                pop = torch.empty(n + extra, H, A, device=dev)
                nz = _noise[i] if _noise is not None else {}
                sr = nz.get("sr")
                si = nz.get("si")
                _lib.check(self.lib.b200pets_icem_sample(
                    n, H, A, float(self.colored_noise_exponent), _lib.ptr(mu), _lib.ptr(var), _lib.ptr(self.lower_bound),
                    _lib.ptr(self.upper_bound), _lib.ptr(sr), _lib.ptr(si), self._seed, base + i, _lib.ptr(pop), stream),
                    "icem_sample")
                if self.elite is not None:
                    if i == self.num_iterations - 1 and i != 0:
                        pop[n].copy_(mu.view(H, A))  # trajectory_opt.py:462-463
                    else:
                        idx = nz.get("keep_perm")
                        if idx is None:
                            idx = torch.randperm(self.elite_num, device=dev)
                        idx = idx[:keep].to(torch.int64).contiguous()
                        _lib.check(self.lib.b200pets_icem_append_elites(
                            keep, H, A, _lib.ptr(self.elite), _lib.ptr(idx), int(i == 0), _lib.ptr(mu),
                            _lib.ptr(var), _lib.ptr(nz.get("end_eps")), self._seed, base + i, _lib.ptr(pop[n:]), stream),
                            "icem_append_elites")
                values = obj_fun(pop)
                if callback is not None:
                    callback(pop, values, i)
                values = values.to(dev, torch.float32).contiguous()
                nbytes = self.lib.b200pets_cem_update_workspace_bytes(pop.shape[0], dims, self.elite_num)
                ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
                _lib.check(self.lib.b200pets_cem_update(
                    pop.shape[0], dims, self.elite_num, float(self.alpha), 0, 0, _lib.ptr(pop), _lib.ptr(values), _lib.ptr(mu),
                    _lib.ptr(var), _lib.ptr(best_val), _lib.ptr(best_sol), None, _lib.ptr(elites_new), _lib.ptr(ws), nbytes,
                    stream), "cem_update")
                self.elite = elites_new.clone()
        out = mu if self.return_mean_elites else best_sol
        return out.view(H, A).clone()



class MPPIOptimizer(Optimizer):
    """Model Predictive Path Integral optimiser, trajectory_opt.py:191-311 (constructor kwargs of mppi.yaml)."""

    def __init__(self, num_iterations: int, population_size: int, gamma: float, sigma: float, beta: float,
                 lower_bound: Sequence[Sequence[float]], upper_bound: Sequence[Sequence[float]], device):
        super().__init__()
        self.planning_horizon = len(lower_bound)
        self.population_size = population_size
        self.action_dimension = len(lower_bound[0])
        self.device = torch.device(device)
        self.mean = torch.zeros((self.planning_horizon, self.action_dimension), device=self.device, dtype=torch.float32)
        self.lower_bound = torch.tensor(lower_bound, device=self.device, dtype=torch.float32).contiguous()
        self.upper_bound = torch.tensor(upper_bound, device=self.device, dtype=torch.float32).contiguous()
        self.var = sigma ** 2 * torch.ones_like(self.lower_bound)  # kept for API parity; unused by the reference's sampler
        self.beta = beta
        self.gamma = gamma
        self.refinements = num_iterations
        self.lib = _lib.load()
        self._seed = int(torch.initial_seed()) & 0xFFFFFFFFFFFFFFFF

    def optimize(self, obj_fun, x0: Optional[torch.Tensor] = None, callback=None, *, _noise=None, **kwargs) -> torch.Tensor:
        H, A, N = self.planning_horizon, self.action_dimension, self.population_size
        dev = self.device
        # `past_action = self.mean[0]` is a view in the reference and the in-place shift below rewrites it: the value
        # used by every refinement is the *shifted* first row (old mean[1]); restated explicitly (lines 250-251).
        self.mean[:-1] = self.mean[1:].clone()
        past_action = self.mean[0].clone()
        pop = torch.empty(N, H, A, device=dev)
        nbytes = self.lib.b200pets_mppi_update_workspace_bytes(N, H * A)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        base = _next_seed_offset(self) * 1024
        with torch.cuda.device(dev):
            stream = _lib.stream_ptr()
            for k in range(self.refinements):
                z = None if _noise is None else _noise[k].to(dev, torch.float32).contiguous()
                _lib.check(self.lib.b200pets_mppi_sample(N, H, A, float(self.beta), _lib.ptr(self.mean), _lib.ptr(past_action),
                                                         _lib.ptr(self.lower_bound), _lib.ptr(self.upper_bound), _lib.ptr(z),
                                                         self._seed, base + k, _lib.ptr(pop), stream), "mppi_sample")
                values = obj_fun(pop).to(dev, torch.float32).contiguous()
                new_mean = torch.empty(H, A, device=dev)
                _lib.check(self.lib.b200pets_mppi_update(N, H * A, float(self.gamma), _lib.ptr(pop), _lib.ptr(values),
                                                         _lib.ptr(new_mean), _lib.ptr(ws), nbytes, stream), "mppi_update")
                if callback is not None:
                    callback(pop, values, k)
                self.mean = new_mean
        return self.mean.clone()


_KNOWN_TARGETS = {"CEMOptimizer": CEMOptimizer, "ICEMOptimizer": ICEMOptimizer, "MPPIOptimizer": MPPIOptimizer}


def _cfg_to_dict(cfg) -> dict:
    return {k: cfg[k] for k in cfg.keys()}


def _instantiate(cfg, **overrides):
    """Minimal stand-in for hydra.utils.instantiate: ``_target_`` names ending in a class we provide map to
    ours (so ``mbrl.planning.CEMOptimizer`` in the shipped YAMLs selects this implementation)."""
    d = _cfg_to_dict(cfg)
    d.update(overrides)
    target = d.pop("_target_")
    d.pop("_recursive_", None)
    name = target.rsplit(".", 1)[-1]
    if name in _KNOWN_TARGETS:
        cls = _KNOWN_TARGETS[name]
    else:
        mod, _, attr = target.rpartition(".")
        cls = getattr(importlib.import_module(mod), attr)
    return cls(**d)


class TrajectoryOptimizer:
    """trajectory_opt.py:490-572."""

    def __init__(self, optimizer_cfg, action_lb: np.ndarray, action_ub: np.ndarray, planning_horizon: int,
                 replan_freq: int = 1, keep_last_solution: bool = True):
        lower = np.tile(action_lb, (planning_horizon, 1)).tolist()
        upper = np.tile(action_ub, (planning_horizon, 1)).tolist()
        self.optimizer: Optimizer = _instantiate(optimizer_cfg, lower_bound=lower, upper_bound=upper)
        device = optimizer_cfg["device"]
        self.initial_solution = ((torch.tensor(action_lb) + torch.tensor(action_ub)) / 2).float().to(device)
        self.initial_solution = self.initial_solution.repeat((planning_horizon, 1)).contiguous()
        self.previous_solution = self.initial_solution.clone()
        self.replan_freq = replan_freq
        self.keep_last_solution = keep_last_solution
        self.horizon = planning_horizon
        self.lib = _lib.load()
        self._pin = None  # pinned staging buffer for the plan, allocated on first use

    def optimize(self, trajectory_eval_fn, callback: Optional[Callable] = None) -> np.ndarray:
        best = self.optimizer.optimize(trajectory_eval_fn, x0=self.previous_solution, callback=callback).contiguous()
        if self.keep_last_solution:
            H, A = best.shape
            with torch.cuda.device(best.device):
                _lib.check(self.lib.b200pets_shift_solution(H, A, self.replan_freq, _lib.ptr(best),
                                                            _lib.ptr(self.initial_solution), _lib.ptr(self.previous_solution),
                                                            _lib.stream_ptr()), "shift_solution")
        if self._pin is None or self._pin.shape != best.shape:
            self._pin = torch.empty(best.shape, dtype=torch.float32).pin_memory()
        self._pin.copy_(best, non_blocking=True)
        torch.cuda.current_stream().synchronize()  # the one device->host boundary (trajectory_opt.py:568)
        return self._pin.numpy().copy()

    def reset(self):
        self.previous_solution = self.initial_solution.clone()


class TrajectoryOptimizerAgent(Agent):
    """trajectory_opt.py:575-716."""

    def __init__(self, optimizer_cfg, action_lb: Sequence[float], action_ub: Sequence[float], planning_horizon: int = 1,
                 replan_freq: int = 1, verbose: bool = False, keep_last_solution: bool = True):
        self.optimizer = TrajectoryOptimizer(optimizer_cfg, np.array(action_lb), np.array(action_ub),
                                             planning_horizon=planning_horizon, replan_freq=replan_freq,
                                             keep_last_solution=keep_last_solution)
        self.optimizer_args = {"optimizer_cfg": optimizer_cfg, "action_lb": np.array(action_lb),
                               "action_ub": np.array(action_ub)}
        self.trajectory_eval_fn = None
        self.actions_to_use: List[np.ndarray] = []
        self.replan_freq = replan_freq
        self.verbose = verbose
        self._fused_env = None
        self._fused_particles = 1

    def set_trajectory_eval_fn(self, trajectory_eval_fn):
        self.trajectory_eval_fn = trajectory_eval_fn
        self._fused_env = None

    def set_model_env(self, model_env, num_particles: int):
        """Bind the objective to ``model_env.evaluate_action_sequences`` (enables the fused CEM plan)."""
        self._fused_env, self._fused_particles = model_env, num_particles
        self.trajectory_eval_fn = lambda obs, seqs: model_env.evaluate_action_sequences(
            seqs, initial_state=obs, num_particles=num_particles)

    def reset(self, planning_horizon: Optional[int] = None):
        if planning_horizon:
            self.optimizer = TrajectoryOptimizer(self.optimizer_args["optimizer_cfg"], self.optimizer_args["action_lb"],
                                                 self.optimizer_args["action_ub"], planning_horizon=planning_horizon,
                                                 replan_freq=self.replan_freq)
        self.optimizer.reset()

    def _objective(self, obs):
        if self._fused_env is not None:
            return _FusedObjective(self._fused_env, np.asarray(obs), self._fused_particles)

        def trajectory_eval_fn(action_sequences):
            return self.trajectory_eval_fn(obs, action_sequences)

        return trajectory_eval_fn

    def act(self, obs: np.ndarray, optimizer_callback: Optional[Callable] = None, **_kwargs) -> np.ndarray:
        if self.trajectory_eval_fn is None:
            raise RuntimeError("Please call `set_trajectory_eval_fn()` before using TrajectoryOptimizerAgent")
        plan_time = 0.0
        if not self.actions_to_use:
            start_time = time.time()
            plan = self.optimizer.optimize(self._objective(obs), callback=optimizer_callback)
            plan_time = time.time() - start_time
            self.actions_to_use.extend([a for a in plan[: self.replan_freq]])
        action = self.actions_to_use.pop(0)
        if self.verbose:
            print(f"Planning time: {plan_time:.3f}")
        return action

    def plan(self, obs: np.ndarray, **_kwargs) -> np.ndarray:
        if self.trajectory_eval_fn is None:
            raise RuntimeError("Please call `set_trajectory_eval_fn()` before using TrajectoryOptimizerAgent")
        return self.optimizer.optimize(self._objective(obs))


_KNOWN_TARGETS["TrajectoryOptimizerAgent"] = TrajectoryOptimizerAgent


def complete_agent_cfg(env, agent_cfg):
    """Fill action bounds from the (model) environment, mbrl/planning/core.py:71-123 for the keys this agent reads."""
    lb = np.asarray(env.action_space.low).tolist()
    ub = np.asarray(env.action_space.high).tolist()
    for key, val in (("action_lb", lb), ("action_ub", ub)):
        if key not in agent_cfg.keys() or agent_cfg[key] in (None, "???"):
            agent_cfg[key] = val
    return agent_cfg


def create_trajectory_optim_agent_for_model(model_env, agent_cfg, num_particles: int = 1) -> TrajectoryOptimizerAgent:
    """trajectory_opt.py:719-749."""
    complete_agent_cfg(model_env, agent_cfg)
    agent = _instantiate(agent_cfg)
    agent.set_model_env(model_env, num_particles)
    return agent


def rollout_model_env(model_env, initial_obs: np.ndarray, plan: Optional[np.ndarray] = None, agent: Optional[Agent] = None,
                      num_samples: int = 1) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Execute ``plan`` (or ``agent.plan``'s, which takes precedence) open loop on the model, ``num_samples`` copies of
    ``initial_obs`` side by side, predictions taken with ``sample=False`` (mbrl/util/common.py:416-454).

    Returns ``(observations [len+1, num_samples, D], rewards [len, num_samples, 1], plan)``.  One ``b200pets_step``
    launch per action; the per-step numpy hand-over is the reference's interface for this diagnostic.
    """
    if agent:
        plan = agent.plan(initial_obs[None, :])
    start = np.tile(initial_obs, (num_samples, 1))
    model_state = model_env.reset(start, return_as_np=True)
    observations, rewards = [start], []
    for action in plan:
        next_obs, reward, _, model_state = model_env.step(np.tile(action, (num_samples, 1)), model_state, sample=False)
        observations.append(next_obs)
        rewards.append(reward)
    return np.stack(observations), np.stack(rewards), plan
