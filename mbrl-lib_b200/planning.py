"""Trajectory optimisers and the MPC agent with the reference's plugin interface
(mbrl/planning/core.py:18-49, mbrl/planning/trajectory_opt.py) over the CUDA CEM / rollout kernels.

* ``CEMOptimizer`` / ``ICEMOptimizer``: same constructor kwargs as the YAML configs pass
  (conf/action_optimizer/cem.yaml, icem.yaml), same ``optimize(obj_fun, x0, callback)`` protocol.  With an
  opaque ``obj_fun`` each iteration is  sample kernel -> obj_fun(population) -> select/refit kernel  and no
  host synchronisation of ours (the reference syncs on ``.item()`` / ``best_values[0] > best_value``).
* When ``obj_fun`` is the ``evaluate_action_sequences`` closure built by
  :func:`create_trajectory_optim_agent_for_model`, ``CEMOptimizer`` runs the whole optimisation as one
  C call (``b200pets_cem_plan_batch``, one observation being the batch of one): every iteration's sample -> rollout ->
  refit is enqueued back to back.
  With a reward or termination callable the kernels do not know it runs the per-iteration loop instead, the
  objective applying the callable to windows of the rollout (``ModelEnv.evaluate_action_sequences``).
* Over PlaNet's latent model (:class:`mbrl_lib_b200.latent.LatentModelEnv`) the fused plan is one
  ``b200pets_latent_cem_plan_batch`` call; iCEM and MPPI evaluate through its ``evaluate_action_sequences``.  For K
  observations the environment's K posteriors plan as one ``b200pets_latent_cem_plan_batch`` call, and MPPI plans
  entry k from posterior k.
* ``ICEMOptimizer`` over that closure (no callback, no callable the kernels do not know) runs the whole optimisation as
  one C call too (``b200pets_icem_plan``), with the per-iteration loop's draws, counters, elites and result.
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

    def optimize_batch(self, obj_funs, x0=None, callback=None, **kwargs):
        """One plan per objective of ``obj_funs`` from the warm starts ``x0 [K, H, A]``.  CEMOptimizer keeps no state
        between calls besides the warm start, and MPPIOptimizer keeps one mean per problem; an optimiser with other state
        (iCEM's kept elites) would have to split it per problem, which is not implemented."""
        raise NotImplementedError(f"{type(self).__name__} does not plan for a batch of observations; "
                                  "CEMOptimizer and MPPIOptimizer are the optimisers that support act_batch")


class _FusedObjective:
    """Callable handed to the optimiser when the objective is ModelEnv.evaluate_action_sequences."""

    def __init__(self, model_env, obs: np.ndarray, num_particles: int):
        self.model_env, self.obs, self.num_particles = model_env, obs, num_particles

    def __call__(self, action_sequences: torch.Tensor) -> torch.Tensor:
        return self.model_env.evaluate_action_sequences(action_sequences, initial_state=self.obs,
                                                        num_particles=self.num_particles)


class _FusedBatchObjective:
    """The objectives of K observations when they all are ModelEnv.evaluate_action_sequences of one environment."""

    def __init__(self, model_env, obs: np.ndarray, num_particles: int):
        self.model_env, self.obs, self.num_particles = model_env, obs, num_particles

    def entries(self) -> List[Callable[[torch.Tensor], torch.Tensor]]:
        env, P = self.model_env, self.num_particles
        if getattr(env, "is_latent", False):  # entry k evaluates from the environment's posterior k
            return [lambda seqs, k=k, o=o: env.evaluate_action_sequences(seqs, o, P, _entry=k) for k, o in enumerate(self.obs)]
        return [_FusedObjective(env, o, P) for o in self.obs]


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
        # the fused plan runs every iteration inside one C call, which cannot call back into Python: with a reward or
        # termination callable the kernels do not know, the loop below evaluates through the objective instead
        if isinstance(obj_fun, _FusedObjective) and callback is None and not obj_fun.model_env.has_external_callables():
            # the plan of one observation is the batch of one
            noise = None if _noise is None else _noise[None]
            model_noise = None if _model_noise is None else tuple(None if t is None else t[None] for t in _model_noise)
            sol = self._optimize_fused(obj_fun, x0[None], noise, model_noise)
            if self.last_values is not None:
                self.last_values = self.last_values[0]
            return sol[0]
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

    def optimize_batch(self, obj_funs, x0: torch.Tensor, callback=None, *, _noise=None, _model_noise=None,
                       **kwargs) -> torch.Tensor:
        """K independent plans from the warm starts ``x0 [K, H, A]``; returns ``[K, H, A]``.  ``obj_funs`` is a
        :class:`_FusedBatchObjective` (the model's objective for K observations) or a list of K objectives.  The model's
        objective with no callback and no reward / termination callable runs as one batched device-resident plan
        (``b200pets_cem_plan_batch``); anything else runs :meth:`optimize` once per entry, each from its own warm start."""
        x0 = x0.to(self.device, torch.float32).contiguous()
        if isinstance(obj_funs, _FusedBatchObjective):
            if callback is None and not obj_funs.model_env.has_external_callables():
                return self._optimize_fused(obj_funs, x0, _noise, _model_noise)
            obj_funs = obj_funs.entries()
        if len(obj_funs) != x0.shape[0]:
            raise ValueError(f"{len(obj_funs)} objectives for {x0.shape[0]} warm starts")
        return torch.stack([self.optimize(f, x0=x0[k], callback=callback) for k, f in enumerate(obj_funs)])

    def _cem_cfg(self) -> _lib.CemCfg:
        """This optimizer's settings as the fused plans' ``b200pets_cem_cfg``."""
        return _lib.CemCfg(self.num_iterations, self.elite_num, float(self.alpha), int(self.return_mean_elites),
                           int(self._clipped_normal))

    def _plan_perms(self, env, prop: str, horizon: int, num_particles: int) -> Optional[torch.Tensor]:
        """The permutations one fused plan draws, ``[iterations, horizon or 1, N * P]`` (None: members drawn in kernel);
        over a BasicEnsemble the per-row member indices of each iteration's evaluation."""
        if prop != "expectation" and env._member_rows():
            return torch.stack([env._eval_perms(prop, self.population_size, horizon, num_particles)
                                for _ in range(self.num_iterations)])
        if prop not in ("random_model", "fixed_model") or not (
                env.ts1 == "perms" or env._few_groups(self.population_size, num_particles)):
            return None
        B = self.population_size * num_particles
        n = horizon if prop == "random_model" else 1
        return torch.stack([torch.stack([torch.randperm(B, device=self.device) for _ in range(n)])
                            for _ in range(self.num_iterations)])

    def _optimize_fused(self, obj, x0, noise, model_noise) -> torch.Tensor:
        """One device-resident plan (``b200pets_cem_plan_batch``, or the latent model's) for the K observations of a
        :class:`_FusedBatchObjective`, or for the one observation of a :class:`_FusedObjective` as K = 1.  ``x0 [K, H, A]``;
        ``noise [K, it, N, H, A]`` and ``model_noise`` (perms, eps), each ``[K, ...]``, replace the draws.  Returns
        ``[K, H, A]``; with ``record_values`` ``last_values`` is ``[K, it, N]``."""
        env = obj.model_env
        batch = isinstance(obj, _FusedBatchObjective)
        if getattr(env, "is_latent", False):  # b200pets_latent_cem_plan_batch, model noise = eps only
            return env.cem_plan(self, x0, obj.num_particles, noise, None if model_noise is None else model_noise[1],
                                batch=batch)
        env._fresh()
        K, H, A = x0.shape
        obs = np.asarray(obj.obs) if batch else np.asarray(obj.obs)[None]
        if obs.ndim != 2 or obs.shape[0] != K:
            raise ValueError(f"observations must be [K={K}, obs_dim], got {tuple(obs.shape)}")
        prop = env._propagation()
        perms = eps = None
        if model_noise is not None:
            perms, eps = model_noise
        if perms is None:
            per = [self._plan_perms(env, prop, H, obj.num_particles) for _ in range(K)]
            perms = None if not per or per[0] is None else torch.stack(per)
        # problem k plans with counter value first + k: the one its own single plan would take k calls later
        rcfg = _lib.RolloutCfg(self.population_size, H, obj.num_particles, _lib.PREC[env.precision_for(prop)], _lib.PROP[prop],
                               _lib.TS1_PERMS if perms is not None else _lib.TS1_TILE_SHUFFLE, env._seed,
                               env._next_offset())
        env._offset += K - 1
        ccfg = self._cem_cfg()
        need = self.lib.b200pets_cem_plan_batch_workspace_bytes(env.staged.handle, C.byref(rcfg), C.byref(ccfg), K)
        if self._plan_ws is None or self._plan_ws.numel() < need:
            self._plan_ws = torch.empty(max(need, 1), dtype=torch.uint8, device=self.device)
        obs0 = env._obs_to_device(obs)
        sol = torch.empty(K, H * A, dtype=torch.float32, device=self.device)
        z = None if noise is None else noise.to(self.device, torch.float32).contiguous()
        if perms is not None:
            perms = perms.to(torch.int64).contiguous()
        self.last_values = None
        if self.record_values:  # per-iteration objective values of the fused plan (diagnostics / tests)
            self.last_values = torch.empty(K, self.num_iterations, self.population_size, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.b200pets_cem_plan_batch(
                env.staged.handle, C.byref(rcfg), C.byref(ccfg), K, _lib.ptr(obs0), _lib.ptr(x0), _lib.ptr(self.lower_bound),
                _lib.ptr(self.upper_bound), _lib.ptr(z), _lib.ptr(eps), _lib.ptr(perms), _lib.ptr(sol),
                _lib.ptr(self.last_values), _lib.ptr(self._plan_ws), self._plan_ws.numel(), _lib.stream_ptr()),
                "cem_plan_batch")
        return sol.view(K, H, A)


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
        self._plan_ws = None
        self.record_values = False
        self.last_values: Optional[List[torch.Tensor]] = None

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
        """trajectory_opt.py:391-487.  Over the model's objective (a non-latent ModelEnv without reward / termination
        callables), with no callback and no injected noise, the whole optimisation is one device-resident call
        (``b200pets_icem_plan``) that leaves the result, the elites, the counters and the torch generator exactly as the
        per-iteration loop below would.  With ``record_values`` ``last_values`` holds each iteration's values."""
        H, A = x0.shape
        if H < 2:  # b200pets_icem_sample refuses it too; checked here before anything is launched
            raise ValueError(f"ICEMOptimizer needs a planning horizon of at least 2, got {H}: coloured noise over a "
                             "one-step series has no frequency above DC to normalise by")
        x0 = x0.to(self.device, torch.float32).contiguous()
        # the fused plan cannot call back into Python: callbacks, injected noise and callables keep the loop
        if (isinstance(obj_fun, _FusedObjective) and callback is None and _noise is None and self.num_iterations >= 1
                and not getattr(obj_fun.model_env, "is_latent", False) and not obj_fun.model_env.has_external_callables()):
            return self._optimize_fused(obj_fun, x0)
        self.last_values = [] if self.record_values else None
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
                if self.last_values is not None:
                    self.last_values.append(values)
        out = mu if self.return_mean_elites else best_sol
        return out.view(H, A).clone()

    def _fused_draws(self, env, prop: str, horizon: int, num_particles: int, sizes: Optional[List[int]] = None):
        """The torch generator draws of one :meth:`optimize` over the model, in the loop's order: per iteration the
        permutation of the kept elites (whenever elites are kept) and then that evaluation's permutations
        (``ModelEnv._eval_perms``).  Returns each iteration's evaluated population, the kept elites' indices
        ``[iterations, keep]`` (None when no iteration keeps any) and each evaluation's permutations (None: members
        drawn in the kernel)."""
        keep = min(self.keep_elite_size, self.elite_num)
        last = self.num_iterations - 1
        rows, index, perms = [], [], []
        for i, n in enumerate(self.population_sizes() if sizes is None else sizes):
            extra, idx = 0, None
            if self.elite is not None or i > 0:
                if i == last and i != 0:
                    extra = 1  # the current mean
                else:
                    extra = keep
                    idx = torch.randperm(self.elite_num, device=self.device)[:keep]
            rows.append(n + extra)
            index.append(idx)
            perms.append(env._eval_perms(prop, n + extra, horizon, num_particles))
        drawn = [t for t in index if t is not None]
        if keep == 0 or not drawn:
            return rows, None, perms
        # the rows of iterations that keep no elites are not read
        return rows, torch.stack([drawn[0] if t is None else t for t in index]).to(torch.int64).contiguous(), perms

    def _optimize_fused(self, obj: _FusedObjective, x0: torch.Tensor) -> torch.Tensor:
        env = obj.model_env
        obs = np.asarray(obj.obs)
        if obs.ndim != 1:
            raise NotImplementedError("pixel observations are outside the GaussianMLP hot path")
        env._fresh()
        H, A = x0.shape
        P, iters = obj.num_particles, self.num_iterations
        prop = env._propagation()
        sizes = self.population_sizes()
        rows, keep_index, perms = self._fused_draws(env, prop, H, P, sizes)
        # iteration i evaluates with the environment's counter first + i, as the loop's i-th evaluation does
        rcfg = _lib.RolloutCfg(0, H, P, _lib.PREC[env.precision_for(prop)], _lib.PROP[prop],
                               _lib.TS1_PERMS if env.ts1 == "perms" else _lib.TS1_TILE_SHUFFLE, env._seed, env._offset + 1)
        env._offset += iters
        icfg = _lib.IcemCfg(iters, self.elite_num, min(self.keep_elite_size, self.elite_num), float(self.alpha),
                            float(self.colored_noise_exponent), int(self.return_mean_elites), self._seed,
                            _next_seed_offset(self))
        sizes = (C.c_int32 * iters)(*sizes)
        need = self.lib.b200pets_icem_plan_workspace_bytes(env.staged.handle, C.byref(rcfg), C.byref(icfg), sizes)
        if self._plan_ws is None or self._plan_ws.numel() < need:
            self._plan_ws = torch.empty(max(need, 1), dtype=torch.uint8, device=self.device)
        perms = [None if p is None else p.to(torch.int64).contiguous() for p in perms]
        perm_ptrs = (C.c_void_p * iters)(*[None if p is None else p.data_ptr() for p in perms])
        obs0 = env._obs_to_device(obs)
        sol = torch.empty(H, A, device=self.device)
        elite = torch.empty(self.elite_num, H, A, device=self.device)
        values = torch.empty(sum(rows), device=self.device) if self.record_values else None
        with torch.cuda.device(self.device):
            _lib.check(self.lib.b200pets_icem_plan(
                env.staged.handle, C.byref(rcfg), C.byref(icfg), sizes, _lib.ptr(obs0), _lib.ptr(x0), _lib.ptr(self.lower_bound),
                _lib.ptr(self.upper_bound), _lib.ptr(self.elite), _lib.ptr(keep_index), perm_ptrs, _lib.ptr(sol),
                _lib.ptr(elite), _lib.ptr(values), _lib.ptr(self._plan_ws), self._plan_ws.numel(), _lib.stream_ptr()),
                "icem_plan")
        self.elite = elite
        self.last_values = None if values is None else list(values.split(rows))
        return sol



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
        self.batch_mean: Optional[torch.Tensor] = None  # [K, H, A] carried means of optimize_batch
        self._plan_batch_ws = None
        self.record_values = False
        self.last_values = None

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

    def optimize_batch(self, obj_funs, x0: Optional[torch.Tensor] = None, callback=None, *, _noise=None, _model_noise=None,
                       **kwargs) -> torch.Tensor:
        """K independent plans, one per objective of ``obj_funs`` (a :class:`_FusedBatchObjective` or a list of K
        objectives); returns ``[K, H, A]``.  Problem k plans as :meth:`optimize` would from its own carried mean
        ``batch_mean[k]``.  The batch's means start at zeros, as ``mean`` does, and are re-created when K changes;
        :meth:`optimize` / ``mean`` and the batch never touch each other's state.  ``x0`` is ignored, as in
        :meth:`optimize`.  The model's objective with no callback and no reward / termination callable runs as one
        device-resident plan (``b200pets_mppi_plan_batch``) in which problem k takes the counter values of the k-th of K
        consecutive single plans; anything else runs :meth:`optimize` once per entry, in order.  With ``record_values``
        the batched plan leaves every refinement's values in ``last_values [K, R, N]``."""
        K = len(obj_funs.obs) if isinstance(obj_funs, _FusedBatchObjective) else len(obj_funs)
        H, A = self.planning_horizon, self.action_dimension
        if self.batch_mean is None or self.batch_mean.shape[0] != K:
            self.batch_mean = torch.zeros((K, H, A), device=self.device, dtype=torch.float32)
        self.last_values = None
        if isinstance(obj_funs, _FusedBatchObjective):
            env = obj_funs.model_env
            if callback is None and not env.has_external_callables() and not getattr(env, "is_latent", False):
                return self._optimize_fused_batch(obj_funs, _noise, _model_noise)
            obj_funs = obj_funs.entries()
        saved = self.mean
        try:
            for k, f in enumerate(obj_funs):
                self.mean = self.batch_mean[k].clone()
                self.batch_mean[k] = self.optimize(f, callback=callback, _noise=None if _noise is None else _noise[k])
        finally:
            self.mean = saved
        return self.batch_mean.clone()

    def _optimize_fused_batch(self, obj: _FusedBatchObjective, noise, model_noise) -> torch.Tensor:
        env = obj.model_env
        env._fresh()
        self.batch_mean = self.batch_mean.to(self.device, torch.float32).contiguous()
        K, H, A = self.batch_mean.shape
        N, P, R = self.population_size, obj.num_particles, self.refinements
        obs = np.asarray(obj.obs)
        if obs.ndim != 2 or obs.shape[0] != K:
            raise ValueError(f"observations must be [K={K}, obs_dim], got {tuple(obs.shape)}")
        prop = env._propagation()
        perms = eps = None
        if model_noise is not None:
            perms, eps = model_noise
        if perms is None and R > 0:
            # the draws of K consecutive single plans, in their order: problem-major, then refinement
            per = [env._eval_perms(prop, N, H, P) for _ in range(K * R)]
            if per[0] is not None:
                perms = torch.stack(per).view(K, R, *per[0].shape)
        # problem k takes optimiser counter first + k and environment counters env_first + k * R + r
        first = _next_seed_offset(self)
        self._offset += K - 1
        rcfg = _lib.RolloutCfg(N, H, P, _lib.PREC[env.precision_for(prop)], _lib.PROP[prop],
                               _lib.TS1_PERMS if perms is not None else _lib.TS1_TILE_SHUFFLE, env._seed, env._offset + 1)
        env._offset += K * R
        mcfg = _lib.MppiCfg(R, float(self.gamma), float(self.beta), self._seed, first)
        need = self.lib.b200pets_mppi_plan_batch_workspace_bytes(env.staged.handle, C.byref(rcfg), C.byref(mcfg), K)
        if self._plan_batch_ws is None or self._plan_batch_ws.numel() < need:
            self._plan_batch_ws = torch.empty(max(need, 1), dtype=torch.uint8, device=self.device)
        obs0 = torch.from_numpy(np.ascontiguousarray(obs, dtype=np.float32)).to(self.device)
        z = None if noise is None else noise.to(self.device, torch.float32).contiguous()
        if eps is not None:
            eps = eps.to(self.device, torch.float32).contiguous()
        if perms is not None:
            perms = perms.to(self.device, torch.int64).contiguous()
        if self.record_values:
            self.last_values = torch.empty(K, R, N, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.b200pets_mppi_plan_batch(
                env.staged.handle, C.byref(rcfg), C.byref(mcfg), K, _lib.ptr(obs0), _lib.ptr(self.batch_mean),
                _lib.ptr(self.lower_bound), _lib.ptr(self.upper_bound), _lib.ptr(z), _lib.ptr(eps), _lib.ptr(perms),
                _lib.ptr(self.last_values), _lib.ptr(self._plan_batch_ws), self._plan_batch_ws.numel(), _lib.stream_ptr()),
                "mppi_plan_batch")
        return self.batch_mean.clone()


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
        self.previous_solutions: Optional[torch.Tensor] = None  # [K, H, A] warm starts of optimize_batch
        self._pin_batch = None

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

    def optimize_batch(self, trajectory_eval_fns, num_problems: int, callback: Optional[Callable] = None) -> np.ndarray:
        """:meth:`optimize` for K observations at once: K plans from K warm starts (kept in ``previous_solutions``,
        created on the first call and re-created when K changes, shifted after each plan with the rule of
        :meth:`optimize`).  Returns the plans ``[K, H, A]`` through one device-to-host copy."""
        K = num_problems
        if self.previous_solutions is None or self.previous_solutions.shape[0] != K:
            self.previous_solutions = self.initial_solution.repeat(K, 1, 1).contiguous()
        best = self.optimizer.optimize_batch(trajectory_eval_fns, x0=self.previous_solutions, callback=callback).contiguous()
        if self.keep_last_solution:
            _, H, A = best.shape
            with torch.cuda.device(best.device):
                for k in range(K):
                    _lib.check(self.lib.b200pets_shift_solution(H, A, self.replan_freq, _lib.ptr(best[k]),
                                                                _lib.ptr(self.initial_solution),
                                                                _lib.ptr(self.previous_solutions[k]), _lib.stream_ptr()),
                               "shift_solution")
        if self._pin_batch is None or self._pin_batch.shape != best.shape:
            self._pin_batch = torch.empty(best.shape, dtype=torch.float32).pin_memory()
        self._pin_batch.copy_(best, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return self._pin_batch.numpy().copy()

    def reset_batch(self, indices: Optional[Sequence[int]] = None):
        """Restore the warm starts of the batch entries ``indices`` (all of them when None).  MPPIOptimizer's carried
        means are kept, as :meth:`reset` keeps ``MPPIOptimizer.mean``."""
        if indices is None or self.previous_solutions is None:
            self.previous_solutions = None
            return
        idx = torch.as_tensor(list(indices), dtype=torch.int64, device=self.previous_solutions.device)
        self.previous_solutions[idx] = self.initial_solution


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
        self._batch_actions: List[np.ndarray] = []  # [K, A] actions of the batch's last plan still to be used

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

    def act_batch(self, obs: np.ndarray, optimizer_callback: Optional[Callable] = None, **_kwargs) -> np.ndarray:
        """:meth:`act` for K observations at once (a vectorised environment, several episodes or seeds): returns the
        actions ``[K, A]``.  Each entry plans as :meth:`act` would, from its own warm start; with the model's objective
        the K plans run as one batched device-resident plan.  With ``replan_freq > 1`` every entry replans at the same
        steps.  The batch keeps its own warm starts and cached actions: :meth:`act` / :meth:`reset` do not touch them,
        :meth:`reset_batch` restores them."""
        if self.trajectory_eval_fn is None:
            raise RuntimeError("Please call `set_trajectory_eval_fn()` before using TrajectoryOptimizerAgent")
        obs = np.asarray(obs)
        K = obs.shape[0]
        if getattr(self._fused_env, "is_latent", False):  # plans from the environment's K posteriors (update_posterior_batch)
            self._fused_env._posterior_batch(K)
        if self._batch_actions and self._batch_actions[0].shape[0] != K:
            self._batch_actions = []
        plan_time = 0.0
        if not self._batch_actions:
            if self._fused_env is not None:
                objective = _FusedBatchObjective(self._fused_env, obs, self._fused_particles)
            else:
                objective = [self._objective(o) for o in obs]
            start_time = time.time()
            plans = self.optimizer.optimize_batch(objective, K, callback=optimizer_callback)
            plan_time = time.time() - start_time
            self._batch_actions = [plans[:, i] for i in range(min(self.replan_freq, plans.shape[1]))]
        actions = self._batch_actions.pop(0)
        if self.verbose:
            print(f"Planning time: {plan_time:.3f}")
        return actions

    def reset_batch(self, indices: Optional[Sequence[int]] = None):
        """Restore the warm starts of the batch entries ``indices`` (every entry when None) and drop the cached actions,
        so that the next :meth:`act_batch` replans.  With MPPIOptimizer the entries' carried means are not cleared, just
        as :meth:`reset` leaves ``MPPIOptimizer.mean`` alone in the reference."""
        self.optimizer.reset_batch(indices)
        self._batch_actions = []


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
