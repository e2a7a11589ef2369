"""``ModelEnv`` with the reference's interface (mbrl/models/model_env.py:15-191) over the CUDA rollout kernels.

Drop-in: same constructor ``(env, model, termination_fn, reward_fn=None, generator=None)``, same
``reset`` / ``step`` / ``evaluate_action_sequences`` signatures, shapes, return types and error behaviour.
Extra keyword-only knobs choose the arithmetic (``precision``) and how TS1 draws members (``ts1``).
Over a BasicEnsemble the rows' members are drawn where the reference draws them, ``torch.randint(E, (B,))`` on the
environment's generator (basic_ensemble.py:122-127, 255-260), and ``ts1`` has no effect.
Constructed over a PlaNet latent model, it returns the latent environment of :mod:`mbrl_lib_b200.latent`.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import numpy as np
import torch

from . import _lib
from .staging import StagedModel


class ModelEnv:
    def __new__(cls, env=None, model=None, *args, **kwargs):
        """A PlaNet latent model (``belief_model``, ``prior_transition_model``, ``reward_model``) gets the latent
        environment, :class:`mbrl_lib_b200.latent.LatentModelEnv`; every other model this class."""
        if cls is ModelEnv and model is not None:
            from .latent import LatentModelEnv, is_latent_model

            if is_latent_model(model):
                return super().__new__(LatentModelEnv)
        return super().__new__(cls)

    def __init__(self, env, model, termination_fn, reward_fn=None, generator: Optional[torch.Generator] = None, *,
                 precision: str = "auto", ts1: str = "tile_shuffle"):
        self.dynamics_model = model
        self.termination_fn = termination_fn
        self.reward_fn = reward_fn
        self.device = torch.device(model.device)
        self.observation_space = env.observation_space
        self.action_space = env.action_space
        self._rng = generator if generator is not None else torch.Generator(device=self.device)
        self._return_as_np = True
        if ts1 not in ("tile_shuffle", "perms"):
            raise ValueError("ts1 must be 'tile_shuffle' (in-kernel member draw) or 'perms' (torch.randperm per step)")
        self.ts1 = ts1
        self.lib = _lib.load()
        self.staged = StagedModel(model, reward_fn, termination_fn)
        self._auto = precision == "auto"
        if precision == "auto":
            precision = "bf16_tc" if self.staged.supports_tc() else "f32"
        self.precision = precision
        self._seed = int(self._rng.initial_seed()) & 0xFFFFFFFFFFFFFFFF
        self._offset = 0
        self._ws: Optional[torch.Tensor] = None
        self._obs_pin: Optional[torch.Tensor] = None
        self._obs_dev: Optional[torch.Tensor] = None
        self._auto_refresh = True  # re-check the staged copy's signature on every call (see hand_off_from)

    # ---- helpers ---------------------------------------------------------------------------------------
    def _propagation(self) -> str:
        pm = getattr(self.staged.mlp, "propagation_method", None)
        if pm is None:
            if len(self.staged.members()) == 1:
                return "expectation"  # single model: plain forward
            raise ValueError("ensemble models need a propagation_method for ModelEnv (gaussian_mlp.py:185-190)")
        if pm not in _lib.PROP:
            raise ValueError(f"Invalid propagation method {pm}.")  # gaussian_mlp.py:216
        return pm

    def precision_for(self, propagation: str) -> str:
        """The kernel a call with ``propagation`` runs on.  ``precision="auto"`` picks the tensor-core kernel only where
        it has a launch plan for that propagation: "expectation" keeps per-row member sums in shared memory, so a model
        the tensor-core kernel covers for TS1 / TSinf can still need the fp32 kernel there.  An explicit precision is
        used as given (and fails loudly where its kernel does not cover the call)."""
        if self._auto and self.precision == "bf16_tc" and not self.staged.supports_tc(propagation):
            return "f32"
        return self.precision

    def _next_offset(self) -> int:
        """Philox stream counter of this environment: one value per API call.  ``b200pets_cem_plan`` derives the
        offsets of its iterations as ``counter * 1024 + it``; single evaluations / steps use ``counter * 1024``
        (:meth:`_call_offset`), so the two kinds of call never share a stream."""
        self._offset += 1
        return self._offset

    def _call_offset(self) -> int:
        return self._next_offset() * 1024

    def _few_groups(self, population: int, particles: int) -> bool:
        """Tile shuffle deals members to groups of 128 rows; with fewer groups than twice the members the draw would
        collapse to (almost) one member for everybody, so such small batches use generated permutations instead
        (exact reference rule, gaussian_mlp.py:202-212)."""
        groups = particles * ((population + 127) // 128)
        return groups < 2 * len(self.staged.members())

    def _member_rows(self) -> bool:
        """True over a BasicEnsemble: each row's member is an index drawn by :meth:`_draw_members`."""
        return self.staged.member_rule == "rows"

    def _draw_members(self, batch: int) -> torch.Tensor:
        """One BasicEnsemble member draw for ``batch`` rows, on this environment's generator (basic_ensemble.py:126)."""
        return torch.randint(len(self.staged.members()), (batch,), generator=self._rng, device=self.device)

    def _workspace(self, nbytes: int) -> torch.Tensor:
        if self._ws is None or self._ws.numel() < nbytes:
            self._ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=self.device)
        return self._ws

    def _obs_to_device(self, initial_state: np.ndarray) -> torch.Tensor:
        """host fp64/fp32 observations of any shape ([D] or [K, D]) -> fp32 device tensor of that shape through a pinned
        staging buffer."""
        host = np.ascontiguousarray(initial_state, dtype=np.float32)
        if self._obs_pin is None or self._obs_pin.numel() != host.size:
            self._obs_pin = torch.empty(host.size, dtype=torch.float32).pin_memory()
            self._obs_dev = torch.empty(host.size, dtype=torch.float32, device=self.device)
            with torch.cuda.device(self.device):
                self._obs_evt = torch.cuda.Event()
        else:
            self._obs_evt.synchronize()  # the previous async H2D copy must have read the pinned buffer before we overwrite it
        self._obs_pin.copy_(torch.from_numpy(host).reshape(-1))
        with torch.cuda.device(self.device):  # copy and event on the model's device / stream, whatever the current one is
            self._obs_dev.copy_(self._obs_pin, non_blocking=True)
            self._obs_evt.record()
        return self._obs_dev.view(host.shape)

    def shuffle_member_assignment(self, population: int, horizon: int, num_particles: int, offset: int,
                                  first_sequence: int = 0, global_population: int = 0) -> torch.Tensor:
        """Row -> member map ``[H, B]`` (positions in the elite list, rows ``r = n * P + p`` of this shard) that the
        kernels use in tile-shuffle mode for Philox ``offset`` (``b200pets_shuffle_member_map``).  Diagnostics /
        parity tests: the oracle consumes it as the reference's per-step assignment (gaussian_mlp.py:202-212)."""
        prop = self._propagation()
        cfg = _lib.RolloutCfg(population, horizon, num_particles, _lib.PREC[self.precision_for(prop)], _lib.PROP[prop],
                              _lib.TS1_TILE_SHUFFLE, self._seed, offset, first_sequence, global_population)
        groups = int(self.lib.b200pets_shuffle_num_groups(C.byref(cfg)))
        M = len(self.staged.members())
        gm = torch.empty(horizon, groups, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.b200pets_shuffle_member_map(C.byref(cfg), M, _lib.ptr(gm), _lib.stream_ptr()),
                       "shuffle_member_map")
        gm = gm.cpu().numpy()
        c_lo = first_sequence // 128
        C_loc = (first_sequence + population - 1) // 128 - c_lo + 1
        assert groups == num_particles * C_loc
        assign = np.full((horizon, population * num_particles), -1, dtype=np.int64)
        for p in range(num_particles):
            for ci in range(C_loc):
                lo = max((c_lo + ci) * 128, first_sequence) - first_sequence
                hi = min((c_lo + ci + 1) * 128, first_sequence + population) - first_sequence
                rows = np.arange(lo, hi) * num_particles + p
                assign[:, rows] = gm[:, p * C_loc + ci][:, None]
        assert (assign >= 0).all()
        return torch.from_numpy(assign)

    # ---- weight hand-off from training (SURVEY.md 8f #3) --------------------------------------------------
    def _fresh(self):
        if self._auto_refresh:
            self.staged.ensure_fresh()

    def push_weights(self):
        """Re-stage the packed device copy NOW (fp32 gather of the elite members + bf16 tensor-core images, a few small kernels on
        the model's stream): what the end of ``ModelTrainer.train`` / ``set_elite`` / ``update_normalizer`` should call."""
        self.staged.ensure_fresh()

    def hand_off_from(self, trainer, model=None):
        """Make training PUSH its result instead of every ``act()`` / ``step()`` polling for it.

        ``trainer`` is the reference's ``mbrl.models.ModelTrainer`` (model_trainer.py:70-214): its ``train`` ends by loading
        the best weights and calling ``model.set_elite`` (:205-214, 288-296), and the training loop of PETS / MBPO calls
        ``update_normalizer`` right before it (mbrl/util/common.py:385-389).  ``train`` is wrapped so that the packed copy
        is re-staged once, when it returns; the dynamics model's ``update_normalizer`` / ``set_elite`` (callable on their
        own) are wrapped the same way.  From then on the planner's hot path no longer walks the parameters' version
        counters (``_auto_refresh`` off): one signature walk per training round instead of one per planned action.
        ``model`` defaults to this environment's dynamics model.  Returns ``trainer``."""
        env = self
        model = model if model is not None else self.dynamics_model

        def _wrap(obj, name):
            fn = getattr(obj, name, None)
            if fn is None:
                return
            if getattr(fn, "_b200pets_pushes", False):  # already wrapped (another ModelEnv of the same model): join its list
                if all(e is not env for e in fn._b200pets_envs):
                    fn._b200pets_envs.append(env)
                return
            envs = [env]

            def pushed(*a, **kw):
                out = fn(*a, **kw)
                for e in envs:
                    e.staged.ensure_fresh()
                return out
            pushed._b200pets_pushes = True
            pushed._b200pets_envs = envs
            pushed.__wrapped__ = fn
            setattr(obj, name, pushed)

        if trainer is not None:
            _wrap(trainer, "train")
        for name in ("update_normalizer", "set_elite", "load"):
            _wrap(model, name)
        self.staged.ensure_fresh()
        self._auto_refresh = False
        return trainer

    # ---- reference API ---------------------------------------------------------------------------------
    def reset(self, initial_obs_batch: np.ndarray, return_as_np: bool = True) -> Dict[str, torch.Tensor]:
        assert len(initial_obs_batch.shape) == 2  # batch, obs_dim  (model_env.py:78-79)
        self._fresh()
        obs = torch.from_numpy(np.ascontiguousarray(initial_obs_batch.astype(np.float32))).to(self.device)
        state = {"obs": obs, "propagation_indices": None}
        if self._propagation() == "fixed_model" and self._member_rows():
            state["propagation_indices"] = self._draw_members(obs.shape[0])  # model.py:405, basic_ensemble.py:255-260
        elif self._propagation() == "fixed_model":
            B, M = obs.shape[0], len(self.staged.members())
            if B % M != 0:  # gaussian_mlp.py:369-373
                raise ValueError("To use GaussianMLP's ensemble propagation, the batch size must "
                                 "be a multiple of the number of models in the ensemble.")
            state["propagation_indices"] = torch.randperm(B, device=self.device)
        self._return_as_np = return_as_np
        return state

    def step(self, actions, model_state: Dict[str, torch.Tensor], sample: bool = False, *,
             _perm: Optional[torch.Tensor] = None, _eps: Optional[torch.Tensor] = None, _offset: Optional[int] = None,
             _out=None):
        assert len(actions.shape) == 2  # batch, action_dim  (model_env.py:108)
        self._fresh()
        with torch.no_grad():
            if isinstance(actions, np.ndarray):
                actions = torch.from_numpy(actions).to(self.device)
            actions = actions.to(torch.float32).contiguous()
            obs = model_state["obs"]
            if isinstance(obs, np.ndarray):
                obs = torch.from_numpy(obs).to(self.device)
            obs = obs.to(torch.float32).contiguous()
            B = obs.shape[0]
            prop = self._propagation()
            perm = _perm
            if perm is None:
                if prop == "fixed_model":
                    perm = model_state.get("propagation_indices")
                    if perm is None:
                        raise ValueError("When using propagation='fixed_model', `propagation_indices` must be provided.")
                elif prop == "random_model" and self._member_rows():
                    perm = self._draw_members(B)
                elif prop == "random_model" and (self.ts1 == "perms" or self._few_groups(B, 1)):
                    perm = torch.randperm(B, device=self.device)
            if perm is not None:
                perm = perm.to(torch.int64).contiguous()
            d = self.staged.desc
            if _out is not None:  # caller-owned output buffers (device-resident rollout loops: mbpo.py)
                next_obs, reward, done = _out
            else:
                next_obs = torch.empty_like(obs)
                reward = torch.empty(B, dtype=torch.float32, device=self.device)
                done = torch.empty(B, dtype=torch.uint8, device=self.device)
            with torch.cuda.device(self.device):
                _lib.check(self.lib.b200pets_step(
                    self.staged.handle, _lib.PREC[self.precision_for(prop)], _lib.PROP[prop], B, _lib.ptr(obs), _lib.ptr(actions),
                    _lib.ptr(perm), _lib.ptr(_eps), self._seed, self._call_offset() if _offset is None else _offset,
                    int(bool(sample)), _lib.ptr(next_obs),
                    _lib.ptr(reward), _lib.ptr(done), _lib.stream_ptr()), "step")
            rewards = reward.view(-1, 1)
            dones = done.view(-1, 1).bool()
            if d.reward_fn == _lib.REWARD["external"]:
                rewards = self.reward_fn(actions, next_obs)
                if _out is not None:
                    reward.copy_(rewards.view(-1))
            if d.term_fn == _lib.TERM["external"]:
                dones = self.termination_fn(actions, next_obs)
                if _out is not None:
                    done.copy_(dones.view(-1))
            next_state = dict(model_state)
            next_state["obs"] = next_obs
            if self._return_as_np:
                return next_obs.cpu().numpy(), rewards.cpu().numpy(), dones.cpu().numpy(), next_state
            return next_obs, rewards, dones, next_state

    def render(self, mode="human"):
        pass

    def has_external_callables(self) -> bool:
        """True when the reward or the termination function is a callable the kernels do not know: evaluations then run
        the rollout in windows and apply the callable once per window (see :meth:`evaluate_action_sequences`)."""
        d = self.staged.desc
        return d.reward_fn == _lib.REWARD["external"] or d.term_fn == _lib.TERM["external"]

    def evaluate_action_sequences(self, action_sequences: torch.Tensor, initial_state: np.ndarray, num_particles: int, *,
                                  _perms: Optional[torch.Tensor] = None, _eps: Optional[torch.Tensor] = None,
                                  _row_returns: Optional[torch.Tensor] = None, _offset: Optional[int] = None,
                                  _shard=(0, 0), _window: Optional[int] = None) -> torch.Tensor:
        """model_env.py:145-191.  Known reward / termination functions run inside the rollout kernel.  A callable the
        kernels do not know is applied to whole windows of steps: the kernel writes every step's next observation, then
        ``reward_fn(act, next_obs)`` / ``termination_fn(act, next_obs)`` are called ONCE per window on all its T * B rows
        (fp32 device tensors, rows in the reference's order: step-major, then ``n * P + p``).  Such callables must
        therefore compute each row from that row alone, as all of mbrl-lib's reward and termination functions do."""
        with torch.no_grad():
            assert len(action_sequences.shape) == 3  # model_env.py:166
            population_size, horizon, action_dim = action_sequences.shape
            assert initial_state.ndim in (1, 3)  # model_env.py:169
            if initial_state.ndim != 1:
                raise NotImplementedError("pixel observations are outside the GaussianMLP hot path")
            self._fresh()
            actions = action_sequences.to(self.device, torch.float32).contiguous()
            prop = self._propagation()
            perms = _perms
            if perms is None:
                perms = self._eval_perms(prop, population_size, horizon, num_particles)
            cfg = _lib.RolloutCfg(population_size, horizon, num_particles, _lib.PREC[self.precision_for(prop)], _lib.PROP[prop],
                                  _lib.TS1_PERMS if perms is not None else _lib.TS1_TILE_SHUFFLE, self._seed,
                                  self._call_offset() if _offset is None else _offset, int(_shard[0]), int(_shard[1]))
            obs0 = self._obs_to_device(initial_state)
            returns = torch.empty(population_size, dtype=torch.float32, device=self.device)
            if perms is not None:
                perms = perms.to(torch.int64).contiguous()
            if self.has_external_callables():
                self._evaluate_with_callables(cfg, actions, obs0, perms, _eps, returns, _row_returns, _window)
                return returns
            need = self.lib.b200pets_eval_workspace_bytes(self.staged.handle, C.byref(cfg))
            ws = self._workspace(need)
            with torch.cuda.device(self.device):
                _lib.check(self.lib.b200pets_eval_sequences(
                    self.staged.handle, C.byref(cfg), _lib.ptr(obs0), _lib.ptr(actions), _lib.ptr(perms), _lib.ptr(_eps),
                    _lib.ptr(returns), _lib.ptr(_row_returns), _lib.ptr(ws), ws.numel(), _lib.stream_ptr()),
                    "eval_sequences")
            return returns

    def _eval_perms(self, prop: str, population: int, horizon: int, num_particles: int) -> Optional[torch.Tensor]:
        """The permutations :meth:`evaluate_action_sequences` draws for one evaluation (None: members drawn in kernel)."""
        B = population * num_particles
        if self._member_rows() and prop != "expectation":
            return torch.stack([self._draw_members(B) for _ in range(horizon if prop == "random_model" else 1)])
        if prop == "fixed_model":
            if B % len(self.staged.members()) != 0:
                raise ValueError("To use GaussianMLP's ensemble propagation, the batch size must "
                                 "be a multiple of the number of models in the ensemble.")
            if self.ts1 == "perms" or self._few_groups(population, num_particles):
                return torch.randperm(B, device=self.device).view(1, B)
        elif prop == "random_model" and (self.ts1 == "perms" or self._few_groups(population, num_particles)):
            return torch.stack([torch.randperm(B, device=self.device) for _ in range(horizon)])
        return None

    def evaluate_action_sequences_batch(self, action_sequences: torch.Tensor, initial_states: np.ndarray, num_particles: int, *,
                                        _perms: Optional[torch.Tensor] = None, _eps: Optional[torch.Tensor] = None,
                                        _row_returns: Optional[torch.Tensor] = None,
                                        _offset: Optional[int] = None) -> torch.Tensor:
        """:meth:`evaluate_action_sequences` for K independent problems in one call: ``action_sequences [K, N, H, A]``
        from ``initial_states [K, D]``, returns ``[K, N]``.  Each problem gets exactly what a single call would give it:
        the same permutation decision, drawn in the same order, and the Philox offset of the k-th of K consecutive
        single calls (the call reserves K counter values).  The rollouts of all problems run in one launch per step
        window, which fills the GPU where one problem's population does not.  Reward or termination callables the
        kernels do not know are not supported here (``NotImplementedError``): call :meth:`evaluate_action_sequences`
        per problem."""
        with torch.no_grad():
            assert len(action_sequences.shape) == 4  # problems, population, horizon, action_dim
            K, population_size, horizon, action_dim = action_sequences.shape
            initial_states = np.asarray(initial_states)
            if initial_states.ndim != 2 or initial_states.shape[0] != K:
                raise ValueError(f"initial_states must be [K={K}, obs_dim], got {tuple(initial_states.shape)}")
            if self.has_external_callables():
                raise NotImplementedError("evaluate_action_sequences_batch runs known reward / termination functions only; "
                                          "with a callable, call evaluate_action_sequences once per problem")
            self._fresh()
            actions = action_sequences.to(self.device, torch.float32).contiguous()
            prop = self._propagation()
            perms = _perms
            if perms is None:
                per = [self._eval_perms(prop, population_size, horizon, num_particles) for _ in range(K)]
                perms = None if not per or per[0] is None else torch.stack(per)
            if perms is not None:
                perms = perms.to(torch.int64).contiguous()
            if _offset is None:
                _offset = self._call_offset()
                self._offset += K - 1  # problem k uses the offset of the k-th of K consecutive calls
            cfg = _lib.RolloutCfg(population_size, horizon, num_particles, _lib.PREC[self.precision_for(prop)], _lib.PROP[prop],
                                  _lib.TS1_PERMS if perms is not None else _lib.TS1_TILE_SHUFFLE, self._seed, _offset, 0, 0)
            obs0 = torch.from_numpy(np.ascontiguousarray(initial_states, dtype=np.float32)).to(self.device)
            returns = torch.empty(K, population_size, dtype=torch.float32, device=self.device)
            need = self.lib.b200pets_eval_batch_workspace_bytes(self.staged.handle, C.byref(cfg), K)
            ws = self._workspace(need)
            with torch.cuda.device(self.device):
                _lib.check(self.lib.b200pets_eval_sequences_batch(
                    self.staged.handle, C.byref(cfg), K, _lib.ptr(obs0), _lib.ptr(actions), _lib.ptr(perms), _lib.ptr(_eps),
                    _lib.ptr(returns), _lib.ptr(_row_returns), _lib.ptr(ws), ws.numel(), _lib.stream_ptr()),
                    "eval_sequences_batch")
            return returns

    def _evaluate_with_callables(self, cfg, actions, obs0, perms, eps, returns, row_returns, window):
        """The evaluation ``cfg`` describes with the caller's reward / termination callables: per window of T steps one
        trajectory launch (next observations, kernel-side reward / done), the callables on the window's T * B rows, and
        the masking / accumulation kernel (model_env.py:178-191).  The row state stays in one workspace throughout."""
        N, H, A = actions.shape
        P = cfg.particles
        B, D = N * P, self.staged.desc.obs_dim
        T = trajectory_window(B, D, A, H) if window is None else max(1, min(int(window), H))
        ws = self._workspace(self.lib.b200pets_trajectory_workspace_bytes(self.staged.handle, C.byref(cfg)))
        next_obs = torch.empty(T, B, D, dtype=torch.float32, device=self.device)
        reward = torch.empty(T, B, dtype=torch.float32, device=self.device)
        done = torch.empty(T, B, dtype=torch.uint8, device=self.device)
        ext_reward = self.staged.desc.reward_fn == _lib.REWARD["external"]
        ext_term = self.staged.desc.term_fn == _lib.TERM["external"]
        with torch.cuda.device(self.device):
            for t0 in range(0, H, T):
                t1 = min(t0 + T, H)
                rows = (t1 - t0) * B
                _lib.check(self.lib.b200pets_eval_trajectory(
                    self.staged.handle, C.byref(cfg), t0, t1, _lib.ptr(obs0), _lib.ptr(actions), _lib.ptr(perms),
                    _lib.ptr(eps), _lib.ptr(next_obs), _lib.ptr(reward), _lib.ptr(done), _lib.ptr(ws), ws.numel(),
                    _lib.stream_ptr()), "eval_trajectory")
                # the reference's action batch of each step, torch.repeat_interleave over particles (model_env.py:181)
                act = actions[:, t0:t1].transpose(0, 1).repeat_interleave(P, dim=1).reshape(rows, A)
                nobs = next_obs[:t1 - t0].view(rows, D)
                if ext_reward:
                    reward[:t1 - t0].view(rows).copy_(self.reward_fn(act, nobs).reshape(rows))
                if ext_term:
                    done[:t1 - t0].view(rows).copy_(self.termination_fn(act, nobs).reshape(rows))
                _lib.check(self.lib.b200pets_trajectory_returns(
                    C.byref(cfg), t0, t1, _lib.ptr(reward), _lib.ptr(done), _lib.ptr(returns), _lib.ptr(row_returns),
                    _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), "trajectory_returns")


# Device memory one window of an evaluation with external callables may take for its next observations, actions, rewards
# and done flags: long horizons over large populations are split so that these stay bounded.
TRAJECTORY_WINDOW_BYTES = 256 << 20


def trajectory_window(batch: int, obs_dim: int, act_dim: int, horizon: int,
                      budget: int = TRAJECTORY_WINDOW_BYTES) -> int:
    """Steps per window: as many as fit ``budget`` bytes of fp32 next observations and actions, fp32 rewards and uint8
    done flags for ``batch`` rows each, at least 1 and at most ``horizon``."""
    per_step = batch * (4 * obs_dim + 4 * act_dim + 4 + 1)
    return max(1, min(horizon, budget // max(per_step, 1)))
