"""PlaNet's latent model behind ``ModelEnv`` (mbrl/models/planet.py, mbrl/models/model_env.py).

:class:`StagedLatentModel` reads the planning half of a ``PlaNetModel`` -- mbrl-lib's own or the container
:class:`mbrl_lib_b200.models.PlaNetModel` -- by attribute: ``belief_model.embedding_layer[0]``, ``belief_model.rnn``,
``prior_transition_model[0]`` / ``[2]``, ``min_std`` and ``reward_model[0]`` / ``[2]`` / ``[4]``.  Like
:class:`~mbrl_lib_b200.staging.StagedModel` it never copies the weights to the host and re-packs its device copy when
a parameter's storage or ``_version`` counter changed, so a training round in between needs no extra call.

:class:`LatentModelEnv` is what ``ModelEnv(env, planet_model, no_termination, generator=rng)`` returns: the reference's
interface over ``b200pets_latent_step`` and ``b200pets_latent_eval_sequences_batch``; ``CEMOptimizer`` plans over it
with one ``b200pets_latent_cem_plan_batch`` call.  A single call is the batch of one.  Every rollout starts at the
model's posterior (``_current_posterior_sample``, ``_current_belief``), which ``update_posterior`` (the conv encoder, run
by the caller once per environment step) sets.

For K environments at once the env itself holds K posteriors: ``update_posterior_batch`` (or ``set_posterior_batch``)
sets them, ``evaluate_action_sequences_batch`` and ``cem_plan(..., batch=True)`` plan from them, and
``TrajectoryOptimizerAgent.act_batch`` plans with them.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional

import numpy as np
import torch

from . import _lib, functions
from .model_env import ModelEnv


def is_latent_model(model) -> bool:
    """Whether ``model`` has PlaNet's attribute layout (the latent path) rather than a GaussianMLP's."""
    return all(hasattr(model, n) for n in ("belief_model", "prior_transition_model", "reward_model"))


def latent_params(model) -> List[torch.Tensor]:
    """The planning parameters of a PlaNet model in the order ``b200pets_latent_model_create`` takes them
    (include/b200pets.h)."""
    emb, rnn = model.belief_model.embedding_layer[0], model.belief_model.rnn
    p1, p2 = model.prior_transition_model[0], model.prior_transition_model[2]
    r1, r2, r3 = model.reward_model[0], model.reward_model[2], model.reward_model[4]
    return [emb.weight, emb.bias, rnn.weight_ih, rnn.weight_hh, rnn.bias_ih, rnn.bias_hh, p1.weight, p1.bias,
            p2.weight, p2.bias, r1.weight, r1.bias, r2.weight, r2.bias, r3.weight, r3.bias]


def _expect_relu(module, where: str):
    if type(module).__name__ != "ReLU":
        raise NotImplementedError(f"{where} is {type(module).__name__}; the latent kernel implements PlaNet's ReLU")


class StagedLatentModel:
    """Owns the C handle of one staged latent model and re-stages it when the source object changed.  ``stage=False``
    only reads the object (description, parameter list, signature) and touches neither the library nor a device."""

    def __init__(self, planet, stage: bool = True):
        if not is_latent_model(planet):
            raise NotImplementedError(f"{type(planet).__name__} has no belief_model / prior_transition_model / reward_model")
        self.src = planet
        self.lib = _lib.load() if stage else None
        emb, rnn = planet.belief_model.embedding_layer, planet.belief_model.rnn
        prior, rew = planet.prior_transition_model, planet.reward_model
        _expect_relu(emb[1], "belief_model.embedding_layer[1]")
        _expect_relu(prior[1], "prior_transition_model[1]")
        _expect_relu(rew[1], "reward_model[1]")
        _expect_relu(rew[3], "reward_model[3]")
        self._modules = (emb[0], rnn, prior[0], prior[2], rew[0], rew[2], rew[4])
        self.device = torch.device(emb[0].weight.device)
        if stage and self.device.type != "cuda":
            raise RuntimeError(f"b200pets runs on a CUDA device; the model lives on {self.device} (no CPU fallback)")
        self.desc = self._describe()
        self.handle: Optional[C.c_void_p] = None
        self._sig = None
        if stage:
            self.ensure_fresh()

    def _describe(self) -> _lib.LatentDesc:
        emb, rnn, p1, p2, r1, r2, r3 = self._modules
        Hb = int(rnn.hidden_size)
        L = int(p2.out_features) // 2
        A = int(emb.in_features) - L
        Hf = int(p1.out_features)
        if (int(emb.out_features), int(rnn.input_size), int(p1.in_features), int(r1.in_features), int(r2.in_features),
                int(r2.out_features), int(r3.in_features), int(r3.out_features), int(r1.out_features)) != \
                (Hb, Hb, Hb, Hb + L, Hf, Hf, Hf, 1, Hf) or A < 1 or not getattr(rnn, "bias", True):
            raise ValueError("the latent model's layer sizes do not chain as PlaNet's do (planet.py:82-114, 231-264)")
        d = _lib.LatentDesc()
        d.action_size, d.latent_size, d.belief_size, d.hidden_size = A, L, Hb, Hf
        d.min_std = float(self.src.min_std)
        return d

    def params(self) -> List[torch.Tensor]:
        """The tensors ``b200pets_latent_model_create`` takes, in its order (include/b200pets.h)."""
        return latent_params(self.src)

    def signature(self):
        sig = [(p.data_ptr(), p._version, tuple(p.shape)) for p in self.params()]
        sig.append(float(self.src.min_std))
        return tuple(sig)

    def ensure_fresh(self):
        sig = self.signature()
        if sig == self._sig:
            return
        desc = self._describe()
        params = self.params()
        for p in params:
            if p.dtype != torch.float32 or not p.is_contiguous() or p.device != self.device:
                raise ValueError("latent model weights must be contiguous float32 tensors on one CUDA device")
        arr = (C.c_void_p * len(params))(*[p.data_ptr() for p in params])
        same = self.handle is not None and all(getattr(desc, f) == getattr(self.desc, f) for f, _ in desc._fields_)
        with torch.cuda.device(self.device):
            stream = _lib.stream_ptr()
            if same:
                _lib.check(self.lib.b200pets_latent_model_refresh(self.handle, arr, stream), "latent_model_refresh")
            else:
                self.close()
                h = C.c_void_p()
                _lib.check(self.lib.b200pets_latent_model_create(C.byref(desc), arr, stream, C.byref(h)),
                           "latent_model_create")
                self.handle = h
        self.desc = desc
        self._sig = sig

    def plan_info(self, rows: int) -> dict:
        """The rollout kernel's launch for ``rows`` rows on the current device (``b200pets_latent_plan_info``)."""
        info = (C.c_int32 * 4)()
        with torch.cuda.device(self.device):
            _lib.check(self.lib.b200pets_latent_plan_info(self.handle, int(rows), info), "latent_plan_info")
        return {"rows_per_cta": info[0], "ctas": info[1], "smem": info[2], "row_bytes": info[3]}

    def posterior(self):
        """``(latent [L], belief [Hb])``: the posterior every planned rollout starts from (planet.py:641-660)."""
        s, h = getattr(self.src, "_current_posterior_sample", None), getattr(self.src, "_current_belief", None)
        if s is None or h is None:
            raise RuntimeError("the latent model has no posterior: call update_posterior(obs) before planning "
                               "(mbrl/algorithms/planet.py:163-170)")
        if s.shape[0] != 1 or h.shape[0] != 1:
            raise ValueError(f"the posterior must hold one state, got latent {tuple(s.shape)} and belief {tuple(h.shape)}")
        return (s.detach().reshape(-1).to(self.device, torch.float32).contiguous(),
                h.detach().reshape(-1).to(self.device, torch.float32).contiguous())

    def close(self):
        if self.handle is not None:
            self.lib.b200pets_latent_model_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class PosteriorBatch:
    """The K posteriors a :class:`LatentModelEnv` plans K observations from, kept apart from the model's own posterior:
    ``latent [K, L]`` and ``belief [K, Hb]`` on ``device``, plus the entries whose next :meth:`update` starts a new
    episode.  Reads the model only in :meth:`update`."""

    def __init__(self, model, latent_size: int, belief_size: int, action_size: int, device):
        self.model, self.L, self.Hb, self.A = model, latent_size, belief_size, action_size
        self.device = torch.device(device)
        self.latent: Optional[torch.Tensor] = None
        self.belief: Optional[torch.Tensor] = None
        self.fresh: Optional[np.ndarray] = None

    def set(self, latent, belief):
        latent = torch.as_tensor(latent).detach().to(self.device, torch.float32).contiguous()
        belief = torch.as_tensor(belief).detach().to(self.device, torch.float32).contiguous()
        K = latent.shape[0] if latent.ndim == 2 else 0
        if K < 1 or latent.shape != (K, self.L) or belief.shape != (K, self.Hb):
            raise ValueError(f"set_posterior_batch: latent {tuple(latent.shape)} and belief {tuple(belief.shape)} must be "
                             f"[K, {self.L}] and [K, {self.Hb}]")
        self.latent, self.belief = latent, belief
        self.fresh = np.zeros(K, dtype=bool)

    def update(self, obs, action=None, rng: Optional[torch.Generator] = None, *,
               _eps: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        """``PlaNetModel.update_posterior`` (planet.py:592-641) for K observations ``obs [K, C, H, W]`` and the actions
        ``action [K, A]`` that led to them, with the model's own ``encoder``, ``belief_model`` and
        ``posterior_transition_model`` and the reference's ``x / 256 - 0.5``.  Entries of a new batch and entries listed
        to :meth:`reset` start from zero latent, belief and action (``action`` may be None only when every entry does).
        The posterior draw is one N(0, 1) ``[K, L]`` from ``rng`` (else the model's ``rng``); ``_eps`` replaces it.
        Returns ``{"latent": [K, L], "belief": [K, Hb]}``."""
        model = self.model
        missing = [n for n in ("encoder", "belief_model", "posterior_transition_model") if not hasattr(model, n)]
        if missing:
            raise NotImplementedError(f"update_posterior_batch runs the model's encoder, belief_model and "
                                      f"posterior_transition_model; this model has no {', '.join(missing)}")
        with torch.no_grad():
            x = torch.as_tensor(obs).float().to(self.device) / 256.0 - 0.5  # planet.py:274-275
            if x.ndim != 4:
                raise ValueError(f"update_posterior_batch: obs must be [K, C, H, W], got {tuple(x.shape)}")
            K = x.shape[0]
            if self.latent is None:
                fresh = np.ones(K, dtype=bool)
            elif self.latent.shape[0] != K:
                raise ValueError(f"update_posterior_batch: {K} observations for a batch of {self.latent.shape[0]} "
                                 "posteriors (reset_posterior_batch() starts a new batch)")
            else:
                fresh = self.fresh
            latent = torch.zeros(K, self.L, device=self.device)
            belief = torch.zeros(K, self.Hb, device=self.device)
            act = torch.zeros(K, self.A, device=self.device)
            if not fresh.all():
                if action is None:
                    raise ValueError("update_posterior_batch: action is None but some entries continue an episode")
                keep = torch.from_numpy(~fresh).to(self.device)[:, None]
                act = torch.where(keep, torch.as_tensor(action).float().to(self.device).reshape(K, self.A), act)
                latent = torch.where(keep, self.latent, latent)
                belief = torch.where(keep, self.belief, belief)
            bm = model.belief_model  # BeliefModel.forward (planet.py:90-101)
            next_belief = bm.rnn(bm.embedding_layer(torch.cat([latent, act], dim=1)), belief)
            params = model.posterior_transition_model(torch.cat([next_belief, model.encoder(x)], dim=1))
            mean, std = params[:, :self.L], params[:, self.L:]
            if _eps is None:
                _eps = torch.randn(mean.size(), dtype=mean.dtype, layout=mean.layout, device=mean.device,
                                   generator=model.rng if rng is None else rng)
            self.set(mean + std * _eps.to(mean.device, mean.dtype), next_belief)
            return {"latent": self.latent, "belief": self.belief}

    def reset(self, indices=None):
        """``indices`` None drops the batch (the next update sets K from its observations); otherwise the listed entries
        start their next :meth:`update` from zero latent, belief and action, as ``reset_posterior()`` followed by
        ``update_posterior(obs, action=None)`` does."""
        if indices is None or self.latent is None:
            self.latent = self.belief = self.fresh = None
            return
        self.fresh[np.asarray(list(indices), dtype=np.int64)] = True

    def get(self, K: Optional[int] = None):
        """``(latent [K, L], belief [K, Hb])``: ``NotImplementedError`` when none is set, ``ValueError`` when ``K``
        differs, ``RuntimeError`` when an entry was reset and not updated since."""
        if self.latent is None:
            raise NotImplementedError("the latent model holds one posterior; to plan for K observations set K posteriors "
                                      "first with update_posterior_batch(obs) or set_posterior_batch")
        if K is not None and K != self.latent.shape[0]:
            raise ValueError(f"{K} problems for a batch of {self.latent.shape[0]} posteriors")
        if self.fresh.any():
            raise RuntimeError(f"entries {np.flatnonzero(self.fresh).tolist()} were reset: call "
                               "update_posterior_batch(obs) before planning")
        return self.latent, self.belief


class LatentModelEnv(ModelEnv):
    """``ModelEnv`` over PlaNet's latent model (model_env.py:15-191 with ``PlaNetModel.sample``).  The states are
    ``{"latent": [B, L], "belief": [B, Hb]}``; rewards come from the reward model and nothing terminates."""

    is_latent = True

    def __init__(self, env, model, termination_fn, reward_fn=None, generator: Optional[torch.Generator] = None, *,
                 precision: str = "f32"):
        if reward_fn is not None:
            raise NotImplementedError("the latent model's rewards come from its reward model; a reward_fn is not "
                                      "supported (mbrl/algorithms/planet.py passes none)")
        if functions.resolve_term(termination_fn) != _lib.TERM["no_termination"]:
            raise NotImplementedError("the latent model plans with no_termination only: its next observation is a latent "
                                      "state that a termination function cannot read")
        if precision not in ("f32", "auto"):
            raise NotImplementedError(f"the latent model runs in fp32 only, not {precision!r}")
        self.dynamics_model = model
        self.termination_fn = termination_fn
        self.reward_fn = None
        self.device = torch.device(model.device)
        self.observation_space = env.observation_space
        self.action_space = env.action_space
        self._rng = generator if generator is not None else torch.Generator(device=self.device)
        self._return_as_np = True
        self.precision = "f32"
        self.lib = _lib.load()
        self.staged = StagedLatentModel(model)
        self._seed = int(self._rng.initial_seed()) & 0xFFFFFFFFFFFFFFFF
        self._offset = 0
        self._ws: Optional[torch.Tensor] = None
        self._auto_refresh = True
        d = self.staged.desc
        self.posteriors = PosteriorBatch(model, d.latent_size, d.belief_size, d.action_size, self.device)

    def has_external_callables(self) -> bool:
        return False

    def reset(self, initial_obs_batch: np.ndarray, return_as_np: bool = True) -> Dict[str, torch.Tensor]:
        """PlaNetModel.reset (planet.py:662-677): the posterior repeated once per row of ``initial_obs_batch``, whose
        content is not read."""
        self._fresh()
        latent, belief = self.staged.posterior()
        B = int(initial_obs_batch.shape[0])
        self._return_as_np = return_as_np
        return {"latent": latent.view(1, -1).repeat(B, 1), "belief": belief.view(1, -1).repeat(B, 1)}

    def step(self, actions, model_state: Dict[str, torch.Tensor], sample: bool = False, *,
             _eps: Optional[torch.Tensor] = None, _offset: Optional[int] = None):
        """One launch of ``b200pets_latent_step``: ``(next_latent, reward [B, 1], dones [B, 1], next_state)``."""
        assert len(actions.shape) == 2  # batch, action_dim  (model_env.py:108)
        self._fresh()
        with torch.no_grad():
            if isinstance(actions, np.ndarray):
                actions = torch.from_numpy(actions)
            actions = actions.to(self.device, torch.float32).contiguous()
            latent = torch.as_tensor(model_state["latent"]).to(self.device, torch.float32).contiguous()
            belief = torch.as_tensor(model_state["belief"]).to(self.device, torch.float32).contiguous()
            B = latent.shape[0]
            d = self.staged.desc
            if actions.shape != (B, d.action_size) or belief.shape != (B, d.belief_size) or latent.shape[1] != d.latent_size:
                raise ValueError(f"step: actions {tuple(actions.shape)}, latent {tuple(latent.shape)} and belief "
                                 f"{tuple(belief.shape)} do not match the model (A {d.action_size}, L {d.latent_size}, "
                                 f"Hb {d.belief_size})")
            eps = None if _eps is None else _eps.to(self.device, torch.float32).contiguous()
            next_latent = torch.empty_like(latent)
            next_belief = torch.empty_like(belief)
            reward = torch.empty(B, dtype=torch.float32, device=self.device)
            with torch.cuda.device(self.device):
                _lib.check(self.lib.b200pets_latent_step(
                    self.staged.handle, B, _lib.ptr(latent), _lib.ptr(belief), _lib.ptr(actions), _lib.ptr(eps), self._seed,
                    self._call_offset() if _offset is None else _offset, int(bool(sample)), _lib.ptr(next_latent),
                    _lib.ptr(next_belief), _lib.ptr(reward), _lib.stream_ptr()), "latent_step")
            rewards = reward.view(-1, 1)
            dones = torch.zeros(B, 1, dtype=torch.bool, device=self.device)  # no_termination
            next_state = {"latent": next_latent, "belief": next_belief}
            if self._return_as_np:
                return next_latent.cpu().numpy(), rewards.cpu().numpy(), dones.cpu().numpy(), next_state
            return next_latent, rewards, dones, next_state

    def _rollout_cfg(self, population: int, horizon: int, num_particles: int, offset: int) -> _lib.RolloutCfg:
        return _lib.RolloutCfg(population, horizon, num_particles, _lib.PREC["f32"], _lib.PROP["expectation"],
                               _lib.TS1_PERMS, self._seed, offset, 0, 0)

    def evaluate_action_sequences(self, action_sequences: torch.Tensor, initial_state: np.ndarray, num_particles: int, *,
                                  _eps: Optional[torch.Tensor] = None, _row_returns: Optional[torch.Tensor] = None,
                                  _offset: Optional[int] = None, _entry: Optional[int] = None) -> torch.Tensor:
        """model_env.py:145-191 as one launch from the posterior: ``initial_state`` (a 1-D or a 3-D pixel observation)
        is only checked for its rank, since PlaNetModel.reset reads nothing but the batch size.  ``_eps [H, B, L]``
        replaces the in-kernel draws; ``_entry`` k starts from the batch's posterior k instead of the model's."""
        with torch.no_grad():
            assert len(action_sequences.shape) == 3  # model_env.py:166
            assert np.ndim(initial_state) in (1, 3)  # model_env.py:169
            self._fresh()
            if _entry is None:
                latent0, belief0 = self.staged.posterior()
            else:
                latent, belief = self._posterior_batch()
                latent0, belief0 = latent[_entry], belief[_entry]
            offset = self._call_offset() if _offset is None else _offset
            return self._evaluate(action_sequences[None], latent0.view(1, -1), belief0.view(1, -1), num_particles, offset,
                                  _eps, _row_returns)[0]

    def _evaluate(self, action_sequences, latent0, belief0, num_particles, offset, eps, row_returns) -> torch.Tensor:
        """One ``b200pets_latent_eval_sequences_batch`` launch: ``action_sequences [K, N, H, A]`` from the posteriors
        ``latent0 [K, L]``, ``belief0 [K, Hb]``, problem k at Philox offset ``offset + k * 1024``; returns ``[K, N]``."""
        K, population_size, horizon, _ = action_sequences.shape
        actions = action_sequences.to(self.device, torch.float32).contiguous()
        cfg = self._rollout_cfg(population_size, horizon, num_particles, offset)
        eps = None if eps is None else eps.to(self.device, torch.float32).contiguous()
        returns = torch.empty(K, population_size, dtype=torch.float32, device=self.device)
        ws = self._workspace(self.lib.b200pets_latent_eval_batch_workspace_bytes(self.staged.handle, C.byref(cfg), K))
        with torch.cuda.device(self.device):
            _lib.check(self.lib.b200pets_latent_eval_sequences_batch(
                self.staged.handle, C.byref(cfg), K, _lib.ptr(latent0), _lib.ptr(belief0), _lib.ptr(actions),
                _lib.ptr(eps), _lib.ptr(returns), _lib.ptr(row_returns), _lib.ptr(ws), ws.numel(), _lib.stream_ptr()),
                "latent_eval_sequences_batch")
        return returns

    # ---- K posteriors (PosteriorBatch) ------------------------------------------------------------------------------
    def set_posterior_batch(self, latent, belief):
        """Set the K posteriors batched planning starts from: ``latent [K, L]``, ``belief [K, Hb]``."""
        self.posteriors.set(latent, belief)

    def update_posterior_batch(self, obs, action=None, rng: Optional[torch.Generator] = None, *,
                               _eps: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        """:meth:`PosteriorBatch.update`: ``PlaNetModel.update_posterior`` for K observations ``obs [K, C, H, W]``."""
        return self.posteriors.update(obs, action, rng, _eps=_eps)

    def reset_posterior_batch(self, indices=None):
        """:meth:`PosteriorBatch.reset`: drop the batch (None) or restart the listed entries."""
        self.posteriors.reset(indices)

    def _posterior_batch(self, K: Optional[int] = None):
        return self.posteriors.get(K)

    def evaluate_action_sequences_batch(self, action_sequences: torch.Tensor, initial_states: np.ndarray, num_particles: int,
                                        *, _eps: Optional[torch.Tensor] = None, _row_returns: Optional[torch.Tensor] = None,
                                        _offset: Optional[int] = None) -> torch.Tensor:
        """:meth:`evaluate_action_sequences` for the K posteriors in one launch: ``action_sequences [K, N, H, A]``, returns
        ``[K, N]``.  Only the leading K of ``initial_states`` is checked.  Problem k gets what a single call from
        posterior k would give at the offset of the k-th of K consecutive calls; ``_eps [K, H, B, L]``,
        ``_row_returns [K, B]``."""
        with torch.no_grad():
            assert len(action_sequences.shape) == 4  # problems, population, horizon, action_dim
            K = action_sequences.shape[0]
            latent0, belief0 = self._posterior_batch(K)
            if np.shape(initial_states)[0] != K:
                raise ValueError(f"{np.shape(initial_states)[0]} initial states for {K} problems")
            self._fresh()
            if _offset is None:
                _offset = self._call_offset()
                self._offset += K - 1  # problem k uses the offset of the k-th of K consecutive calls
            return self._evaluate(action_sequences, latent0, belief0, num_particles, _offset, _eps, _row_returns)

    def shuffle_member_assignment(self, *args, **kwargs):
        raise NotImplementedError("the latent model has no ensemble members")

    def cem_plan(self, optimizer, x0: torch.Tensor, num_particles: int, noise: Optional[torch.Tensor] = None,
                 eps: Optional[torch.Tensor] = None, *, batch: bool = False) -> torch.Tensor:
        """``optimizer`` (a CEMOptimizer) over :meth:`evaluate_action_sequences` from the warm starts ``x0 [K, H, A]`` as
        one ``b200pets_latent_cem_plan_batch`` call: K = 1 from the model's posterior, or with ``batch`` from the K
        posteriors.  Problem k plans with counter value first + k, the one its own single plan would take k calls later.
        ``noise [K, it, N, H, A]`` / ``eps [K, it, H, B, L]`` replace the population / model draws; with
        ``record_values`` ``last_values`` is ``[K, it, N]``."""
        K, H, A = x0.shape
        if batch:
            latent0, belief0 = self._posterior_batch(K)
            self._fresh()
        else:
            self._fresh()
            latent0, belief0 = (t.view(1, -1) for t in self.staged.posterior())
        rcfg = self._rollout_cfg(optimizer.population_size, H, num_particles, self._next_offset())
        self._offset += K - 1
        ccfg = optimizer._cem_cfg()
        ws = self._workspace(self.lib.b200pets_latent_cem_plan_batch_workspace_bytes(self.staged.handle, C.byref(rcfg),
                                                                                      C.byref(ccfg), K))
        x0 = x0.to(self.device, torch.float32).contiguous()
        sol = torch.empty(K, H * A, dtype=torch.float32, device=self.device)
        z = None if noise is None else noise.to(self.device, torch.float32).contiguous()
        if eps is not None:
            eps = eps.to(self.device, torch.float32).contiguous()
        optimizer.last_values = None
        if optimizer.record_values:
            optimizer.last_values = torch.empty(K, optimizer.num_iterations, optimizer.population_size, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.b200pets_latent_cem_plan_batch(
                self.staged.handle, C.byref(rcfg), C.byref(ccfg), K, _lib.ptr(latent0), _lib.ptr(belief0), _lib.ptr(x0),
                _lib.ptr(optimizer.lower_bound), _lib.ptr(optimizer.upper_bound), _lib.ptr(z), _lib.ptr(eps), _lib.ptr(sol),
                _lib.ptr(optimizer.last_values), _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), "latent_cem_plan_batch")
        return sol.view(K, H, A)
