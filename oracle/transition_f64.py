"""Float64 restatement of one ``ModelEnv.step`` over ``OneDTransitionRewardModel(GaussianMLP)`` -- TEST INFRASTRUCTURE.

The checker of the per-element transition tests (tests/test_gpu_transitions.py): given rows, their member positions (or
expectation) and the injected N(0,1) draws, it returns every column of ``next_obs`` and the learned reward column in
float64.  Unlike :class:`pets_oracle.OracleModel` (fp32, the reference's own arithmetic) it keeps everything in float64
and rounds to fp32 only where the reference casts, so the difference to a kernel is the kernel's own rounding:

* model input (one_dim_tr_model.py:103-116, util/math.py:129-143): obs_process and concatenation in float64; with fp64
  statistics, normalise in float64 and round to fp32 (the reference's ``.float()``); with fp32 statistics, normalise in
  fp32 as the reference does; without a normaliser the input is the fp32 tensor the reference feeds the model;
* MLP (gaussian_mlp.py:140-154): float64 with the member's weights, the activation (slope included) as given;
* ``bf16=True``: the operands of the tensor-core kernel -- input and every hidden activation rounded to bf16 from their
  float64 value, weights rounded to bf16, each bias split into bf16 hi + lo -- accumulated in float64;
* noise (gaussian_mlp.py:156-177, math: model.py:426-473): the two soft logvar clamps in float64, then
  ``mean + sqrt(exp(lv)) * eps``; expectation averages the mean and the clamped logvar over the members;
* outputs (one_dim_tr_model.py:245-289): the delta add-back honours ``target_is_delta`` and ``no_delta_list``; the
  learned reward is the last output column.

Known reward / termination functions are not part of the transition: tests apply ``pets_oracle.REWARD_FNS`` /
``TERM_FNS`` to the kernel's own fp32 ``next_obs`` (:func:`known_reward`, :func:`known_done`).
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np
import torch


def bf16_round(x) -> np.ndarray:
    """Round float64 values to the nearest bf16 (ties to even), returned as float64.  Exact for every finite value in
    bf16's normal range, which is where the model's operands live."""
    x = np.ascontiguousarray(x, dtype=np.float64)
    bits = x.view(np.uint64)
    lsb = (bits >> np.uint64(45)) & np.uint64(1)
    out = (bits + np.uint64((1 << 44) - 1) + lsb) & ~np.uint64((1 << 45) - 1)
    return out.view(np.float64)


def _softplus(x):
    return np.logaddexp(0.0, x)


def _proc(name: Optional[str], s: np.ndarray) -> np.ndarray:
    """pets_oracle.OBS_PROCESS in float64."""
    if name is None:
        return s
    if name == "halfcheetah":
        return np.concatenate([s[:, 1:2], np.sin(s[:, 2:3]), np.cos(s[:, 2:3]), s[:, 3:]], axis=1)
    if name == "cartpole":
        return np.concatenate([np.sin(s[:, 1:2]), np.cos(s[:, 1:2]), s[:, :1], s[:, 2:]], axis=1)
    raise ValueError(name)


class TransitionF64:
    """One model step in float64.  ``spec`` gives the structure (synthetic.CaseSpec); ``arrays`` the numbers
    (synthetic.make_model_arrays layout).  ``members`` (ensemble indices in elite order), ``slope`` (LeakyReLU),
    ``no_delta`` and ``target_is_delta`` default to the spec's; :meth:`from_model` reads all of them from a live model."""

    def __init__(self, spec, arrays, *, members: Optional[Sequence[int]] = None, slope: float = 0.01,
                 no_delta: Optional[Sequence[int]] = None, target_is_delta: Optional[bool] = None):
        self.spec = spec
        self.members = list(members) if members is not None else (
            list(spec.elites) if spec.elites is not None else list(range(spec.ensemble_size)))
        self.slope = float(slope)
        self.no_delta = list(spec.no_delta_list if no_delta is None else no_delta)
        self.target_is_delta = spec.target_is_delta if target_is_delta is None else bool(target_is_delta)
        self.W = [np.asarray(w, dtype=np.float64)[self.members] for w in arrays["weights"]]
        self.b = [np.asarray(b, dtype=np.float64)[self.members, 0] for b in arrays["biases"]]
        self.Wb = [bf16_round(w) for w in self.W]
        bh = [bf16_round(b) for b in self.b]
        self.bb = [h + bf16_round(b - h) for h, b in zip(bh, self.b)]
        self.min_lv = np.asarray(arrays["min_logvar"], dtype=np.float64).reshape(-1)
        self.max_lv = np.asarray(arrays["max_logvar"], dtype=np.float64).reshape(-1)
        self.norm_mean = self.norm_std = None
        if arrays.get("norm_mean") is not None:
            self.norm_mean = np.asarray(arrays["norm_mean"]).reshape(-1)
            self.norm_std = np.asarray(arrays["norm_std"]).reshape(-1)

    @classmethod
    def from_model(cls, spec, model):
        """Everything the step depends on read from a ``OneDTransitionRewardModel(GaussianMLP)`` object (models.py or
        mbrl-lib's): weights, elite list, normaliser, logvar bounds, activation slope, delta options."""
        mlp = model.model
        layers = [seq[0] for seq in mlp.hidden_layers] + [mlp.mean_and_logvar]
        arrays = {"weights": [l.weight.detach().float().cpu().numpy() for l in layers],
                  "biases": [l.bias.detach().float().cpu().numpy() for l in layers],
                  "min_logvar": np.zeros((1, spec.out_size)), "max_logvar": np.zeros((1, spec.out_size))}
        if not mlp.deterministic:
            arrays["min_logvar"] = mlp.min_logvar.detach().float().cpu().numpy()
            arrays["max_logvar"] = mlp.max_logvar.detach().float().cpu().numpy()
        norm = getattr(model, "input_normalizer", None)
        if norm is not None:
            arrays["norm_mean"] = norm.mean.detach().cpu().numpy()
            arrays["norm_std"] = norm.std.detach().cpu().numpy()
        act = mlp.hidden_layers[0][1]
        slope = float(getattr(act, "negative_slope", 0.0))
        el = mlp.elite_models
        members = list(el) if el is not None else list(range(int(mlp.num_members)))
        return cls(spec, arrays, members=members, slope=slope, no_delta=list(model.no_delta_list or []),
                   target_is_delta=model.target_is_delta)

    # ---- pieces ----------------------------------------------------------------------------------------------
    def model_input(self, obs, act) -> np.ndarray:
        obs = np.asarray(obs, dtype=np.float32).astype(np.float64)
        x = np.concatenate([_proc(self.spec.obs_process, obs), np.asarray(act, dtype=np.float32).astype(np.float64)], axis=1)
        if self.norm_mean is None:
            return x.astype(np.float32).astype(np.float64)
        if self.norm_mean.dtype == np.float64:
            return ((x - self.norm_mean) / self.norm_std).astype(np.float32).astype(np.float64)
        x32 = x.astype(np.float32)
        return ((x32 - self.norm_mean.astype(np.float32)) / self.norm_std.astype(np.float32)).astype(np.float64)

    def _act(self, h):
        a = self.spec.activation
        if a == "relu":
            return np.maximum(h, 0.0)
        if a == "silu":
            return h / (1.0 + np.exp(-h))
        if a == "leaky_relu":
            return np.where(h >= 0.0, h, self.slope * h)
        raise ValueError(a)

    def mlp(self, x, mpos: int, bf16: bool = False):
        """Rows x [R, in] through member position ``mpos``: mean [R, out], clamped logvar [R, out] (None if
        deterministic)."""
        W, b = (self.Wb, self.bb) if bf16 else (self.W, self.b)
        h = x
        nl = len(W)
        for li in range(nl):
            if bf16:
                h = bf16_round(h)
            h = h @ W[li][mpos] + b[li][mpos]
            if li < nl - 1:
                h = self._act(h)
        out = self.spec.out_size
        if self.spec.deterministic:
            return h, None
        mean, lv = h[:, :out], h[:, out:]
        lv = self.max_lv - _softplus(self.max_lv - lv)
        lv = self.min_lv + _softplus(lv - self.min_lv)
        return mean, lv

    # ---- the step ---------------------------------------------------------------------------------------------
    def step(self, obs, act, members, eps, sample: bool = True, bf16: bool = False):
        """obs [R, D] (fp32 values), act [R, A], members [R] member positions (index into the elite list) or None for
        expectation, eps [R, out] or None.  Returns next_obs [R, D] and the learned reward [R] (None without one),
        float64."""
        sp = self.spec
        x = self.model_input(obs, act)
        R = x.shape[0]
        if members is None:
            means, lvs = zip(*[self.mlp(x, m, bf16) for m in range(len(self.members))])
            mean = np.mean(means, axis=0)
            lv = None if lvs[0] is None else np.mean(lvs, axis=0)
        else:
            members = np.asarray(members)
            mean = np.empty((R, sp.out_size))
            lv = None if sp.deterministic else np.empty((R, sp.out_size))
            for m in np.unique(members):
                rows = np.nonzero(members == m)[0]
                mm, ll = self.mlp(x[rows], int(m), bf16)
                mean[rows] = mm
                if lv is not None:
                    lv[rows] = ll
        if sp.deterministic or not sample:
            preds = mean
        else:
            preds = mean + np.sqrt(np.exp(lv)) * np.asarray(eps, dtype=np.float64)
        nobs = preds[:, :sp.obs_dim]
        if self.target_is_delta:
            o = np.asarray(obs, dtype=np.float32).astype(np.float64)
            keep = np.ones(sp.obs_dim, bool)
            keep[list(self.no_delta)] = False
            nobs = np.where(keep, nobs + o, nobs)
        rew = preds[:, -1] if sp.learned_rewards else None
        return nobs, rew


def known_reward(name: str, act, next_obs) -> np.ndarray:
    """``pets_oracle.REWARD_FNS[name]`` in float64 on the kernel's fp32 next observations: [R]."""
    from . import pets_oracle as po

    a = torch.from_numpy(np.asarray(act, dtype=np.float32).astype(np.float64))
    o = torch.from_numpy(np.asarray(next_obs, dtype=np.float32).astype(np.float64))
    return po.REWARD_FNS[name](a, o).double().numpy().reshape(-1)


def known_done(name: str, act, next_obs) -> np.ndarray:
    """``pets_oracle.TERM_FNS[name]`` on fp32 tensors, as the reference applies it: bool [R]."""
    from . import pets_oracle as po

    a = torch.from_numpy(np.asarray(act, dtype=np.float32))
    o = torch.from_numpy(np.asarray(next_obs, dtype=np.float32))
    return po.TERM_FNS[name](a, o).numpy().reshape(-1)


def assignment_from_perm(perm, num_members: int) -> np.ndarray:
    """Row -> member position of the reference's split of a permutation (gaussian_mlp.py:202-212): row perm[i] goes
    to member i // (B / M)."""
    perm = np.asarray(perm)
    B = perm.shape[0]
    out = np.empty(B, np.int64)
    out[perm] = np.arange(B) // (B // num_members)
    return out
