"""Staging a ``OneDTransitionRewardModel(GaussianMLP)`` or ``OneDTransitionRewardModel(BasicEnsemble)`` for the kernels
(``b200pets_model_create``).

Reads the live ``nn.Parameter`` s / normaliser tensors of the user's model object (mbrl-lib's or the
containers in :mod:`models`), never copies them to the host, and keeps the packed device copy as a cache
keyed on (parameter storage, version counters, elite list, normaliser tensor identity) because
``ModelTrainer.train`` mutates weights in place and ``Normalizer.update_stats`` *replaces* its tensors
between ``act()`` calls (mbrl/models/model_trainer.py:153,288-296; mbrl/util/math.py:114-127).

A BasicEnsemble (``model.members``: E one-member GaussianMLPs) is staged from a stacked ``[E, K, N]`` device copy of its
members' layers that this object owns, refreshed by device-to-device copies when the signature changes; its rows pick
their member by index (``B200PETS_MEMBER_ROWS``): every member is used and there is no elite list
(basic_ensemble.py:262-266).
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional

import numpy as np
import torch

from . import _lib, functions


def mark_trained(mlp):
    """Record that kernels rewrote ``mlp``'s parameters in place: their writes bypass torch's ``_version`` counters, so
    :class:`mbrl_lib_b200.ModelTrainer` bumps this count, which every staged copy's signature includes."""
    mlp._b200pets_trained = getattr(mlp, "_b200pets_trained", 0) + 1


def _is_member_list(model) -> bool:
    members = getattr(model, "members", None)
    return members is not None and len(members) > 0 and all(
        hasattr(m, "hidden_layers") and hasattr(m, "mean_and_logvar") for m in members)


def _check_members(members) -> None:
    """The BasicEnsembles the kernels cover: one-member GaussianMLPs of one shape, activation and ``deterministic``
    flag, and (probabilistic members) equal log-variance bounds."""
    m0 = members[0]
    def shape(m):
        return ([tuple(seq[0].weight.shape) for seq in m.hidden_layers] + [tuple(m.mean_and_logvar.weight.shape)],
                type(m.hidden_layers[0][1]).__name__, getattr(m.hidden_layers[0][1], "negative_slope", None),
                bool(m.deterministic))
    for i, m in enumerate(members):
        if int(m.mean_and_logvar.weight.shape[0]) != 1:
            raise NotImplementedError(f"BasicEnsemble member {i} has ensemble_size {int(m.mean_and_logvar.weight.shape[0])}; "
                                      "the fused path covers one-member GaussianMLPs")
        if shape(m) != shape(m0):
            raise NotImplementedError(f"BasicEnsemble member {i} differs from member 0 in layer shapes, activation or "
                                      "deterministic; the fused path needs identical members")
    if not m0.deterministic:
        for i, m in enumerate(members[1:], 1):
            if not (torch.equal(m.min_logvar.detach(), m0.min_logvar.detach())
                    and torch.equal(m.max_logvar.detach(), m0.max_logvar.detach())):
                raise NotImplementedError(f"BasicEnsemble member {i} has log-variance bounds other than member 0's "
                                          "(learn_logvar_bounds=True); the fused path needs equal bounds")


def _activation_of(module) -> tuple:
    name = type(module).__name__
    if name == "ReLU":
        return _lib.ACT["relu"], 0.0
    if name == "SiLU":
        return _lib.ACT["silu"], 0.0
    if name == "LeakyReLU":
        return _lib.ACT["leaky_relu"], float(module.negative_slope)
    raise NotImplementedError(f"activation {name} has no device implementation (known: ReLU, SiLU, LeakyReLU)")


class StagedModel:
    """Owns the C handle of one staged model and re-stages it when the source object changed."""

    member_mlps: Optional[List] = None  # BasicEnsemble: its member GaussianMLPs (None: a GaussianMLP ensemble)
    _stacked: Optional[List[torch.Tensor]] = None  # BasicEnsemble: [E, K, N] weights and [E, 1, N] biases per layer

    def __init__(self, dynamics_model, reward_fn=None, termination_fn=None, stage: bool = True):
        """``stage=False`` only reads the source object (description, layer list, members, signature) and touches
        neither the library nor a device: that is how the duck-typing contract is checked against real
        ``mbrl.models`` objects on a CPU-only host (tests/test_reference_objects.py)."""
        self.lib = _lib.load() if stage else None
        self.src = dynamics_model
        mlp = getattr(dynamics_model, "model", None)
        self.member_mlps = list(mlp.members) if mlp is not None and _is_member_list(mlp) else None
        if self.member_mlps is None and (mlp is None or not hasattr(mlp, "hidden_layers") or not hasattr(mlp, "mean_and_logvar")):
            raise NotImplementedError(
                "the fused path covers OneDTransitionRewardModel(GaussianMLP) and OneDTransitionRewardModel(BasicEnsemble); got "
                f"{type(dynamics_model).__name__}({type(mlp).__name__ if mlp is not None else None})")
        if self.member_mlps is not None:
            _check_members(self.member_mlps)
        self.mlp = mlp
        head = self.member_mlps[0] if self.member_mlps is not None else mlp
        dev = torch.device(head.mean_and_logvar.weight.device)
        if stage and dev.type != "cuda":
            raise RuntimeError(f"b200pets runs on a CUDA device; the model lives on {dev} (no CPU fallback)")
        self.device = dev
        self.reward_id = functions.resolve_reward(reward_fn)
        self.term_id = functions.resolve_term(termination_fn) if termination_fn is not None else _lib.TERM["no_termination"]
        self.handle: Optional[C.c_void_p] = None
        self._sig = None
        self._structure = None
        if stage:
            self.ensure_fresh()

    # ---- description -----------------------------------------------------------------------------------
    @property
    def member_rule(self) -> str:
        """"rows" for a BasicEnsemble (``perms`` carries per-row member indices), "perm" for a GaussianMLP ensemble."""
        return "rows" if self.member_mlps is not None else "perm"

    def _head(self):
        """The GaussianMLP whose layer shapes, activation and logvar bounds describe the model."""
        return self.member_mlps[0] if self.member_mlps is not None else self.mlp

    @staticmethod
    def _mlp_layers(mlp) -> List:
        return [seq[0] for seq in mlp.hidden_layers] + [mlp.mean_and_logvar]

    def _layers(self) -> List:
        return self._mlp_layers(self._head())

    def members(self) -> List[int]:
        if self.member_mlps is not None:
            return list(range(len(self.member_mlps)))
        el = getattr(self.mlp, "elite_models", None)
        return list(el) if el is not None else list(range(int(self.mlp.num_members)))

    def _describe(self) -> _lib.ModelDesc:
        m, w = self._head(), self.src
        layers = self._layers()
        act, slope = _activation_of(m.hidden_layers[0][1])
        d = _lib.ModelDesc()
        d.ensemble_size = len(self.member_mlps) if self.member_mlps is not None else int(layers[0].weight.shape[0])
        d.member_rule = _lib.MEMBER_RULE[self.member_rule]
        d.num_members = len(self.members())
        d.in_size = int(m.in_size)
        d.out_size = int(m.out_size)
        d.hid_size = int(layers[0].weight.shape[2])
        d.num_hidden = len(layers) - 1
        d.activation, d.leaky_slope = act, slope
        d.obs_process = functions.resolve_obs_process(getattr(w, "obs_process_fn", None))
        d.learned_rewards = int(bool(w.learned_rewards))
        d.target_is_delta = int(bool(w.target_is_delta))
        d.deterministic = int(bool(m.deterministic))
        d.obs_dim = d.out_size - d.learned_rewards
        d.act_dim = d.in_size - d.obs_dim - (1 if d.obs_process == _lib.PROC["cartpole"] else 0)
        d.reward_fn = self.reward_id
        d.term_fn = self.term_id
        norm = getattr(w, "input_normalizer", None)
        d.norm_mode = 0 if norm is None else (2 if norm.mean.dtype == torch.float64 else 1)
        if not d.learned_rewards and d.reward_fn == _lib.REWARD["learned"]:
            raise ValueError("reward_fn is None but the model does not learn rewards")
        return d

    def _signature(self):
        sig = []
        for mlp in (self.member_mlps if self.member_mlps is not None else [self.mlp]):
            for layer in self._mlp_layers(mlp):
                for p in (layer.weight, layer.bias):
                    sig.append((p.data_ptr(), p._version, tuple(p.shape)))
            if not mlp.deterministic:
                for p in (mlp.min_logvar, mlp.max_logvar):
                    sig.append((p.data_ptr(), p._version))
            if mlp is not self.mlp:
                sig.append(getattr(mlp, "_b200pets_trained", 0))
        norm = getattr(self.src, "input_normalizer", None)
        if norm is not None:
            sig.append((id(norm.mean), norm.mean.data_ptr(), norm.mean._version, id(norm.std), norm.std._version))
        sig.append(tuple(self.members()))
        sig.append(getattr(self.mlp, "_b200pets_trained", 0))
        return tuple(sig)

    # ---- staging ---------------------------------------------------------------------------------------
    def ensure_fresh(self):
        sig = self._signature()
        if sig == self._sig:
            return
        if self.member_mlps is not None and self._sig is not None:
            _check_members(self.member_mlps)
        desc = self._describe()
        structure = tuple(getattr(desc, f[0]) for f in desc._fields_) + tuple(getattr(self.src, "no_delta_list", []) or [])
        mlps = self.member_mlps if self.member_mlps is not None else [self.mlp]
        for mlp in mlps:
            for layer in self._mlp_layers(mlp):
                for p in (layer.weight, layer.bias):
                    if p.dtype != torch.float32 or not p.is_contiguous() or p.device != self.device:
                        raise ValueError("ensemble weights must be contiguous float32 tensors on one CUDA device")
        if self.member_mlps is not None:
            ptrs = self._stack_members()
        else:
            ptrs = [(layer.weight.data_ptr(), layer.bias.data_ptr()) for layer in self._layers()]
        n = len(ptrs)
        W = (C.c_void_p * n)(*[w for w, _ in ptrs])
        Bv = (C.c_void_p * n)(*[b for _, b in ptrs])
        members = self.members()
        mem = (C.c_int32 * len(members))(*members)
        norm = getattr(self.src, "input_normalizer", None)
        nm = ns = None
        if norm is not None:
            nm_np = np.ascontiguousarray(norm.mean.detach().double().cpu().numpy().reshape(-1))
            ns_np = np.ascontiguousarray(norm.std.detach().double().cpu().numpy().reshape(-1))
            nm = nm_np.ctypes.data_as(C.POINTER(C.c_double))
            ns = ns_np.ctypes.data_as(C.POINTER(C.c_double))
        mn = mx = None
        head = self._head()
        if not head.deterministic:
            mn_np = np.ascontiguousarray(head.min_logvar.detach().float().cpu().numpy().reshape(-1))
            mx_np = np.ascontiguousarray(head.max_logvar.detach().float().cpu().numpy().reshape(-1))
            mn = mn_np.ctypes.data_as(C.POINTER(C.c_float))
            mx = mx_np.ctypes.data_as(C.POINTER(C.c_float))
        with torch.cuda.device(self.device):
            stream = _lib.stream_ptr()  # the model's device's current stream, not the caller's current device's
            if self.handle is not None and structure == self._structure:
                _lib.check(self.lib.b200pets_model_refresh(self.handle, W, Bv, mem, nm, ns, mn, mx, stream), "model_refresh")
            else:
                self.close()
                nd = list(getattr(self.src, "no_delta_list", []) or [])
                nd_arr = (C.c_int32 * max(len(nd), 1))(*nd)
                h = C.c_void_p()
                _lib.check(self.lib.b200pets_model_create(C.byref(desc), W, Bv, mem, nm, ns, mn, mx, nd_arr, len(nd), stream,
                                                          C.byref(h)), "model_create")
                self.handle = h
                self._structure = structure
        self.desc = desc
        self._sig = sig

    def _stack_members(self) -> List[tuple]:
        """Copy every member's layers into this object's stacked ``[E, K, N]`` / ``[E, 1, N]`` device tensors (device to
        device, on the model's device's current stream); returns their (weight, bias) pointers per layer."""
        E = len(self.member_mlps)
        per = [self._mlp_layers(m) for m in self.member_mlps]
        if self._stacked is None or [tuple(t.shape) for t in self._stacked] != [
                (E, *tuple(p.shape)[1:]) for layer in per[0] for p in (layer.weight, layer.bias)]:
            self._stacked = [torch.empty((E, *tuple(p.shape)[1:]), dtype=torch.float32, device=self.device)
                             for layer in per[0] for p in (layer.weight, layer.bias)]
        with torch.no_grad(), torch.cuda.device(self.device):
            for li in range(len(per[0])):
                torch.cat([p[li].weight for p in per], dim=0, out=self._stacked[2 * li])
                torch.cat([p[li].bias for p in per], dim=0, out=self._stacked[2 * li + 1])
        return [(self._stacked[2 * li].data_ptr(), self._stacked[2 * li + 1].data_ptr()) for li in range(len(per[0]))]

    def supports_tc(self, propagation: Optional[str] = None) -> bool:
        """Whether the tensor-core kernel covers this model; with ``propagation``, whether it has a launch plan for
        that propagation method ("expectation" needs more shared memory than the other two)."""
        if propagation is None:
            return bool(self.lib.b200pets_model_supports_tc(self.handle))
        return self.plan_info(propagation)["kslice"] > 0

    def plan_info(self, propagation: str) -> dict:
        """Launch plans of the rollout kernels for this model on the current device (``b200pets_model_plan_info``)."""
        info = (C.c_int32 * 4)()
        with torch.cuda.device(self.device):
            _lib.check(self.lib.b200pets_model_plan_info(self.handle, _lib.PROP[propagation], info), "model_plan_info")
        return {"kslice": info[0], "nstages": info[1], "tc_smem": info[2], "f32_rows": info[3]}

    def close(self):
        if self.handle is not None:
            self.lib.b200pets_model_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
