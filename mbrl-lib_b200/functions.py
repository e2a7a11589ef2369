"""Named reward / termination / observation-preprocessing functions and their kernel ids.

The reference passes these as Python callables (``reward_fn(act, next_obs)``, ``termination_fn(act,
next_obs)``, ``obs_process_fn(obs)``; mbrl/env/reward_fns.py, mbrl/env/termination_fns.py,
mbrl/env/pets_halfcheetah.py:91-121, mbrl/env/pets_cartpole.py:78-101).  The kernels implement the shipped
ones as device functions selected by id; :func:`resolve_reward` / :func:`resolve_term` map a callable (ours
or mbrl-lib's own, matched by module + name) to that id.  Anything else is "external": the kernels still
advance the model and the caller's callable is applied to their device tensors (per step in ``ModelEnv.step``, per
window of steps in ``ModelEnv.evaluate_action_sequences``).

The torch bodies below are the host-visible definitions of the same functions (used for external/hybrid
evaluation and by users who want the callables); they run on whatever device their inputs live on.
"""
from __future__ import annotations

import math
from typing import Callable, Dict, Optional

import torch

from . import _lib


def _named(kind: str, name: str):
    def deco(fn):
        fn.b200pets_kind = kind
        fn.b200pets_name = name
        return fn

    return deco


# ---- termination ------------------------------------------------------------------------------------------
@_named("term", "no_termination")
def no_termination(act, next_obs):
    return torch.zeros(next_obs.shape[0], 1, dtype=torch.bool, device=next_obs.device)


@_named("term", "cartpole")
def term_cartpole(act, next_obs):
    x, th = next_obs[:, 0], next_obs[:, 2]
    lim = 12 * 2 * math.pi / 360
    return (~((x > -2.4) & (x < 2.4) & (th > -lim) & (th < lim)))[:, None]


@_named("term", "inverted_pendulum")
def term_inverted_pendulum(act, next_obs):
    return (~(torch.isfinite(next_obs).all(-1) & (next_obs[:, 1].abs() <= 0.2)))[:, None]


@_named("term", "hopper")
def term_hopper(act, next_obs):
    ok = (torch.isfinite(next_obs).all(-1) & (next_obs[:, 1:].abs() < 100).all(-1)
          & (next_obs[:, 0] > 0.7) & (next_obs[:, 1].abs() < 0.2))
    return (~ok)[:, None]


@_named("term", "walker2d")
def term_walker2d(act, next_obs):
    h, a = next_obs[:, 0], next_obs[:, 1]
    return (~((h > 0.8) & (h < 2.0) & (a > -1.0) & (a < 1.0)))[:, None]


@_named("term", "ant")
def term_ant(act, next_obs):
    x = next_obs[:, 0]
    return (~(torch.isfinite(next_obs).all(-1) & (x >= 0.2) & (x <= 1.0)))[:, None]


@_named("term", "humanoid")
def term_humanoid(act, next_obs):
    z = next_obs[:, 0]
    return ((z < 1.0) | (z > 2.0))[:, None]


# ---- reward -----------------------------------------------------------------------------------------------
@_named("reward", "cartpole")
def reward_cartpole(act, next_obs):
    return (~term_cartpole(act, next_obs)).float().view(-1, 1)


@_named("reward", "inverted_pendulum")
def reward_inverted_pendulum(act, next_obs):
    return (~term_inverted_pendulum(act, next_obs)).float().view(-1, 1)


@_named("reward", "cartpole_pets")
def reward_cartpole_pets(act, next_obs):
    x0, th = next_obs[:, :1], next_obs[:, 1:2]
    ee = torch.cat([x0 - 0.6 * th.sin(), -0.6 * th.cos() - 0.6], dim=1)
    return (torch.exp(-(ee ** 2).sum(dim=1) / 0.36) - 0.01 * (act ** 2).sum(dim=1)).view(-1, 1)


@_named("reward", "halfcheetah")
def reward_halfcheetah(act, next_obs):
    return (next_obs[:, 0] - 0.1 * act.square().sum(dim=1)).view(-1, 1)


@_named("reward", "pusher")
def reward_pusher(act, next_obs):
    goal = torch.tensor([0.45, -0.05, -0.323], device=next_obs.device)
    tip, obj = next_obs[:, 14:17], next_obs[:, 17:20]
    cost = 0.5 * (tip - obj).abs().sum(dim=1) + 1.25 * (goal - obj).abs().sum(dim=1) + 0.1 * (act ** 2).sum(dim=1)
    return -cost.view(-1, 1)


# ---- observation pre-processing ---------------------------------------------------------------------------
@_named("proc", "halfcheetah")
def proc_halfcheetah(state):
    return torch.cat([state[..., 1:2], torch.sin(state[..., 2:3]), torch.cos(state[..., 2:3]), state[..., 3:]], dim=-1)


@_named("proc", "cartpole")
def proc_cartpole(state):
    return torch.cat([torch.sin(state[..., 1:2]), torch.cos(state[..., 1:2]), state[..., :1], state[..., 2:]], dim=-1)


REWARD_FNS: Dict[str, Callable] = {"cartpole": reward_cartpole, "cartpole_pets": reward_cartpole_pets,
                                   "inverted_pendulum": reward_inverted_pendulum, "halfcheetah": reward_halfcheetah,
                                   "pusher": reward_pusher}
TERM_FNS: Dict[str, Callable] = {"no_termination": no_termination, "cartpole": term_cartpole,
                                 "inverted_pendulum": term_inverted_pendulum, "hopper": term_hopper,
                                 "walker2d": term_walker2d, "ant": term_ant, "humanoid": term_humanoid}
OBS_PROCESS_FNS: Dict[Optional[str], Optional[Callable]] = {None: None, "halfcheetah": proc_halfcheetah,
                                                            "cartpole": proc_cartpole}


def _ref_name(fn, module_suffix: str, table) -> Optional[str]:
    """Name of an mbrl-lib callable (e.g. ``mbrl.env.reward_fns.halfcheetah``) if it is one the kernels know."""
    mod = getattr(fn, "__module__", "") or ""
    name = getattr(fn, "__name__", "")
    if mod.endswith(module_suffix) and name in table:
        return name
    return None


def resolve_reward(fn) -> int:
    if fn is None:
        return _lib.REWARD["learned"]
    if getattr(fn, "b200pets_kind", None) == "reward":
        return _lib.REWARD[fn.b200pets_name]
    name = _ref_name(fn, "reward_fns", _lib.REWARD)
    return _lib.REWARD[name] if name else _lib.REWARD["external"]


def resolve_term(fn) -> int:
    if getattr(fn, "b200pets_kind", None) == "term":
        return _lib.TERM[fn.b200pets_name]
    name = _ref_name(fn, "termination_fns", _lib.TERM)
    return _lib.TERM[name] if name else _lib.TERM["external"]


def resolve_obs_process(fn) -> int:
    if fn is None:
        return _lib.PROC[None]
    if getattr(fn, "b200pets_kind", None) == "proc":
        return _lib.PROC[fn.b200pets_name]
    qual = getattr(fn, "__qualname__", "")
    if "HalfCheetahEnv." in qual and "preprocess" in qual:
        return _lib.PROC["halfcheetah"]
    if "CartPoleEnv." in qual and "preprocess" in qual:
        return _lib.PROC["cartpole"]
    raise NotImplementedError(
        f"obs_process_fn {fn!r} has no device implementation (known: HalfCheetahEnv.preprocess_fn, "
        "CartPoleEnv.preprocess_fn); the fused path needs it inside the kernel")
