"""CPU checks for evaluations with reward / termination callables the kernels do not know."""
import dataclasses

import numpy as np
import pytest
import torch

from mbrl_lib_b200 import synthetic as syn
from mbrl_lib_b200.model_env import TRAJECTORY_WINDOW_BYTES, trajectory_window


def _window_bytes(batch, obs_dim, act_dim, steps):
    return steps * batch * (4 * obs_dim + 4 * act_dim + 4 + 1)


@pytest.mark.parametrize("batch,obs_dim,act_dim,horizon", [
    (10000, 17, 6, 30),        # PETS HalfCheetah (pop 500 x 20 particles): the whole horizon in one window
    (20000, 45, 17, 40),       # iCEM Humanoid, truncated observation
    (20000, 376, 17, 40),      # iCEM Humanoid-v4 dims
    (1280000, 17, 6, 30),      # 64 000 sequences x 20 particles
    (2000000, 376, 17, 100),   # one step alone is above the budget
    (1, 1, 1, 1), (4, 1, 1, 1000)])
def test_trajectory_window_rule(batch, obs_dim, act_dim, horizon):
    T = trajectory_window(batch, obs_dim, act_dim, horizon)
    assert 1 <= T <= horizon
    if _window_bytes(batch, obs_dim, act_dim, 1) <= TRAJECTORY_WINDOW_BYTES:
        assert _window_bytes(batch, obs_dim, act_dim, T) <= TRAJECTORY_WINDOW_BYTES
        # as long as possible: one more step would leave the budget (or the horizon)
        assert T == horizon or _window_bytes(batch, obs_dim, act_dim, T + 1) > TRAJECTORY_WINDOW_BYTES
    else:
        assert T == 1
    if (batch, obs_dim, horizon) == (10000, 17, 30):
        assert T == horizon


def test_trajectory_window_budget_argument():
    assert trajectory_window(100, 10, 2, 50, budget=0) == 1
    per_step = 100 * (4 * 10 + 4 * 2 + 5)
    assert trajectory_window(100, 10, 2, 50, budget=7 * per_step) == 7
    assert trajectory_window(100, 10, 2, 50, budget=7 * per_step - 1) == 6


def test_custom_termination_is_reached(monkeypatch):
    """The bound termination of tests/test_gpu_callables.py::test_custom_functions_match_oracle ends part of the
    rollouts of its inputs early and leaves the others running, so that test exercises the masking."""
    from oracle import pets_oracle as po
    from test_gpu_callables import bound_termination, goal_reward

    monkeypatch.setitem(po.REWARD_FNS, "test_goal", goal_reward)
    monkeypatch.setitem(po.TERM_FNS, "test_bound", bound_termination)
    spec = dataclasses.replace(syn.CASES["halfcheetah"], reward_fn="test_goal", term_fn="test_bound")
    arrays = syn.make_model_arrays(spec)
    inp = syn.make_rollout_inputs(spec)
    m = po.OracleModel(spec, arrays)
    B = spec.batch
    obs = torch.from_numpy(np.tile(inp["obs0"], (B, 1)).astype(np.float32))
    dead = torch.zeros(B, 1, dtype=torch.bool)
    first = np.full(B, -1)
    with torch.no_grad():
        for t in range(spec.horizon):
            a = torch.repeat_interleave(torch.from_numpy(inp["actions"][:, t]), spec.particles, dim=0)
            obs, _, done = m.step(obs, a, torch.from_numpy(inp["perms"][t]), torch.from_numpy(inp["eps"][t]))
            first[(done[:, 0] & ~dead[:, 0]).numpy()] = t
            dead |= done
    frac = dead.float().mean().item()
    print(f"{frac:.3f} of the rows terminate; first terminations at steps {np.unique(first[first >= 0])[:10]}")
    assert 0.1 < frac < 0.9, frac
    assert (first > 0).any()  # some rows run a while before they terminate
