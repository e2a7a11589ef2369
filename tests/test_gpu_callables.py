"""Reward and termination callables the kernels do not know (``functions.resolve_* == "external"``).

``ModelEnv.evaluate_action_sequences`` then rolls the model out in windows of steps (b200pets_eval_trajectory writes
every step's next observation), calls the callables once per window on all of its rows, and applies the reference's
termination masking and sums on the device (b200pets_trajectory_returns).  Checked here:

* the existing parity cases, with their reward / termination wrapped in plain lambdas, against the same goldens and
  oracle at the same bars as tests/test_gpu_parity.py;
* lambda against in-kernel function with the same Philox keys: bit-identical returns where only the termination is a
  callable or the reward derives from the termination, within 1e-5 of scale for continuous rewards;
* splitting the horizon into windows changes nothing, bit for bit;
* functions the kernels do not have (a goal-distance reward, a bound termination) against the oracle, also under tile
  shuffle with the exported member map;
* the agent: CEM's closed loop reaches the goal with a custom reward, iCEM and MPPI return valid actions;
* the reference's own ModelEnv with the same lambdas and draws.
"""
import dataclasses
import os

import numpy as np
import pytest
import torch

from mbrl_lib_b200 import synthetic as syn
from test_gpu_parity import (CONTINUOUS, DEV, DISCRETE, TC_CONTINUOUS, _Env, assert_close_continuous,
                             assert_close_discrete, gpu_returns, oracle_returns)

pytestmark = pytest.mark.gpu

TC_DISCRETE = ["cartpole", "hopper_tsinf", "walker_ant", "ant_learned_fn", "relu_expectation"]


def _wrap(fn):
    """A plain lambda around ``fn``: resolves to "external", so the kernels cannot run it."""
    return None if fn is None else (lambda act, next_obs: fn(act, next_obs))


def make_env(name, precision, ts1="perms", reward=True, term=True, spec=None, arrays=None):
    """The parity case ``name`` with its reward (``reward``) and / or termination (``term``) as lambdas."""
    import mbrl_lib_b200 as bp
    from mbrl_lib_b200 import functions

    spec = spec or syn.CASES[name]
    arrays = arrays if arrays is not None else syn.make_model_arrays(spec)
    model = bp.model_from_arrays(spec, arrays, DEV)
    rew = functions.REWARD_FNS[spec.reward_fn] if spec.reward_fn else None
    trm = functions.TERM_FNS[spec.term_fn]
    env = bp.ModelEnv(_Env(spec), model, _wrap(trm) if term else trm, _wrap(rew) if reward else rew,
                      generator=torch.Generator(device=DEV), precision=precision, ts1=ts1)
    return spec, arrays, env


# ---- 1. existing goldens through callables -----------------------------------------------------------------
@pytest.mark.parametrize("name", CONTINUOUS)
def test_callables_f32_match_oracle_and_golden(golden_dir, name):
    spec, arrays, env = make_env(name, "f32")
    assert env.has_external_callables()
    inp = syn.make_rollout_inputs(spec)
    got = gpu_returns(env, spec, inp)
    assert_close_continuous(got, oracle_returns(spec, arrays, inp), 2e-4)
    gold = np.load(os.path.join(golden_dir, f"rollout_{name}.npz"))
    assert str(gold["input_sum"]) == syn.checksum(inp)
    assert_close_continuous(got, gold["returns"], 2e-4)


@pytest.mark.parametrize("name", DISCRETE)
def test_callables_f32_discrete_rewards(golden_dir, name):
    spec, arrays, env = make_env(name, "f32")
    inp = syn.make_rollout_inputs(spec)
    got = gpu_returns(env, spec, inp)
    gold = np.load(os.path.join(golden_dir, f"rollout_{name}.npz"))
    assert_close_discrete(got, gold["returns"], spec.particles)


@pytest.mark.parametrize("name", TC_CONTINUOUS)
def test_callables_tc_match_oracle(golden_dir, name):
    spec, arrays, env = make_env(name, "bf16_tc")
    inp = syn.make_rollout_inputs(spec)
    got = gpu_returns(env, spec, inp)
    assert_close_continuous(got, oracle_returns(spec, arrays, inp, bf16=True), 5e-3)
    gold = np.load(os.path.join(golden_dir, f"rollout_{name}.npz"))
    assert_close_continuous(got, gold["returns"], 2e-2)


def _assert_tc_discrete(got, orc, gold):
    """The bars of test_gpu_parity.py::test_rollout_tc_discrete_rewards."""
    d_o = np.abs(got - orc)
    assert (d_o > 1e-2 * np.maximum(1.0, np.abs(orc))).mean() <= 0.01
    assert d_o.mean() <= 1e-4 * max(1.0, float(np.abs(orc).mean()))
    diff = np.abs(got - gold)
    assert (diff > 1e-2 * np.maximum(1.0, np.abs(gold))).mean() <= 0.06
    assert diff.mean() <= 5e-3 * max(1.0, np.abs(gold).mean())


@pytest.mark.parametrize("name", TC_DISCRETE)
def test_callables_tc_discrete_rewards(golden_dir, name):
    spec, arrays, env = make_env(name, "bf16_tc")
    inp = syn.make_rollout_inputs(spec)
    got = gpu_returns(env, spec, inp)
    gold = np.load(os.path.join(golden_dir, f"rollout_{name}.npz"))
    _assert_tc_discrete(got, oracle_returns(spec, arrays, inp, bf16=True), gold["returns"])


# ---- 2. same draws as the in-kernel functions ----------------------------------------------------------------
# (case, how members are drawn): tile shuffle and explicit per-step permutations under TS1, TSinf with the in-kernel
# draw, expectation
SAME_DRAWS = [("halfcheetah_small", "tile_shuffle"), ("halfcheetah_small", "perms"), ("cartpole", "tile_shuffle"),
              ("cartpole", "perms"), ("hopper_tsinf", "tile_shuffle"), ("ant_learned_fn", "tile_shuffle"),
              ("silu_expectation", None), ("relu_expectation", None)]


@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
@pytest.mark.parametrize("name,mode", SAME_DRAWS)
def test_callables_use_the_in_kernel_draws(name, mode, precision):
    spec = syn.CASES[name]
    inp = syn.make_rollout_inputs(spec)
    acts = torch.from_numpy(inp["actions"]).to(DEV)
    perms = torch.from_numpy(inp["perms"]).to(DEV) if mode == "perms" else None
    offset = 13 * 1024

    def run(reward, term):
        _, _, env = make_env(name, precision, ts1="tile_shuffle", reward=reward, term=term)
        env._few_groups = lambda *a: False  # the in-kernel member draw also at these small populations
        rr = torch.empty(spec.batch, device=DEV)
        out = env.evaluate_action_sequences(acts, inp["obs0"], spec.particles, _perms=perms, _offset=offset, _row_returns=rr)
        torch.cuda.synchronize()
        return out.cpu().numpy(), rr.cpu().numpy()

    base, base_rows = run(False, False)
    assert np.isfinite(base).all()
    # only the termination is a callable: the kernel's reward column and the callable's done are the kernel's own
    got, rows = run(False, True)
    assert np.array_equal(got, base) and np.array_equal(rows, base_rows)
    if spec.reward_fn is None:
        return
    got, rows = run(True, True)
    if spec.reward_fn in ("cartpole", "inverted_pendulum"):  # rewards that derive from the termination rule
        assert np.array_equal(got, base) and np.array_equal(rows, base_rows)
    else:  # torch's arithmetic for the reward formula against the device function's
        assert_close_continuous(got, base, 1e-5)


# ---- 3. window invariance -------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
@pytest.mark.parametrize("name,mode", [("halfcheetah", "tile_shuffle"), ("halfcheetah_small", "perms"),
                                       ("hopper_tsinf", "tile_shuffle"), ("silu_expectation", None)])
def test_windows_are_bit_identical(name, mode, precision):
    spec, _, env = make_env(name, precision, ts1="tile_shuffle")
    env._few_groups = lambda *a: False
    H = max(spec.horizon, 12)  # windows of 7 steps leave a shorter last window
    inp = syn.make_rollout_inputs(spec, horizon=H)
    acts = torch.from_numpy(inp["actions"]).to(DEV)
    perms = torch.from_numpy(inp["perms"]).to(DEV) if mode == "perms" else None
    out = {}
    for w in (1, 7, H):
        rr = torch.empty(spec.batch, device=DEV)
        ret = env.evaluate_action_sequences(acts, inp["obs0"], spec.particles, _perms=perms, _offset=17 * 1024,
                                            _row_returns=rr, _window=w)
        torch.cuda.synchronize()
        out[w] = (ret.cpu().numpy(), rr.cpu().numpy())
    for w in (1, 7):
        assert np.array_equal(out[w][0], out[H][0]), w
        assert np.array_equal(out[w][1], out[H][1]), w
    assert np.isfinite(out[H][0]).all()


# ---- 4. functions the kernels do not have ----------------------------------------------------------------------
GOAL = torch.tensor([0.5, -0.25, 0.75])


def goal_reward(act, next_obs):
    """Negative distance of the first three observation words to a goal, minus an action cost."""
    d = next_obs[:, :3] - GOAL.to(next_obs.device)
    return -(d.square().sum(dim=1).sqrt() + 0.05 * act.square().sum(dim=1)).view(-1, 1)


def bound_termination(act, next_obs):
    """Ends an episode once the second observation word leaves [-0.8, 0.8]."""
    return (next_obs[:, 1].abs() > 0.8).view(-1, 1)


@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
@pytest.mark.parametrize("ts1", ["tile_shuffle", "perms"])
def test_custom_functions_match_oracle(monkeypatch, precision, ts1):
    import mbrl_lib_b200 as bp
    from oracle import pets_oracle as po

    monkeypatch.setitem(po.REWARD_FNS, "test_goal", goal_reward)
    monkeypatch.setitem(po.TERM_FNS, "test_bound", bound_termination)
    spec = dataclasses.replace(syn.CASES["halfcheetah"], reward_fn="test_goal", term_fn="test_bound")
    arrays = syn.make_model_arrays(spec)
    env = bp.ModelEnv(_Env(spec), bp.model_from_arrays(spec, arrays, DEV), bound_termination, goal_reward,
                      generator=torch.Generator(device=DEV), precision=precision, ts1=ts1)
    assert env.has_external_callables()
    env._few_groups = lambda *a: False
    inp = syn.make_rollout_inputs(spec)
    acts = torch.from_numpy(inp["actions"]).to(DEV)
    eps = torch.from_numpy(inp["eps"]).to(DEV)
    offset = 19 * 1024
    oracle = po.OracleModel(spec, arrays)
    oracle.emulate_bf16 = precision == "bf16_tc"
    if ts1 == "perms":
        got = env.evaluate_action_sequences(acts, inp["obs0"], spec.particles, _perms=torch.from_numpy(inp["perms"]).to(DEV),
                                            _eps=eps, _offset=offset)
        ref = oracle.evaluate_action_sequences(torch.from_numpy(inp["actions"]), inp["obs0"], spec.particles,
                                               torch.from_numpy(inp["perms"]), torch.from_numpy(inp["eps"]))
    else:
        # the particles of a sequence sit in different shuffle groups and draw their members independently
        got = env.evaluate_action_sequences(acts, inp["obs0"], spec.particles, _eps=eps, _offset=offset)
        assign = env.shuffle_member_assignment(spec.population, spec.horizon, spec.particles, offset)
        ref = oracle.evaluate_action_sequences(torch.from_numpy(inp["actions"]), inp["obs0"], spec.particles, None,
                                               torch.from_numpy(inp["eps"]), assign=assign)
    torch.cuda.synchronize()
    got, ref = got.cpu().numpy(), ref.numpy()
    assert np.isfinite(got).all()  # (tests/test_callables_cpu.py: the bound ends part of these rollouts early)
    if precision == "f32":
        assert_close_discrete(got, ref, spec.particles)
    else:  # a state near the bound may flip a particle at bf16 (same rule as the tensor-core discrete cases)
        d_o = np.abs(got - ref)
        assert (d_o > 1e-2 * np.maximum(1.0, np.abs(ref))).mean() <= 0.02
        assert d_o.mean() <= 1e-3 * max(1.0, float(np.abs(ref).mean()))


# ---- 5. the agent ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
def test_closed_loop_mpc_with_custom_reward_reaches_goal(precision):
    """test_gpu_scale.py::test_closed_loop_mpc_reaches_goal with the reward given as a lambda: agent.act runs CEM's
    per-iteration loop over the windowed evaluation."""
    import mbrl_lib_b200 as bp
    from mbrl_lib_b200 import functions
    from test_gpu_parity import _Env as Env
    from test_gpu_scale import _line_world

    class _Spec:
        obs_dim, act_dim, action_lb, action_ub = 1, 1, -1.0, 1.0

    env = bp.ModelEnv(Env(_Spec), _line_world(DEV), functions.no_termination, lambda act, next_obs: -next_obs.abs(),
                      generator=torch.Generator(device=DEV), precision=precision, ts1="tile_shuffle")
    assert env.has_external_callables()
    cfg = {"_target_": "mbrl.planning.TrajectoryOptimizerAgent", "planning_horizon": 5, "replan_freq": 1,
           "optimizer_cfg": {"_target_": "mbrl.planning.CEMOptimizer", "num_iterations": 4, "elite_ratio": 0.1,
                             "population_size": 256, "alpha": 0.1, "device": DEV, "return_mean_elites": True}}
    agent = bp.create_trajectory_optim_agent_for_model(env, cfg, num_particles=2)
    pos, total = 1.0, 0.0
    for _ in range(18):
        a = float(np.clip(agent.act(np.array([pos])), -1, 1)[0])
        pos = pos + 0.1 * a
        total += -abs(pos)
    assert abs(pos) < 0.12, pos
    assert total > -7.5, total


@pytest.mark.parametrize("optimizer", ["ICEMOptimizer", "MPPIOptimizer"])
def test_icem_and_mppi_agents_with_callables(optimizer):
    import mbrl_lib_b200 as bp

    spec, _, env = make_env("halfcheetah_small", "auto", ts1="tile_shuffle")
    assert env.has_external_callables()
    opt = {"ICEMOptimizer": {"num_iterations": 3, "elite_ratio": 0.1, "population_size": 100, "population_decay_factor": 1.3,
                             "colored_noise_exponent": 2.0, "keep_elite_frac": 0.3, "alpha": 0.1, "return_mean_elites": True},
           "MPPIOptimizer": {"num_iterations": 3, "population_size": 100, "gamma": 0.9, "sigma": 1.0, "beta": 0.9}}[optimizer]
    cfg = {"_target_": "mbrl.planning.TrajectoryOptimizerAgent", "planning_horizon": spec.horizon, "replan_freq": 1,
           "verbose": False, "optimizer_cfg": {"_target_": f"mbrl.planning.{optimizer}", "device": DEV, **opt}}
    agent = bp.create_trajectory_optim_agent_for_model(env, cfg, num_particles=spec.particles)
    obs0 = syn.make_rollout_inputs(spec, with_noise=False)["obs0"]
    for _ in range(2):
        a = agent.act(obs0)
        assert a.shape == (spec.act_dim,) and np.isfinite(a).all()
        assert (a >= spec.action_lb - 1e-6).all() and (a <= spec.action_ub + 1e-6).all()


# ---- 6. the reference itself -----------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["halfcheetah_small", "cartpole", "hopper_tsinf", "pets_halfcheetah_small", "ant_learned_fn"])
@pytest.mark.parametrize("precision,tol", [("f32", 2e-4), ("bf16_tc", 2e-2)])
def test_reference_model_env_with_callables(name, precision, tol):
    """The reference's ModelEnv and ours on the same real reference model, both with the reference's own reward /
    termination functions wrapped in lambdas, fed the same draws (test_reference_objects.py's bars)."""
    import mbrl_lib_b200 as bp
    from test_reference_objects import _Feed, _real_model, mbrl

    if mbrl is None:
        pytest.skip("reference not importable here")
    spec, arrays, ref_env = _real_model(name, DEV)
    rew, trm = _wrap(ref_env.reward_fn), _wrap(ref_env.termination_fn)
    ref_env.reward_fn, ref_env.termination_fn = rew, trm
    inp = syn.make_rollout_inputs(spec)
    acts = torch.from_numpy(inp["actions"]).to(DEV)
    perms = torch.from_numpy(inp["perms"]).to(DEV)
    eps = torch.from_numpy(inp["eps"]).to(DEV)
    feed_perms = [] if spec.propagation == "expectation" else [perms[t] for t in range(perms.shape[0])]
    feed_norm = [] if spec.deterministic else [eps[t] for t in range(spec.horizon)]
    with _Feed(feed_perms, feed_norm):
        want = ref_env.evaluate_action_sequences(acts, inp["obs0"], spec.particles).float().cpu().numpy()
    env = bp.ModelEnv(ref_env, ref_env.dynamics_model, trm, rew, generator=torch.Generator(device=DEV),
                      precision=precision, ts1="perms")
    assert env.has_external_callables()
    if precision == "bf16_tc" and not env.staged.supports_tc():
        pytest.skip("dims outside the tensor-core plan")
    got = env.evaluate_action_sequences(acts, inp["obs0"], spec.particles, _perms=perms, _eps=eps).cpu().numpy()
    scale = max(1.0, float(np.abs(want).max()))
    if spec.term_fn != "no_termination" or spec.reward_fn in ("cartpole",):
        frac = float((np.abs(got - want) > tol * scale).mean())
        assert frac <= 0.02, f"{frac:.3f} of sequences differ"
    else:
        np.testing.assert_allclose(got, want, atol=tol * scale, rtol=0)
