"""Planning for a batch of observations: K independent problems in one call.

Problem k of a batched evaluation or CEM plan gives, bit for bit, what the single call gives for its inputs made with
the Philox offset the batch assigns to it (evaluation: ``offset + k * 1024``; plan: counter ``offset + k``).  A batch
may run a different CTA shape from the single calls (the shape follows the total tile count), which a row's results do
not depend on, so equality here also covers 64-row against 128-row CTAs and launches with more tiles than SMs.
"""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

from mbrl_lib_b200 import synthetic as syn
from test_gpu_parity import DEV, make_env
from test_gpu_scale import _line_world
from test_gpu_tiles import _sm_count, _tc_tiles

pytestmark = pytest.mark.gpu


def _problems(spec, K, seed=0):
    """K different initial states and action sequences of ``spec``'s shape."""
    g = np.random.default_rng(seed)
    inp = syn.make_rollout_inputs(spec, with_noise=False)
    obs = np.stack([inp["obs0"] + (0.1 * k) * g.standard_normal(spec.obs_dim) for k in range(K)])
    acts = g.uniform(spec.action_lb, spec.action_ub, (K, spec.population, spec.horizon, spec.act_dim)).astype(np.float32)
    return obs, torch.from_numpy(acts).to(DEV)


# name, propagation mode, horizon: TS1 with tile shuffle, TS1 with injected permutations (and noise), TSinf with an
# injected permutation, expectation, and a synthetic model with an odd hidden width (143)
EVAL_CASES = [("halfcheetah", "tile_shuffle", 6), ("halfcheetah", "perms", 4), ("hopper_tsinf", "perms", None),
              ("silu_expectation", "expectation", None), ("plan_hid143", "tile_shuffle", None)]


@pytest.mark.parametrize("K", [1, 3, 9])
@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
@pytest.mark.parametrize("name,mode,horizon", EVAL_CASES)
def test_batched_evaluation_equals_single_evaluations(name, mode, horizon, precision, K):
    spec, _, env = make_env(name, precision, ts1="tile_shuffle" if mode == "tile_shuffle" else "perms")
    if horizon:
        spec = dataclasses.replace(spec, horizon=horizon)
    env._few_groups = lambda *a: False
    N, H, P = spec.population, spec.horizon, spec.particles
    B = N * P
    if name == "halfcheetah" and precision == "bf16_tc":  # 80 tiles: 64-row CTAs alone, 128-row CTAs from K = 2 on
        assert (_tc_tiles(spec, "tile_shuffle") * K < _sm_count()) == (K == 1)
    obs, acts = _problems(spec, K)
    perms = eps = None
    if mode == "perms":
        g = torch.Generator().manual_seed(7)
        nperm = 1 if spec.propagation == "fixed_model" else H
        perms = torch.stack([torch.stack([torch.randperm(B, generator=g) for _ in range(nperm)]) for _ in range(K)]).to(DEV)
        if name == "halfcheetah":
            eps = torch.randn(K, H, B, spec.out_size, generator=g).to(DEV)
    base = 40 * 1024
    rows = torch.empty(K, B, device=DEV)
    got = env.evaluate_action_sequences_batch(acts, obs, P, _perms=perms, _eps=eps, _row_returns=rows, _offset=base)
    torch.cuda.synchronize()
    for k in range(K):
        rr = torch.empty(B, device=DEV)
        ref = env.evaluate_action_sequences(acts[k], obs[k], P, _perms=None if perms is None else perms[k],
                                            _eps=None if eps is None else eps[k], _row_returns=rr, _offset=base + k * 1024)
        torch.cuda.synchronize()
        assert np.isfinite(ref.cpu().numpy()).all()
        assert torch.equal(got[k], ref), f"problem {k}: {(got[k] != ref).sum().item()} of {N} returns differ"
        assert torch.equal(rows[k], rr), f"problem {k}: row returns differ"


def test_batched_evaluation_draws_the_callers_counter_values():
    """Without an explicit offset a batch takes K consecutive counter values: the same as K single calls."""
    spec, _, env = make_env("halfcheetah", "bf16_tc", ts1="tile_shuffle")
    spec = dataclasses.replace(spec, horizon=4)
    obs, acts = _problems(spec, 3)
    env._offset = 10
    got = env.evaluate_action_sequences_batch(acts, obs, spec.particles)
    assert env._offset == 13
    env._offset = 10
    ref = torch.stack([env.evaluate_action_sequences(acts[k], obs[k], spec.particles) for k in range(3)])
    assert torch.equal(got, ref)


def _cem_pair(spec, K, iters, rme, clipped, precision="bf16_tc"):
    """(batched plan, [single plans]) with the solution and every iteration's values of each problem."""
    import mbrl_lib_b200 as bp
    from mbrl_lib_b200.planning import _FusedBatchObjective, _FusedObjective

    _, _, env = make_env(spec.name, precision, ts1="tile_shuffle")
    env._few_groups = lambda *a: False
    H, A = spec.horizon, spec.act_dim
    lb, ub = np.full((H, A), spec.action_lb).tolist(), np.full((H, A), spec.action_ub).tolist()
    opt = bp.CEMOptimizer(iters, 0.1, spec.population, lb, ub, 0.1, DEV, return_mean_elites=rme, clipped_normal=clipped)
    opt.record_values = True
    obs, _ = _problems(spec, K)
    x0 = torch.from_numpy(np.random.default_rng(3).uniform(-0.5, 0.5, (K, H, A)).astype(np.float32)).to(DEV)
    env._offset = 100
    sol = opt.optimize_batch(_FusedBatchObjective(env, obs, spec.particles), x0=x0).clone()
    vals = opt.last_values.clone()
    assert env._offset == 100 + K
    singles = []
    for k in range(K):
        env._offset = 100 + k
        s = opt.optimize(_FusedObjective(env, obs[k], spec.particles), x0=x0[k]).clone()
        singles.append((s, opt.last_values.clone()))
    torch.cuda.synchronize()
    return (sol, vals), singles


@pytest.mark.parametrize("rme,clipped", [(True, False), (False, False), (True, True), (False, True)])
def test_batched_plan_equals_single_plans(rme, clipped):
    """HalfCheetah, pop 500 x 20 particles, H 30, 4 problems (one 320-tile rollout per iteration on 128-row CTAs)."""
    spec = syn.CASES["halfcheetah"]
    (sol, vals), singles = _cem_pair(spec, 4, 5, rme, clipped)
    for k, (s, v) in enumerate(singles):
        assert torch.isfinite(s).all()
        assert torch.equal(vals[k], v), f"problem {k}: values differ at iterations {(vals[k] != v).any(1).nonzero().flatten().tolist()}"
        assert torch.equal(sol[k], s), f"problem {k}: solutions differ"


@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
def test_batched_plan_above_the_single_cta_refit(precision):
    """2 100 sequences: sample and refit kernels once per problem around the batched rollout."""
    spec = dataclasses.replace(syn.CASES["halfcheetah"], population=2100, horizon=6, particles=4)
    (sol, vals), singles = _cem_pair(spec, 2, 3, True, False, precision)
    for k, (s, v) in enumerate(singles):
        assert torch.equal(vals[k], v) and torch.equal(sol[k], s), f"problem {k} differs"


def _agent(env, particles, replan_freq=1, horizon=10, pop=256, optimizer="CEMOptimizer", **opt):
    import mbrl_lib_b200 as bp

    ocfg = {"_target_": f"mbrl.planning.{optimizer}", "device": DEV, "num_iterations": 3, "elite_ratio": 0.1,
            "population_size": pop, "alpha": 0.1, "return_mean_elites": True, **opt}
    cfg = {"_target_": "mbrl.planning.TrajectoryOptimizerAgent", "planning_horizon": horizon, "replan_freq": replan_freq,
           "optimizer_cfg": ocfg}
    return bp.create_trajectory_optim_agent_for_model(env, cfg, num_particles=particles)


def test_act_batch_equals_per_entry_act():
    """Consecutive steps with replan_freq 2 (warm-start shift, cached actions) and a reset of one entry in between:
    entry k of act_batch equals act of its own agent run with the counter value the batch gave entry k."""
    spec, _, env_b = make_env("halfcheetah", "bf16_tc", ts1="tile_shuffle")
    _, _, env_s = make_env("halfcheetah", "bf16_tc", ts1="tile_shuffle")
    K, P = 3, spec.particles
    agent_b = _agent(env_b, P, replan_freq=2)
    singles = [_agent(env_s, P, replan_freq=2) for _ in range(K)]
    g = np.random.default_rng(5)
    for step in range(7):
        obs = g.standard_normal((K, spec.obs_dim))
        if step == 4:
            agent_b.reset_batch([1])
            singles[1].reset()
            for a in singles:  # the batch replans every entry at its next call
                a.actions_to_use.clear()
        base = env_b._offset
        got = agent_b.act_batch(obs)
        replanned = env_b._offset != base
        assert got.shape == (K, spec.act_dim)
        for k, a in enumerate(singles):
            if replanned:
                assert not a.actions_to_use
                env_s._offset = base + k
            else:
                assert a.actions_to_use
            ref = a.act(obs[k])
            assert np.array_equal(got[k], ref), (step, k)


@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
def test_closed_loop_batch_reaches_goal(precision):
    """The line world of test_closed_loop_mpc_reaches_goal from 8 start positions, all driven through act_batch."""
    import mbrl_lib_b200 as bp
    from mbrl_lib_b200 import functions
    from test_gpu_parity import _Env

    class _Spec:
        obs_dim, act_dim, action_lb, action_ub = 1, 1, -1.0, 1.0

    env = bp.ModelEnv(_Env(_Spec), _line_world(DEV), functions.no_termination, None, generator=torch.Generator(device=DEV),
                      precision=precision, ts1="tile_shuffle")
    agent = _agent(env, 2, horizon=5, num_iterations=4)
    pos = np.linspace(-1.0, 1.0, 8)
    for _ in range(18):
        a = np.clip(agent.act_batch(pos[:, None]), -1, 1)[:, 0]
        pos = pos + 0.1 * a
    assert (np.abs(pos) < 0.12).all(), pos


def test_icem_act_batch_is_not_implemented():
    spec, _, env = make_env("halfcheetah_small", "bf16_tc", ts1="tile_shuffle")
    agent = _agent(env, spec.particles, optimizer="ICEMOptimizer", population_decay_factor=1.3, colored_noise_exponent=2.0,
                   keep_elite_frac=0.3)
    with pytest.raises(NotImplementedError, match="CEMOptimizer"):
        agent.act_batch(np.zeros((2, spec.obs_dim)))


def test_act_batch_with_a_reward_callable_equals_single_acts():
    """A lambda reward: the batch plans entry by entry, in order, each from its own warm start."""
    from test_gpu_callables import make_env as make_callable_env

    spec, _, env_b = make_callable_env("halfcheetah_small", "bf16_tc", ts1="tile_shuffle", term=False)
    _, _, env_s = make_callable_env("halfcheetah_small", "bf16_tc", ts1="tile_shuffle", term=False)
    assert env_b.has_external_callables()
    K = 3
    obs = np.random.default_rng(2).standard_normal((K, spec.obs_dim))
    agent_b, agent_s = _agent(env_b, spec.particles, pop=spec.population), _agent(env_s, spec.particles, pop=spec.population)
    torch.manual_seed(0)
    got = agent_b.act_batch(obs)
    torch.manual_seed(0)
    for k in range(K):
        agent_s.reset()
        assert np.array_equal(got[k], agent_s.act(obs[k])), k
    with pytest.raises(NotImplementedError):
        env_b.evaluate_action_sequences_batch(torch.zeros(K, 8, spec.horizon, spec.act_dim, device=DEV), obs, spec.particles)


def test_bad_batches_are_refused():
    from mbrl_lib_b200 import _lib

    spec, _, env = make_env("halfcheetah_small", "bf16_tc", ts1="tile_shuffle")
    N, H, A, D, P = spec.population, spec.horizon, spec.act_dim, spec.obs_dim, spec.particles
    with pytest.raises(ValueError, match="num_problems must be at least 1"):
        env.evaluate_action_sequences_batch(torch.zeros(0, N, H, A, device=DEV), np.zeros((0, D)), P)
    with pytest.raises(ValueError, match="initial_states"):
        env.evaluate_action_sequences_batch(torch.zeros(2, N, H, A, device=DEV), np.zeros((3, D)), P)
    lib = _lib.load()
    cfg = _lib.RolloutCfg(N, H, P, _lib.PREC["bf16_tc"], _lib.PROP["random_model"], _lib.TS1_TILE_SHUFFLE, 1, 1024, 8, 2 * N)
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=DEV)
    out = torch.empty(2, N, device=DEV)
    obs0, acts = torch.zeros(2, D, device=DEV), torch.zeros(2, N, H, A, device=DEV)
    with pytest.raises(NotImplementedError, match="cannot be sharded"):
        _lib.check(lib.b200pets_eval_sequences_batch(env.staged.handle, C.byref(cfg), 2, _lib.ptr(obs0), _lib.ptr(acts), None,
                                                     None, _lib.ptr(out), None, _lib.ptr(ws), ws.numel(), _lib.stream_ptr()))
    ccfg = _lib.CemCfg(2, 4, 0.1, 1, 0)
    cfg.first_sequence, cfg.global_population = 0, 0
    with pytest.raises(ValueError, match="num_problems must be at least 1"):
        _lib.check(lib.b200pets_cem_plan_batch(env.staged.handle, C.byref(cfg), C.byref(ccfg), 0, _lib.ptr(obs0), _lib.ptr(acts),
                                               _lib.ptr(acts), _lib.ptr(acts), None, None, None, _lib.ptr(out), None, _lib.ptr(ws),
                                               ws.numel(), _lib.stream_ptr()))
