"""Planning for a batch of observations with MPPI: K independent MPPIOptimizer plans in one device-resident call.

Problem k of a batched MPPI plan gives, bit for bit, the k-th of K consecutive single ``MPPIOptimizer.optimize`` calls
over ``ModelEnv.evaluate_action_sequences``, from its own carried mean: population noise with optimiser counter
``first + k``, the rollout of refinement r with environment counter ``env_first + k * R + r``, and permutations drawn
from the torch RNG in the order the single plans draw them.  Every refinement's values (after the NaN rule), the plans
and the carried means are compared with ``torch.equal``.
"""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

from mbrl_lib_b200 import synthetic as syn
from test_gpu_batch import _problems
from test_gpu_parity import DEV, make_env
from test_gpu_tiles import _sm_count, _tc_tiles

pytestmark = pytest.mark.gpu

R, GAMMA, SIGMA, BETA = 5, 0.9, 1.0, 0.9  # conf/overrides/pets_mppi_halfcheetah.yaml
MPPI_HALFCHEETAH = dataclasses.replace(syn.CASES["halfcheetah"], population=350)  # pop 350 x 20 particles x H 30


def _mppi(spec, iters=R):
    import mbrl_lib_b200 as bp

    H, A = spec.horizon, spec.act_dim
    lb, ub = np.full((H, A), spec.action_lb).tolist(), np.full((H, A), spec.action_ub).tolist()
    return bp.MPPIOptimizer(iters, spec.population, GAMMA, SIGMA, BETA, lb, ub, DEV)


def _means(K, spec, seed=3):
    """A different non-zero carried mean per problem."""
    m = np.random.default_rng(seed).uniform(-0.5, 0.5, (K, spec.horizon, spec.act_dim)).astype(np.float32)
    return torch.from_numpy(m).to(DEV)


class _Objective:
    """The single path's objective: evaluate_action_sequences of one observation, refinement r with eps[r] (or none)."""

    def __init__(self, env, obs, particles, eps=None):
        self.env, self.obs, self.particles, self.eps, self.r = env, obs, particles, eps, 0

    def __call__(self, pop):
        eps = None if self.eps is None else self.eps[self.r]
        self.r += 1
        return self.env.evaluate_action_sequences(pop, initial_state=self.obs, num_particles=self.particles, _eps=eps)


def _check_pair(spec, env, K, noise=None, eps=None, torch_seed=None):
    """Batched plan against K consecutive single plans at the counter values the batch gave each problem."""
    from mbrl_lib_b200.planning import _FusedBatchObjective

    P = spec.particles
    opt = _mppi(spec)
    opt.record_values = True
    obs, _ = _problems(spec, K)
    m0 = _means(K, spec)
    opt.batch_mean = m0.clone()
    env._offset, opt._offset = 100, 50
    if torch_seed is not None:
        torch.manual_seed(torch_seed)
    got = opt.optimize_batch(_FusedBatchObjective(env, obs, P), _noise=noise,
                             _model_noise=None if eps is None else (None, eps)).clone()
    vals = opt.last_values.clone()
    carried = opt.batch_mean.clone()
    assert vals.shape == (K, R, spec.population)
    assert env._offset == 100 + K * R and opt._offset == 50 + K
    if torch_seed is not None:
        torch.manual_seed(torch_seed)
    for k in range(K):
        env._offset, opt._offset = 100 + k * R, 50 + k
        opt.mean = m0[k].clone()
        seen = []
        s = opt.optimize(_Objective(env, obs[k], P, None if eps is None else eps[k]),
                         callback=lambda pop, v, r: seen.append(v.clone()), _noise=None if noise is None else noise[k])
        torch.cuda.synchronize()
        v = torch.stack(seen)
        assert torch.isfinite(s).all()
        assert torch.equal(vals[k], v), f"problem {k}: values differ at refinements {(vals[k] != v).any(1).nonzero().flatten().tolist()}"
        assert torch.equal(got[k], s), f"problem {k}: plans differ"
        assert torch.equal(carried[k], opt.mean), f"problem {k}: carried means differ"
    assert not torch.equal(got[0], m0[0])


@pytest.mark.parametrize("K", [1, 3, 8])
@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
def test_batched_mppi_plan_equals_single_plans(precision, K):
    """pets_mppi_halfcheetah: 60 tiles per rollout, so K = 1 runs 64-row CTAs and K = 3, 8 run 128-row CTAs with more
    tiles than SMs."""
    spec = MPPI_HALFCHEETAH
    _, _, env = make_env("halfcheetah", precision, ts1="tile_shuffle")
    env._few_groups = lambda *a: False
    if precision == "bf16_tc":
        assert (_tc_tiles(spec, "tile_shuffle") * K < _sm_count()) == (K == 1)
    _check_pair(spec, env, K)


@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
def test_batched_mppi_plan_ts1_perms_with_injected_noise(precision):
    """TS1 with torch.randperm permutations from a seeded RNG, injected population noise z and model noise eps."""
    spec = dataclasses.replace(MPPI_HALFCHEETAH, horizon=8)
    _, _, env = make_env("halfcheetah", precision, ts1="perms")
    K, N, H, A, B = 3, spec.population, spec.horizon, spec.act_dim, spec.population * spec.particles
    g = torch.Generator().manual_seed(11)
    z = torch.randn(K, R, N, H, A, generator=g).clamp(-2, 2).to(DEV)
    eps = torch.randn(K, R, H, B, spec.out_size, generator=g).to(DEV)
    _check_pair(spec, env, K, noise=z, eps=eps, torch_seed=5)


@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
@pytest.mark.parametrize("name,ts1", [("hopper_tsinf", "perms"), ("silu_expectation", "tile_shuffle"),
                                      ("halfcheetah_small", "tile_shuffle")])
def test_batched_mppi_plan_propagation_modes(name, ts1, precision):
    """TSinf with one permutation per evaluation, expectation, and a population so small that _few_groups makes the
    single path draw permutations (halfcheetah_small: 5 shuffle groups for 5 members)."""
    spec, _, env = make_env(name, precision, ts1=ts1)
    if name == "halfcheetah_small":
        assert env._few_groups(spec.population, spec.particles)
    _check_pair(spec, env, 3, torch_seed=9)


def _mppi_agent(env, particles, replan_freq=1, horizon=10, pop=256):
    import mbrl_lib_b200 as bp

    ocfg = {"_target_": "mbrl.planning.MPPIOptimizer", "device": DEV, "num_iterations": R, "population_size": pop,
            "gamma": GAMMA, "sigma": SIGMA, "beta": BETA}
    cfg = {"_target_": "mbrl.planning.TrajectoryOptimizerAgent", "planning_horizon": horizon, "replan_freq": replan_freq,
           "optimizer_cfg": ocfg}
    return bp.create_trajectory_optim_agent_for_model(env, cfg, num_particles=particles)


def test_mppi_act_batch_equals_per_entry_act():
    """Seven steps with replan_freq 2 and reset_batch([1]) after four: entry k of act_batch equals act of its own agent
    (its own MPPIOptimizer) run at the counter values the batch gave entry k.  The means carry across calls and across
    the reset, which leaves them alone as reset() leaves MPPIOptimizer.mean."""
    spec, _, env_b = make_env("halfcheetah", "bf16_tc", ts1="tile_shuffle")
    _, _, env_s = make_env("halfcheetah", "bf16_tc", ts1="tile_shuffle")
    K, P = 3, spec.particles
    agent_b = _mppi_agent(env_b, P, replan_freq=2)
    singles = [_mppi_agent(env_s, P, replan_freq=2) for _ in range(K)]
    opt_b = agent_b.optimizer.optimizer
    g = np.random.default_rng(5)
    plans = 0
    for step in range(7):
        obs = g.standard_normal((K, spec.obs_dim))
        if step == 4:
            means = opt_b.batch_mean.clone()
            agent_b.reset_batch([1])
            assert torch.equal(opt_b.batch_mean, means)
            singles[1].reset()
            for a in singles:  # the batch replans every entry at its next call
                a.actions_to_use.clear()
        base, opt_base = env_b._offset, getattr(opt_b, "_offset", 0)
        got = agent_b.act_batch(obs)
        replanned = env_b._offset != base
        plans += replanned
        assert got.shape == (K, spec.act_dim)
        for k, a in enumerate(singles):
            if replanned:
                assert env_b._offset == base + K * R
                assert not a.actions_to_use
                env_s._offset, a.optimizer.optimizer._offset = base + k * R, opt_base + k
            else:
                assert a.actions_to_use
            ref = a.act(obs[k])
            assert np.array_equal(got[k], ref), (step, k)
    assert plans == 4
    for k, a in enumerate(singles):
        assert torch.equal(opt_b.batch_mean[k], a.optimizer.optimizer.mean), k


def test_mppi_act_batch_with_a_reward_callable_equals_single_acts():
    """A lambda reward: the batch runs MPPIOptimizer.optimize entry by entry, in order, each on its own mean; the
    single path's mean is left as it was."""
    from test_gpu_callables import make_env as make_callable_env

    spec, _, env_b = make_callable_env("halfcheetah_small", "bf16_tc", ts1="tile_shuffle", term=False)
    _, _, env_s = make_callable_env("halfcheetah_small", "bf16_tc", ts1="tile_shuffle", term=False)
    assert env_b.has_external_callables()
    K = 3
    agent_b = _mppi_agent(env_b, spec.particles, horizon=spec.horizon, pop=spec.population)
    agent_s = _mppi_agent(env_s, spec.particles, horizon=spec.horizon, pop=spec.population)
    opt_b, opt_s = agent_b.optimizer.optimizer, agent_s.optimizer.optimizer
    single_mean = _means(1, spec, seed=8)[0]
    opt_b.mean = single_mean.clone()
    g = np.random.default_rng(2)
    means = [torch.zeros(spec.horizon, spec.act_dim, device=DEV) for _ in range(K)]
    for step in range(2):
        obs = g.standard_normal((K, spec.obs_dim))
        torch.manual_seed(step)
        got = agent_b.act_batch(obs)
        torch.manual_seed(step)
        for k in range(K):
            agent_s.reset()
            opt_s.mean = means[k]
            assert np.array_equal(got[k], agent_s.act(obs[k])), (step, k)
            means[k] = opt_s.mean
            assert torch.equal(opt_b.batch_mean[k], means[k]), (step, k)
    assert torch.equal(opt_b.mean, single_mean)


def test_mppi_zero_refinements_return_the_shifted_means():
    from mbrl_lib_b200.planning import _FusedBatchObjective, _FusedObjective

    spec, _, env = make_env("halfcheetah_small", "bf16_tc", ts1="tile_shuffle")
    K = 4
    opt = _mppi(spec, iters=0)
    m0 = _means(K, spec)
    opt.batch_mean = m0.clone()
    obs, _ = _problems(spec, K)
    env._offset = 7
    got = opt.optimize_batch(_FusedBatchObjective(env, obs, spec.particles))
    assert env._offset == 7
    assert torch.equal(got, torch.cat([m0[:, 1:], m0[:, -1:]], 1))
    for k in range(K):
        opt.mean = m0[k].clone()
        assert torch.equal(opt.optimize(_FusedObjective(env, obs[k], spec.particles)), got[k])


def test_mppi_tsinf_batch_not_a_multiple_of_the_members_is_refused_before_any_launch():
    from mbrl_lib_b200.planning import _FusedBatchObjective, _FusedObjective

    spec, _, env = make_env("hopper_tsinf", "f32", ts1="tile_shuffle")
    spec = dataclasses.replace(spec, population=31, particles=5)  # 155 rows over 2 members
    assert (spec.population * spec.particles) % len(env.staged.members()) != 0
    opt = _mppi(spec)
    m0 = _means(2, spec)
    opt.batch_mean = m0.clone()
    obs, _ = _problems(spec, 2)
    env._offset = 3
    with pytest.raises(ValueError, match="multiple of the number of models"):
        opt.optimize_batch(_FusedBatchObjective(env, obs, spec.particles))
    torch.cuda.synchronize()
    assert torch.equal(opt.batch_mean, m0) and env._offset == 3
    with pytest.raises(ValueError, match="multiple of the number of models"):
        opt.optimize(_FusedObjective(env, obs[0], spec.particles))


def test_bad_mppi_batches_are_refused():
    from mbrl_lib_b200 import _lib
    from test_gpu_callables import make_env as make_callable_env

    spec, _, env = make_env("halfcheetah_small", "bf16_tc", ts1="tile_shuffle")
    N, H, A, D, P, K = spec.population, spec.horizon, spec.act_dim, spec.obs_dim, spec.particles, 2
    lib = _lib.load()
    cfg = _lib.RolloutCfg(N, H, P, _lib.PREC["bf16_tc"], _lib.PROP["random_model"], _lib.TS1_TILE_SHUFFLE, 1, 1, 0, 0)
    mcfg = _lib.MppiCfg(R, GAMMA, BETA, 1, 1)
    need = lib.b200pets_mppi_plan_batch_workspace_bytes(env.staged.handle, C.byref(cfg), C.byref(mcfg), K)
    assert need > 0
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    obs0, mean = torch.zeros(K, D, device=DEV), torch.zeros(K, H, A, device=DEV)
    lb, ub = -torch.ones(H, A, device=DEV), torch.ones(H, A, device=DEV)

    def call(handle=env.staged.handle, cfg=cfg, mcfg=mcfg, K=K, obs0=obs0, mean=mean, lb=lb, ws=ws, nbytes=need):
        _lib.check(lib.b200pets_mppi_plan_batch(handle, C.byref(cfg), C.byref(mcfg), K, _lib.ptr(obs0), _lib.ptr(mean),
                                                _lib.ptr(lb), _lib.ptr(ub), None, None, None, None, _lib.ptr(ws), nbytes,
                                                _lib.stream_ptr()), "mppi_plan_batch")

    with pytest.raises(ValueError, match="num_problems must be at least 1"):
        call(K=0)
    sharded = _lib.RolloutCfg(N, H, P, _lib.PREC["bf16_tc"], _lib.PROP["random_model"], _lib.TS1_TILE_SHUFFLE, 1, 1, 8, 2 * N)
    with pytest.raises(NotImplementedError, match="cannot be sharded"):
        call(cfg=sharded)
    for kw in ({"obs0": None}, {"mean": None}, {"lb": None}, {"ws": None}):
        with pytest.raises(ValueError, match="null argument"):
            call(**kw)
    with pytest.raises(ValueError, match="workspace too small"):
        call(nbytes=need - 1)
    with pytest.raises(ValueError, match="num_iterations must not be negative"):
        call(mcfg=_lib.MppiCfg(-1, GAMMA, BETA, 1, 1))
    _, _, env_cb = make_callable_env("halfcheetah_small", "bf16_tc", ts1="tile_shuffle", term=False)
    with pytest.raises(NotImplementedError, match="external reward/termination callables"):
        call(handle=env_cb.staged.handle)
    torch.cuda.synchronize()
    assert torch.equal(mean, torch.zeros(K, H, A, device=DEV))  # nothing was launched
