"""Planning PlaNet's latent model for K observations at once (b200pets_latent_eval_sequences_batch,
b200pets_latent_cem_plan_batch, LatentModelEnv's K posteriors and TrajectoryOptimizerAgent.act_batch over them).

Problem k of a batch must give, bit for bit, what the single call gives from posterior k with the Philox counter the
batch assigns it: offset + k * 1024 for an evaluation, counter offset + k for a plan.
* Evaluation: K in {1, 3, 9}, in-kernel and injected draws, distinct posteriors, at PlaNet's sizes with a population of
  1000 and at an odd model size with N 37, P 3 (N * P not a multiple of the tile).  NaN sentinels past the batch.
* Tiles: a batch's rows per CTA come from plan_info(K * N * P); on a 132-SM card K = 4 at a population of 1000 runs 32
  rows per CTA where one problem runs 8.
* CEM plan: solution and values against K single plans, on both refit routes (population <= 2048 with >= 2 elites, and
  2500), return_mean_elites and clipped normal on and off.
* Agent: the shipped PlaNet agent and CEM configs, keep_last_solution off and on, reset_batch; MPPI from the K
  posteriors against K single MPPI plans; the refusals.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import mbrl_lib_b200 as bp
from mbrl_lib_b200 import _lib, functions, models, planning

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SIZES = {"planet": (6, 30, 200, 200), "odd": (1, 7, 37, 45)}


class _Box:
    def __init__(self, lo_, hi, shape):
        self.low, self.high, self.shape = np.full(shape, lo_, np.float32), np.full(shape, hi, np.float32), shape


class _Env:
    def __init__(self, A):
        self.observation_space = _Box(0, 255, (3, 64, 64))
        self.action_space = _Box(-1.0, 1.0, (A,))


def _model(size, seed=0):
    A, L, Hb, Hf = SIZES[size]
    torch.manual_seed(seed)
    return models.PlaNetModel(A, L, Hb, Hf, device=DEV)


def _env(model, seed=5):
    gen = torch.Generator(device=DEV)
    gen.manual_seed(seed)
    return bp.ModelEnv(_Env(model.action_size), model, functions.no_termination, generator=gen)


def _posteriors(model, K, seed=1):
    g = np.random.default_rng(seed)
    latent = torch.from_numpy(g.standard_normal((K, model.latent_state_size)).astype(np.float32)).to(DEV)
    belief = torch.from_numpy(np.tanh(g.standard_normal((K, model.belief_size))).astype(np.float32)).to(DEV)
    return latent, belief


# ---- evaluation -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [1, 3, 9])
@pytest.mark.parametrize("size,N,P,H", [("planet", 1000, 1, 12), ("odd", 37, 3, 5)])
@pytest.mark.parametrize("injected", [False, True])
def test_evaluation_equals_single_calls(K, size, N, P, H, injected):
    model = _model(size)
    env = _env(model)
    A, L = model.action_size, model.latent_state_size
    latent, belief = _posteriors(model, K, seed=K)
    env.set_posterior_batch(latent, belief)
    g = torch.Generator(device=DEV)
    g.manual_seed(K * 10 + N)
    acts = torch.rand(K, N, H, A, device=DEV, generator=g) * 2 - 1
    eps = torch.randn(K, H, N * P, L, device=DEV, generator=g) if injected else None
    rows = torch.empty(K, N * P, device=DEV)
    env._offset = 20
    got = env.evaluate_action_sequences_batch(acts, np.zeros((K, 3, 64, 64)), P, _eps=eps, _row_returns=rows)
    assert env._offset == 20 + K and got.shape == (K, N)
    for k in range(K):
        model.set_posterior(latent[k], belief[k])
        want_rows = torch.empty(N * P, device=DEV)
        want = env.evaluate_action_sequences(acts[k], np.zeros((3, 64, 64)), P, _offset=(21 + k) * 1024,
                                             _eps=None if eps is None else eps[k], _row_returns=want_rows)
        assert torch.equal(got[k], want), k
        assert torch.equal(rows[k], want_rows), k


def test_evaluation_writes_nothing_past_the_batch():
    model = _model("odd")
    env = _env(model)
    lib = _lib.load()
    K, N, P, H = 3, 37, 3, 4
    B = N * P
    latent, belief = _posteriors(model, K)
    acts = torch.rand(K, N, H, 1, device=DEV) * 2 - 1
    cfg = env._rollout_cfg(N, H, P, 7 * 1024)
    rows = torch.full((K * B + 64,), float("nan"), device=DEV)
    returns = torch.full((K * N + 64,), float("nan"), device=DEV)
    ws = torch.empty(lib.b200pets_latent_eval_batch_workspace_bytes(env.staged.handle, C.byref(cfg), K), dtype=torch.uint8,
                     device=DEV)
    _lib.check(lib.b200pets_latent_eval_sequences_batch(env.staged.handle, C.byref(cfg), K, _lib.ptr(latent),
                                                        _lib.ptr(belief), _lib.ptr(acts), None, _lib.ptr(returns),
                                                        _lib.ptr(rows), _lib.ptr(ws), ws.numel(), _lib.stream_ptr()))
    assert torch.isfinite(rows[:K * B]).all() and torch.isnan(rows[K * B:]).all()
    assert torch.isfinite(returns[:K * N]).all() and torch.isnan(returns[K * N:]).all()


def test_a_batch_takes_its_tile_from_all_its_rows():
    model = _model("planet")
    env = _env(model)
    sms = torch.cuda.get_device_properties(0).multi_processor_count

    def rule(rows):
        r = 1
        while r < -(-rows // sms) and r < 32:
            r *= 2
        return r

    for K in (1, 4):
        info = env.staged.plan_info(K * 1000)
        assert info["rows_per_cta"] == rule(K * 1000), (K, info)
    if sms == 132:
        assert env.staged.plan_info(1000)["rows_per_cta"] == 8 and env.staged.plan_info(4000)["rows_per_cta"] == 32
    # the K = 4 batch on that tile still gives each problem its single call's bits
    K, N, H = 4, 1000, 12
    latent, belief = _posteriors(model, K, seed=4)
    env.set_posterior_batch(latent, belief)
    acts = torch.rand(K, N, H, 6, device=DEV) * 2 - 1
    got = env.evaluate_action_sequences_batch(acts, np.zeros((K, 3)), 1, _offset=3 * 1024)
    for k in (0, K - 1):
        model.set_posterior(latent[k], belief[k])
        assert torch.equal(got[k], env.evaluate_action_sequences(acts[k], np.zeros(3), 1, _offset=(3 + k) * 1024))


# ---- CEM plan ---------------------------------------------------------------------------------------------------------
def _cem(N, it, H, A, clipped, rme, alpha=0.1):
    return planning.CEMOptimizer(num_iterations=it, elite_ratio=0.1, population_size=N, lower_bound=[[-1.0] * A] * H,
                                 upper_bound=[[1.0] * A] * H, alpha=alpha, device=DEV, return_mean_elites=rme,
                                 clipped_normal=clipped)


@pytest.mark.parametrize("N,P", [(1000, 1), (300, 2), (2500, 1)])  # 2500: outside the single-CTA refit
@pytest.mark.parametrize("rme", [True, False])
@pytest.mark.parametrize("clipped", [True, False])
def test_cem_plan_equals_single_plans(N, P, rme, clipped):
    model = _model("planet")
    env = _env(model)
    K, it, H, A, L = 3, 3, 5, 6, 30
    latent, belief = _posteriors(model, K, seed=N)
    env.set_posterior_batch(latent, belief)
    opt = _cem(N, it, H, A, clipped, rme)
    opt.record_values = True
    g = torch.Generator(device=DEV)
    g.manual_seed(N + rme)
    injected = N == 300
    z = torch.randn(K, it, N, H, A, device=DEV, generator=g) if injected else None
    eps = torch.randn(K, it, H, N * P, L, device=DEV, generator=g) if injected else None
    x0 = (torch.rand(K, H, A, device=DEV, generator=g) - 0.5).contiguous()
    env._offset = 40
    sol = opt.optimize_batch(planning._FusedBatchObjective(env, np.zeros((K, 3, 64, 64)), P), x0, _noise=z,
                             _model_noise=(None, eps))
    assert env._offset == 40 + K and sol.shape == (K, H, A)
    values = opt.last_values.clone()
    for k in range(K):
        model.set_posterior(latent[k], belief[k])
        env._offset = 40 + k
        want = opt.optimize(planning._FusedObjective(env, np.zeros((3, 64, 64)), P), x0[k],
                            _noise=None if z is None else z[k], _model_noise=(None, None if eps is None else eps[k]))
        assert torch.equal(sol[k], want), k
        assert torch.equal(values[k], opt.last_values), k


# ---- agent ------------------------------------------------------------------------------------------------------------
CEM_CFG = {"_target_": "mbrl.planning.CEMOptimizer", "num_iterations": 10, "elite_ratio": 0.1, "population_size": 1000,
           "alpha": 0.0, "lower_bound": "???", "upper_bound": "???", "return_mean_elites": True, "device": DEV,
           "clipped_normal": True}
MPPI_CFG = {"_target_": "mbrl.planning.MPPIOptimizer", "num_iterations": 3, "gamma": 10.0, "population_size": 200,
            "sigma": 1.0, "beta": 0.9, "lower_bound": "???", "upper_bound": "???", "device": DEV}
ICEM_CFG = {"_target_": "mbrl.planning.ICEMOptimizer", "num_iterations": 3, "elite_ratio": 0.1, "population_size": 200,
            "population_decay_factor": 1.25, "colored_noise_exponent": 2.0, "keep_elite_frac": 0.1, "alpha": 0.1,
            "lower_bound": "???", "upper_bound": "???", "return_mean_elites": True, "population_size_module": None,
            "device": DEV}


def _agent(env, optimizer_cfg, keep_last_solution=False, H=12):
    cfg = {"_target_": "mbrl.planning.TrajectoryOptimizerAgent", "action_lb": "???", "action_ub": "???",
           "planning_horizon": H, "optimizer_cfg": dict(optimizer_cfg), "replan_freq": 1,
           "keep_last_solution": keep_last_solution, "verbose": False}
    return bp.create_trajectory_optim_agent_for_model(env, cfg)


@pytest.mark.parametrize("keep", [False, True])
def test_act_batch_equals_single_acts(keep):
    model = _model("planet", seed=2)
    env = _env(model)
    K = 3
    latent, belief = _posteriors(model, K, seed=7)
    obs = np.random.default_rng(0).integers(0, 255, (K, 3, 64, 64), dtype=np.uint8)
    agent = _agent(env, CEM_CFG, keep)
    env.set_posterior_batch(latent, belief)
    env._offset = 100
    got = [agent.act_batch(obs), agent.act_batch(obs)]
    assert got[0].shape == (K, 6) and env._offset == 100 + 2 * K
    agent.reset_batch([1])
    init = agent.optimizer.initial_solution
    assert torch.equal(agent.optimizer.previous_solutions[1], init)
    assert torch.equal(agent.optimizer.previous_solutions[0], init) != keep  # a kept warm start has moved
    got.append(agent.act_batch(obs))
    for k in range(K):
        single = _agent(env, CEM_CFG, keep)
        model.set_posterior(latent[k], belief[k])
        for step in range(2):
            env._offset = 100 + step * K + k
            assert np.array_equal(single.act(obs[k]), got[step][k]), (k, step)
        if k == 1:
            single.reset()
        env._offset = 100 + 2 * K + k
        assert np.array_equal(single.act(obs[k]), got[2][k]), (k, "after reset_batch")


def test_mppi_act_batch_plans_each_entry_from_its_posterior(monkeypatch):
    def unreachable(*_a, **_kw):
        raise AssertionError("the ensemble's batched MPPI plan was reached with a latent model")

    monkeypatch.setattr(planning.MPPIOptimizer, "_optimize_fused_batch", unreachable)
    model = _model("planet", seed=4)
    env = _env(model)
    K = 3
    latent, belief = _posteriors(model, K, seed=8)
    obs = np.zeros((K, 3, 64, 64), np.uint8)
    agent = _agent(env, MPPI_CFG)
    env.set_posterior_batch(latent, belief)
    env._offset = 10
    got = agent.act_batch(obs)
    single = _agent(env, MPPI_CFG)
    env._offset = 10
    for k in range(K):
        model.set_posterior(latent[k], belief[k])
        single.optimizer.optimizer.mean.zero_()  # the batch's entries start from zero means, as a fresh optimiser
        assert np.array_equal(single.act(obs[k]), got[k]), k


def test_update_posterior_batch_then_act_batch():
    enc = ((3, 32, 4, 2), (32, 64, 4, 2), (64, 128, 4, 2), (128, 256, 4, 2))  # planet.yaml
    dec = ((1024, 1, 1), ((1024, 128, 5, 2), (128, 64, 5, 2), (64, 32, 6, 2), (32, 3, 6, 2)))
    torch.manual_seed(0)
    model = models.PlaNetModel(6, 30, 200, 200, device=DEV, obs_shape=(3, 64, 64), obs_encoding_size=1024,
                               encoder_config=enc, decoder_config=dec)
    model.set_posterior(torch.zeros(30), torch.zeros(200))
    env = _env(model)
    agent = _agent(env, CEM_CFG)
    K = 4
    obs = np.random.default_rng(3).integers(0, 255, (K, 3, 64, 64), dtype=np.uint8)
    post = env.update_posterior_batch(obs)
    assert post["latent"].shape == (K, 30) and post["belief"].shape == (K, 200)
    a = agent.act_batch(obs)
    assert a.shape == (K, 6) and np.isfinite(a).all()
    env.update_posterior_batch(obs, torch.from_numpy(a))
    env.reset_posterior_batch([2])
    with pytest.raises(RuntimeError, match="reset"):
        agent.act_batch(obs)
    env.update_posterior_batch(obs, torch.from_numpy(a))
    assert agent.act_batch(obs).shape == (K, 6)
    assert torch.equal(model._current_posterior_sample, torch.zeros(1, 30, device=DEV))  # the model's own is untouched


def test_refusals():
    model = _model("odd")
    env = _env(model)
    agent = _agent(env, dict(CEM_CFG, population_size=50), H=3)
    with pytest.raises(NotImplementedError, match="one posterior"):
        agent.act_batch(np.zeros((2, 3, 64, 64)))
    with pytest.raises(NotImplementedError, match="one posterior"):
        env.evaluate_action_sequences_batch(torch.zeros(2, 4, 3, 1, device=DEV), np.zeros((2, 3)), 1)
    env.set_posterior_batch(*_posteriors(model, 2))
    with pytest.raises(ValueError, match="batch of 2"):
        agent.act_batch(np.zeros((3, 3, 64, 64)))
    with pytest.raises(ValueError, match="batch of 2"):
        env.evaluate_action_sequences_batch(torch.zeros(3, 4, 3, 1, device=DEV), np.zeros((3, 3)), 1)
    with pytest.raises(ValueError, match="initial states"):
        env.evaluate_action_sequences_batch(torch.zeros(2, 4, 3, 1, device=DEV), np.zeros((3, 3)), 1)
    with pytest.raises(NotImplementedError, match="batch of observations"):
        _agent(env, ICEM_CFG, H=3).act_batch(np.zeros((2, 3, 64, 64)))
    with pytest.raises(NotImplementedError, match="encoder"):
        env.update_posterior_batch(np.zeros((2, 3, 64, 64)))
    assert agent.act_batch(np.zeros((2, 3, 64, 64))).shape == (2, 1)
