"""PlaNet's latent model on the device (csrc/latent.cu) against the float64 oracle (oracle/latent_f64.py).

* Step (b200pets_latent_step), deterministic and with injected draws: every column of latent, belief and reward at
  PlaNet's sizes (A 6, L 30, Hb 200, Hf 200), an odd size (A 1, L 7, Hb 37, Hf 45) and the largest size the row limit
  accepts (Hb = Hf = 1203 at L 30, A 6), B in {1, 7, 1000, 4099}.  Bar: 3e-5 of max(1, |column|).
* evaluate_action_sequences with injected draws, N in {1, 37, 1000}, P in {1, 4}, H in {1, 12, 50}, returns and row
  returns.  Bar: 1e-4 of max(1, |returns|).
* In-kernel draws equal a numpy Philox restatement of the RNG_STREAM_LATENT counter layout (common.cuh), per row and
  step; they differ from call to call.
* The CEM plan equals, bit for bit, the chain  cem_sample -> evaluate_action_sequences -> cem_update  with the plan's
  offsets, with injected and with in-kernel draws, and the float64 CEM plan at the planet_cheetah_run planner config.
* Drop-in: the shipped PlaNet agent config over the reference's PlaNetModel (oracle/_ref, skipped without it) and over
  the local container; iCEM and MPPI through their loops.  Re-staging after an optimizer step.  Refusals.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import mbrl_lib_b200 as bp
from baseline import reference_arm as ra
from mbrl_lib_b200 import _lib, functions, latent, models, planning
from oracle import latent_f64 as lo

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
mbrl, REF_SRC = ra.import_reference()
needs_ref = pytest.mark.skipif(mbrl is None, reason=f"reference not importable here: {REF_SRC}")

SIZES = {"planet": (6, 30, 200, 200), "odd": (1, 7, 37, 45), "largest": (6, 30, 1203, 1203)}
STEP_BAR, EVAL_BAR = 3e-5, 1e-4
RNG_STREAM_LATENT = 0x60000
PLANET_CHEETAH = {"num_iterations": 10, "elite_ratio": 0.1, "population_size": 1000, "alpha": 0.0, "horizon": 12}


class _Box:
    def __init__(self, lo_, hi, shape):
        self.low, self.high, self.shape = np.full(shape, lo_, np.float32), np.full(shape, hi, np.float32), shape


class _Env:
    def __init__(self, A):
        self.observation_space = _Box(0, 255, (3, 64, 64))
        self.action_space = _Box(-1.0, 1.0, (A,))


def _model(size, seed=0):
    A, L, Hb, Hf = SIZES[size] if isinstance(size, str) else size
    torch.manual_seed(seed)
    m = models.PlaNetModel(A, L, Hb, Hf, device=DEV)  # torch's default initialisation: activations stay O(1)
    g = np.random.default_rng(seed + 1)
    m.set_posterior(g.standard_normal(L), np.tanh(g.standard_normal(Hb)))
    return m


def _env(model, seed=5):
    gen = torch.Generator(device=DEV)
    gen.manual_seed(seed)
    return bp.ModelEnv(_Env(model.action_size), model, functions.no_termination, generator=gen)


def _err(got, want):
    got = got.detach().cpu().double().numpy() if torch.is_tensor(got) else np.asarray(got, np.float64)
    return float(np.max(np.abs(got - want)) / max(1.0, float(np.max(np.abs(want)))))


def _post(model):
    return model._current_posterior_sample[0].cpu().numpy(), model._current_belief[0].cpu().numpy()


# ---- numpy Philox (common.cuh) ------------------------------------------------------------------------------------
M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    c0, c1, c2, c3 = np.broadcast_arrays(*(np.asarray(c, np.uint64) for c in (c0, c1, c2, c3)))
    k0, k1 = int(k0), int(k1)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c0, np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ np.uint64(k0), p1 & M32, (p0 >> np.uint64(32)) ^ c3 ^ np.uint64(k1), p0 & M32
        k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
    return c0, c1, c2, c3


def latent_draws64(B, L, t, seed, offset):
    """[B, L] draws of step t: lane j & 3 of the Box-Muller block at counter (row, t, RNG_STREAM_LATENT | j >> 2,
    low word of offset) under key seed ^ (high word of offset)."""
    key = (seed ^ (offset & 0xFFFFFFFF00000000)) & 0xFFFFFFFFFFFFFFFF
    rows, j = np.arange(B)[:, None], np.arange(L)[None, :]
    r = philox4x32_10(rows, t, RNG_STREAM_LATENT | (j >> 2), offset & 0xFFFFFFFF, key & 0xFFFFFFFF, key >> 32)
    u = [((x >> np.uint64(8)).astype(np.float64) + 0.5) / 16777216.0 for x in r]
    lane = np.broadcast_to(j & 3, (B, L))
    ur, ua = np.where(lane < 2, u[0], u[2]), np.where(lane < 2, u[1], u[3])
    rad, ang = np.sqrt(-2.0 * np.log(ur)), 2.0 * np.pi * ua
    return np.where(lane & 1, rad * np.sin(ang), rad * np.cos(ang))


# ---- step ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("size", list(SIZES))
@pytest.mark.parametrize("B", [1, 7, 1000, 4099])
def test_step_matches_float64(size, B):
    model = _model(size)
    env = _env(model)
    A, L, Hb, _ = SIZES[size]
    g = np.random.default_rng(B)
    s0, h0 = g.standard_normal((B, L)).astype(np.float32), np.tanh(g.standard_normal((B, Hb))).astype(np.float32)
    act = np.clip(g.standard_normal((B, A)), -1, 1).astype(np.float32)
    eps = g.standard_normal((B, L)).astype(np.float32)
    p = lo.params_of(model)
    state = {"latent": torch.from_numpy(s0).to(DEV), "belief": torch.from_numpy(h0).to(DEV)}
    env.reset(np.zeros((B, 1)), return_as_np=False)
    for sample, e in ((False, None), (True, eps)):
        nl, rew, done, nxt = env.step(torch.from_numpy(act).to(DEV), state, sample=sample,
                                      _eps=None if e is None else torch.from_numpy(e).to(DEV))
        ws, wh, wr = lo.step(p, s0, h0, act, e)
        assert rew.shape == (B, 1) and done.shape == (B, 1) and not done.any()
        assert torch.equal(nl, nxt["latent"])
        for what, got, want in (("latent", nl, ws), ("belief", nxt["belief"], wh), ("reward", rew[:, 0], wr)):
            for c in range(want.shape[1] if want.ndim == 2 else 1):
                gc, wc = (got[:, c], want[:, c]) if want.ndim == 2 else (got, want)
                err = _err(gc, wc)
                assert err <= STEP_BAR, f"{size} B={B} sample={sample} {what}[{c}]: {err:.2e}"


def test_step_returns_numpy_by_default():
    model = _model("odd")
    env = _env(model)
    st = env.reset(np.zeros((3, 7)))
    nl, rew, done, nxt = env.step(np.zeros((3, 1), np.float32), st, sample=True)
    assert isinstance(nl, np.ndarray) and nl.shape == (3, 7) and rew.shape == (3, 1) and done.dtype == bool
    assert torch.is_tensor(nxt["belief"]) and nxt["belief"].shape == (3, 37)


# ---- evaluation ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [1, 37, 1000])
@pytest.mark.parametrize("P", [1, 4])
@pytest.mark.parametrize("H", [1, 12, 50])
def test_evaluate_matches_float64(N, P, H):
    model = _model("planet", seed=N + P + H)
    env = _env(model)
    g = np.random.default_rng(N * 100 + P * 10 + H)
    acts = np.clip(g.standard_normal((N, H, 6)), -1, 1).astype(np.float32)
    eps = g.standard_normal((H, N * P, 30)).astype(np.float32)
    rows = torch.empty(N * P, device=DEV)
    got = env.evaluate_action_sequences(torch.from_numpy(acts).to(DEV), np.zeros((3, 64, 64), np.uint8), P,
                                        _eps=torch.from_numpy(eps).to(DEV), _row_returns=rows)
    want, want_rows = lo.evaluate(lo.params_of(model), *_post(model), acts, P, eps)
    assert _err(got, want) <= EVAL_BAR, _err(got, want)
    assert _err(rows, want_rows) <= EVAL_BAR, _err(rows, want_rows)


def test_in_kernel_draws_follow_the_counter_layout():
    model = _model("odd")
    env = _env(model, seed=123)
    N, P, H = 50, 3, 4
    g = np.random.default_rng(0)
    acts = np.clip(g.standard_normal((N, H, 1)), -1, 1).astype(np.float32)
    offset = (7 << 32) + 5 * 1024  # a high word too: it goes into the key
    rows = torch.empty(N * P, device=DEV)
    env.evaluate_action_sequences(torch.from_numpy(acts).to(DEV), np.zeros(3), P, _offset=offset, _row_returns=rows)
    eps = np.stack([latent_draws64(N * P, 7, t, env._seed, offset) for t in range(H)])
    _, want_rows = lo.evaluate(lo.params_of(model), *_post(model), acts, P, eps)
    assert _err(rows, want_rows) <= EVAL_BAR
    # one step: step 0 of the same counter layout
    B = 64
    s0 = torch.randn(B, 7, device=DEV)
    h0 = torch.tanh(torch.randn(B, 37, device=DEV))
    a0 = torch.rand(B, 1, device=DEV) * 2 - 1
    env._return_as_np = False
    nl, _, _, _ = env.step(a0, {"latent": s0, "belief": h0}, sample=True, _offset=offset)
    ws, _, _ = lo.step(lo.params_of(model), s0.cpu().numpy(), h0.cpu().numpy(), a0.cpu().numpy(),
                       latent_draws64(B, 7, 0, env._seed, offset))
    assert _err(nl, ws) <= STEP_BAR
    # consecutive calls draw from fresh counters
    n1, _, _, _ = env.step(a0, {"latent": s0, "belief": h0}, sample=True)
    n2, _, _, _ = env.step(a0, {"latent": s0, "belief": h0}, sample=True)
    assert not torch.equal(n1, n2)
    r1 = env.evaluate_action_sequences(torch.from_numpy(acts).to(DEV), np.zeros(3), P)
    r2 = env.evaluate_action_sequences(torch.from_numpy(acts).to(DEV), np.zeros(3), P)
    assert not torch.equal(r1, r2)


# ---- CEM plan --------------------------------------------------------------------------------------------------------
def _cem(env_model, N, it, clipped=True, alpha=0.1, rme=True):
    return planning.CEMOptimizer(num_iterations=it, elite_ratio=0.1, population_size=N,
                                 lower_bound=[[-1.0] * env_model.action_size] * 5,
                                 upper_bound=[[1.0] * env_model.action_size] * 5, alpha=alpha, device=DEV,
                                 return_mean_elites=rme, clipped_normal=clipped)


def _chain(env, opt, P, O, x0, z, eps):
    """The plan as separate calls: cem_sample -> evaluate_action_sequences -> cem_update, offsets O * 1024 + it."""
    lib = _lib.load()
    H, A = x0.shape
    dims, N, k = H * A, opt.population_size, opt.elite_num
    mu = x0.reshape(-1).clone()
    disp = torch.ones(dims, device=DEV) if opt._clipped_normal else \
        (((opt.upper_bound - opt.lower_bound) ** 2) / 16).reshape(-1).contiguous()
    best_val = torch.full((1,), float("-inf"), device=DEV)
    best_sol = torch.zeros(dims, device=DEV)
    pop = torch.empty(N, H, A, device=DEV)
    ws = torch.empty(lib.b200pets_cem_update_workspace_bytes(N, dims, k), dtype=torch.uint8, device=DEV)
    values = []
    stream = _lib.stream_ptr()
    for i in range(opt.num_iterations):
        off = O * 1024 + i
        zi = None if z is None else z[i].contiguous()
        _lib.check(lib.b200pets_cem_sample(N, dims, _lib.ptr(mu), _lib.ptr(disp), _lib.ptr(opt.lower_bound),
                                           _lib.ptr(opt.upper_bound), _lib.ptr(zi), env._seed, off,
                                           int(opt._clipped_normal), _lib.ptr(pop), stream))
        v = env.evaluate_action_sequences(pop, np.zeros(3), P, _offset=off, _eps=None if eps is None else eps[i])
        _lib.check(lib.b200pets_cem_update(N, dims, k, float(opt.alpha), 1, int(opt._clipped_normal), _lib.ptr(pop),
                                           _lib.ptr(v), _lib.ptr(mu), _lib.ptr(disp), _lib.ptr(best_val),
                                           _lib.ptr(best_sol), None, None, _lib.ptr(ws), ws.numel(), stream))
        values.append(v.clone())
    return (mu if opt.return_mean_elites else best_sol).view(H, A), torch.stack(values)


@pytest.mark.parametrize("N,P", [(1000, 1), (300, 4), (2500, 1)])  # 2500: above the single-CTA refit (three launches)
@pytest.mark.parametrize("injected", [False, True])
@pytest.mark.parametrize("rme", [True, False])
def test_cem_plan_equals_the_chain(N, P, injected, rme):
    model = _model("planet")
    env = _env(model)
    it, H = 4, 5
    opt = _cem(model, N, it, rme=rme)
    opt.record_values = True
    g = torch.Generator(device=DEV)
    g.manual_seed(N)
    z = torch.randn(it, N, H, 6, device=DEV, generator=g) if injected else None
    eps = torch.randn(it, H, N * P, 30, device=DEV, generator=g) if injected else None
    x0 = torch.zeros(H, 6, device=DEV)
    env._offset = 40
    sol = opt.optimize(planning._FusedObjective(env, np.zeros((3, 64, 64)), P), x0, _noise=z, _model_noise=(None, eps))
    assert env._offset == 41
    want_sol, want_values = _chain(env, opt, P, 41, x0, z, eps)
    assert torch.equal(opt.last_values, want_values)
    assert torch.equal(sol, want_sol)


def test_cem_plan_matches_float64_at_planet_cheetah_run():
    c = PLANET_CHEETAH
    model = _model("planet", seed=3)
    env = _env(model)
    N, H, it = c["population_size"], c["horizon"], c["num_iterations"]
    opt = planning.CEMOptimizer(num_iterations=it, elite_ratio=c["elite_ratio"], population_size=N,
                                lower_bound=[[-1.0] * 6] * H, upper_bound=[[1.0] * 6] * H, alpha=c["alpha"], device=DEV,
                                return_mean_elites=True, clipped_normal=True)
    g = np.random.default_rng(9)
    z = g.standard_normal((it, N, H, 6)).astype(np.float32)
    eps = g.standard_normal((it, H, N, 30)).astype(np.float32)
    sol = opt.optimize(planning._FusedObjective(env, np.zeros((3, 64, 64)), 1), torch.zeros(H, 6, device=DEV),
                       _noise=torch.from_numpy(z).to(DEV), _model_noise=(None, torch.from_numpy(eps).to(DEV)))
    want = lo.cem_plan(lo.params_of(model), *_post(model), np.zeros((H, 6)), -np.ones((H, 6)), np.ones((H, 6)), it,
                       c["elite_ratio"], N, c["alpha"], z, eps)
    err = float(np.max(np.abs(sol.cpu().numpy() - want)))
    assert err <= 1e-3, err


# ---- drop-in ---------------------------------------------------------------------------------------------------------
def _agent_cfg(optimizer_cfg, H=12):
    return {"_target_": "mbrl.planning.TrajectoryOptimizerAgent", "action_lb": "???", "action_ub": "???",
            "planning_horizon": H, "optimizer_cfg": optimizer_cfg, "replan_freq": 1, "keep_last_solution": False,
            "verbose": False}


CEM_CFG = {"_target_": "mbrl.planning.CEMOptimizer", "num_iterations": 10, "elite_ratio": 0.1, "population_size": 1000,
           "alpha": 0.0, "lower_bound": "???", "upper_bound": "???", "return_mean_elites": True, "device": DEV,
           "clipped_normal": True}
ICEM_CFG = {"_target_": "mbrl.planning.ICEMOptimizer", "num_iterations": 3, "elite_ratio": 0.1, "population_size": 200,
            "population_decay_factor": 1.25, "colored_noise_exponent": 2.0, "keep_elite_frac": 0.1, "alpha": 0.1,
            "lower_bound": "???", "upper_bound": "???", "return_mean_elites": True, "population_size_module": None,
            "device": DEV}
MPPI_CFG = {"_target_": "mbrl.planning.MPPIOptimizer", "num_iterations": 3, "gamma": 10.0, "population_size": 200,
            "sigma": 1.0, "beta": 0.9, "lower_bound": "???", "upper_bound": "???", "device": DEV}


def _act_checks(env, obs):
    for cfg in (CEM_CFG, ICEM_CFG, MPPI_CFG):
        agent = bp.create_trajectory_optim_agent_for_model(env, _agent_cfg(dict(cfg)))
        a = agent.act(obs)
        assert a.shape == (env.action_space.shape[0],) and np.isfinite(a).all(), cfg["_target_"]
        assert (a >= -1.0).all() and (a <= 1.0).all(), (cfg["_target_"], a)


def test_agent_over_the_local_container():
    model = _model("planet")
    env = _env(model)
    assert isinstance(env, latent.LatentModelEnv)
    _act_checks(env, np.random.default_rng(0).integers(0, 255, (3, 64, 64), dtype=np.uint8))


@needs_ref
def test_agent_over_the_reference_planet_model():
    model = mbrl.models.PlaNetModel(
        obs_shape=(3, 64, 64), obs_encoding_size=1024,
        encoder_config=((3, 32, 4, 2), (32, 64, 4, 2), (64, 128, 4, 2), (128, 256, 4, 2)),
        decoder_config=((1024, 1, 1), ((1024, 128, 5, 2), (128, 64, 5, 2), (64, 32, 6, 2), (32, 3, 6, 2))),
        latent_state_size=30, action_size=6, belief_size=200, hidden_size_fcs=200, device=DEV)
    rng = torch.Generator(device=DEV)
    obs = np.random.default_rng(1).integers(0, 255, (3, 64, 64), dtype=np.uint8)
    model.update_posterior(obs, rng=rng)  # the conv encoder, as mbrl/algorithms/planet.py:163 runs it
    env = bp.ModelEnv(_Env(6), model, mbrl.env.termination_fns.no_termination, generator=rng)
    assert isinstance(env, latent.LatentModelEnv)
    _act_checks(env, obs)
    # the same evaluation as the reference's ModelEnv with the draws fed to its torch.randn
    N, H = 64, 12
    acts = torch.rand(N, H, 6, device=DEV) * 2 - 1
    eps = torch.randn(H, N, 30, device=DEV)
    got = env.evaluate_action_sequences(acts, obs, 1, _eps=eps)
    ref_env = mbrl.models.ModelEnv(_Env(6), model, mbrl.env.termination_fns.no_termination, generator=rng)
    queue = list(eps)
    orig = torch.randn
    torch.randn = lambda *a, **kw: queue.pop(0)
    try:
        want = ref_env.evaluate_action_sequences(acts, obs, 1)
    finally:
        torch.randn = orig
    assert _err(got, want.cpu().double().numpy()) <= EVAL_BAR


# ---- re-staging, plan info, refusals ---------------------------------------------------------------------------------
def test_restaging_after_an_optimizer_step():
    model = _model("odd")
    env = _env(model)
    acts = torch.rand(20, 6, 1, device=DEV) * 2 - 1
    eps = torch.randn(6, 20, 7, device=DEV)
    env.evaluate_action_sequences(acts, np.zeros(3), 1, _eps=eps)
    opt = torch.optim.Adam(model.parameters(), lr=0.05)
    loss = sum((p ** 2).sum() for p in latent.latent_params(model))
    loss.backward()
    opt.step()  # in place: same storage, new version counters
    got = env.evaluate_action_sequences(acts, np.zeros(3), 1, _eps=eps)
    want, _ = lo.evaluate(lo.params_of(model), *_post(model), acts.cpu().numpy(), 1, eps.cpu().numpy())
    assert _err(got, want) <= EVAL_BAR


def test_plan_info_spreads_a_planet_population_over_the_sms():
    env = _env(_model("planet"))
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    info = env.staged.plan_info(1000)
    want = 1
    while want < -(-1000 // sms) and want < 32:
        want *= 2
    assert info["rows_per_cta"] == want and info["ctas"] == -(-1000 // want)
    assert info["smem"] >= want * info["row_bytes"]
    if sms == 132:
        assert (info["rows_per_cta"], info["ctas"]) == (8, 125)
    assert env.staged.plan_info(1)["rows_per_cta"] == 1


def test_refusals():
    with pytest.raises(NotImplementedError, match="limit"):
        _env(_model((6, 30, 1204, 1204)))
    model = _model("odd")
    with pytest.raises(NotImplementedError, match="reward_fn"):
        bp.ModelEnv(_Env(1), model, functions.no_termination, functions.reward_halfcheetah)
    with pytest.raises(NotImplementedError, match="no_termination"):
        bp.ModelEnv(_Env(1), model, functions.term_hopper)
    env = _env(model)
    agent = bp.create_trajectory_optim_agent_for_model(env, _agent_cfg(dict(CEM_CFG, population_size=50), H=3))
    with pytest.raises(NotImplementedError, match="one posterior"):
        agent.act_batch(np.zeros((2, 3, 64, 64)))
    with pytest.raises(NotImplementedError, match="one posterior"):
        env.evaluate_action_sequences_batch(torch.zeros(2, 4, 3, 1, device=DEV), np.zeros((2, 3)), 1)
    model.reset_posterior()
    with pytest.raises(RuntimeError, match="update_posterior"):
        env.evaluate_action_sequences(torch.zeros(4, 3, 1, device=DEV), np.zeros(3), 1)
