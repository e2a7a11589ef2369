"""Full-size / size-independent properties on the GPU (BASELINE.json configs 2, 4, 5) where the oracle is too slow to
be the checker: determinism, top-k invariants of the radix-select path, conservation checks of the MBPO step."""
import numpy as np
import pytest
import torch

from mbrl_lib_b200 import synthetic as syn
from test_gpu_parity import DEV, make_env

pytestmark = pytest.mark.gpu


def _refit_values(N, k, seed):
    """Returns with every hazard of the selection: NaN (-> -1e-10), +inf among the elites, -inf, and the k-th value in
    the middle of a run of k exact zeros of both signs, so the selection ends inside a tie."""
    g = np.random.default_rng(seed)
    v = g.standard_normal(N).astype(np.float32)
    order = g.permutation(N)
    hi, zeros, rest = order[:k // 2], order[k // 2:k // 2 + k], order[k // 2 + k:]
    v[hi] = np.abs(v[hi]) + 1.0
    v[hi[:2]] = np.inf
    v[zeros] = np.where(g.random(zeros.size) < 0.5, np.float32(0.0), np.float32(-0.0))
    v[rest] = -np.abs(v[rest]) - 1e-3
    v[rest[:max(3, N // 977)]] = np.nan
    v[rest[-3:]] = -np.inf
    return v


# (population, dims, k, unbiased, use_std, elites_out): run_select's three kernels --
#   n <= 2048 with k * dims * 4 <= 150 KB: the single-CTA refit with the elite rows in shared memory;
#   n <= 2048 with larger elite sets: cem_select_kernel's counting rank (config 3's iCEM refit: pop 1000, k 100, 40 x 17),
#     and with dims > 1241 its partial sums in the global workspace;
#   n > 2048: cem_select_kernel's radix select (config 5's scale), again also with global partial sums.
REFIT_SHAPES = {
    "single_cta": (500, 180, 50, 1, 0, True),
    "counting_config3": (1000, 680, 100, 1, 1, True),
    "counting_global_partials": (1500, 1300, 40, 0, 0, False),
    # iCEM's flags (biased variance, no std, elite rows out) at bench config 3's first and last populations
    "counting_icem_first": (1030, 680, 100, 0, 0, True),
    "counting_icem_last": (356, 680, 100, 0, 0, True),
    "radix_config5": (64000, 36, 6400, 1, 0, False),
    "radix_global_partials": (5000, 1300, 60, 0, 1, True),
}


def test_large_population_refit_matches_torch():
    """config 5 scale: N = 64 000, k = 6 400 goes through the radix-select path (checker: _check_refit)."""
    _check_refit("radix_config5")


@pytest.mark.parametrize("branch", [b for b in REFIT_SHAPES if b != "radix_config5"])
def test_refit_branches_match_float64(branch):
    """The other kernels run_select dispatches to (see REFIT_SHAPES), with the same checker."""
    _check_refit(branch)


def _check_refit(branch):
    """b200pets_cem_update against a float64 restatement of trajectory_opt.py:170-186: elites = the first k of the
    stable order by (-value, index) (the header's "ties broken by lowest index", -0.0 equal to +0.0), momentum-blended
    mean / (unbiased) variance or std, best value / row, elite rows by descending value."""
    from mbrl_lib_b200 import _lib

    lib = _lib.load()
    N, dims, k, unbiased, use_std, with_elites = REFIT_SHAPES[branch]
    alpha = 0.1
    vals = _refit_values(N, k, seed=N + dims)
    g = np.random.default_rng(dims)
    pop = g.standard_normal((N, dims)).astype(np.float32)
    mu0 = g.standard_normal(dims).astype(np.float32)
    disp0 = (0.5 + g.random(dims)).astype(np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)  # noqa: E731
    pop_d, v_d, mu, disp = t(pop), t(vals), t(mu0), t(disp0)
    best_v = torch.full((1,), float("-inf"), device=DEV)
    best_s = torch.zeros(dims, device=DEV)
    idx = torch.empty(k, dtype=torch.int32, device=DEV)
    elites = torch.full((k, dims), float("nan"), device=DEV) if with_elites else None
    nbytes = lib.b200pets_cem_update_workspace_bytes(N, dims, k)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    _lib.check(lib.b200pets_cem_update(N, dims, k, alpha, unbiased, use_std, _lib.ptr(pop_d), _lib.ptr(v_d), _lib.ptr(mu),
                                       _lib.ptr(disp), _lib.ptr(best_v), _lib.ptr(best_s), _lib.ptr(idx), _lib.ptr(elites),
                                       _lib.ptr(ws), nbytes, _lib.stream_ptr()))
    torch.cuda.synchronize()
    ref = np.where(np.isnan(vals), np.float32(-1e-10), vals)
    assert np.array_equal(v_d.cpu().numpy(), ref)  # NaN rule applied in place
    key = ref + np.float32(0.0)  # -0.0 -> +0.0
    order = np.lexsort((np.arange(N), -key))  # stable: by descending value, then ascending index
    want = np.sort(order[:k])
    got = idx.cpu().numpy()
    assert np.array_equal(got, want), (f"{np.setdiff1d(got, want).size} selected indices differ; "
                                       f"values of the extra ones {ref[np.setdiff1d(got, want)][:8]}")
    elite = pop[order[:k]].astype(np.float64)
    var = elite.var(0, ddof=1 if unbiased else 0)
    nd = np.sqrt(var) if use_std else var
    np.testing.assert_allclose(mu.cpu().numpy(), alpha * mu0 + (1 - alpha) * elite.mean(0), rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(disp.cpu().numpy(), alpha * disp0 + (1 - alpha) * nd, rtol=1e-4, atol=1e-5)
    assert float(best_v) == float(key[order[0]])  # +inf, lowest index of the two
    assert np.array_equal(best_s.cpu().numpy(), pop[order[0]])
    if with_elites:  # descending value, lower index first on ties: exactly the stable order's first k rows
        assert np.array_equal(elites.cpu().numpy(), pop[order[:k]])


@pytest.mark.parametrize("precision", ["bf16_tc", "f32"])
def test_rollout_is_deterministic_at_scale(precision):
    spec, arrays, env = make_env("halfcheetah", precision, ts1="tile_shuffle")
    N = 4000 if precision == "bf16_tc" else 1000
    g = np.random.default_rng(0)
    acts = torch.from_numpy(g.uniform(-1, 1, (N, spec.horizon, spec.act_dim)).astype(np.float32)).to(DEV)
    obs0 = syn.make_rollout_inputs(spec, with_noise=False)["obs0"]
    env._offset = 100
    r1 = env.evaluate_action_sequences(acts, obs0, spec.particles)
    env._offset = 100
    r2 = env.evaluate_action_sequences(acts, obs0, spec.particles)
    assert torch.equal(r1, r2) and bool(torch.isfinite(r1).all())  # same Philox (seed, offset) => bit-identical
    env._offset = 101
    r3 = env.evaluate_action_sequences(acts, obs0, spec.particles)
    assert not torch.equal(r1, r3)


@pytest.mark.parametrize("precision", ["bf16_tc", "f32"])
def test_mbpo_step_full_size(precision):
    """config 4: 100 000 start states x 1 step (mbpo.py:31-63).  Mean prediction (sample=False) must equal the model
    applied row by row: check a random subset against the oracle, and conservation properties on all rows."""
    from oracle import pets_oracle as po

    spec, arrays, env = make_env("mbpo_halfcheetah", precision, ts1="tile_shuffle")
    B = 100000
    inp = syn.make_step_inputs(spec, B)
    state = env.reset(inp["obs"], return_as_np=False)
    act = torch.from_numpy(inp["act"]).to(DEV)
    perm = torch.from_numpy(inp["perm"]).to(DEV)
    nobs, rew, done, _ = env.step(act, state, sample=False, _perm=perm)
    assert nobs.shape == (B, spec.obs_dim) and rew.shape == (B, 1) and done.shape == (B, 1)
    assert bool(torch.isfinite(nobs).all()) and not bool(done.any())  # no_termination
    # a slice of member 0's rows, checked against the oracle's member MLP
    M = len(spec.elites)
    rows = perm[: B // M][:256].cpu()
    m = po.OracleModel(spec, arrays)
    m.emulate_bf16 = precision == "bf16_tc"
    x = m.model_input(torch.from_numpy(inp["obs"])[rows], torch.from_numpy(inp["act"])[rows])
    mean, _ = m.mlp(x.unsqueeze(0).expand(M, -1, -1).contiguous())
    pred = mean[0]
    ref_nobs = pred[:, :-1] + torch.from_numpy(inp["obs"])[rows]
    tol = 2e-4 if precision == "f32" else 5e-3
    scale = max(1.0, float(ref_nobs.abs().max()))
    assert float((nobs[rows.to(DEV)].cpu() - ref_nobs).abs().max()) <= tol * scale
    assert float((rew[rows.to(DEV)].cpu()[:, 0] - pred[:, -1]).abs().max()) <= tol * scale


def test_icem_over_model_runs_and_improves():
    """config 3 shape family: iCEM (coloured noise, decaying population, kept elites) driving the model rollout."""
    import mbrl_lib_b200 as bp

    spec, arrays, env = make_env("humanoid_trunc", "auto", ts1="tile_shuffle")
    H, A = spec.horizon, spec.act_dim
    lb, ub = np.full((H, A), spec.action_lb).tolist(), np.full((H, A), spec.action_ub).tolist()
    opt = bp.ICEMOptimizer(4, 0.1, 350, 1.3, 2.0, lb, ub, 0.3, 0.1, DEV, return_mean_elites=False, population_size_module=5)
    obs0 = syn.make_rollout_inputs(spec, with_noise=False)["obs0"]
    best = []

    def obj(pop):
        return env.evaluate_action_sequences(pop, obs0, spec.particles)

    sol = opt.optimize(obj, x0=torch.zeros(H, A, device=DEV), callback=lambda p, v, i: best.append(float(v.max())))
    assert sol.shape == (H, A) and bool(torch.isfinite(sol).all())
    assert float(sol.min()) >= spec.action_lb - 1e-6 and float(sol.max()) <= spec.action_ub + 1e-6
    assert opt.elite.shape == (opt.elite_num, H, A)
    assert max(best[1:]) >= best[0] - 0.05  # later generations are at least as good as the first (noisy objective)
    sol2 = opt.optimize(obj, x0=torch.zeros(H, A, device=DEV))  # second call: shifted elites of the previous plan
    assert bool(torch.isfinite(sol2).all())


def _line_world(device):
    """A hand-built deterministic 'ensemble' that is exactly a 1-D point mass (ReLU pairs encode identity / abs):
    next_pos = pos + 0.1 * a, learned reward = -|next_pos|.  Plays the role of the reference's MockLineEnv
    integration test (tests/algorithms/test_algorithms.py:44-68) without needing model training."""
    import mbrl_lib_b200 as bp

    mlp = bp.GaussianMLP(2, 2, device, num_layers=1, ensemble_size=2, hid_size=32, deterministic=True,
                         propagation_method="random_model", activation="relu")
    w0 = torch.zeros(2, 2, 32)
    w0[:, 1, 0], w0[:, 1, 1] = 1.0, -1.0                      # relu(a), relu(-a)
    w0[:, 0, 2], w0[:, 1, 2] = 1.0, 0.1                       # relu(pos + 0.1 a)
    w0[:, 0, 3], w0[:, 1, 3] = -1.0, -0.1                     # relu(-(pos + 0.1 a))
    w1 = torch.zeros(2, 32, 2)
    w1[:, 0, 0], w1[:, 1, 0] = 0.1, -0.1                      # delta = 0.1 a
    w1[:, 2, 1], w1[:, 3, 1] = -1.0, -1.0                     # reward = -|pos + 0.1 a|
    with torch.no_grad():
        mlp.hidden_layers[0][0].weight.copy_(w0)
        mlp.hidden_layers[0][0].bias.zero_()
        mlp.mean_and_logvar.weight.copy_(w1)
        mlp.mean_and_logvar.bias.zero_()
    return bp.OneDTransitionRewardModel(mlp, target_is_delta=True, normalize=False, learned_rewards=True)


@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
def test_closed_loop_mpc_reaches_goal(precision):
    """Behavioural check of the whole agent loop on the GPU (act -> fused CEM plan -> warm-start shift -> act ...)."""
    import mbrl_lib_b200 as bp
    from mbrl_lib_b200 import functions
    from test_gpu_parity import _Env

    class _Spec:
        obs_dim, act_dim, action_lb, action_ub = 1, 1, -1.0, 1.0

    model = _line_world(DEV)
    env = bp.ModelEnv(_Env(_Spec), model, functions.no_termination, None, generator=torch.Generator(device=DEV),
                      precision=precision, ts1="tile_shuffle")
    cfg = {"_target_": "mbrl.planning.TrajectoryOptimizerAgent", "planning_horizon": 5, "replan_freq": 1,
           "optimizer_cfg": {"_target_": "mbrl.planning.CEMOptimizer", "num_iterations": 4, "elite_ratio": 0.1,
                             "population_size": 256, "alpha": 0.1, "device": DEV, "return_mean_elites": True}}
    agent = bp.create_trajectory_optim_agent_for_model(env, cfg, num_particles=2)
    pos, total = 1.0, 0.0
    for _ in range(18):
        a = float(np.clip(agent.act(np.array([pos])), -1, 1)[0])
        pos = pos + 0.1 * a  # the true environment is the same point mass
        total += -abs(pos)
    assert abs(pos) < 0.12, pos            # started at 1.0, can move 0.1 per step
    assert total > -7.5, total             # an agent that never moves collects -18


@pytest.mark.gpu
def test_rollout_model_env_matches_oracle_open_loop():
    """util/common.py:416-454 on the CUDA step kernel vs. the oracle stepping the same plan (TSinf, sample=False)."""
    import mbrl_lib_b200 as bp
    from oracle import pets_oracle as po

    spec, arrays, env = make_env("hopper_tsinf", "f32")
    S, L = 3 * spec.num_models, 6
    rng = np.random.default_rng(5)
    obs0 = rng.standard_normal(spec.obs_dim).astype(np.float32)
    plan = rng.uniform(spec.action_lb, spec.action_ub, size=(L, spec.act_dim)).astype(np.float32)
    torch.manual_seed(11)
    obs, rew, got_plan = bp.rollout_model_env(env, obs0, plan, None, num_samples=S)
    assert obs.shape == (L + 1, S, spec.obs_dim) and rew.shape == (L, S, 1) and got_plan is plan
    torch.manual_seed(11)
    perm = torch.randperm(S, device="cuda").cpu()  # the draw ModelEnv.reset made
    m = po.OracleModel(spec, arrays)
    o = torch.from_numpy(np.tile(obs0, (S, 1)))
    for t in range(L):
        o, r, _ = m.step(o, torch.from_numpy(np.tile(plan[t], (S, 1))), perm, None, sample=False)
        scale = max(1.0, float(o.abs().max()))
        assert np.abs(obs[t + 1] - o.numpy()).max() <= 5e-4 * scale
        assert np.abs(rew[t] - r.numpy().reshape(S, 1)).max() <= 5e-4 * max(1.0, float(r.abs().max()))
