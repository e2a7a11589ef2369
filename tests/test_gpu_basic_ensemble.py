"""Planning over a BasicEnsemble: per-row member indices bucketed into member tiles on the device.

* the bucketing kernel (``b200pets_member_slots``) against numpy's stable argsort and bincount;
* ``step`` and ``evaluate_action_sequences`` with injected indices and noise, row by row against the float64 transition
  with every row's own member (uneven member counts, B not a multiple of M or of 128);
* a BasicEnsemble whose members are the slices of a GaussianMLP ensemble gives, bit for bit, what the GaussianMLP path
  gives when its rows' indices are the reference's split of the permutation the GaussianMLP path is given;
* fused iCEM plans equal their per-iteration loop, batched CEM and MPPI plans equal single plans with the same draws,
  and a closed MPC loop reaches its goal;
* ``ModelEnv.step`` over mbrl-lib's own BasicEnsemble matches mbrl-lib's ``ModelEnv.step``.
"""
import dataclasses

import numpy as np
import pytest
import torch

from mbrl_lib_b200 import synthetic as syn
from oracle.transition_f64 import TransitionF64, assignment_from_perm
from test_gpu_parity import DEV, _Env
from test_gpu_transitions import BAR, compare_step

pytestmark = pytest.mark.gpu


def _lib():
    from mbrl_lib_b200 import _lib

    return _lib, _lib.load()


def _member_slots(idx: np.ndarray, M: int):
    _l, lib = _lib()
    K, B = idx.shape
    d_idx = torch.from_numpy(idx.astype(np.int64)).to(DEV)
    slots = torch.full((K, B), -7, dtype=torch.int64, device=DEV)
    offs = torch.full((K, M + 1), -7, dtype=torch.int32, device=DEV)
    _l.check(lib.b200pets_member_slots(K, B, M, _l.ptr(d_idx), _l.ptr(slots), _l.ptr(offs), _l.stream_ptr()), "member_slots")
    torch.cuda.synchronize()
    return slots.cpu().numpy(), offs.cpu().numpy()


def _expected(idx, M):
    key = np.where((idx >= 0) & (idx < M), idx, M)
    order = np.argsort(key, kind="stable")
    counts = np.bincount(key, minlength=M + 1)[:M]
    return order, np.concatenate([[0], np.cumsum(counts)])


def _indices(kind, B, M, g):
    if kind == "uniform":
        return g.integers(0, M, B)
    if kind == "one_member":
        return np.full(B, M - 1)
    if kind == "empty_members":  # only even members
        return 2 * g.integers(0, (M + 1) // 2, B)
    bad = g.integers(0, M, B)  # out of range
    bad[g.random(B) < 0.2] = -1
    bad[g.random(B) < 0.1] = M + 3
    return bad


@pytest.mark.parametrize("kind", ["uniform", "one_member", "empty_members", "out_of_range"])
@pytest.mark.parametrize("M", [1, 2, 5, 7])
@pytest.mark.parametrize("B", [1, 3, 127, 128, 129, 10_000, 100_000])
def test_member_slots_match_stable_argsort(B, M, kind):
    g = np.random.default_rng(B * 31 + M)
    idx = np.stack([_indices(kind, B, M, g) for _ in range(3)])  # three problems in one launch
    slots, offs = _member_slots(idx, M)
    for k in range(3):
        order, off = _expected(idx[k], M)
        assert np.array_equal(slots[k], order), k
        assert np.array_equal(offs[k], off), k


# ---- models ------------------------------------------------------------------------------------------------------
def _spec(name, propagation):
    """The case with every member used: the GaussianMLP ensemble and the BasicEnsemble of its slices are one model."""
    s = syn.CASES[name]
    return dataclasses.replace(s, propagation=propagation, elites=None)


def _envs(spec, arrays=None):
    import mbrl_lib_b200 as bp
    from mbrl_lib_b200 import functions
    from mbrl_lib_b200.models import basic_ensemble_from_arrays

    arrays = syn.make_model_arrays(spec) if arrays is None else arrays
    rew = functions.REWARD_FNS[spec.reward_fn] if spec.reward_fn else None
    term = functions.TERM_FNS[spec.term_fn]
    out = []
    for build in (bp.model_from_arrays, basic_ensemble_from_arrays):
        env = bp.ModelEnv(_Env(spec), build(spec, arrays, DEV), term, rew, generator=torch.Generator(device=DEV),
                          precision="f32", ts1="perms")
        out.append(env)
    assert out[1].staged.member_rule == "rows"
    return arrays, out[0], out[1]


PROPS = ["random_model", "fixed_model", "expectation"]


@pytest.mark.parametrize("prop", PROPS)
@pytest.mark.parametrize("name", ["halfcheetah_small", "hopper_tsinf", "plan_hid143"])
def test_step_equals_gaussian_mlp_path(name, prop):
    spec = _spec(name, prop)
    _, env_g, env_b = _envs(spec)
    M = spec.ensemble_size
    for rpm in (1, 127, 129):
        B = M * rpm
        inp = syn.make_step_inputs(spec, B)
        perm = torch.from_numpy(inp["perm"]).to(DEV)
        idx = torch.from_numpy(assignment_from_perm(inp["perm"], M)).to(DEV)
        eps = None if spec.deterministic else torch.from_numpy(inp["eps"]).to(DEV)
        sg = env_g.reset(inp["obs"], return_as_np=False)
        sb = env_b.reset(inp["obs"], return_as_np=False)
        use = prop != "expectation"
        g = env_g.step(inp["act"], sg, sample=True, _perm=perm if use else None, _eps=eps, _offset=5 * 1024)
        b = env_b.step(inp["act"], sb, sample=True, _perm=idx if use else None, _eps=eps, _offset=5 * 1024)
        for x, y in zip(g[:3], b[:3]):
            assert torch.equal(x, y), (rpm, prop)
        assert torch.isfinite(g[0]).all()


@pytest.mark.parametrize("prop", PROPS)
@pytest.mark.parametrize("name", ["halfcheetah_small", "hopper_tsinf", "silu_expectation"])
def test_evaluation_equals_gaussian_mlp_path(name, prop):
    spec = _spec(name, prop)
    _, env_g, env_b = _envs(spec)
    M, N, H, P = spec.ensemble_size, spec.population, spec.horizon, spec.particles
    N = N - N % M if (N * P) % M else N
    B = N * P
    inp = syn.make_rollout_inputs(spec, population=N)
    acts = torch.from_numpy(inp["actions"]).to(DEV)
    g = torch.Generator().manual_seed(7)
    nperm = H if prop == "random_model" else 1
    perms = torch.stack([torch.randperm(B, generator=g) for _ in range(nperm)])
    idx = torch.from_numpy(np.stack([assignment_from_perm(p.numpy(), M) for p in perms])).to(DEV)
    use = prop != "expectation"
    rg, rb = torch.empty(B, device=DEV), torch.empty(B, device=DEV)
    vg = env_g.evaluate_action_sequences(acts, inp["obs0"], P, _perms=perms.to(DEV) if use else None, _row_returns=rg, _offset=9 * 1024)
    vb = env_b.evaluate_action_sequences(acts, inp["obs0"], P, _perms=idx if use else None, _row_returns=rb, _offset=9 * 1024)
    assert torch.isfinite(vg).all()
    assert torch.equal(rg, rb) and torch.equal(vg, vb)


@pytest.mark.parametrize("prop", PROPS)
@pytest.mark.parametrize("name", ["halfcheetah_small", "plan_hid143", "humanoid_v4"])
def test_step_matches_float64_with_uneven_members(name, prop):
    """Per-row members drawn uniformly (uneven counts), B not a multiple of M or of 128; rows with an index outside
    [0, M) come back NaN and leave the other rows as they are."""
    spec = _spec(name, prop)
    arrays, _, env_b = _envs(spec)
    M = spec.ensemble_size
    ck = TransitionF64(spec, arrays, members=list(range(M)))
    g = np.random.default_rng(11)
    for B in (1, 3, 1000, 4099):
        inp = syn.make_step_inputs(spec, B)
        idx = g.integers(0, M, B)
        if prop != "expectation" and B > 3:
            idx[:: 97] = M  # out of range
        eps = None if spec.deterministic else inp["eps"]
        state = env_b.reset(inp["obs"], return_as_np=True)
        nobs, rew, done, _ = env_b.step(inp["act"], state, sample=True,
                                        _perm=torch.from_numpy(idx).to(DEV) if prop != "expectation" else None,
                                        _eps=None if eps is None else torch.from_numpy(eps).to(DEV), _offset=3 * 1024)
        ok = (idx < M) if prop != "expectation" else np.ones(B, bool)
        assert np.isnan(nobs[~ok]).all() and np.isnan(rew[~ok]).all()
        rows = np.nonzero(ok)[0]
        err = compare_step(spec, ck, inp["obs"][rows], inp["act"][rows], None if prop == "expectation" else idx[rows],
                           None if eps is None else eps[rows], nobs[rows], rew[rows, 0], done[rows, 0], False)
        assert err["next_obs"] <= BAR["f32"] and err["reward"] <= BAR["f32"] and err["done"] == 0, (B, err)


def test_reset_draws_like_the_reference():
    """``reset`` draws fixed_model's indices with one ``randint(M, (B,))`` on the environment's generator (the step's
    random_model draw is checked against the reference's own step below)."""
    spec = _spec("halfcheetah_small", "fixed_model")
    _, _, env = _envs(spec)
    M, B = spec.ensemble_size, 37
    env._rng.manual_seed(123)
    state = env.reset(np.zeros((B, spec.obs_dim), np.float32), return_as_np=False)
    ref = torch.Generator(device=DEV).manual_seed(123)
    assert torch.equal(state["propagation_indices"], torch.randint(M, (B,), generator=ref, device=DEV))


def _cem(env, spec, K, iters):
    import mbrl_lib_b200 as bp
    from mbrl_lib_b200.planning import _FusedBatchObjective, _FusedObjective

    H, A = spec.horizon, spec.act_dim
    lb, ub = np.full((H, A), spec.action_lb).tolist(), np.full((H, A), spec.action_ub).tolist()
    opt = bp.CEMOptimizer(iters, 0.1, spec.population, lb, ub, 0.1, DEV, return_mean_elites=True)
    opt.record_values = True
    g = np.random.default_rng(2)
    obs = np.stack([0.1 * k * g.standard_normal(spec.obs_dim) for k in range(K)])
    x0 = torch.from_numpy(g.uniform(-0.5, 0.5, (K, H, A)).astype(np.float32)).to(DEV)
    env._offset = 100
    env._rng.manual_seed(77)
    sol = opt.optimize_batch(_FusedBatchObjective(env, obs, spec.particles), x0=x0).clone()
    vals = opt.last_values.clone()
    env._rng.manual_seed(77)
    singles = []
    for k in range(K):
        env._offset = 100 + k
        singles.append((opt.optimize(_FusedObjective(env, obs[k], spec.particles), x0=x0[k]).clone(),
                        opt.last_values.clone()))
    return sol, vals, singles


@pytest.mark.parametrize("K", [1, 3])
@pytest.mark.parametrize("prop", ["random_model", "fixed_model"])
def test_batched_cem_plan_equals_single_plans(prop, K):
    spec = dataclasses.replace(_spec("halfcheetah", prop), population=203, horizon=8, particles=6)
    _, _, env = _envs(spec)
    sol, vals, singles = _cem(env, spec, K, 3)
    for k, (s, v) in enumerate(singles):
        assert torch.isfinite(s).all()
        assert torch.equal(vals[k], v) and torch.equal(sol[k], s), k


def test_closed_loop_reaches_goal():
    """The line world of test_gpu_scale as a BasicEnsemble of its two members, driven by agent.act (fused CEM)."""
    import mbrl_lib_b200 as bp
    from mbrl_lib_b200 import functions
    from test_gpu_scale import _line_world

    src = _line_world(DEV).model
    members = []
    for e in range(2):
        m = bp.GaussianMLP(2, 2, DEV, num_layers=1, ensemble_size=1, hid_size=32, deterministic=True, activation="relu")
        with torch.no_grad():
            for dst, s in ((m.hidden_layers[0][0], src.hidden_layers[0][0]), (m.mean_and_logvar, src.mean_and_logvar)):
                dst.weight.copy_(s.weight[e:e + 1])
                dst.bias.copy_(s.bias[e:e + 1])
        members.append(m)
    model = bp.OneDTransitionRewardModel(bp.BasicEnsemble(members, "random_model"), target_is_delta=True, normalize=False,
                                         learned_rewards=True)

    class _Spec:
        obs_dim, act_dim, action_lb, action_ub = 1, 1, -1.0, 1.0

    env = bp.ModelEnv(_Env(_Spec), model, functions.no_termination, None, generator=torch.Generator(device=DEV))
    ocfg = {"_target_": "mbrl.planning.CEMOptimizer", "device": DEV, "num_iterations": 4, "elite_ratio": 0.1,
            "population_size": 255, "alpha": 0.1, "return_mean_elites": True}
    agent = bp.create_trajectory_optim_agent_for_model(
        env, {"_target_": "mbrl.planning.TrajectoryOptimizerAgent", "planning_horizon": 5, "replan_freq": 1,
              "optimizer_cfg": ocfg}, num_particles=3)
    pos = 0.9
    for _ in range(18):
        pos += 0.1 * float(np.clip(agent.act(np.array([pos])), -1, 1)[0])
    assert abs(pos) < 0.12, pos


# ---- tensor-core kernel and every fp32 tile plan -------------------------------------------------------------------
def _step_rows_check(spec, env, arrays, precision, batches, seed=13):
    """step with uneven per-row members against the float64 transition (bf16-rounded operands on the tensor cores)."""
    M = spec.ensemble_size
    ck = TransitionF64(spec, arrays, members=list(range(M)))
    g = np.random.default_rng(seed)
    prop = spec.propagation
    for B in batches:
        inp = syn.make_step_inputs(spec, B)
        idx = g.integers(0, M, B)
        eps = None if spec.deterministic else inp["eps"]
        state = env.reset(inp["obs"], return_as_np=True)
        nobs, rew, done, _ = env.step(inp["act"], state, sample=True,
                                      _perm=torch.from_numpy(idx).to(DEV) if prop != "expectation" else None,
                                      _eps=None if eps is None else torch.from_numpy(eps).to(DEV), _offset=7 * 1024)
        rows = np.unique(np.concatenate([np.arange(min(B, 600)), np.arange(0, B, max(1, B // 600)), [B - 1]]))
        err = compare_step(spec, ck, inp["obs"][rows], inp["act"][rows], None if prop == "expectation" else idx[rows],
                           None if eps is None else eps[rows], nobs[rows], rew[rows, 0], done[rows, 0], precision == "bf16_tc")
        assert err["next_obs"] <= BAR[precision] and err["reward"] <= BAR[precision] and err["done"] == 0, (B, err)


@pytest.mark.parametrize("prop", PROPS)
@pytest.mark.parametrize("name", ["halfcheetah_small", "plan_hid143"])
def test_tensor_core_step_matches_float64(name, prop):
    """B = 1000 (fewer tiles than SMs: 64-row CTAs) and B = 40 000 (more: 128-row CTAs)."""
    from test_gpu_tiles import _sm_count

    import mbrl_lib_b200 as bp
    from mbrl_lib_b200 import functions
    from mbrl_lib_b200.models import basic_ensemble_from_arrays

    spec = _spec(name, prop)
    arrays = syn.make_model_arrays(spec)
    rew = functions.REWARD_FNS[spec.reward_fn] if spec.reward_fn else None
    env = bp.ModelEnv(_Env(spec), basic_ensemble_from_arrays(spec, arrays, DEV), functions.TERM_FNS[spec.term_fn], rew,
                      generator=torch.Generator(device=DEV), precision="bf16_tc")
    if not env.staged.supports_tc(prop):
        pytest.skip("no tensor-core plan for this propagation")
    assert (1000 + 127) // 128 + spec.ensemble_size - 1 < _sm_count() < 40000 // 128
    _step_rows_check(spec, env, arrays, "bf16_tc", (1000, 40000))


@pytest.mark.parametrize("prop", ["random_model", "fixed_model"])
def test_tensor_core_evaluation_equals_gaussian_mlp_path(prop):
    import mbrl_lib_b200 as bp
    from mbrl_lib_b200 import functions
    from mbrl_lib_b200.models import basic_ensemble_from_arrays

    spec = _spec("halfcheetah_small", prop)
    arrays = syn.make_model_arrays(spec)
    rew = functions.REWARD_FNS[spec.reward_fn] if spec.reward_fn else None
    envs = [bp.ModelEnv(_Env(spec), b(spec, arrays, DEV), functions.TERM_FNS[spec.term_fn], rew,
                        generator=torch.Generator(device=DEV), precision="bf16_tc", ts1="perms")
            for b in (bp.model_from_arrays, basic_ensemble_from_arrays)]
    M, H, P = spec.ensemble_size, spec.horizon, spec.particles
    for N in (7 * 6, 7 * 400):  # B a multiple of the 7 members, as the GaussianMLP path needs
        B = N * P
        inp = syn.make_rollout_inputs(spec, population=N)
        acts = torch.from_numpy(inp["actions"]).to(DEV)
        g = torch.Generator().manual_seed(N)
        perms = torch.stack([torch.randperm(B, generator=g) for _ in range(H if prop == "random_model" else 1)])
        idx = torch.from_numpy(np.stack([assignment_from_perm(p.numpy(), M) for p in perms])).to(DEV)
        rows = [torch.empty(B, device=DEV) for _ in envs]
        for env, pm, r in zip(envs, (perms.to(DEV), idx), rows):
            env.evaluate_action_sequences(acts, inp["obs0"], P, _perms=pm, _row_returns=r, _offset=11 * 1024)
        assert torch.isfinite(rows[0]).all() and torch.equal(rows[0], rows[1]), N


def test_every_f32_tile_plan_matches_float64():
    """The fp32 kernel's 64-, 32- and 16-row tiles (the widest models the shared memory takes at each)."""
    import mbrl_lib_b200 as bp
    from mbrl_lib_b200 import functions
    from mbrl_lib_b200.models import basic_ensemble_from_arrays

    seen = {}
    for name in syn.CASES:
        spec = _spec(name, "random_model")
        if spec.ensemble_size < 2:
            continue
        arrays = syn.make_model_arrays(spec)
        rew = functions.REWARD_FNS[spec.reward_fn] if spec.reward_fn else None
        env = bp.ModelEnv(_Env(spec), basic_ensemble_from_arrays(spec, arrays, DEV), functions.TERM_FNS[spec.term_fn], rew,
                          generator=torch.Generator(device=DEV), precision="f32")
        rows = env.staged.plan_info("random_model")["f32_rows"]
        if rows in seen:
            continue
        seen[rows] = name
        _step_rows_check(spec, env, arrays, "f32", (3, 1001))
    print(seen)
    assert set(seen) == {64, 32, 16}, seen


# ---- fused plans against their loops -------------------------------------------------------------------------------
def _compare_fused_and_loop(env, fused, loop, obs, P, x0):
    """Both optimisers from the same counters and the same state of the environment's generator."""
    from mbrl_lib_b200.planning import _FusedObjective

    obj = _FusedObjective(env, obs, P)
    # the environment's generator draws the members, torch's default CUDA generator iCEM's kept-elite permutations
    rng, cuda_rng, offset = env._rng.get_state(), torch.cuda.get_rng_state(), env._offset
    got = fused.optimize(obj, x0=x0).clone(), [v.clone() for v in fused.last_values]
    after = env._rng.get_state(), env._offset
    env._rng.set_state(rng)
    torch.cuda.set_rng_state(cuda_rng)
    env._offset = offset
    seen = []
    sol = loop.optimize(lambda seqs: obj(seqs), x0=x0, callback=lambda pop, v, i: seen.append(v.clone())).clone()
    ref = sol, [v.clone() for v in loop.last_values] if loop.last_values is not None else seen
    assert env._offset == after[1] and torch.equal(env._rng.get_state(), after[0])
    assert len(got[1]) == len(ref[1]) == loop.num_iterations
    for i, (v, r) in enumerate(zip(got[1], ref[1])):
        assert torch.equal(v, r), f"values of iteration {i} differ"
    assert torch.isfinite(got[0]).all() and torch.equal(got[0], ref[0])


@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
@pytest.mark.parametrize("prop", ["random_model", "fixed_model"])
def test_fused_icem_plan_equals_the_loop(prop, precision):
    import mbrl_lib_b200 as bp

    spec = _spec("halfcheetah_small", prop)
    _, _, env = _envs(spec)
    env.precision = precision
    H, A, P = 10, spec.act_dim, 5
    lb, ub = np.full((H, A), spec.action_lb).tolist(), np.full((H, A), spec.action_ub).tolist()
    fused, loop = (bp.ICEMOptimizer(5, 0.1, 200, 1.3, 2.0, lb, ub, 0.3, 0.1, DEV, return_mean_elites=True,
                                    population_size_module=7) for _ in range(2))
    for o in (fused, loop):
        o.record_values = True
    obs = syn.make_rollout_inputs(spec, with_noise=False)["obs0"]
    g = np.random.default_rng(1)
    env._offset = 40
    for _ in range(2):  # a cold and a warm-started plan (kept elites)
        x0 = torch.from_numpy(g.uniform(-0.3, 0.3, (H, A)).astype(np.float32)).to(DEV)
        _compare_fused_and_loop(env, fused, loop, obs, P, x0)


@pytest.mark.parametrize("prop", ["random_model", "fixed_model"])
def test_batched_mppi_plan_equals_single_plans(prop):
    import mbrl_lib_b200 as bp
    from mbrl_lib_b200.planning import _FusedBatchObjective

    spec = dataclasses.replace(_spec("halfcheetah_small", prop), horizon=8, population=203, particles=6)
    _, _, env = _envs(spec)
    K, R, P, H, A = 3, 3, spec.particles, spec.horizon, spec.act_dim
    lb, ub = np.full((H, A), spec.action_lb).tolist(), np.full((H, A), spec.action_ub).tolist()
    opt = bp.MPPIOptimizer(R, spec.population, 0.9, 1.0, 0.3, lb, ub, DEV)
    g = np.random.default_rng(4)
    obs = g.standard_normal((K, spec.obs_dim))
    m0 = torch.from_numpy(g.uniform(-0.5, 0.5, (K, H, A)).astype(np.float32)).to(DEV)
    opt.batch_mean = m0.clone()
    env._offset, opt._offset = 100, 50
    env._rng.manual_seed(9)
    got = opt.optimize_batch(_FusedBatchObjective(env, obs, P)).clone()
    env._rng.manual_seed(9)
    for k in range(K):
        env._offset, opt._offset = 100 + k * R, 50 + k
        opt.mean = m0[k].clone()
        s = opt.optimize(lambda pop, k=k: env.evaluate_action_sequences(pop, initial_state=obs[k], num_particles=P))
        assert torch.isfinite(s).all() and torch.equal(got[k], s), k


# ---- against the reference ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("prop", ["random_model", "fixed_model", "expectation"])
def test_step_over_the_reference_basic_ensemble_matches_reference_step(prop):
    """Our ModelEnv over mbrl-lib's own BasicEnsemble on cuda against mbrl-lib's ModelEnv.step, same
    propagation_indices (random_model: the same generator state), sample=False."""
    from baseline import reference_arm as ra

    mbrl, src = ra.import_reference()
    if mbrl is None:
        pytest.skip(f"reference not importable here: {src}")
    import mbrl.models as mm

    import mbrl_lib_b200 as bp
    from mbrl_lib_b200 import functions

    spec = _spec("halfcheetah_small", prop)
    arrays = syn.make_model_arrays(spec)
    cfg = {"_target_": "mbrl.models.GaussianMLP", "device": DEV, "num_layers": spec.num_layers, "in_size": spec.in_size,
           "out_size": spec.out_size, "ensemble_size": 1, "hid_size": spec.hid_size, "deterministic": False,
           "activation_fn_cfg": {"_target_": "torch.nn.SiLU" if spec.activation == "silu" else "torch.nn.ReLU"}}
    ens = mm.BasicEnsemble(spec.ensemble_size, DEV, cfg, propagation_method=prop)
    with torch.no_grad():
        for e, m in enumerate(ens.members):
            for li, lin in enumerate([seq[0] for seq in m.hidden_layers] + [m.mean_and_logvar]):
                lin.weight.copy_(torch.from_numpy(arrays["weights"][li][e:e + 1]))
                lin.bias.copy_(torch.from_numpy(arrays["biases"][li][e:e + 1]))
            m.min_logvar.copy_(torch.from_numpy(arrays["min_logvar"]))
            m.max_logvar.copy_(torch.from_numpy(arrays["max_logvar"]))
    model = mm.OneDTransitionRewardModel(ens, target_is_delta=spec.target_is_delta, normalize=False,
                                         learned_rewards=spec.learned_rewards, no_delta_list=list(spec.no_delta_list) or None)
    rew, term = functions.REWARD_FNS[spec.reward_fn] if spec.reward_fn else None, functions.TERM_FNS[spec.term_fn]
    ours = bp.ModelEnv(_Env(spec), model, term, rew, generator=torch.Generator(device=DEV), precision="f32")
    ref = mm.ModelEnv(_Env(spec), model, term, rew, generator=torch.Generator(device=DEV))
    B = 1001
    inp = syn.make_step_inputs(spec, B)
    for env in (ours, ref):
        env._rng.manual_seed(21)
    s_ours, s_ref = ours.reset(inp["obs"], return_as_np=False), ref.reset(inp["obs"], return_as_np=False)
    if prop == "fixed_model":
        assert torch.equal(s_ours["propagation_indices"], s_ref["propagation_indices"])
    act = torch.from_numpy(inp["act"]).to(DEV)
    got = ours.step(act, s_ours, sample=False)
    want = ref.step(act, s_ref, sample=False)
    for x, y, what in zip(got[:2], want[:2], ("next_obs", "reward")):
        x, y = torch.as_tensor(x).float().cpu(), torch.as_tensor(y).float().cpu()
        assert torch.allclose(x, y, rtol=1e-4, atol=1e-4), (what, (x - y).abs().max())
