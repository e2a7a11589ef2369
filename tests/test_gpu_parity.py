"""GPU parity tests: the CUDA path (through the C ABI / the reference-shaped Python boundary) against the
oracle on the same seeded, injected-noise inputs, and against the golden vectors of the imported reference.

Tolerances (stated):
  * fp32 SIMT path      : |diff| <= 2e-4 * max(1, |ref|)   per-sequence returns (summation order only)
  * bf16 tensor-core    : <= 5e-3 * max(1, max|ref|) against the oracle run with bf16-rounded operands, and
                          <= 2e-2 * max(1, max|ref|) against the fp32 reference (bf16 quantisation of operands)
  * discrete rewards    : termination thresholds can flip a particle; at most 2 % of sequences may differ and
                          none by more than 2 particles' worth
"""
import os

import numpy as np
import pytest
import torch

from mbrl_lib_b200 import synthetic as syn

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
CONTINUOUS = ["halfcheetah_small", "pets_halfcheetah_small", "humanoid_trunc", "cartpole_pets", "pusher_det", "halfcheetah",
              "humanoid_v4", "tc_hid64", "tc_wide", "tc_shallow", "silu_expectation"] + syn.PLAN_CASES
DISCRETE = ["cartpole", "relu_expectation", "hopper_tsinf", "walker_ant", "ant_learned_fn"]
# the cases the tensor-core kernel is compared with the oracle on: every continuous-reward case it has a plan for
TC_CONTINUOUS = ["halfcheetah_small", "pets_halfcheetah_small", "humanoid_trunc", "cartpole_pets", "pusher_det", "halfcheetah",
                 "tc_hid64", "tc_wide", "tc_shallow", "silu_expectation"] + \
                [n for n in syn.PLAN_CASES if not n.startswith("plan_f32_")]


class _Env:
    def __init__(self, spec):
        class _Box:
            def __init__(self, lo, hi, n):
                self.low = np.full(n, lo, dtype=np.float32)
                self.high = np.full(n, hi, dtype=np.float32)
                self.shape = (n,)

        self.observation_space = _Box(-np.inf, np.inf, spec.obs_dim)
        self.action_space = _Box(spec.action_lb, spec.action_ub, spec.act_dim)


def make_env(name, precision, ts1="perms"):
    import mbrl_lib_b200 as bp
    from mbrl_lib_b200 import functions

    spec = syn.CASES[name]
    arrays = syn.make_model_arrays(spec)
    model = bp.model_from_arrays(spec, arrays, DEV)
    rew = functions.REWARD_FNS[spec.reward_fn] if spec.reward_fn else None
    term = functions.TERM_FNS[spec.term_fn]
    env = bp.ModelEnv(_Env(spec), model, term, rew, generator=torch.Generator(device=DEV), precision=precision, ts1=ts1)
    return spec, arrays, env


def oracle_returns(spec, arrays, inp, bf16=False):
    from oracle import pets_oracle as po

    m = po.OracleModel(spec, arrays)
    m.emulate_bf16 = bf16
    return m.evaluate_action_sequences(torch.from_numpy(inp["actions"]), inp["obs0"], spec.particles,
                                       torch.from_numpy(inp["perms"]), torch.from_numpy(inp["eps"])).numpy()


def gpu_returns(env, spec, inp):
    perms = None if spec.propagation == "expectation" else torch.from_numpy(inp["perms"]).to(DEV)
    eps = None if spec.deterministic else torch.from_numpy(inp["eps"]).to(DEV)
    out = env.evaluate_action_sequences(torch.from_numpy(inp["actions"]).to(DEV), inp["obs0"], spec.particles,
                                        _perms=perms, _eps=eps)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def assert_close_continuous(got, ref, tol):
    scale = max(1.0, float(np.abs(ref).max()))
    err = np.abs(got - ref).max()
    print(f"max |diff| {err:.3e} = {err / scale:.2e} of scale {scale:.3g} (bar {tol:.0e})")
    assert np.isfinite(got).all()
    assert err <= tol * scale, f"max |diff| {err:.3e} > {tol:.1e} * {scale:.3g}"


def assert_close_discrete(got, ref, particles, tol=2e-4):
    diff = np.abs(got - ref)
    bad = diff > tol * np.maximum(1.0, np.abs(ref))
    assert np.isfinite(got).all()
    assert bad.mean() <= 0.02, f"{bad.sum()} of {bad.size} sequences differ"
    assert diff.mean() <= 0.01 * max(1.0, float(np.abs(ref).mean())), diff.mean()


# ----------------------------------------------------------------------------------------------------------
def test_library_on_h100():
    from mbrl_lib_b200 import _lib
    import ctypes as C

    lib = _lib.load()
    sm, ma, mi = C.c_int32(), C.c_int32(), C.c_int32()
    _lib.check(lib.b200pets_device_info(C.byref(sm), C.byref(ma), C.byref(mi)))
    assert (ma.value, mi.value) == (9, 0), f"built for sm_90a, running on sm_{ma.value}{mi.value}"


@pytest.mark.parametrize("k,n", [(16, 16), (32, 208), (208, 208), (208, 64), (256, 256), (64, 48),
                                 (-16, 16), (-32, 208), (-208, 208), (-208, 64), (-256, 256), (-208, 112)])
def test_umma_selftest(k, n):
    """The tensor-core GEMM building block (wgmma.mma_async on sm_90a) through the no-swizzle canonical layouts,
    descriptors, weight ring and accumulator fragments used by the rollout kernel."""
    from mbrl_lib_b200 import _lib

    lib = _lib.load()
    ka = abs(k)  # negative k: A written as bf16 pairs per thread and row
    g = torch.Generator().manual_seed(ka * 1000 + n)
    a = torch.randn(128, ka, generator=g)
    b = torch.randn(n, ka, generator=g)
    ad, bd = a.to(DEV), b.to(DEV)
    d = torch.zeros(128, n, device=DEV)
    _lib.check(lib.b200pets_selftest_wgmma(k, n, _lib.ptr(ad), _lib.ptr(bd), _lib.ptr(d), _lib.stream_ptr()))
    torch.cuda.synchronize()
    ref = a.bfloat16().float() @ b.bfloat16().float().t()
    err = (d.cpu() - ref).abs().max().item()
    assert err <= 1e-3 * max(1.0, ref.abs().max().item()), f"k={k} n={n} max err {err}"


@pytest.mark.parametrize("name", CONTINUOUS)
def test_rollout_f32_matches_oracle_and_golden(golden_dir, name):
    spec, arrays, env = make_env(name, "f32")
    inp = syn.make_rollout_inputs(spec)
    got = gpu_returns(env, spec, inp)
    assert_close_continuous(got, oracle_returns(spec, arrays, inp), 2e-4)
    gold = np.load(os.path.join(golden_dir, f"rollout_{name}.npz"))
    assert str(gold["input_sum"]) == syn.checksum(inp)
    assert_close_continuous(got, gold["returns"], 2e-4)


@pytest.mark.parametrize("name", DISCRETE)
def test_rollout_f32_discrete_rewards(golden_dir, name):
    spec, arrays, env = make_env(name, "f32")
    inp = syn.make_rollout_inputs(spec)
    got = gpu_returns(env, spec, inp)
    gold = np.load(os.path.join(golden_dir, f"rollout_{name}.npz"))
    assert_close_discrete(got, gold["returns"], spec.particles)


@pytest.mark.parametrize("name", TC_CONTINUOUS)
def test_rollout_tc_matches_oracle(golden_dir, name):
    spec, arrays, env = make_env(name, "bf16_tc")
    inp = syn.make_rollout_inputs(spec)
    got = gpu_returns(env, spec, inp)
    assert_close_continuous(got, oracle_returns(spec, arrays, inp, bf16=True), 5e-3)
    gold = np.load(os.path.join(golden_dir, f"rollout_{name}.npz"))
    assert_close_continuous(got, gold["returns"], 2e-2)


@pytest.mark.parametrize("name", ["cartpole", "hopper_tsinf", "walker_ant", "ant_learned_fn", "relu_expectation"])
def test_rollout_tc_discrete_rewards(golden_dir, name):
    spec, arrays, env = make_env(name, "bf16_tc")
    inp = syn.make_rollout_inputs(spec)
    got = gpu_returns(env, spec, inp)
    gold = np.load(os.path.join(golden_dir, f"rollout_{name}.npz"))
    # against the oracle run with bf16-rounded operands the discrete outcomes must agree (measured: 0 of the sequences differ,
    # mean |diff| <= 2.2e-6, tests/prof_tolerances.py) ...
    orc = oracle_returns(spec, arrays, inp, bf16=True)
    d_o = np.abs(got - orc)
    assert (d_o > 1e-2 * np.maximum(1.0, np.abs(orc))).mean() <= 0.01
    assert d_o.mean() <= 1e-4 * max(1.0, float(np.abs(orc).mean()))
    # ... and against the fp32 golden only a state near a termination threshold may flip (measured: 3 % of cartpole's
    # sequences, none elsewhere; mean |diff| <= 1.5e-3)
    diff = np.abs(got - gold["returns"])
    assert (diff > 1e-2 * np.maximum(1.0, np.abs(gold["returns"]))).mean() <= 0.06
    assert diff.mean() <= 5e-3 * max(1.0, np.abs(gold["returns"]).mean())


@pytest.mark.parametrize("precision,tol", [("f32", 2e-4), ("bf16_tc", 2e-2)])
@pytest.mark.parametrize("name,batch", [("mbpo_halfcheetah_small", 1000), ("cartpole", 500)])
def test_step_matches_golden(golden_dir, name, batch, precision, tol):
    spec, arrays, env = make_env(name, precision)
    inp = syn.make_step_inputs(spec, batch)
    gold = np.load(os.path.join(golden_dir, f"step_{name}.npz"))
    assert str(gold["input_sum"]) == syn.checksum(inp)
    state = env.reset(inp["obs"], return_as_np=True)
    nobs, rew, done, _ = env.step(inp["act"], state, sample=True, _perm=torch.from_numpy(inp["perm"]).to(DEV),
                                  _eps=torch.from_numpy(inp["eps"]).to(DEV))
    assert isinstance(nobs, np.ndarray) and rew.shape == (batch, 1) and done.shape == (batch, 1) and done.dtype == bool
    scale = max(1.0, np.abs(gold["next_obs"]).max())
    assert np.abs(nobs - gold["next_obs"]).max() <= tol * scale
    if spec.reward_fn in ("cartpole",):
        assert (rew != gold["reward"]).mean() <= 0.02
        assert (done != gold["done"]).mean() <= 0.02
    else:
        assert np.abs(rew - gold["reward"]).max() <= tol * scale
        assert (done == gold["done"]).all()


def test_step_returns_tensors_and_mean_prediction():
    spec, arrays, env = make_env("mbpo_halfcheetah_small", "f32")
    inp = syn.make_step_inputs(spec, 500)
    state = env.reset(inp["obs"], return_as_np=False)
    perm = torch.from_numpy(inp["perm"][inp["perm"] < 500][:500].copy()).to(DEV)
    perm = torch.argsort(torch.argsort(perm))  # a permutation of 0..499
    a = torch.from_numpy(inp["act"]).to(DEV)
    n1, r1, d1, _ = env.step(a, state, sample=False, _perm=perm)
    n2, r2, d2, _ = env.step(a, state, sample=False, _perm=perm)
    assert torch.is_tensor(n1) and n1.device.type == "cuda"
    assert torch.equal(n1, n2) and torch.equal(r1, r2)  # deterministic=True path draws nothing
    from oracle import pets_oracle as po

    m = po.OracleModel(spec, arrays)
    on, orw, _ = m.step(torch.from_numpy(inp["obs"]), torch.from_numpy(inp["act"]), perm.cpu(), None, sample=False)
    assert (n1.cpu() - on).abs().max() <= 2e-4 * max(1.0, on.abs().max().item())
    assert (r1.cpu() - orw).abs().max() <= 2e-4 * max(1.0, orw.abs().max().item())


def test_batch_not_multiple_of_members_raises():
    spec, arrays, env = make_env("halfcheetah_small", "f32")
    acts = torch.zeros(3, 4, spec.act_dim, device=DEV)  # 3 * 1 rows for 5 members
    with pytest.raises(ValueError, match="multiple of the number of models"):
        env.evaluate_action_sequences(acts, np.zeros(spec.obs_dim), 1)


# ---- optimisers ------------------------------------------------------------------------------------------
def _quad(target):
    return lambda pop: -((pop - target) ** 2).sum(dim=(1, 2)) + 0.3 * torch.sin(3.0 * pop).sum(dim=(1, 2))


@pytest.mark.parametrize("tag,clipped,ret_mean", [("trunc_best", False, False), ("trunc_mean", False, True),
                                                  ("clipped_best", True, False)])
def test_cem_optimizer_matches_reference(golden_dir, tag, clipped, ret_mean):
    import mbrl_lib_b200 as bp

    g = np.load(os.path.join(golden_dir, f"cem_{tag}.npz"))
    t = lambda k: torch.from_numpy(g[k]).to(DEV)  # noqa: E731
    opt = bp.CEMOptimizer(int(g["iters"]), float(g["elite_ratio"]), int(g["N"]), g["lb"].tolist(), g["ub"].tolist(),
                          float(g["alpha"]), DEV, return_mean_elites=ret_mean, clipped_normal=clipped)
    trace = []
    sol = opt.optimize(_quad(t("target")), x0=t("x0"), callback=lambda p, v, i: trace.append((p.clone(), v.clone())),
                       _noise=t("z"))
    for i, (p, v) in enumerate(trace):
        np.testing.assert_allclose(p.cpu().numpy(), g["pops"][i], rtol=2e-5, atol=2e-6)
        np.testing.assert_allclose(v.cpu().numpy(), g["values"][i], rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(sol.cpu().numpy(), g["solution"], rtol=2e-5, atol=2e-6)


def test_icem_optimizer_matches_reference(golden_dir):
    import mbrl_lib_b200 as bp

    g = np.load(os.path.join(golden_dir, "icem.npz"))
    t = lambda k: torch.from_numpy(g[k]).to(DEV)  # noqa: E731
    iters = int(g["iters"])
    opt = bp.ICEMOptimizer(iters, float(g["elite_ratio"]), int(g["pop0"]), float(g["decay"]), float(g["beta"]),
                           g["lb"].tolist(), g["ub"].tolist(), float(g["keep_frac"]), float(g["alpha"]), DEV,
                           return_mean_elites=False, population_size_module=int(g["module"]))
    assert opt.population_sizes() == g["sizes"].tolist() and opt.keep_elite_size == int(g["keep"])
    for call in range(2):
        noise = []
        for i in range(iters):
            d = {"sr": t(f"c{call}_sr{i}"), "si": t(f"c{call}_si{i}")}
            if f"c{call}_perm{i}" in g:
                d["keep_perm"] = t(f"c{call}_perm{i}")
            if i == 0 and f"c{call}_end_eps" in g:
                d["end_eps"] = t(f"c{call}_end_eps")
            noise.append(d)
        trace = []
        sol = opt.optimize(_quad(t("target")), x0=t("x0"), callback=lambda p, v, i: trace.append((p.clone(), v.clone())),
                           _noise=noise)
        for i, (p, v) in enumerate(trace):
            np.testing.assert_allclose(p.cpu().numpy(), g[f"c{call}_pop{i}"], rtol=1e-4, atol=2e-5)
        np.testing.assert_allclose(sol.cpu().numpy(), g[f"sol{call}"], rtol=1e-4, atol=2e-5)
        # both order the elite set by descending value, and the next call's keep_perm indexes into that order
        np.testing.assert_allclose(opt.elite.cpu().numpy(), g[f"c{call}_elite"], rtol=1e-4, atol=2e-5)


def test_mppi_optimizer_matches_reference(golden_dir):
    import mbrl_lib_b200 as bp

    g = np.load(os.path.join(golden_dir, "mppi.npz"))
    t = lambda k: torch.from_numpy(g[k]).to(DEV)  # noqa: E731
    opt = bp.MPPIOptimizer(int(g["iters"]), int(g["N"]), float(g["gamma"]), float(g["sigma"]), float(g["beta"]),
                           g["lb"].tolist(), g["ub"].tolist(), DEV)
    for call in range(2):  # the second call exercises the shifted mean / past action
        trace = []
        sol = opt.optimize(_quad(t("target")), callback=lambda p, v, k: trace.append(p.clone()), _noise=t(f"z{call}"))
        for k, p in enumerate(trace):
            np.testing.assert_allclose(p.cpu().numpy(), g[f"pops{call}"][k], rtol=2e-5, atol=2e-6)
        np.testing.assert_allclose(sol.cpu().numpy(), g[f"sol{call}"], rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("precision,tol", [("f32", 5e-4), ("bf16_tc", 2e-3)])
def test_fused_cem_plan_matches_reference(golden_dir, precision, tol):
    """CEMOptimizer.optimize over ModelEnv.evaluate_action_sequences as ONE C call, injected noise."""
    import mbrl_lib_b200 as bp
    from mbrl_lib_b200.planning import _FusedObjective

    g = np.load(os.path.join(golden_dir, "cem_model.npz"))
    spec, arrays, env = make_env("halfcheetah_small", precision)
    inp = syn.make_rollout_inputs(spec)
    iters = int(g["iters"])
    nz = syn.make_cem_noise(spec, iters)
    assert str(g["noise_sum"]) == syn.checksum(nz)
    H, A = spec.horizon, spec.act_dim
    lb = np.full((H, A), spec.action_lb).tolist()
    ub = np.full((H, A), spec.action_ub).tolist()
    opt = bp.CEMOptimizer(iters, 0.1, spec.population, lb, ub, 0.1, DEV, return_mean_elites=True)
    opt.record_values = True
    obj = _FusedObjective(env, inp["obs0"], spec.particles)
    sol = opt.optimize(obj, x0=torch.zeros(H, A, device=DEV), _noise=torch.from_numpy(nz["z"]).to(DEV),
                       _model_noise=(torch.from_numpy(nz["perms"]).to(DEV), torch.from_numpy(nz["eps"]).to(DEV)))
    torch.cuda.synchronize()
    vals = opt.last_values.cpu().numpy()
    scale = max(1.0, np.abs(g["values"]).max())
    assert np.abs(vals[0] - g["values"][0]).max() <= tol * scale  # first iteration: identical population
    if precision == "f32":
        assert np.abs(vals - g["values"]).max() <= tol * scale
        np.testing.assert_allclose(sol.cpu().numpy(), g["solution"], rtol=1e-3, atol=1e-3)
    else:
        assert np.abs(vals - g["values"]).max() <= tol * scale  # measured 2.1e-4 of scale (tests/prof_tolerances.py)
        # elite membership did not flip on this case (measured max |diff| 1.2e-7); a flip would move the mean by ~1e-2
        assert np.abs(sol.cpu().numpy() - g["solution"]).max() <= 1e-3


# ---- in-kernel RNG: distribution-level checks ------------------------------------------------------------
def test_truncated_normal_sampler_statistics():
    import mbrl_lib_b200 as bp

    N, H, A = 4096, 8, 4
    lb = np.full((H, A), -10.0).tolist()
    ub = np.full((H, A), 10.0).tolist()
    opt = bp.CEMOptimizer(1, 0.1, N, lb, ub, 0.1, DEV)
    pops = []
    opt.optimize(lambda p: p.sum(dim=(1, 2)), x0=torch.zeros(H, A, device=DEV), callback=lambda p, v, i: pops.append(p.clone()))
    z = pops[0].cpu().numpy() / np.sqrt(20.0 ** 2 / 16)  # initial variance ((ub - lb)^2)/16
    assert np.abs(z).max() <= 2.0 + 1e-5  # tests/core/test_common_utils.py:419-423
    assert abs(z.mean()) < 0.02
    assert abs(z.var() - 0.7737) < 0.03  # variance of N(0,1) truncated to [-2, 2]
    opt.optimize(lambda p: p.sum(dim=(1, 2)), x0=torch.zeros(H, A, device=DEV), callback=lambda p, v, i: pops.append(p.clone()))
    assert not torch.equal(pops[0], pops[1])  # fresh draws on the next call


@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
def test_in_kernel_noise_matches_injected_in_distribution(precision):
    """Philox model noise + tile-shuffle TS1 vs injected noise + permutations: same return distribution."""
    spec, arrays, env_inj = make_env("halfcheetah", precision)
    _, _, env_rng = make_env("halfcheetah", precision, ts1="tile_shuffle")
    inp = syn.make_rollout_inputs(spec)
    r_inj = gpu_returns(env_inj, spec, inp)
    r_rng = env_rng.evaluate_action_sequences(torch.from_numpy(inp["actions"]).to(DEV), inp["obs0"], spec.particles).cpu().numpy()
    r_rng2 = env_rng.evaluate_action_sequences(torch.from_numpy(inp["actions"]).to(DEV), inp["obs0"], spec.particles).cpu().numpy()
    assert np.isfinite(r_rng).all()
    assert not np.array_equal(r_rng, r_rng2)  # new Philox offset per call
    # With this synthetic (untrained, strongly disagreeing) ensemble two *reference-semantics* evaluations with
    # independent permutations are uncorrelated per sequence (measured: corr ~ 0), so the check is on the
    # distribution over the population: mean (member mixture + noise scale) and spread.
    se = max(np.std(r_inj) / np.sqrt(len(r_inj)), 1e-3)
    assert abs(r_inj.mean() - r_rng.mean()) <= 6 * se + 0.02 * abs(r_inj.mean())
    assert 0.7 <= np.std(r_rng) / np.std(r_inj) <= 1.4


def test_humanoid_v4_dims_use_fp32_path():
    """376-dim observations exceed the tensor-core plan (K, N <= 256): precision='auto' must pick the fp32 kernel,
    and asking for the tensor-core path must fail loudly rather than fall back silently."""
    spec, arrays, env = make_env("humanoid_v4", "auto")
    assert env.precision == "f32" and not env.staged.supports_tc()
    _, _, env_tc = make_env("humanoid_v4", "bf16_tc")
    inp = syn.make_rollout_inputs(spec)
    with pytest.raises(NotImplementedError):
        gpu_returns(env_tc, spec, inp)


def test_launch_plans_are_covered():
    """The kernels pick their launch plan from the model's shape at run time (b200pets_model_plan_info reports it, from
    the same code as the launchers).  The cases the oracle comparisons run must together reach every plan class:
    tensor-core ring slices of 1-4 K steps, rings of two, three and more slots, accumulator widths around the 128-column
    split, the bias-one columns at either side of the accumulator's end, 256-column layers, the deepest model, and the
    fp32 kernel's 64 / 32 / 16-row tiles in each of its row mappings."""
    from test_gpu_shuffle import SHUFFLE_CASES

    f32_modes = {"perms": set(), "tile_shuffle": set(), "expectation": set()}
    tc = {"kslice": set(), "slots": set(), "hid_np": set(), "out_np": set(), "hid_mod16": set(), "kp0": set(), "hid_kp": set(),
          "hidden_layers": set(), "deterministic": set(), "exp_kslice": set()}
    tc_cases = set(TC_CONTINUOUS) | {c[0] for c in SHUFFLE_CASES if c[1] == "bf16_tc"}
    f32_shuffle = {c[0] for c in SHUFFLE_CASES if c[1] == "f32"}
    print()
    for name, spec in syn.CASES.items():
        _, _, env = make_env(name, "f32")
        plan = env.staged.plan_info(spec.propagation)
        print(f"{name:24s} {spec.propagation:13s} {plan}")
        rows = plan["f32_rows"]
        assert rows in (16, 32, 64), (name, plan)
        if name in CONTINUOUS:
            f32_modes["expectation" if spec.propagation == "expectation" else "perms"].add(rows)
        if name in f32_shuffle:
            f32_modes["tile_shuffle"].add(rows)
        if name not in tc_cases:
            continue
        assert plan["kslice"] > 0 and plan["nstages"] >= 2 and plan["tc_smem"] > 0, (name, plan)
        hid_np = -(-spec.hid_size // 16) * 16
        out_np = -(-spec.out_size // 16) * 16 * (1 if spec.deterministic else 2)
        tc["kslice"].add(plan["kslice"])
        tc["slots"].add(min(plan["nstages"], 4))
        tc["hid_np"].add(hid_np)
        tc["out_np"].add(out_np)
        tc["hid_mod16"].add(spec.hid_size % 16)
        tc["kp0"].add(-(-(spec.in_size + 2) // 16) * 16)  # input + two bias-one columns, padded to a K step
        tc["hid_kp"].add(-(-(spec.hid_size + 2) // 16) * 16)
        tc["hidden_layers"].add(spec.num_layers)
        tc["deterministic"].add(spec.deterministic)
        if spec.propagation == "expectation":
            tc["exp_kslice"].add(plan["kslice"])
    assert tc["kslice"] >= {1, 2, 3, 4}, tc["kslice"]
    assert tc["slots"] >= {2, 3, 4}, tc["slots"]  # 4 stands for four or more
    assert tc["hid_np"] >= {16, 128, 144, 256}, tc["hid_np"]
    assert 256 in tc["out_np"] and True in tc["deterministic"]
    assert tc["hid_mod16"] >= {0, 14, 15}, tc["hid_mod16"]
    assert 256 in tc["kp0"] and 256 in tc["hid_kp"]
    assert 7 in tc["hidden_layers"]  # B200PETS_MAX_LAYERS - 1
    assert min(tc["exp_kslice"]) < 4, tc["exp_kslice"]
    for mode, seen in f32_modes.items():
        assert seen >= {16, 32, 64}, (mode, seen)


def test_auto_precision_follows_the_propagation_plan():
    """A model the tensor-core kernel covers for TS1 but not for "expectation" (whose per-row member sums take shared
    memory the weight ring needs): precision="auto" must run expectation calls on the fp32 kernel, at its bar, and an
    explicit "bf16_tc" must still refuse them loudly."""
    import dataclasses

    import mbrl_lib_b200 as bp
    from mbrl_lib_b200 import functions
    from oracle import pets_oracle as po

    spec = syn.CaseSpec("auto_expectation_fallback", obs_dim=100, act_dim=8, propagation="expectation",
                        population=20, horizon=4, particles=5)
    arrays = syn.make_model_arrays(spec)
    model = bp.model_from_arrays(spec, arrays, DEV)
    env = bp.ModelEnv(_Env(spec), model, functions.no_termination, functions.REWARD_FNS[spec.reward_fn],
                      generator=torch.Generator(device=DEV), precision="auto")
    assert env.staged.plan_info("random_model")["kslice"] > 0
    assert env.staged.plan_info("expectation")["kslice"] == 0
    inp = syn.make_rollout_inputs(spec)
    got = gpu_returns(env, spec, inp)
    assert_close_continuous(got, oracle_returns(spec, arrays, inp), 2e-4)
    st = syn.make_step_inputs(spec, 100)
    state = env.reset(st["obs"], return_as_np=True)
    nobs, rew, _, _ = env.step(st["act"], state, sample=True, _eps=torch.from_numpy(st["eps"]).to(DEV))
    on, orw, _ = po.OracleModel(spec, arrays).step(torch.from_numpy(st["obs"]), torch.from_numpy(st["act"]), None,
                                                   torch.from_numpy(st["eps"]))
    scale = max(1.0, float(on.abs().max()))
    assert np.abs(nobs - on.numpy()).max() <= 2e-4 * scale
    assert np.abs(rew - orw.numpy()).max() <= 2e-4 * scale
    assert env.precision == "bf16_tc" and env.precision_for("expectation") == "f32"
    # the same model under TS1 keeps the tensor-core kernel
    ts1 = dataclasses.replace(spec, propagation="random_model")
    env_ts1 = bp.ModelEnv(_Env(ts1), bp.model_from_arrays(ts1, arrays, DEV), functions.no_termination,
                          functions.REWARD_FNS[spec.reward_fn], precision="auto")
    assert env_ts1.precision_for("random_model") == "bf16_tc"
    env_tc = bp.ModelEnv(_Env(spec), model, functions.no_termination, functions.REWARD_FNS[spec.reward_fn],
                         precision="bf16_tc")
    with pytest.raises(NotImplementedError):
        gpu_returns(env_tc, spec, inp)


def test_warm_start_shift_matches_reference_rule():
    """TrajectoryOptimizer.optimize keeps best.roll(-replan_freq) with the tail reset (trajectory_opt.py:563-567)."""
    from mbrl_lib_b200 import _lib
    from oracle import pets_oracle as po

    lib = _lib.load()
    H, A = 7, 3
    best = torch.arange(H * A, dtype=torch.float32, device=DEV).view(H, A)
    init = torch.tensor([0.5, -0.5, 0.25], device=DEV)
    for replan in (1, 2, 7):
        prev = torch.empty(H, A, device=DEV)
        _lib.check(lib.b200pets_shift_solution(H, A, replan, _lib.ptr(best), _lib.ptr(init), _lib.ptr(prev), _lib.stream_ptr()))
        ref = po.shift_solution(best.cpu(), replan, init.cpu())
        assert torch.equal(prev.cpu(), ref)


def test_agent_act_end_to_end():
    """TrajectoryOptimizerAgent.act through create_trajectory_optim_agent_for_model (fused plan)."""
    import mbrl_lib_b200 as bp

    spec, arrays, env = make_env("halfcheetah_small", "auto", ts1="tile_shuffle")
    cfg = {"_target_": "mbrl.planning.TrajectoryOptimizerAgent", "planning_horizon": spec.horizon, "replan_freq": 1,
           "verbose": False,
           "optimizer_cfg": {"_target_": "mbrl.planning.CEMOptimizer", "num_iterations": 3, "elite_ratio": 0.1,
                             "population_size": spec.population, "alpha": 0.1, "device": DEV,
                             "return_mean_elites": True}}
    agent = bp.create_trajectory_optim_agent_for_model(env, cfg, num_particles=spec.particles)
    inp = syn.make_rollout_inputs(spec)
    a1 = agent.act(inp["obs0"])
    assert a1.shape == (spec.act_dim,) and np.isfinite(a1).all()
    assert (a1 >= spec.action_lb - 1e-6).all() and (a1 <= spec.action_ub + 1e-6).all()
    plan = agent.plan(inp["obs0"])
    assert plan.shape == (spec.horizon, spec.act_dim)
    agent.reset()
    bare = bp.TrajectoryOptimizerAgent(cfg["optimizer_cfg"], [-1.0] * spec.act_dim, [1.0] * spec.act_dim, spec.horizon)
    with pytest.raises(RuntimeError, match="set_trajectory_eval_fn"):
        bare.act(inp["obs0"])


def test_cem_improves_objective_rosenbrock():
    """CEM on Rosenbrock (notebooks/cem_rosenbrock_ex.ipynb): optimum (1, 1)."""
    import mbrl_lib_b200 as bp

    opt = bp.CEMOptimizer(60, 0.1, 1000, [[-2.0, -2.0]], [[2.0, 2.0]], 0.1, DEV, return_mean_elites=True)

    def neg_rosen(p):
        x, y = p[:, 0, 0], p[:, 0, 1]
        return -((1 - x) ** 2 + 100 * (y - x ** 2) ** 2)

    sol = opt.optimize(neg_rosen, x0=torch.zeros(1, 2, device=DEV)).cpu().numpy().reshape(-1)
    # the reference's CEM (oracle, same settings) stalls in the valley around (0.6, 0.37): same behaviour expected
    assert 0.4 <= sol[0] <= 1.1 and abs(sol[1] - sol[0] ** 2) < 0.05, sol
    assert -((1 - sol[0]) ** 2 + 100 * (sol[1] - sol[0] ** 2) ** 2) > -0.5  # objective at x0 = (0, 0) is -1


@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
@pytest.mark.parametrize("ts1", ["perms", "tile_shuffle"])
def test_reference_known_answer_closed_form(golden_dir, precision, ts1):
    """The reference's known-answer test of evaluate_action_sequences (tests/core/test_models.py:365-385):
    next_obs = obs + a, reward = next_obs => return = H(H+1)/2 * a for H, P in 1..9, a in {1, 2}, bit-exact.
    The model is the hand-built ReLU ensemble the imported reference was run on (tests/golden/kat_counter_world.npz)."""
    import mbrl_lib_b200 as bp
    from mbrl_lib_b200 import functions

    spec, arrays = syn.counter_world()
    gold = np.load(os.path.join(golden_dir, "kat_counter_world.npz"))
    assert str(gold["model_sum"]) == syn.checksum(arrays)
    model = bp.model_from_arrays(spec, arrays, DEV)
    env = bp.ModelEnv(_Env(spec), model, functions.no_termination, None, generator=torch.Generator(device=DEV),
                      precision=precision, ts1=ts1)
    N = 4
    for P in range(1, 10):
        for H in range(1, 10):
            for a in (1.0, 2.0):
                ret = env.evaluate_action_sequences(torch.full((N, H, 1), a, device=DEV), np.zeros(1), P)
                want = gold["returns"][P - 1, H - 1, int(a) - 1]
                assert want == H * (H + 1) / 2 * a
                assert torch.equal(ret.cpu(), torch.full((N,), float(want))), (P, H, a, ret)
