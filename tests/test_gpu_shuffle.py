"""Exact parity of the PRODUCTION TS1 mode (in-kernel "tile shuffle", the mode bench.py times) against the oracle.

The kernels export the member every shuffle group uses at every step (b200pets_shuffle_member_map); the oracle
consumes it as the reference's row -> member assignment (gaussian_mlp.py:202-212 with the permutation replaced by
the map it induces, ``OracleModel.forward_assigned``, itself pinned to the golden-pinned permutation path by
tests/test_oracle_golden.py).  Model noise is injected, so the comparison is at the same bars as the explicit-
permutation tests: 2e-4 (fp32 kernel) / 5e-3 against the bf16-operand oracle (tensor-core kernel), at BASELINE
config 2's FULL size (pop 500 x 20 particles x 30 steps), for one evaluation and for the fused CEM plan
(b200pets_cem_plan: the call bench.py's `value` times).

Also here: shard invariance (the property that makes multi-GPU results independent of the number of GPUs), the
distribution-level equivalence of the tile-shuffle law and the reference's randperm law (two-sample KS over 200
draws each), and ShardedCEMOptimizer == CEMOptimizer on the union population (two shards on one GPU).
"""
import dataclasses
import threading

import numpy as np
import pytest
import torch

from mbrl_lib_b200 import synthetic as syn
from test_gpu_parity import DEV, assert_close_continuous, assert_close_discrete, make_env

pytestmark = pytest.mark.gpu


def _oracle(spec, arrays, bf16):
    from oracle import pets_oracle as po

    m = po.OracleModel(spec, arrays)
    m.emulate_bf16 = bf16
    return m


def _eval_shuffle(env, spec, inp, offset, shard=(0, 0), rows=False, eps=None, actions=None):
    acts = torch.from_numpy(inp["actions"] if actions is None else actions).to(DEV)
    e = None if spec.deterministic else torch.from_numpy(inp["eps"] if eps is None else eps).to(DEV)
    rr = torch.empty(acts.shape[0] * spec.particles, device=DEV) if rows else None
    out = env.evaluate_action_sequences(acts, inp["obs0"], spec.particles, _eps=e, _row_returns=rr, _offset=offset,
                                        _shard=shard)
    torch.cuda.synchronize()
    return (rr if rows else out).cpu().numpy()


TOL = {"f32": 2e-4, "bf16_tc": 5e-3}
# (case, precision, population or None for the case's own).  The fp32 kernel splits a 128-row shuffle group into 2, 4 or
# 8 tiles (64, 32 or 16 rows); the populations of the wide fp32-only models are large enough to fill more than one tile of
# their group.
SHUFFLE_CASES = [(n, p, None) for n in ["halfcheetah", "pets_halfcheetah_small", "humanoid_trunc", "tc_hid64", "cartpole_pets"]
                 for p in ("f32", "bf16_tc")] + \
                [("plan_f32_hid512", "f32", None), ("humanoid_v4", "f32", 70), ("plan_hid143", "f32", None),
                 ("plan_hid143", "bf16_tc", None), ("plan_k3", "bf16_tc", None), ("plan_ring2", "bf16_tc", None),
                 ("plan_k1_out256", "bf16_tc", None), ("plan_hid14_deep", "bf16_tc", None),
                 ("plan_logvar_extreme", "bf16_tc", None), ("plan_logvar_extreme", "f32", None)]


@pytest.mark.parametrize("name,precision,population", SHUFFLE_CASES,
                         ids=[f"{n}-{p}-{TOL[p]}" + (f"-pop{pop}" if pop else "") for n, p, pop in SHUFFLE_CASES])
def test_tile_shuffle_matches_oracle(name, precision, population):
    tol = TOL[precision]
    spec, arrays, env = make_env(name, precision, ts1="tile_shuffle")
    env._few_groups = lambda *a: False  # always the in-kernel draw, also for the small parity cases
    if population is not None:
        spec = dataclasses.replace(spec, population=population)
    inp = syn.make_rollout_inputs(spec)
    offset = 7 * 1024
    got = _eval_shuffle(env, spec, inp, offset)
    assign = env.shuffle_member_assignment(spec.population, spec.horizon, spec.particles, offset)
    M = spec.num_models
    assert assign.min() >= 0 and assign.max() < M
    if name == "halfcheetah":  # uniform member draw per (group, step): 80 groups x 30 steps = 2 400 draws over 5 members
        frac = np.bincount(assign.numpy().reshape(-1), minlength=M) / assign.numel()
        assert np.abs(frac - 1.0 / M).max() < 0.05, frac
    ref = _oracle(spec, arrays, precision == "bf16_tc").evaluate_action_sequences(
        torch.from_numpy(inp["actions"]), inp["obs0"], spec.particles, None, torch.from_numpy(inp["eps"]),
        assign=assign).numpy()
    assert_close_continuous(got, ref, tol)


@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
@pytest.mark.parametrize("name", ["cartpole", "hopper_tsinf"])
def test_tile_shuffle_tsinf_matches_oracle(name, precision):
    """TSinf without an injected permutation: one member per shuffle group for the whole horizon."""
    spec, arrays, env = make_env(name, precision, ts1="tile_shuffle")
    env._few_groups = lambda *a: False
    inp = syn.make_rollout_inputs(spec)
    offset = 3 * 1024
    got = _eval_shuffle(env, spec, inp, offset)
    assign = env.shuffle_member_assignment(spec.population, spec.horizon, spec.particles, offset)
    assert bool((assign == assign[:1]).all())  # fixed for the horizon
    ref = _oracle(spec, arrays, precision == "bf16_tc").evaluate_action_sequences(
        torch.from_numpy(inp["actions"]), inp["obs0"], spec.particles, None, torch.from_numpy(inp["eps"]),
        assign=assign[:1]).numpy()
    if precision == "f32":
        assert_close_discrete(got, ref, spec.particles)
    else:  # discrete rewards: a state near a termination threshold may flip a particle at bf16
        diff = np.abs(got - ref)
        assert (diff > 1e-2 * np.maximum(1.0, np.abs(ref))).mean() <= 0.05
        assert abs(got.mean() - ref.mean()) <= 0.02 * max(1.0, abs(ref.mean()))


@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
def test_shard_invariance_bit_exact(precision):
    """Rows evaluated as shards [0,180) + [180,500) of a global population of 500 (shard boundary inside a shuffle
    group) equal the unsharded evaluation BIT FOR BIT, with in-kernel Philox noise and member draws: every draw is
    keyed by global indices (SURVEY.md section 8e)."""
    spec, arrays, env = make_env("halfcheetah", precision, ts1="tile_shuffle")
    inp = syn.make_rollout_inputs(spec, with_noise=False)
    N, P = spec.population, spec.particles
    offset = 11 * 1024

    def run(lo, hi):
        acts = torch.from_numpy(inp["actions"][lo:hi]).to(DEV)
        rr = torch.empty((hi - lo) * P, device=DEV)
        ret = env.evaluate_action_sequences(acts, inp["obs0"], P, _row_returns=rr, _offset=offset, _shard=(lo, N))
        torch.cuda.synchronize()
        return ret.cpu().numpy(), rr.cpu().numpy()

    full, full_rows = run(0, N)
    a, a_rows = run(0, 180)
    b, b_rows = run(180, N)
    assert np.array_equal(np.concatenate([a_rows, b_rows]), full_rows)
    assert np.array_equal(np.concatenate([a, b]), full)
    assert np.isfinite(full).all() and np.unique(full).size > N // 2


CEM_PLAN_SHAPES = [(p, tol, n, h) for n, h in [(500, 30), (2100, 8)] for p, tol in [("f32", 5e-4), ("bf16_tc", 5e-3)]]


@pytest.mark.parametrize("precision,tol,population,horizon", CEM_PLAN_SHAPES,
                         ids=[f"{p}-{tol}" + ("" if n == 500 else f"-pop{n}-h{h}") for p, tol, n, h in CEM_PLAN_SHAPES])
def test_fused_cem_plan_tile_shuffle_matches_oracle(precision, tol, population, horizon):
    """b200pets_cem_plan (the call bench.py's `value` times) in its production mode -- tile shuffle -- at config 2's
    full size, population noise and model noise injected, against the oracle's CEM over the oracle rollout with the
    exported per-iteration member maps.  A population above 2048 takes the plan's other refit: particle mean, then the
    radix select."""
    import mbrl_lib_b200 as bp
    from mbrl_lib_b200.planning import _FusedObjective
    from oracle import pets_oracle as po

    spec, arrays, env = make_env("halfcheetah", precision, ts1="tile_shuffle")
    spec = dataclasses.replace(spec, population=population, horizon=horizon)
    inp = syn.make_rollout_inputs(spec, with_noise=False)
    iters = 2
    nz = syn.make_cem_noise(spec, iters)
    H, A, N, P = spec.horizon, spec.act_dim, spec.population, spec.particles
    lb = np.full((H, A), spec.action_lb).tolist()
    ub = np.full((H, A), spec.action_ub).tolist()
    opt = bp.CEMOptimizer(iters, 0.1, N, lb, ub, 0.1, DEV, return_mean_elites=True)
    opt.record_values = True
    call = env._offset + 1  # the Philox call counter cem_plan will take
    sol = opt.optimize(_FusedObjective(env, inp["obs0"], P), x0=torch.zeros(H, A, device=DEV),
                       _noise=torch.from_numpy(nz["z"]).to(DEV), _model_noise=(None, torch.from_numpy(nz["eps"]).to(DEV)))
    torch.cuda.synchronize()
    vals = opt.last_values.cpu().numpy()
    assigns = [env.shuffle_member_assignment(N, H, P, call * 1024 + it) for it in range(iters)]
    oracle = _oracle(spec, arrays, precision == "bf16_tc")
    ref_vals = []

    def obj(pop, i):
        v = oracle.evaluate_action_sequences(pop, inp["obs0"], P, None, torch.from_numpy(nz["eps"][i]), assign=assigns[i])
        ref_vals.append(v.numpy())
        return v

    lbt, ubt = torch.tensor(lb), torch.tensor(ub)
    ref_sol = po.cem_optimize(obj, torch.zeros(H, A), lbt, ubt, iters, 0.1, N, 0.1, torch.from_numpy(nz["z"]),
                              return_mean_elites=True)
    scale = max(1.0, np.abs(ref_vals[0]).max())
    assert np.abs(vals[0] - ref_vals[0]).max() <= tol * scale  # iteration 0: identical population
    if precision == "f32":
        assert np.abs(vals[1] - ref_vals[1]).max() <= tol * scale
        np.testing.assert_allclose(sol.cpu().numpy(), ref_sol.numpy(), rtol=1e-3, atol=1e-3)
    else:  # an elite at the selection threshold may flip at bf16: the refit moves by at most 1 of 50 elites
        assert np.abs(sol.cpu().numpy() - ref_sol.numpy()).max() <= 0.05


@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
def test_mbpo_step_tile_shuffle_full_size_sampled(precision):
    """config 4 at full size (100 000 start states, sample=True, injected noise), tile-shuffle member draw: a strided
    subset of rows against the oracle with the exported member of each row."""
    spec, arrays, env = make_env("mbpo_halfcheetah", precision, ts1="tile_shuffle")
    B = 100000
    inp = syn.make_step_inputs(spec, B)
    state = env.reset(inp["obs"], return_as_np=False)
    offset = 5 * 1024
    eps = torch.from_numpy(inp["eps"]).to(DEV)
    nobs, rew, done, _ = env.step(torch.from_numpy(inp["act"]).to(DEV), state, sample=True, _eps=eps, _offset=offset)
    torch.cuda.synchronize()
    assign = env.shuffle_member_assignment(B, 1, 1, offset)[0]
    frac = np.bincount(assign.numpy(), minlength=spec.num_models) / B  # 782 independent group draws over 5 members
    assert np.abs(frac - 1.0 / spec.num_models).max() < 0.06, frac
    rows = np.arange(0, B, 97)[:1030]  # the oracle checks batch % members == 0 like the reference (gaussian_mlp.py:195-200)
    oracle = _oracle(spec, arrays, precision == "bf16_tc")
    on, orw, _ = oracle.step(torch.from_numpy(inp["obs"][rows]), torch.from_numpy(inp["act"][rows]), None,
                             torch.from_numpy(inp["eps"][rows]), sample=True, assign=assign[rows])
    tol = 2e-4 if precision == "f32" else 5e-3
    scale = max(1.0, on.abs().max().item())
    assert (nobs.cpu()[rows] - on).abs().max().item() <= tol * scale
    assert (rew.cpu()[rows] - orw).abs().max().item() <= tol * scale
    assert not bool(done.any())


def test_tile_shuffle_law_matches_reference_law_ks():
    """The tile-shuffle law (an independent uniform member per (shuffle group, step)) against the reference's law
    (a fresh randperm of all rows per step): per-sequence return distributions over 200 independent draws each,
    two-sample Kolmogorov-Smirnov per sequence.  Under equality the p-values are uniform: at most 5 % of the
    sequences may reject at the 1 % level and the mean p-value must sit near 0.5."""
    from scipy import stats

    spec, arrays, env_perm = make_env("halfcheetah", "bf16_tc", ts1="perms")
    _, _, env_shuf = make_env("halfcheetah", "bf16_tc", ts1="tile_shuffle")
    env_shuf._seed = 0x5EED5EED  # independent Philox key: the two samples must not share their model noise
    N, H, P, draws = 256, 8, spec.particles, 200
    inp = syn.make_rollout_inputs(spec, population=N, horizon=H, with_noise=False)
    acts = torch.from_numpy(inp["actions"]).to(DEV)
    g = torch.Generator(device=DEV).manual_seed(1)
    ret_perm = np.empty((draws, N), np.float32)
    ret_shuf = np.empty((draws, N), np.float32)
    for d in range(draws):
        perms = torch.stack([torch.randperm(N * P, device=DEV, generator=g) for _ in range(H)])
        ret_perm[d] = env_perm.evaluate_action_sequences(acts, inp["obs0"], P, _perms=perms).cpu().numpy()
        ret_shuf[d] = env_shuf.evaluate_action_sequences(acts, inp["obs0"], P).cpu().numpy()
    assert np.isfinite(ret_perm).all() and np.isfinite(ret_shuf).all()
    # the member draw matters for this (untrained, disagreeing) ensemble: across-draw spread is far above noise level
    assert ret_perm.std(axis=0).mean() > 1e-3
    pvals = np.array([stats.ks_2samp(ret_perm[:, n], ret_shuf[:, n]).pvalue for n in range(N)])
    # p-values of neighbouring sequences are correlated (they share draws), hence the slack around uniformity
    assert (pvals < 0.01).mean() <= 0.08, f"{(pvals < 0.01).mean():.3f} of sequences reject at 1 %"
    assert 0.3 <= pvals.mean() <= 0.7, pvals.mean()
    # first two moments of the per-sequence return, pooled over sequences
    np.testing.assert_allclose(ret_shuf.mean(axis=0), ret_perm.mean(axis=0), atol=5 * ret_perm.std(axis=0).max() / np.sqrt(draws))
    ratio = ret_shuf.std(axis=0) / ret_perm.std(axis=0)
    assert 0.9 <= np.median(ratio) <= 1.1, np.median(ratio)


@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
def test_sharded_cem_equals_unsharded_plan(precision):
    """ShardedCEMOptimizer over two shards (two threads on one GPU, the all-gather replaced by an in-process exchange)
    produces the plan CEMOptimizer produces on the union population for the same seed: population noise, model noise
    and member draws are keyed by global indices and the refit sums the elites in global index order."""
    import mbrl_lib_b200 as bp
    from mbrl_lib_b200.dist import ShardedCEMOptimizer
    from mbrl_lib_b200.planning import _FusedObjective

    spec = syn.CASES["halfcheetah"]
    H, A, N, P = spec.horizon, spec.act_dim, spec.population, spec.particles
    lb, ub = np.full((H, A), spec.action_lb).tolist(), np.full((H, A), spec.action_ub).tolist()
    inp = syn.make_rollout_inputs(spec, with_noise=False)
    iters = 3
    _, _, env = make_env("halfcheetah", precision, ts1="tile_shuffle")
    ref_opt = bp.CEMOptimizer(iters, 0.1, N, lb, ub, 0.1, DEV, return_mean_elites=True)
    ref_opt.record_values = True
    ref = ref_opt.optimize(_FusedObjective(env, inp["obs0"], P), x0=torch.zeros(H, A, device=DEV)).cpu().numpy()
    ref_vals = ref_opt.last_values.cpu().numpy()

    world = 2
    slots = [None] * world
    barrier = threading.Barrier(world)
    sols, vals, errs = [None] * world, [None] * world, []

    def worker(rank):
        try:
            torch.cuda.set_device(0)
            _, _, env_r = make_env("halfcheetah", precision, ts1="tile_shuffle")

            def gather(rec):
                torch.cuda.synchronize()
                slots[rank] = rec.clone()
                barrier.wait()
                out = torch.cat([slots[r] for r in range(world)], dim=0)
                barrier.wait()
                return out

            opt = ShardedCEMOptimizer(iters, 0.1, N, lb, ub, 0.1, DEV, return_mean_elites=True, rank=rank, world=world,
                                      gather=gather)
            opt.record_values = True
            sols[rank] = opt.optimize(_FusedObjective(env_r, inp["obs0"], P), x0=torch.zeros(H, A, device=DEV)).cpu().numpy()
            vals[rank] = opt.last_values.cpu().numpy()
        except Exception as e:  # pragma: no cover
            errs.append(e)
            barrier.abort()

    threads = [threading.Thread(target=worker, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=120)
    assert not errs, errs
    assert np.array_equal(sols[0], sols[1])  # every rank holds the same plan without a broadcast
    assert np.array_equal(np.concatenate([vals[0], vals[1]], axis=1), ref_vals)  # per-sequence returns, every iteration
    assert np.array_equal(sols[0], ref)


@pytest.mark.parametrize("precision,tol", [("f32", 2e-4), ("bf16_tc", 2e-2)])
def test_mbpo_device_rollout_loop_matches_oracle(precision, tol):
    """rollout_model_and_populate_sac_buffer (mbpo.py:31-63) with obs / predictions / accum_dones resident on the device
    and one ordered compaction at the end, against the oracle stepping the same loop with the same injected draws:
    per-step predictions within the kernel's bar, and the packed transitions EXACTLY the `~accum_dones` rows of the
    device's own per-step arrays, in the order of the reference's add_batch calls."""
    from mbrl_lib_b200 import mbpo
    from oracle import pets_oracle as po

    spec, arrays, env = make_env("mbpo_hopper_small", precision, ts1="perms")
    B, k = 1024, 4
    inp = syn.make_step_inputs(spec, B)
    inp["obs"][:, 1:] *= 0.1  # most rows start inside hopper's alive region (|angle| < 0.2, height > 0.7)
    g = np.random.default_rng(5)
    Wp = (0.3 * g.standard_normal((spec.obs_dim, spec.act_dim))).astype(np.float32)
    perms = [g.permutation(B).astype(np.int64) for _ in range(k)]
    eps = [g.standard_normal((B, spec.out_size)).astype(np.float32) for _ in range(k)]
    Wd = torch.from_numpy(Wp).to(DEV)

    class _Agent:
        def act_torch(self, obs, sample):
            return torch.tanh(obs @ Wd)

    staging = {}
    noise = [(torch.from_numpy(perms[i]).to(DEV), torch.from_numpy(eps[i]).to(DEV)) for i in range(k)]
    obs_p, act_p, nxt_p, rew_p, done_p, counts = mbpo.rollout_on_device(env, inp["obs"], _Agent(), True, k, _noise=noise,
                                                                         _staging=staging)
    oracle = _oracle(spec, arrays, False)
    batches, full = po.mbpo_rollout(oracle, inp["obs"], lambda o: torch.tanh(o @ torch.from_numpy(Wp)), k,
                                    [torch.from_numpy(p) for p in perms], [torch.from_numpy(e) for e in eps])
    st = {kk: v.cpu().numpy() for kk, v in staging.items()}
    # (1) the model steps: rows alive on BOTH sides follow the oracle within the kernel's bar
    both = np.ones(B, bool)
    for i in range(k):
        on, orw, od, okeep = full[i]
        both &= okeep & st["alive"][i].astype(bool)
        scale = max(1.0, np.abs(on[both]).max())
        assert np.abs(st["next_obs"][i][both] - on[both]).max() <= tol * scale, i
        assert np.abs(st["reward"][i][both] - orw[both]).max() <= tol * scale, i
        assert (st["done"][i][both].astype(bool) != od[both]).mean() <= (0.002 if precision == "f32" else 0.02)
        both &= ~(st["done"][i].astype(bool) ^ od)  # a row whose termination flipped at a threshold leaves the comparison
    assert both.sum() > 0 and st["alive"][k - 1].sum() < B  # the mask is exercised: some rows died, some survive
    # (2) the compaction: exactly the alive rows of the device's per-step arrays, in (step, row) order
    lo = 0
    for i in range(k):
        keep = st["alive"][i].astype(bool)
        n = int(keep.sum())
        assert counts[i] == n
        src_obs = st["obs0"] if i == 0 else st["next_obs"][i - 1]
        assert np.array_equal(obs_p[lo:lo + n], src_obs[keep])
        assert np.array_equal(act_p[lo:lo + n], st["act"][i][keep])
        assert np.array_equal(nxt_p[lo:lo + n], st["next_obs"][i][keep])
        assert np.array_equal(rew_p[lo:lo + n], st["reward"][i][keep])
        assert np.array_equal(done_p[lo:lo + n], st["done"][i][keep])
        if i + 1 < k:  # accum_dones |= dones (mbpo.py:62)
            assert np.array_equal(st["alive"][i + 1].astype(bool), keep & ~st["done"][i].astype(bool))
        lo += n
    assert lo == len(obs_p)
    if precision == "f32":  # same row sets as the oracle's add_batch calls when no threshold flipped
        if all(np.array_equal(st["alive"][i].astype(bool), full[i][3]) for i in range(k)):
            for i, (bo, ba, bn, br, bd) in enumerate(batches):
                assert len(bo) == counts[i]


def test_mbpo_populate_sac_buffer_api():
    """Drop-in signature of mbrl/algorithms/mbpo.py:31-63 with stand-in replay buffers; numpy agent fallback."""
    from mbrl_lib_b200 import mbpo

    spec, arrays, env = make_env("mbpo_hopper_small", "auto", ts1="tile_shuffle")
    B = 2048
    inp = syn.make_step_inputs(spec, B)
    inp["obs"][:, 1:] *= 0.1

    class _Batch:
        def astuple(self):
            return (inp["obs"], None, None, None, None, None)

    class _Replay:
        def sample(self, n):
            assert n == B
            return _Batch()

    class _Sac:
        def __init__(self):
            self.calls = []

        def add_batch(self, obs, action, next_obs, reward, terminated, truncated):
            assert obs.shape[1] == spec.obs_dim and action.shape[1] == spec.act_dim and next_obs.shape == obs.shape
            assert reward.shape == (len(obs),) and terminated.dtype == bool and truncated.dtype == bool and not truncated.any()
            self.calls.append(len(obs))

    class _NumpyAgent:
        def act(self, obs, sample=False, batched=False):
            assert batched and isinstance(obs, np.ndarray)
            return np.tanh(obs[:, :spec.act_dim]).astype(np.float32)

    sac = _Sac()
    mbpo.rollout_model_and_populate_sac_buffer(env, _Replay(), _NumpyAgent(), sac, True, 3, B)
    assert len(sac.calls) == 3 and sac.calls[0] == B and sac.calls[0] >= sac.calls[1] >= sac.calls[2] > 0
