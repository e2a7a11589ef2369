"""The rollout kernels' in-kernel draws by counter: the Gaussian output noise (RNG_STREAM_EPS) and the tile-shuffle member
(RNG_STREAM_MEMBER), and production rollouts with no injected draws against float64.

Every other float64 comparison of a rollout injects its noise, and takes the member map from the same device function the
rollout calls.  Here nothing is injected (no eps; a permutation only where the explicit-permutation mode is the subject),
and the draws are restated in numpy from the layout common.cuh documents:

* output noise: column o of row r at step t is lane o & 3 of philox_normal4(r, t, RNG_STREAM_EPS | (o >> 2), low word of
  off) under rng_key(seed, off); r the global row (seq0 + n) * P + p (under a permutation the row, not the slot), t = 0
  and P = 1 for ModelEnv.step, off = offset + k * 1024 for problem k of a batch;
* member: the elite position (x * M) >> 32, x word 0 of Philox at (low word of gt, t, RNG_STREAM_MEMBER, low word of off)
  under key (low word of s, high word of s ^ high word of gt), s = rng_key(seed, off), gt = p * C_glob + global
  sequence // 128 (row // 128 for ModelEnv.step), t = 0 under fixed_model.

1. Probe models (zero weights on a registered shape, so both kernels keep their launch plan; biases bf16 holds exactly):
   the member probe (deterministic, member e predicts e + 1 in column 0 and the learned-reward column) reads back the
   member of every (step, row), compared with torch.equal to the restatement and to ModelEnv.shuffle_member_assignment;
   the noise probe (mean 0, absolute targets, logvar biases inside and outside [min_logvar, max_logvar], per member under
   expectation) reads back sd * z, and z = next_obs / sd64 is compared with the restated draw.  Both kernels at each CTA
   shape they launch (tensor-core 64- and 128-row CTAs, fp32 64 / 32 / 16-row tiles), out % 4 of 0, 1 and 3, one window
   and single-step windows, offsets 0, 29 * 1024, 2^32 - 1024, 2^32 and 2^32 + 29 * 1024 (the last has the low word of
   29 * 1024: only the key tells them apart), a shard whose first sequence is not a multiple of 128, ModelEnv.step at
   1, 127, 128, 129 and 25 000 rows per member, consecutive steps of mbpo.rollout_on_device, and
   b200pets_eval_sequences_batch with K = 3 from 2^32 - 1024 (per-row returns at H = 1 read the learned column).
2. Negative controls: the restatement at t + 1, with the local row, with the slot for the row, with lane and word
   swapped, without the particle, with the key missing the offset's high word, with every problem at the first
   problem's offset, and for members with t not zeroed under TSinf and gt without p.
3. The law the reference draws with (torch.normal, randperm): recovered draws against N(0, 1) (KS) and uncorrelated
   across neighbouring rows, particles, steps, column groups, consecutive calls and batch problems; members uniform,
   particles of a sequence agreeing at 1 / M, constant over t under TSinf, consecutive TS1 steps agreeing at 1 / M.
4. Production rollouts (registered models, no injection) teacher-forced against oracle/transition_f64.py driven by the
   restated draws and member map, with per-row totals of b200pets_eval_sequences bit-equal to the trajectory's.

Bars:
  * members: equal (torch.equal), in the probe's read-back and in the exported map;
  * draws: |z - z_ref| <= 1e-4 * max(1, |z_ref|) beyond the radius slack of test_gpu_icem_draws (the kernel's __logf
    radius may be off by 2 * 2^-21.41 / r; u is rounded as the kernel rounds it): test_gpu_cem_kernels' Philox
    known-answer bar, for the fast log and sincos intrinsics and the tensor-core kernel's approximate sd;
  * production: test_gpu_transitions.BAR (2e-5 fp32, 2e-3 bf16_tc) of max(1, |ref|) beyond sd times the radius slack of
    each draw; done flags equal; per-row totals bit-equal;
  * negative controls: noise controls more than 100 times the draw bar, or NaN (outputs are NaN-filled, so an unwritten
    element fails); member controls differ from the read-back in at least 40 % of the elements they cover (a wrong draw
    agrees with the right one at 1 / M = 20 %);
  * law: KS p > 1e-3 and |corr| < 0.03 over at least 40 000 pairs; member frequencies chi-square p > 1e-3, agreement
    rates within 0.015 of 1 / M.
Measured on an H100 80GB HBM3 (700 W power limit): recovered draws 1.2e-6 to 2.3e-6 of max(1, |z|) beyond the slack
(every probe, both kernels); every member equal; production fp32 8.9e-7 and bf16_tc 2.4e-4 (plan_logvar_extreme) of
max(1, |ref|) beyond the allowance, 0 done flags and 0 per-row totals differ; noise controls 4.0 to 5.6 (over 10 000 times
the bar), member controls 45 % to 85 % of the elements; KS p 0.81, |corr| at most 0.0018, chi-square p 0.84 (TS1) and
1.0 (TSinf), agreement rates 0.199 to 0.200.  The file's wall time there: 40 s (28 s of tests).
"""
import dataclasses
import functools

import numpy as np
import pytest
import torch
from scipy import stats

import test_gpu_transitions as tt
from mbrl_lib_b200 import synthetic as syn
from oracle.transition_f64 import TransitionF64
from test_gpu_cem_kernels import philox4x32_10
from test_gpu_icem_draws import M32, philox_normal4_f32u, radius_slack, rng_key
from test_gpu_parity import DEV
from test_gpu_tiles import _sm_count, _tc_tiles

pytestmark = pytest.mark.gpu

RNG_STREAM_EPS, RNG_STREAM_MEMBER = 0x10000, 0x20000  # common.cuh
DRAW_BAR = 1e-4
CONTROL_FACTOR = 100.0
MEMBER_CONTROL_MIN = 0.4
OFFSETS = [0, 29 * 1024, (1 << 32) - 1024, 1 << 32, (1 << 32) + 29 * 1024]
SHARD_OFFSET = (1 << 32) + 29 * 1024
BATCH_OFFSET = (1 << 32) - 1024  # problems 0, 1, 2 at 2^32 - 1024, 2^32, 2^32 + 1024: across the key change
# raw logvar biases (bf16-exact): min_logvar is about -10 and max_logvar about 0.5 (synthetic.make_model_arrays)
LOGVARS = (-30.0, -12.0, -6.0, -3.0, -1.0, 0.0, 1.0, 2.5)


# ---- numpy restatement of the two streams -------------------------------------------------------------------------
def eps_draws(rows, t, out, seed, off, key=None, swap=False):
    """z [R, out] of rows `rows` (the Philox row word) at step t, and the radius slack of each draw.  `key` and `swap`
    (lane o >> 2, word o & 3) build negative controls."""
    o = np.arange(out)[None, :]
    word, lane = (o & 3, (o >> 2) & 3) if swap else (o >> 2, o & 3)
    rows = np.asarray(rows, np.int64).astype(np.uint64)[:, None] & np.uint64(M32)
    g, (u0, u2) = philox_normal4_f32u(rows, t, RNG_STREAM_EPS | word, off & M32, rng_key(seed, off) if key is None else key)
    lane = np.broadcast_to(lane, g.shape[1:])
    return np.take_along_axis(g, lane[None], axis=0)[0], radius_slack(np.where(lane < 2, u0, u2))


def row_keys(N, P, seq0=0, local=False, drop_p=False):
    """The Philox row word of local rows r = n * P + p: the global row (seq0 + n) * P + p (controls: the local row, or
    the particle dropped)."""
    n, p = np.arange(N)[:, None], np.arange(P)[None, :]
    return (((0 if local else seq0) + n) * P + (0 if drop_p else 1) * p).reshape(-1)


@functools.lru_cache(maxsize=8)
def traj_draws(N, P, H, out, seed, off, seq0=0, t_shift=0, local=False, drop_p=False, key=None, swap=False):
    """z, slack [H, N * P, out] of a trajectory."""
    r = row_keys(N, P, seq0, local, drop_p)
    zs, ss = zip(*[eps_draws(r, t + t_shift, out, seed, off, key, swap) for t in range(H)])
    return np.stack(zs), np.stack(ss)


def slot_draws(perms, H, out, seed, off, seq0, P):
    """Control: the draws keyed by the slot a row sits in (perms [H or 1, B]) instead of the row."""
    zs = []
    for t in range(H):
        perm = perms[min(t, perms.shape[0] - 1)]
        slot = np.empty_like(perm)
        slot[perm] = np.arange(perm.size)
        zs.append(eps_draws(slot + seq0 * P, t, out, seed, off)[0])
    return np.stack(zs)


def member_pos(gt, t, M, seed, off, key=None):
    gt = np.asarray(gt, np.int64).astype(np.uint64)
    assert (gt >> np.uint64(32) == 0).all()  # the key's gt word is then 0
    s = rng_key(seed, off) if key is None else key
    x = philox4x32_10(gt, t, RNG_STREAM_MEMBER, off & M32, s & M32, s >> 32)[0]
    return ((x * np.uint64(M)) >> np.uint64(32)).astype(np.int64)


def traj_members(N, P, H, M, seed, off, fixed, seq0=0, n_glob=0, t_shift=0, local=False, drop_p=False, key=None):
    """Elite positions [H, N * P] of a tile-shuffle trajectory."""
    C_glob = -(-(n_glob or N) // 128)
    n, p = np.arange(N)[:, None], np.arange(P)[None, :]
    gt = ((0 if drop_p else 1) * p * C_glob + ((0 if local else seq0) + n) // 128).reshape(-1)
    return np.stack([member_pos(gt, 0 if fixed else t + t_shift, M, seed, off, key) for t in range(H)])


# ---- probes -------------------------------------------------------------------------------------------------------
def probe(base, kind, propagation=None, **changes):
    """(spec, arrays) of a probe on registered shape `base`: zero weights, absolute targets.  kind "member":
    deterministic, member e's mean bias e + 1 in column 0 and the learned-reward column; kind "noise": mean bias 0,
    logvar bias LOGVARS[(o + 3 e) % 8] in column o under expectation, LOGVARS[o % 8] (every member) otherwise."""
    b = syn.CASES[base]
    spec = dataclasses.replace(b, target_is_delta=False, deterministic=kind == "member",
                               propagation=propagation or b.propagation, **changes)
    arrays = syn.make_model_arrays(spec)
    for a in arrays["weights"] + arrays["biases"]:
        a[...] = 0.0
    last, out = arrays["biases"][-1], spec.out_size
    for e in range(spec.ensemble_size):
        if kind == "member":
            last[e, 0, 0] = e + 1
            if spec.learned_rewards:
                last[e, 0, out - 1] = e + 1
        else:
            shift = 3 * e if spec.propagation == "expectation" else 0
            last[e, 0, out:] = [LOGVARS[(o + shift) % len(LOGVARS)] for o in range(out)]
    return spec, arrays


def elites(spec):
    return np.asarray(spec.elites if spec.elites is not None else range(spec.ensemble_size))


def probe_sd(spec, arrays):
    """sd [out] of the noise probe in float64: the two soft clamps of every elite's logvar, averaged under expectation."""
    raw = arrays["biases"][-1][elites(spec), 0, spec.out_size:].astype(np.float64)
    mn, mx = (np.asarray(arrays[k], np.float64).reshape(-1) for k in ("min_logvar", "max_logvar"))
    lv = mx - np.logaddexp(0.0, mx - raw)
    lv = mn + np.logaddexp(0.0, lv - mn)
    return np.sqrt(np.exp(lv.mean(0)))


def outputs(spec, nobs, rew):
    """Every model output column [..., out]: next_obs and, with a learned reward, the reward."""
    nobs = np.asarray(nobs, np.float64)
    return np.concatenate([nobs, np.asarray(rew, np.float64)[..., None]], -1) if spec.learned_rewards else nobs


def z_error(got, sd, z, slack):
    """max (|got / sd - z| - slack) / max(1, |z|); NaN (an unwritten element) stays NaN."""
    zg = np.asarray(got, np.float64) / sd
    return float(np.max(np.maximum(np.abs(zg - z) - slack, 0.0) / np.maximum(1.0, np.abs(z))))


def _worst(*errs):
    return float(np.max(errs))


def _modes(spec):
    return ["expectation"] if spec.propagation == "expectation" else ["perms", "shuffle"]


def _trajectory(env, spec, mode, windows, offset, shard=(0, 0)):
    inp = syn.make_rollout_inputs(spec)  # actions and obs0; the permutations where mode is "perms"; eps unused
    nobs, rew, done, assign, _ = tt.run_trajectory(env, spec, inp, mode, windows, offset, inject_eps=False, shard=shard)
    return inp, nobs, rew, assign


# ---- 1. noise probe: trajectories -----------------------------------------------------------------------------------
# name -> (registered shape, propagation, population, horizon, particles); out = out_size
NOISE = {
    "halfcheetah": ("halfcheetah", None, 300, 3, 20),  # out 17; fp32 64-row tiles, tensor-core 64-row CTAs (60 tiles)
    "halfcheetah_many_tiles": ("halfcheetah", None, 1500, 2, 20),  # 240 tiles: tensor-core 128-row CTAs
    "hopper_tsinf": ("hopper_tsinf", None, 300, 4, 6),  # out 12 (learned reward), fixed_model
    "plan_in254": ("plan_in254", None, 200, 3, 4),  # out 11
    "silu_expectation": ("silu_expectation", None, 300, 3, 4),  # out 17, 5 members with different logvars
    "relu_expectation": ("relu_expectation", None, 150, 3, 4),  # out 11, 3 members
    "plan_f32_hid512": ("plan_f32_hid512", None, 200, 3, 4),  # fp32 32-row tiles
    "humanoid_v4": ("humanoid_v4", None, 150, 2, 5),  # out 377 (learned reward), fp32 16-row tiles
}
NOISE_RUNS = [(n, p) for n, c in NOISE.items() for p in ("f32", "bf16_tc") if not (p == "bf16_tc" and c[0] in tt.NO_TC)]


def noise_probe(name):
    base, prop, N, H, P = NOISE[name]
    return probe(base, "noise", prop, population=N, horizon=H, particles=P)


def _f32_rows(env, spec):
    return env.staged.plan_info(spec.propagation)["f32_rows"]


@pytest.mark.parametrize("name,precision", NOISE_RUNS, ids=[f"{n}-{p}" for n, p in NOISE_RUNS])
def test_noise_probe_trajectories_follow_the_counter_layout(name, precision):
    spec, arrays = noise_probe(name)
    _, env = tt.make_env(spec, arrays, precision)
    N, H, P, out = spec.population, spec.horizon, spec.particles, spec.out_size
    sd = probe_sd(spec, arrays)
    if precision == "f32":
        want = {"plan_f32_hid512": 32, "humanoid_v4": 16}.get(name, 64)
        assert _f32_rows(env, spec) == want, env.staged.plan_info(spec.propagation)
    elif name.startswith("halfcheetah"):  # the CTA shape: 64-row CTAs below one tile per SM, 128-row above
        assert (_tc_tiles(spec, "tile_shuffle") > _sm_count()) == (name == "halfcheetah_many_tiles")
    worst, runs = 0.0, 0
    for mode in _modes(spec):
        for windows in ("one", "steps"):
            for off in OFFSETS:
                _, nobs, rew, _ = _trajectory(env, spec, mode, windows, off)
                z, slack = traj_draws(N, P, H, out, env._seed, off)
                worst = _worst(worst, z_error(outputs(spec, nobs, rew), sd, z, slack))
                runs += 1
        # a shard [70, 70 + N / 2) of the population: the first sequence is not a multiple of 128
        seq0, n = 70, N // 2
        sh = dataclasses.replace(spec, population=n)
        _, nobs, rew, _ = _trajectory(env, sh, mode, "one", SHARD_OFFSET, shard=(seq0, N))
        z, slack = traj_draws(n, P, H, out, env._seed, SHARD_OFFSET, seq0)
        worst = _worst(worst, z_error(outputs(spec, nobs, rew), sd, z, slack))
        runs += 1
    print(f"{name} {precision}: {runs} trajectories, out {out}, recovered draws {worst:.2e} of max(1, |z|) beyond the "
          f"radius slack (bar {DRAW_BAR:.0e})")
    assert worst <= DRAW_BAR


# ---- 1. member probe: trajectories ---------------------------------------------------------------------------------
MEMBER_BASE = "mbpo_halfcheetah_small"  # 7 members, elites (0, 2, 3, 5, 6), learned reward
MEMBER = {"ts1": ("random_model", 300, 6, 20), "tsinf": ("fixed_model", 300, 6, 20)}


def member_probe(prop, N, H, P):
    return probe(MEMBER_BASE, "member", prop, population=N, horizon=H, particles=P)


def member_values(spec, pos):
    """What the member probe writes for elite positions `pos`: the member's index + 1."""
    return (elites(spec)[pos] + 1).astype(np.float32)


def check_members(spec, nobs, rew, pos, what):
    want = torch.from_numpy(member_values(spec, pos))
    assert torch.equal(torch.from_numpy(np.ascontiguousarray(nobs[..., 0])), want), what
    assert torch.equal(torch.from_numpy(np.ascontiguousarray(rew)), want), what


@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
@pytest.mark.parametrize("prop", list(MEMBER))
def test_member_probe_trajectories_follow_the_counter_layout(prop, precision):
    propagation, N, H, P = MEMBER[prop]
    spec, arrays = member_probe(propagation, N, H, P)
    _, env = tt.make_env(spec, arrays, precision)
    M, fixed, runs = spec.num_models, propagation == "fixed_model", 0
    for windows in ("one", "steps"):
        for off in OFFSETS:
            _, nobs, rew, assign = _trajectory(env, spec, "shuffle", windows, off)
            pos = traj_members(N, P, H, M, env._seed, off, fixed)
            assert np.array_equal(assign, pos), f"exported map, offset {off}"
            check_members(spec, nobs, rew, pos, f"{windows} window(s), offset {off}")
            runs += 1
    seq0, n = 70, N // 2
    sh = dataclasses.replace(spec, population=n)
    _, nobs, rew, assign = _trajectory(env, sh, "shuffle", "one", SHARD_OFFSET, shard=(seq0, N))
    pos = traj_members(n, P, H, M, env._seed, SHARD_OFFSET, fixed, seq0, N)
    assert np.array_equal(assign, pos), "exported map of the shard"
    check_members(spec, nobs, rew, pos, "shard")
    print(f"{prop} {precision}: {runs + 1} trajectories, every member equal to the restatement and the exported map")


# ---- 1. ModelEnv.step, mbpo.rollout_on_device, batches ---------------------------------------------------------------
STEP_ROWS_PER_MEMBER = (1, 127, 128, 129, 25000)


def _step(env, spec, B, mode, off, g):
    """ModelEnv.step (sampled) over B rows from zero observations: outputs [B, out]."""
    obs = np.zeros((B, spec.obs_dim), np.float32)
    act = np.zeros((B, spec.act_dim), np.float32)
    perm = torch.from_numpy(g.permutation(B)).to(DEV) if mode == "perms" else None
    state = env.reset(obs, return_as_np=True)
    nobs, rew, _, _ = env.step(act, state, sample=True, _perm=perm, _offset=off)
    return nobs, rew[:, 0]


@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
def test_step_draws_follow_the_counter_layout(precision):
    """b200pets_step: row r draws at (r, 0) whatever the row mapping (in-kernel member, permutation, expectation), at
    1 to 25 000 rows per member; the member probe's members at gt = r // 128."""
    g = np.random.default_rng(5)
    worst, runs = 0.0, 0
    for prop, modes in (("random_model", ("shuffle", "perms")), ("expectation", ("expectation",))):
        spec, arrays = probe(MEMBER_BASE, "noise", prop)
        _, env = tt.make_env(spec, arrays, precision)
        sd = probe_sd(spec, arrays)
        M = spec.num_models
        for i, rpm in enumerate(STEP_ROWS_PER_MEMBER):
            B, off = M * rpm, OFFSETS[i % len(OFFSETS)]
            z, slack = traj_draws(B, 1, 1, spec.out_size, env._seed, off)
            for mode in modes:
                nobs, rew = _step(env, spec, B, mode, off, g)
                worst = _worst(worst, z_error(outputs(spec, nobs, rew), sd, z[0], slack[0]))
                runs += 1
    print(f"step {precision}: {runs} steps, recovered draws {worst:.2e} of max(1, |z|) beyond the radius slack "
          f"(bar {DRAW_BAR:.0e})")
    assert worst <= DRAW_BAR
    spec, arrays = probe(MEMBER_BASE, "member", "random_model")
    _, env = tt.make_env(spec, arrays, precision)
    M = spec.num_models
    for i, rpm in enumerate(STEP_ROWS_PER_MEMBER):
        B, off = M * rpm, OFFSETS[i % len(OFFSETS)]
        nobs, rew = _step(env, spec, B, "shuffle", off, g)
        pos = member_pos(np.arange(B) // 128, 0, M, env._seed, off)
        assert np.array_equal(env.shuffle_member_assignment(B, 1, 1, off)[0].numpy(), pos), B
        check_members(spec, nobs, rew, pos, f"step of {B} rows")


class _ZeroAgent:
    def __init__(self, A):
        self.A = A

    def act_torch(self, obs, sample):
        return torch.zeros(obs.shape[0], self.A, device=obs.device)


MBPO_FIRST = (1 << 22) - 1  # the first step's offset is 2^32 - 1024, the second 2^32


def mbpo_steps(precision, steps=4, rows_per_member=129):
    """mbpo.rollout_on_device on the noise probe: outputs [steps, B, out] of its consecutive ModelEnv.step calls and
    the offsets they drew at."""
    from mbrl_lib_b200 import mbpo

    spec, arrays = probe(MEMBER_BASE, "noise", "random_model")
    _, env = tt.make_env(spec, arrays, precision)
    B = spec.num_models * rows_per_member
    env._offset = MBPO_FIRST - 1
    st = {}
    mbpo.rollout_on_device(env, np.zeros((B, spec.obs_dim), np.float32), _ZeroAgent(spec.act_dim), True, steps, _staging=st)
    torch.cuda.synchronize()
    got = outputs(spec, st["next_obs"].cpu().numpy(), st["reward"].cpu().numpy())
    return spec, arrays, env, got, [(MBPO_FIRST + i) * 1024 for i in range(steps)]


@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
def test_mbpo_rollout_steps_each_draw_at_their_own_offset(precision):
    spec, arrays, env, got, offs = mbpo_steps(precision)
    sd, B = probe_sd(spec, arrays), got.shape[1]
    worst = 0.0
    for i, off in enumerate(offs):
        z, slack = traj_draws(B, 1, 1, spec.out_size, env._seed, off)
        worst = _worst(worst, z_error(got[i], sd, z[0], slack[0]))
    print(f"mbpo rollout {precision}: {len(offs)} steps, recovered draws {worst:.2e} (bar {DRAW_BAR:.0e})")
    assert worst <= DRAW_BAR
    z0, slack0 = traj_draws(B, 1, 1, spec.out_size, env._seed, offs[0])
    bad = _worst(*[z_error(got[i], sd, z0[0], slack0[0]) for i in range(1, len(offs))])
    print(f"control 'every step at the first step's offset': {bad:.2e} against bar {DRAW_BAR:.0e}")
    assert not bad <= CONTROL_FACTOR * DRAW_BAR, bad


def batch_rows(env, spec, K, offset=BATCH_OFFSET):
    """b200pets_eval_sequences_batch at H = 1: per-row returns [K, B], the learned column of step 0."""
    N, P = spec.population, spec.particles
    inp = syn.make_rollout_inputs(spec, with_noise=False)
    acts = torch.from_numpy(np.stack([inp["actions"]] * K)).to(DEV)
    rr = torch.full((K * N * P,), float("nan"), device=DEV)
    env.evaluate_action_sequences_batch(acts, np.stack([inp["obs0"]] * K), P, _row_returns=rr, _offset=offset)
    torch.cuda.synchronize()
    return rr.cpu().numpy().reshape(K, N * P).astype(np.float64)


def batch_noise(spec, seed, K, offsets):
    """The restated learned-column draws of problem k at offsets[k]: z, slack [K, B]."""
    B, o = spec.population * spec.particles, spec.out_size - 1
    zs, ss = zip(*[(z[0, :, o], s[0, :, o]) for z, s in (traj_draws(spec.population, spec.particles, 1, spec.out_size,
                                                                     seed, off) for off in offsets)])
    return np.stack(zs), np.stack(ss)


BATCH_SHAPE = dict(population=300, horizon=1, particles=4)
K_BATCH = 3


@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
def test_batch_problems_draw_at_their_own_offsets(precision):
    """Problem k of b200pets_eval_sequences_batch draws its noise and members at offset + k * 1024 under the key of that
    offset: from 2^32 - 1024 the three problems straddle the key's change."""
    offs = [BATCH_OFFSET + k * 1024 for k in range(K_BATCH)]
    spec, arrays = probe(MEMBER_BASE, "noise", "random_model", **BATCH_SHAPE)
    _, env = tt.make_env(spec, arrays, precision)
    sd = probe_sd(spec, arrays)[-1]
    got = batch_rows(env, spec, K_BATCH)
    z, slack = batch_noise(spec, env._seed, K_BATCH, offs)
    err = z_error(got, sd, z, slack)
    bad = z_error(got, sd, *batch_noise(spec, env._seed, K_BATCH, [BATCH_OFFSET] * K_BATCH)[:1], slack)
    print(f"batch {precision}: learned-column draws {err:.2e} (bar {DRAW_BAR:.0e}); control 'every problem at the "
          f"first offset' {bad:.2e}")
    assert err <= DRAW_BAR
    assert not bad <= CONTROL_FACTOR * DRAW_BAR, bad
    spec, arrays = probe(MEMBER_BASE, "member", "random_model", **BATCH_SHAPE)
    _, env = tt.make_env(spec, arrays, precision)
    got = batch_rows(env, spec, K_BATCH)
    N, P, M = spec.population, spec.particles, spec.num_models
    pos = np.stack([traj_members(N, P, 1, M, env._seed, off, False)[0] for off in offs])
    assert torch.equal(torch.from_numpy(got), torch.from_numpy(member_values(spec, pos).astype(np.float64)))
    wrong = np.stack([traj_members(N, P, 1, M, env._seed, BATCH_OFFSET, False)[0]] * K_BATCH)
    frac = float((member_values(spec, wrong) != got).mean())
    print(f"batch {precision}: members equal; control 'every problem at the first offset' differs in {frac:.2f}")
    assert frac >= MEMBER_CONTROL_MIN, frac


# ---- 2. negative controls -------------------------------------------------------------------------------------------
CONTROL_SHAPE = dict(population=300, horizon=4, particles=20)
SEQ0, N_SHARD = 100, 150  # the shard [100, 250) of 300 sequences: its local chunk differs from the global one for 100
NOISE_CONTROLS = {
    "t + 1": dict(t_shift=1),
    "local row": dict(local=True),
    "slot for the row": dict(slot=True),
    "lane and word swapped": dict(swap=True),
    "particle dropped": dict(drop_p=True),
    "key without the offset's high word": dict(key="seed"),
}


@functools.lru_cache(maxsize=2)
def control_noise_run(precision):
    """The noise probe on a shard under TS1 permutations, at an offset above 2^32."""
    spec, arrays = probe("halfcheetah", "noise", None, **CONTROL_SHAPE)
    _, env = tt.make_env(spec, arrays, precision)
    sh = dataclasses.replace(spec, population=N_SHARD)
    inp, nobs, rew, _ = _trajectory(env, sh, "perms", "one", SHARD_OFFSET, shard=(SEQ0, spec.population))
    return sh, probe_sd(spec, arrays), env._seed, inp["perms"], outputs(sh, nobs, rew)


@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
@pytest.mark.parametrize("kind", list(NOISE_CONTROLS))
def test_noise_negative_controls_fail_the_bar(kind, precision):
    spec, sd, seed, perms, got = control_noise_run(precision)
    N, H, P, out = spec.population, spec.horizon, spec.particles, spec.out_size
    z, slack = traj_draws(N, P, H, out, seed, SHARD_OFFSET, SEQ0)
    right = z_error(got, sd, z, slack)
    assert right <= DRAW_BAR
    kw = dict(NOISE_CONTROLS[kind])
    if kw.pop("slot", False):
        zc = slot_draws(perms, H, out, seed, SHARD_OFFSET, SEQ0, P)
    else:
        if kw.get("key") == "seed":
            kw["key"] = seed
        zc = traj_draws(N, P, H, out, seed, SHARD_OFFSET, SEQ0, **kw)[0]
    err = _worst(right, z_error(got, sd, zc, slack))
    print(f"noise control '{kind}' ({precision}): {err:.2e} against bar {DRAW_BAR:.0e}")
    assert not err <= CONTROL_FACTOR * DRAW_BAR, err


def test_noise_control_of_an_unwritten_element_fails():
    spec, sd, seed, _, got = control_noise_run("f32")
    z, slack = traj_draws(spec.population, spec.particles, spec.horizon, spec.out_size, seed, SHARD_OFFSET, SEQ0)
    got = got.copy()
    got[-1, -1, -1] = np.nan
    assert np.isnan(z_error(got, sd, z, slack))


MEMBER_CONTROLS = {  # kind -> (propagation, restatement changes)
    "t + 1": ("random_model", dict(t_shift=1)),
    "local row": ("random_model", dict(local=True)),
    "gt without p": ("random_model", dict(drop_p=True)),
    "key without the offset's high word": ("random_model", dict(key="seed")),
    "t not zeroed under TSinf": ("fixed_model", dict(fixed=False)),
}


@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
@pytest.mark.parametrize("kind", list(MEMBER_CONTROLS))
def test_member_negative_controls_fail(kind, precision):
    prop, kw = MEMBER_CONTROLS[kind]
    N, H, P = CONTROL_SHAPE["population"], CONTROL_SHAPE["horizon"], CONTROL_SHAPE["particles"]
    spec, arrays = member_probe(prop, N, H, P)
    _, env = tt.make_env(spec, arrays, precision)
    sh = dataclasses.replace(spec, population=N_SHARD)
    _, nobs, rew, _ = _trajectory(env, sh, "shuffle", "one", SHARD_OFFSET, shard=(SEQ0, N))
    M, fixed = spec.num_models, prop == "fixed_model"
    pos = traj_members(N_SHARD, P, H, M, env._seed, SHARD_OFFSET, fixed, SEQ0, N)
    check_members(spec, nobs, rew, pos, "right restatement")
    kw = dict(kw)
    if kw.get("key") == "seed":
        kw["key"] = env._seed
    fixed = kw.pop("fixed", fixed)
    wrong = traj_members(N_SHARD, P, H, M, env._seed, SHARD_OFFSET, fixed, SEQ0, N, **kw)
    frac = float((member_values(spec, wrong) != nobs[..., 0]).mean())
    print(f"member control '{kind}' ({precision}): differs in {frac:.2f} of the elements (right: 0)")
    assert frac >= MEMBER_CONTROL_MIN, frac


# ---- 3. the law -------------------------------------------------------------------------------------------------------
CORR_MAX = 0.03


def _corr(a, b):
    a, b = np.ravel(a), np.ravel(b)
    assert a.size >= 40000, a.size
    return float(np.corrcoef(a, b)[0, 1])


def test_noise_law():
    """Recovered draws of a 10 000-row trajectory, the next call's and a batch of three 40 000-row problems."""
    spec, arrays = probe("halfcheetah", "noise", None, population=500, horizon=4, particles=20)
    _, env = tt.make_env(spec, arrays, "f32")
    sd = probe_sd(spec, arrays)
    N, H, P, out = spec.population, spec.horizon, spec.particles, spec.out_size
    runs = []
    for off in (40 * 1024, 41 * 1024):  # consecutive calls
        _, nobs, rew, _ = _trajectory(env, spec, "shuffle", "one", off)
        zg = outputs(spec, nobs, rew) / sd
        z, slack = traj_draws(N, P, H, out, env._seed, off)
        assert z_error(zg * sd, sd, z, slack) <= DRAW_BAR
        runs.append(zg.reshape(H, N, P, out))
    zg = runs[0]
    ks = stats.kstest(zg.ravel(), "norm").pvalue
    corr = {"neighbouring sequences": _corr(zg[:, :-1], zg[:, 1:]),
            "particles of a sequence": _corr(zg[:, :, :-1], zg[:, :, 1:]),
            "steps": _corr(zg[:-1], zg[1:]),
            "column groups (o, o + 4)": _corr(zg[..., :-4], zg[..., 4:]),
            "consecutive calls": _corr(runs[0], runs[1])}
    bspec, barrays = probe(MEMBER_BASE, "noise", "random_model", population=8000, horizon=1, particles=5)
    _, benv = tt.make_env(bspec, barrays, "f32")
    zb = batch_rows(benv, bspec, K_BATCH) / probe_sd(bspec, barrays)[-1]
    corr["batch problems"] = _corr(zb[:-1], zb[1:])
    print(f"KS p {ks:.3f} over {zg.size} draws; " + ", ".join(f"{k} {v:+.4f}" for k, v in corr.items()))
    assert ks > 1e-3
    assert all(abs(v) < CORR_MAX for v in corr.values()), corr


def _agree(a, b):
    return float((a == b).mean())


def test_member_law():
    """The in-kernel map (b200pets_shuffle_member_map) of 6 400 sequences x 20 particles x 30 steps: one draw per
    (group, step) under TS1, per group under TSinf."""
    N, H, P = 6400, 30, 20
    for prop in ("random_model", "fixed_model"):
        spec, arrays = member_probe(prop, N, H, P)
        _, env = tt.make_env(spec, arrays, "f32")
        M = spec.num_models
        assign = env.shuffle_member_assignment(N, H, P, 29 * 1024).numpy()
        groups = assign.reshape(H, N // 128, 128, P)[:, :, 0, :]  # [H, chunk, particle]: one draw per group
        if prop == "fixed_model":
            assert (assign == assign[:1]).all(), "TSinf members change over t"
            draws = groups[0]
        else:
            draws = groups
        chi = stats.chisquare(np.bincount(draws.ravel(), minlength=M)).pvalue
        pairs = [_agree(draws[..., p], draws[..., q]) for p in range(P) for q in range(p + 1, P)]
        particles = float(np.mean(pairs))
        line = f"{prop}: chi-square p {chi:.3f} over {draws.size} draws, particles of a sequence agree {particles:.4f}"
        assert chi > 1e-3 and abs(particles - 1 / M) < 0.015, line
        if prop == "random_model":
            steps = _agree(groups[:-1], groups[1:])
            line += f", consecutive steps agree {steps:.4f}"
            assert abs(steps - 1 / M) < 0.015, line
        print(line + f" (1 / M = {1 / M:.3f})")


# ---- 4. production rollouts against float64 ---------------------------------------------------------------------------
PRODUCTION = ["halfcheetah_small", "hopper_tsinf", "silu_expectation", "mbpo_hopper_small", "plan_logvar_extreme",
              "halfcheetah"]
PROD_OFFSET = (1 << 32) + 29 * 1024


@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
@pytest.mark.parametrize("name", PRODUCTION)
def test_production_rollout_matches_float64_with_in_kernel_draws(name, precision):
    spec = syn.CASES[name]
    arrays = syn.make_model_arrays(spec)
    model, env = tt.make_env(spec, arrays, precision)
    N, H, P, M = spec.population, spec.horizon, spec.particles, spec.num_models
    mode = "expectation" if spec.propagation == "expectation" else "shuffle"
    inp = syn.make_rollout_inputs(spec, with_noise=False)
    nobs, rew, done, assign, eval_rows = tt.run_trajectory(env, spec, inp, mode, "one", PROD_OFFSET, inject_eps=False)
    if mode == "shuffle":
        pos = traj_members(N, P, H, M, env._seed, PROD_OFFSET, spec.propagation == "fixed_model")
        assert np.array_equal(assign, pos)
    else:
        pos = None
    z, slack = traj_draws(N, P, H, spec.out_size, env._seed, PROD_OFFSET)
    ck = TransitionF64.from_model(spec, model)
    err = tt.check_trajectory(spec, ck, inp, nobs, rew, done, pos, precision == "bf16_tc", mode, eps=z, slack=slack)
    tt.assert_within(err, precision)
    differ = int((eval_rows() != tt.masked_row_totals(rew, done)).sum())
    print(f"{name}: per-row totals of eval_sequences differ from the trajectory's in {differ} rows")
    assert differ == 0
