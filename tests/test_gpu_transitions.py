"""Every column of every model step: the rollout and step kernels against a float64 transition, row by row.

The parity tests check a rollout through its particle-mean returns.  A return hides most of what a rollout kernel
computes: the last step's observation, and every observation column the reward function does not read (those enter
only through the next step's first layer).  Here the kernels' own outputs are compared element by element with
oracle/transition_f64.py (pinned on the CPU by tests/test_transition_checker.py):

* teacher forcing: step t's reference starts from the kernel's own ``next_obs`` of step t - 1 (``obs0`` at t = 0), so
  errors do not accumulate and each row is checked on its own.  Large launches check a strided subset of rows that
  includes the first and last row (and the 64-row halves) of every 128-row tile, of every shuffle group and of every
  member's slot range;
* ``b200pets_eval_trajectory`` (the ``TRAJ = true`` kernels the reward / termination callables read) over every case
  in ``synthetic.CASES``, at fp32 and on the tensor-core kernel wherever it has a plan for the case's propagation, with
  every member draw the case's propagation allows (injected permutations, the in-kernel tile-shuffle draw with its
  exported map, expectation), as one window and as single-step windows (the carried-state path);
* per-row totals of ``b200pets_eval_sequences`` (the ``TRAJ = false`` kernels ``bench.py`` times) equal, bit for bit,
  the masked sum of the trajectory's own reward / done with the same draws (model_env.py:183-188);
* ``ModelEnv.step`` (``b200pets_step``, MBPO's model step) over the same cases at 1, 127, 128 and 129 rows per member,
  ``sample=False``, and a batch with more 128-row tiles than SMs;
* model options no registered case has: ``target_is_delta=False``, several ``no_delta_list`` indices on a learned
  reward model, LeakyReLU slope 0.2, a deterministic model under TSinf and under expectation, an observation of 1e3;
* ``b200pets_model_refresh`` after weights, elite order, normaliser and logvar bounds all change;
* negative controls: a checker with one deliberate error (slope, ``no_delta_list``, member position, ``eps`` column)
  must fail the bar.

Bars, per element of ``next_obs`` and of the reward, relative to max(1, |ref|).  tests/prof_transitions.py prints the
worst values; measured on an H100 80GB HBM3 at a 700 W power limit, over every case, kernel, member draw and window:
  * fp32 kernel against the float64 step: worst 1.0e-6 (reward, plan_in254 step) and 3.1e-6 with an observation of 1e3
    (fp32 sums of a ~1e2 first-layer term); bar 2e-5;
  * tensor-core kernel against the bf16-operand float64 step: worst 3.4e-4 (plan_k1_out256 step; most cases 5e-5 to
    2e-4); bar 2e-3.  The observation of 1e3 has its own row rule (:func:`assert_large_input_rows`);
  * ``done`` equal to the termination function on the kernel's own ``next_obs``, bit for bit (0 differ everywhere), and
    the per-row totals of the two kernel instantiations equal bit for bit (0 rows differ everywhere);
  * negative controls: 2.5e-2 (slope), 0.73 (no_delta_list), 0.25 (member), 0.58 (eps columns), at both kernels.
"""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

from mbrl_lib_b200 import synthetic as syn
from oracle.transition_f64 import TransitionF64, assignment_from_perm, known_done, known_reward
from test_gpu_parity import DEV, _Env
from test_gpu_tiles import TILE, _sm_count, _tc_tiles

pytestmark = pytest.mark.gpu

BAR = {"f32": 2e-5, "bf16_tc": 2e-3}
# registered cases the tensor-core kernel has no launch plan for (their propagation): the fp32 kernel only
NO_TC = {"humanoid_v4", "plan_f32_hid512", "plan_f32_hid512_exp", "plan_f32_humanoid_exp"}
# rows of the float64 reference per step beyond the tile / group / slot edges
STRIDED_ROWS = 768
SHUFFLE_OFFSET = 29 * 1024


def _spec(name):
    spec = syn.CASES[name]
    if name == "mbpo_halfcheetah":  # config 4 is 100 000 states: 25 000 keep 196 tiles of 128 rows
        spec = dataclasses.replace(spec, population=25000)
    return spec


def _modes(spec, step=False):
    """Member draws of the case's propagation: injected permutations (TS1 per step / TSinf at reset), the in-kernel
    tile-shuffle draw, or expectation.  A TSinf step always takes the caller's propagation indices
    (gaussian_mlp.py:208-211)."""
    if spec.propagation == "expectation":
        return ["expectation"]
    return ["perms"] if step and spec.propagation == "fixed_model" else ["perms", "shuffle"]


def make_env(spec, arrays, precision, slope=None):
    import mbrl_lib_b200 as bp
    from mbrl_lib_b200 import functions

    model = bp.model_from_arrays(spec, arrays, DEV)
    if slope is not None:
        for seq in model.model.hidden_layers:
            seq[1] = torch.nn.LeakyReLU(slope)
    rew = functions.REWARD_FNS[spec.reward_fn] if spec.reward_fn else None
    env = bp.ModelEnv(_Env(spec), model, functions.TERM_FNS[spec.term_fn], rew, generator=torch.Generator(device=DEV),
                      precision=precision, ts1="tile_shuffle")
    env._few_groups = lambda *a: False  # the in-kernel member draw at every population
    if precision == "bf16_tc":
        assert env.staged.supports_tc(spec.propagation), spec.name
    return model, env


# ---- rows ------------------------------------------------------------------------------------------------------
def _edges(lo, hi):
    """First and last row of every 128-row tile of [lo, hi) and of each of its 64-row halves."""
    out = []
    for k in range(lo, hi, TILE // 2):
        out += [k, min(k + TILE // 2, hi) - 1]
    return out


def check_rows(N, P, M, perm=None):
    """Rows r = n * P + p checked at one step: a strided subset plus the tile edges of every row mapping the kernels
    use -- 128-row tiles in row order (expectation, step tile shuffle), shuffle groups (particle p of 128 consecutive
    sequences) and, under a permutation, the tiles of every member's slot range (slot i holds row perm[i])."""
    B = N * P
    if B <= 2 * STRIDED_ROWS:
        return np.arange(B)
    s = set(range(0, B, B // STRIDED_ROWS)) | {B - 1}
    s.update(_edges(0, B))
    for p in range(P):
        for c in range(0, N, TILE):
            s.update([c * P + p, (min(c + TILE, N) - 1) * P + p, (min(c + TILE // 2, N) - 1) * P + p])
    if perm is not None:
        for m in range(M):
            s.update(perm[_edges(m * (B // M), (m + 1) * (B // M))].tolist())
    return np.array(sorted(s))


def _rel(got, ref, allow=0.0):
    got = np.asarray(got, np.float64).reshape(ref.shape[0], -1)
    allow = np.reshape(allow, (ref.shape[0], -1)) if np.ndim(allow) else allow
    ref = ref.reshape(ref.shape[0], -1)
    return (np.maximum(np.abs(got - ref) - allow, 0.0) / np.maximum(1.0, np.abs(ref))).max(axis=1)


def compare_step(spec, ck, obs, act, members, eps, nobs, rew, done, bf16, sample=True, slack=None):
    """Worst relative error of next_obs and reward of these rows, the number of done flags that differ, and every row's
    worst error ("rows").  `slack` [rows, out] (in-kernel draws): how far each draw may be off; an element may then
    differ from the reference by that times its sd beyond the bar (the checker's output moved by `slack` in place of
    the draws, less its output at zero draws)."""
    ref_obs, ref_rew = ck.step(obs, act, members, eps, sample=sample, bf16=bf16)
    a_obs = a_rew = 0.0
    if slack is not None:
        hi_obs, hi_rew = ck.step(obs, act, members, slack, sample=sample, bf16=bf16)
        lo_obs, lo_rew = ck.step(obs, act, members, np.zeros_like(slack), sample=sample, bf16=bf16)
        a_obs = np.abs(hi_obs - lo_obs)
        a_rew = 0.0 if hi_rew is None else np.abs(hi_rew - lo_rew)
    if spec.reward_fn is not None:  # a known function on the kernel's own next_obs (it wins over a learned column)
        ref_rew, a_rew = known_reward(spec.reward_fn, act, nobs), 0.0
    bad_done = int((known_done(spec.term_fn, act, nobs) != done.astype(bool)).sum())
    e_obs, e_rew = _rel(nobs, ref_obs, a_obs), _rel(rew, ref_rew, a_rew)
    return {"next_obs": float(e_obs.max()), "reward": float(e_rew.max()), "done": bad_done,
            "rows": np.maximum(e_obs, e_rew)}


def _worst(acc, err):
    for k, v in err.items():
        if k == "rows":
            acc[k] = np.concatenate([acc[k], v]) if k in acc else v
        else:
            acc[k] = max(acc.get(k, 0), v)
    return acc


# ---- trajectories --------------------------------------------------------------------------------------------------
def run_trajectory(env, spec, inp, mode, windows, offset=SHUFFLE_OFFSET, inject_eps=True, shard=(0, 0)):
    """b200pets_eval_trajectory over [0, H) as one window ("one") or H single-step windows ("steps").  Returns next_obs
    [H, B, D], reward [H, B], done [H, B], the row -> member map [H, B] (None for expectation) and a closure that runs
    b200pets_eval_sequences with the same configuration and draws (per-row totals).  With `inject_eps` False the
    kernels draw their own noise (a NULL eps); `shard` is (first sequence, global population) of a sharded evaluation
    whose population is spec.population."""
    from mbrl_lib_b200 import _lib

    lib, h = env.lib, env.staged.handle
    N, H, P, D = spec.population, spec.horizon, spec.particles, spec.obs_dim
    B = N * P
    prop = spec.propagation
    perms = torch.from_numpy(inp["perms"]).to(DEV) if mode == "perms" else None
    eps = None if spec.deterministic or not inject_eps else torch.from_numpy(inp["eps"]).to(DEV)
    acts = torch.from_numpy(inp["actions"]).to(DEV)
    obs0 = torch.from_numpy(np.asarray(inp["obs0"], np.float32)).to(DEV)
    cfg = _lib.RolloutCfg(N, H, P, _lib.PREC[env.precision], _lib.PROP[prop],
                          _lib.TS1_PERMS if perms is not None else _lib.TS1_TILE_SHUFFLE, env._seed, offset, *shard)
    ws = torch.empty(lib.b200pets_trajectory_workspace_bytes(h, C.byref(cfg)), dtype=torch.uint8, device=DEV)
    nobs = torch.full((H, B, D), float("nan"), device=DEV)
    rew = torch.full((H, B), float("nan"), device=DEV)
    done = torch.full((H, B), 7, dtype=torch.uint8, device=DEV)
    spans = [(0, H)] if windows == "one" else [(t, t + 1) for t in range(H)]
    for t0, t1 in spans:
        _lib.check(lib.b200pets_eval_trajectory(h, C.byref(cfg), t0, t1, _lib.ptr(obs0), _lib.ptr(acts), _lib.ptr(perms),
                                                _lib.ptr(eps), _lib.ptr(nobs[t0]), _lib.ptr(rew[t0]), _lib.ptr(done[t0]),
                                                _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), "eval_trajectory")
    torch.cuda.synchronize()
    M = spec.num_models
    if mode == "perms":
        assign = np.stack([assignment_from_perm(inp["perms"][min(t, inp["perms"].shape[0] - 1)], M) for t in range(H)])
    elif mode == "shuffle":
        assign = env.shuffle_member_assignment(N, H, P, offset, *shard).numpy()
    else:
        assign = None

    def eval_rows():
        wsz = lib.b200pets_eval_workspace_bytes(h, C.byref(cfg))
        w = torch.empty(wsz, dtype=torch.uint8, device=DEV)
        ret = torch.empty(N, device=DEV)
        rows = torch.empty(B, device=DEV)
        _lib.check(lib.b200pets_eval_sequences(h, C.byref(cfg), _lib.ptr(obs0), _lib.ptr(acts), _lib.ptr(perms), _lib.ptr(eps),
                                               _lib.ptr(ret), _lib.ptr(rows), _lib.ptr(w), w.numel(), _lib.stream_ptr()),
                   "eval_sequences")
        torch.cuda.synchronize()
        return rows.cpu().numpy()

    return nobs.cpu().numpy(), rew.cpu().numpy(), done.cpu().numpy(), assign, eval_rows


def check_trajectory(spec, ck, inp, nobs, rew, done, assign, bf16, mode, eps=None, slack=None):
    """Teacher-forced comparison of every step: worst errors over steps and checked rows (`slack` [H, B, out]: see
    compare_step)."""
    N, H, P, M = spec.population, spec.horizon, spec.particles, spec.num_models
    B = N * P
    eps = inp.get("eps") if eps is None else eps
    obs0 = np.asarray(inp["obs0"], np.float32)
    acc = {}
    for t in range(H):
        perm = inp["perms"][min(t, inp["perms"].shape[0] - 1)] if mode == "perms" else None
        rows = check_rows(N, P, M, perm)
        obs = np.broadcast_to(obs0, (rows.size, obs0.size)) if t == 0 else nobs[t - 1, rows]
        act = inp["actions"][rows // P, t]
        e = None if spec.deterministic else eps[t, rows]
        mem = None if assign is None else assign[t, rows]
        s = None if slack is None or spec.deterministic else slack[t, rows]
        _worst(acc, compare_step(spec, ck, obs, act, mem, e, nobs[t, rows], rew[t, rows], done[t, rows], bf16, slack=s))
    assert np.isfinite(nobs).all() and np.isfinite(rew).all() and (done <= 1).all()
    return acc


def masked_row_totals(rew, done):
    """model_env.py:183-188 in fp32 with the kernels' order of operations: a reward after termination counts 0."""
    tot = np.zeros(rew.shape[1], np.float32)
    dead = np.zeros(rew.shape[1], bool)
    for t in range(rew.shape[0]):
        tot = (tot + np.where(dead, np.float32(0), rew[t])).astype(np.float32)
        dead |= done[t].astype(bool)
    return tot


def trajectory_errors(name, precision, mode, windows, spec=None, arrays=None, slope=None, obs0=None, link=False):
    spec = spec or _spec(name)
    arrays = arrays if arrays is not None else syn.make_model_arrays(spec)
    model, env = make_env(spec, arrays, precision, slope)
    inp = syn.make_rollout_inputs(spec)
    if obs0 is not None:
        inp["obs0"] = obs0
    nobs, rew, done, assign, eval_rows = run_trajectory(env, spec, inp, mode, windows)
    ck = TransitionF64.from_model(spec, model)
    err = check_trajectory(spec, ck, inp, nobs, rew, done, assign, precision == "bf16_tc", mode)
    if link:
        got = eval_rows()
        want = masked_row_totals(rew, done)
        err["link_rows_differ"] = int((got != want).sum())
    return err, (spec, model, env, inp, nobs, rew, done, assign)


def assert_within(err, precision):
    bar = BAR[precision]
    print(f"{precision}: next_obs {err['next_obs']:.2e}, reward {err['reward']:.2e} of max(1, |ref|) (bar {bar:.0e}), "
          f"done differ {err['done']}")
    assert err["next_obs"] <= bar and err["reward"] <= bar, err
    assert err["done"] == 0, err


TRAJ = [(n, p, m) for n in syn.CASES for p in ("f32", "bf16_tc") for m in _modes(syn.CASES[n])
        if not (p == "bf16_tc" and n in NO_TC)]


@pytest.mark.parametrize("windows", ["one", "steps"])
@pytest.mark.parametrize("name,precision,mode", TRAJ, ids=[f"{n}-{p}-{m}" for n, p, m in TRAJ])
def test_trajectory_matches_float64_step(name, precision, mode, windows):
    err, _ = trajectory_errors(name, precision, mode, windows, link=windows == "one")
    assert_within(err, precision)
    if windows == "one":  # the TRAJ = false kernel's per-row totals: the same rows, bit for bit
        assert err["link_rows_differ"] == 0, err


def test_no_tc_list_is_exact():
    """NO_TC names exactly the registered cases without a tensor-core plan for their propagation."""
    for name, spec in syn.CASES.items():
        _, env = make_env(spec, syn.make_model_arrays(spec), "f32")
        assert env.staged.supports_tc(spec.propagation) == (name not in NO_TC), name


# ---- ModelEnv.step ---------------------------------------------------------------------------------------------
ROWS_PER_MEMBER = (1, 127, 128, 129)


def step_errors(name, precision, mode):
    """``ModelEnv.step`` at 1 / 127 / 128 / 129 rows per member (sampled and, at 129, the mean prediction) and at a
    batch with more 128-row tiles than the device has SMs; worst errors over all of them."""
    spec = _spec(name)
    arrays = syn.make_model_arrays(spec)
    model, env = make_env(spec, arrays, precision)
    ck = TransitionF64.from_model(spec, model)
    M = spec.num_models
    sms = _sm_count()
    big = TILE * -(-(sms + 1) // M) + 5
    acc = {}
    runs = [(r, True) for r in ROWS_PER_MEMBER] + [(129, False), (big, True)]
    for i, (rpm, sample) in enumerate(runs):
        B = M * rpm
        if rpm == big:
            tiles = _tc_tiles(dataclasses.replace(spec, population=B, particles=1),
                              {"perms": "ts1_perms", "shuffle": "tile_shuffle", "expectation": "expectation"}[mode])
            assert tiles > sms, tiles
        inp = syn.make_step_inputs(spec, B)
        perm = torch.from_numpy(inp["perm"]).to(DEV) if mode == "perms" else None
        eps = None if spec.deterministic else torch.from_numpy(inp["eps"]).to(DEV)
        offset = (31 + i) * 1024
        state = env.reset(inp["obs"], return_as_np=True)
        nobs, rew, done, _ = env.step(inp["act"], state, sample=sample, _perm=perm, _eps=eps, _offset=offset)
        if mode == "perms":
            members = assignment_from_perm(inp["perm"], M)
        elif mode == "shuffle":
            members = env.shuffle_member_assignment(B, 1, 1, offset)[0].numpy()
        else:
            members = None
        rows = check_rows(B, 1, M, inp["perm"] if mode == "perms" else None)
        e = None if spec.deterministic else inp["eps"][rows]
        _worst(acc, compare_step(spec, ck, inp["obs"][rows], inp["act"][rows], None if members is None else members[rows],
                                 e, nobs[rows], rew[rows, 0], done[rows, 0], precision == "bf16_tc", sample=sample))
        assert np.isfinite(nobs).all() and np.isfinite(rew).all()
    return acc


STEP = [(n, p, m) for n in syn.CASES for p in ("f32", "bf16_tc") for m in _modes(syn.CASES[n], step=True)
        if not (p == "bf16_tc" and n in NO_TC)]


@pytest.mark.parametrize("name,precision,mode", STEP, ids=[f"{n}-{p}-{m}" for n, p, m in STEP])
def test_step_matches_float64_step(name, precision, mode):
    assert_within(step_errors(name, precision, mode), precision)


# ---- model options no registered case has ------------------------------------------------------------------------
def _obs0_large(spec):
    o = syn.make_rollout_inputs(spec, with_noise=False)["obs0"].copy()
    o[3] = 1e3
    return o


# name -> (base case, CaseSpec changes, LeakyReLU slope, obs0 builder)
OPTIONS = {
    "absolute_targets": ("halfcheetah_small", {"target_is_delta": False}, None, None),
    "no_delta_learned": ("tc_hid64", {"no_delta_list": (0, 4, 8)}, None, None),
    "leaky_slope_0.2": ("cartpole", {}, 0.2, None),
    "det_tsinf": ("pusher_det", {"propagation": "fixed_model"}, None, None),
    "det_expectation": ("pusher_det", {"propagation": "expectation"}, None, None),
    "obs_1e3": ("halfcheetah_small", {}, None, _obs0_large),
}


def option_case(opt):
    base, changes, slope, obs0 = OPTIONS[opt]
    spec = dataclasses.replace(syn.CASES[base], name=f"{base}_{opt}", **changes)
    arrays = syn.make_model_arrays(syn.CASES[base])
    return spec, arrays, slope, (obs0(spec) if obs0 else None)


def option_errors(opt, precision, mode=None):
    spec, arrays, slope, obs0 = option_case(opt)
    mode = mode or _modes(spec)[-1]
    return trajectory_errors(spec.name, precision, mode, "one", spec=spec, arrays=arrays, slope=slope, obs0=obs0)


@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
@pytest.mark.parametrize("opt", list(OPTIONS))
def test_model_option_matches_float64_step(opt, precision):
    err, (spec, model, env, *_) = option_errors(opt, precision)
    assert env.staged.desc.target_is_delta == int(spec.target_is_delta)
    if opt == "obs_1e3" and precision == "bf16_tc":
        assert_large_input_rows(err)
    else:
        assert_within(err, precision)


def assert_large_input_rows(err):
    """The tensor-core kernel with an observation of 1e3: the normalised input is ~1e3 and the hidden activations reach
    ~1e2, where one bf16 step is 0.5.  An activation whose fp32 sum (kernel) and float64 sum (checker) straddle a bf16
    rounding boundary then rounds to neighbouring bf16 values, and the row's outputs move by up to ~1e-2.  Such flips
    are isolated rows; a wrong kernel moves every row.  Measured (halfcheetah_small, 200 rows x 12 steps): median row
    8.3e-7, 1.5 % of rows above 2e-3, worst 8.2e-3; the fp32 kernel on the same input stays within 3.1e-6."""
    rows = err["rows"]
    frac = float((rows > BAR["bf16_tc"]).mean())
    print(f"bf16_tc, observation 1e3: median row {np.median(rows):.2e}, {frac:.4f} of rows above {BAR['bf16_tc']:.0e}, "
          f"worst {rows.max():.2e}, done differ {err['done']}")
    assert np.median(rows) <= 1e-5, np.median(rows)
    assert frac <= 0.05, frac
    assert rows.max() <= 4e-2, rows.max()
    assert err["done"] == 0


# ---- refresh -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
def test_refresh_restages_every_input(precision):
    """After a passing comparison the model changes in place: every weight and bias, the elite order (same count), the
    normaliser tensors (replaced), the logvar bounds.  push_weights re-stages it through b200pets_model_refresh (the
    handle stays); the kernels must then match a checker built from the new model, and no longer the old one."""
    spec = syn.CASES["halfcheetah_small"]
    arrays = syn.make_model_arrays(spec)
    model, env = make_env(spec, arrays, precision)
    inp = syn.make_rollout_inputs(spec)
    bf16 = precision == "bf16_tc"

    def compare(ck):
        nobs, rew, done, assign, _ = run_trajectory(env, spec, inp, "shuffle", "one")
        return check_trajectory(spec, ck, inp, nobs, rew, done, assign, bf16, "shuffle")

    old = TransitionF64.from_model(spec, model)
    assert_within(compare(old), precision)
    handle = env.staged.handle.value
    g = torch.Generator(device=DEV).manual_seed(3)
    mlp = model.model
    with torch.no_grad():
        for layer in [s[0] for s in mlp.hidden_layers] + [mlp.mean_and_logvar]:
            layer.weight.add_(0.05 * torch.randn(layer.weight.shape, device=DEV, generator=g) * layer.weight.std())
            layer.bias.add_(0.05 * torch.randn(layer.bias.shape, device=DEV, generator=g))
        mlp.min_logvar.add_(-0.5)
        mlp.max_logvar.add_(-0.25)
    model.set_elite([6, 5, 3, 2, 0])
    norm = model.input_normalizer
    norm.mean = norm.mean + 0.1 * torch.randn(norm.mean.shape, device=DEV, generator=g, dtype=norm.mean.dtype)
    norm.std = norm.std * (1.0 + 0.1 * torch.rand(norm.std.shape, device=DEV, generator=g, dtype=norm.std.dtype))
    env.push_weights()
    assert env.staged.handle.value == handle  # re-staged in place, not re-created
    new = TransitionF64.from_model(spec, model)
    assert new.members == [6, 5, 3, 2, 0]
    assert_within(compare(new), precision)
    stale = compare(old)
    assert stale["next_obs"] > 10 * BAR[precision], stale


# ---- negative controls -----------------------------------------------------------------------------------------
def _control_error(kind, precision):
    """Worst next_obs error against a checker with one deliberate error."""
    if kind == "slope":
        err, (spec, model, env, inp, nobs, rew, done, assign) = option_errors("leaky_slope_0.2", precision)
        assert_within(err, precision)
        ck = TransitionF64.from_model(spec, model)
        ck.slope = 0.01
    elif kind == "no_delta":
        err, (spec, model, env, inp, nobs, rew, done, assign) = option_errors("no_delta_learned", precision)
        assert_within(err, precision)
        ck = TransitionF64.from_model(spec, model)
        ck.no_delta = []
    else:
        err, (spec, model, env, inp, nobs, rew, done, assign) = trajectory_errors(
            "halfcheetah_small", precision, "shuffle", "one")
        assert_within(err, precision)
        ck = TransitionF64.from_model(spec, model)
    mode = "shuffle"  # every control case draws its members in the kernel
    eps = inp.get("eps")
    if kind == "member":
        assign = (assign + 1) % spec.num_models
    if kind == "eps":
        eps = np.roll(eps, 1, axis=-1)
    bad = check_trajectory(spec, ck, inp, nobs, rew, done, assign, precision == "bf16_tc", mode, eps=eps)
    return max(bad["next_obs"], bad["reward"])


@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
@pytest.mark.parametrize("kind", ["slope", "no_delta", "member", "eps"])
def test_negative_controls_fail_the_bar(kind, precision):
    e = _control_error(kind, precision)
    print(f"{kind}: {e:.2e} against bar {BAR[precision]:.0e}")
    assert e > BAR[precision], e
