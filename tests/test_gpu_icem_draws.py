"""iCEM's in-kernel draws by counter, and the fused iCEM plan (``b200pets_icem_plan``) against float64 with those draws.

The fused plan always draws its coloured noise and its kept elites' fresh last action in the kernel.  Here:

1. Known answers: ``b200pets_icem_sample`` with ``sr = si = NULL`` and ``b200pets_icem_append_elites`` with
   ``shift = 1, end_eps = NULL`` against a numpy restatement of the two Philox streams (cem.cu icem_noise_element and
   icem_append_element, common.cuh rng_key), at three seeds, the offsets ``c * 1024 + i`` both plan paths form and an
   offset above 2^32 whose counter word equals a smaller one's (only the key tells them apart); H 2, 3, 8, 41 and
   A 1, 5, 17, at populations whose element counts end on, or one or two elements past, a thread-block edge.
   Negative controls (offset + 1, the other stream word, the sequence or kept row off by one, the noise word with
   k and ad swapped, the key without the offset's high word, the source elite as the counter) must miss the bar by
   orders of magnitude.
2. The fused plan over the model against the per-iteration loop, bit for bit over three consecutive calls, and
   against oracle/pets_oracle.py icem_optimize in float64, driven by the restated draws of every iteration, the
   kept-elite permutations the host drew (replayed from the saved torch generator state) and the recorded values:
   pets_icem_cartpole's shapes and bench config 3's humanoid_trunc on the fp32 and the tensor-core rollout.
3. The single-CTA refit's limits (at most 2 048 rows, an elite set of at most 150 KB, at least 2 elites), with a case
   on each side of each.  Every case asserts its branch twice: from the limits, and from the kernels the plan launched.
   The branch is chosen once per plan, from the workspace's largest population: sizes[i] + max(keep, 1) over the
   iterations (api.cu icem_layout), whether or not elites are carried in.  So a first call (no kept elites) and the
   calls after it always take the same branch: a plan whose first population fits 2 048 rows but whose kept elites
   take it past them runs the chain in every call, the first included, as call_1_above_2048_rows asserts.
4. Coloured noise at horizons 64 to 150 (up to 76 frequencies), with injected and with in-kernel normals.

Bars (stated; the measured maxima are printed with -s):
  * coloured noise: |got - ref| <= 1e-5 * sqrt(var) * max(1, |y|), test_gpu_optimizers' bar, with injected normals;
  * in-kernel draws are held to the same bars beyond a per-draw slack.  The restatement rounds u as the kernel's
    u32_to_unit does ((float)(x >> 8) + 0.5f rounds to even in fp32 from 2^23 up, and the top word gives u = 1,
    radius 0), so what remains is the logarithm: the kernel's Box-Muller radius is sqrt(-2 __logf(u)), and CUDA bounds
    __logf's absolute error by 2^-21.41, so a draw of radius r may be off by 2 * 2^-21.41 / r (and never by more than
    sqrt(2 * 2^-21.41)).  This matters only for u within ~1e-5 of 1: on an H100, 6 of 5.1 million draws have
    r < 1e-3, and the worst of them is off by 1.3e-4 (|dz| * r stays at 8e-8 there).  A series gets the slack of its
    K draws, weighted as they enter y;
  * end action: the draw recovered from it, (v - mu) / sqrt(var), within 1e-4 * max(1, |e|) of the restated normal
    (test_gpu_cem_kernels' Philox known-answer bar, for the fast log and sincos intrinsics).  The shifted rows must be
    bit-equal;
  * plans: fused plan and loop bit-equal; every population, the elite set in order and the solution within
    2e-5 * max(1, max|ref|) of the oracle (run_icem_against_oracle's bar), beyond a first-order bound of what the
    draws' slack can move them by (_DrivenDraws);
  * negative controls: more than 1 000 times the bar, or NaN.  Every error measure keeps a NaN, so an element a
    kernel never writes (the tests fill outputs with NaN) fails its bar.
Tied values are common where a population has about 2 000 sequences of a short horizon: the H 4 cases below meet a
few per plan (2 to 6 so far).  The oracle gets them ranked by index, as the kernels rank them (torch.topk states no
order), so that the elite set's order, and with it which rows the kept-elite permutation picks, is defined.
Measured maxima on an H100 80GB HBM3 (700 W limit), in the units of each bar: in-kernel coloured noise 1.4e-6 beyond
the slack (H 2 to 41) and 1.5e-7 (H 64 to 150); injected coloured noise at H 64 to 150 1.2e-6, so the 1e-5 bar holds
there too (the error grows with the number of frequencies summed: 8.6e-7 at H <= 41); end action 1.4e-6; plans 7.1e-7
beyond their allowance, which reached 1.8e-4; negative controls 2.6 to 4.8, and NaN for the unwritten elements.
"""
import dataclasses
import re

import numpy as np
import pytest
import torch

from mbrl_lib_b200 import synthetic as syn
from test_gpu_cem_kernels import ELITE_SMEM_BYTES, K_SMALL_N, philox4x32_10
from test_gpu_icem_plan import _cartpole_env, _optimizer
from test_gpu_optimizers import _Driven, _dev, _icem_sample, _report, colored64
from test_gpu_parity import DEV, _Env, make_env

pytestmark = pytest.mark.gpu

RNG_STREAM_ICEM = 0x40000  # common.cuh
M32 = 0xFFFFFFFF
NOISE_BAR, DRAW_BAR, PLAN_BAR = 1e-5, 1e-4, 2e-5
OPT_SEED = 0x5DEECE66D


# ---- numpy restatement of the two iCEM streams ---------------------------------------------------------------------
def rng_key(seed, offset):
    """common.cuh rng_key: the offset's low word goes into a counter word, its high word into the key."""
    return (seed ^ (offset & 0xFFFFFFFF00000000)) & 0xFFFFFFFFFFFFFFFF


def _unit(x):
    """common.cuh u32_to_unit: (float)(x >> 8) + 0.5f rounds in fp32, to even from x >> 8 = 2^23 up (the top word gives
    exactly 1, whose radius is 0); the scale by 2^-24 is exact."""
    return ((x >> np.uint64(8)).astype(np.float32) + np.float32(0.5)).astype(np.float64) / 16777216.0


def philox_normal4_f32u(c0, c1, c2, c3, key):
    """common.cuh philox_normal4: two Box-Muller pairs from the four words of one block, u rounded as the kernel rounds
    it and the rest in float64.  Returns the four lanes and the two radii's u (lanes 0, 1 and lanes 2, 3)."""
    u = [_unit(x) for x in philox4x32_10(c0, c1, c2, c3, key & M32, key >> 32)]
    r0, r1 = np.sqrt(-2.0 * np.log(u[0])), np.sqrt(-2.0 * np.log(u[2]))
    a0, a1 = 2.0 * np.pi * u[1], 2.0 * np.pi * u[3]
    return np.stack([r0 * np.cos(a0), r0 * np.sin(a0), r1 * np.cos(a1), r1 * np.sin(a1)]), (u[0], u[2])


def icem_normals(n, H, A, seed, offset, stream=0, first=0, swap_word=False, key=None, radii=False):
    """sr, si [n, A, K] as icem_noise_element draws them: lanes 0 and 1 of the Philox block at counter (sequence,
    ad * K + k, RNG_STREAM_ICEM, low word of offset) under rng_key(seed, offset).  The other arguments build the
    negative controls; with `radii` the u of each pair's radius follows."""
    K = H // 2 + 1
    ni = (first + np.arange(n))[:, None, None]
    ad, k = np.arange(A)[None, :, None], np.arange(K)[None, None, :]
    word = k * A + ad if swap_word else ad * K + k
    g, (u0, _) = philox_normal4_f32u(ni, word, RNG_STREAM_ICEM | stream, offset & M32,
                                     rng_key(seed, offset) if key is None else key)
    return (g[0], g[1], u0) if radii else (g[0], g[1])


def icem_end_eps(rows, A, seed, offset, stream=1, key=None, radii=False):
    """e [len(rows), A] as icem_append_element draws the fresh last action of kept row j: lane ad & 3 of the Philox
    block at counter (j, ad >> 2, RNG_STREAM_ICEM | 1, low word of offset) under rng_key(seed, offset).  `rows` are the
    counters (np.arange(keep) for the kernel's layout); with `radii` the u of each draw's radius follows."""
    j = np.asarray(rows)[:, None]
    ad = np.arange(A)[None, :]
    g, (u0, u2) = philox_normal4_f32u(j, ad >> 2, RNG_STREAM_ICEM | stream, offset & M32,
                                      rng_key(seed, offset) if key is None else key)
    e = np.take_along_axis(g, np.broadcast_to(ad & 3, g.shape[1:])[None], axis=0)[0]
    return (e, np.where((ad & 3) < 2, u0, u2)) if radii else e


# ---- what the kernel's fast logarithm allows ---------------------------------------------------------------------
# The kernel's Box-Muller radius is sqrt(-2 __logf(u)).  The restatement rounds u exactly as the kernel does, but takes
# the logarithm in float64.  CUDA bounds |__logf(u) - log(u)| by 2^-21.41 on [0.5, 2], so r^2 is off by up to twice that
# and r by up to 2 * 2^-21.41 / r, and by no more than sqrt(2 * 2^-21.41) however small r is: a draw whose u is within
# ~1e-6 of 1 (radius ~1e-3) may be off by ~1e-4 however right its counter.  On an H100 |dz| * r stays at 8e-8 down to
# r = 5e-4 (|dz| 1.3e-4 there).  The bars below are met beyond this per-draw slack; a wrong counter moves a draw by
# order 1.
LOGF_ERR = 2.0 ** -21.41


def radius_slack(u):
    r = np.sqrt(np.abs(-2.0 * np.log(u)))  # u = 1 gives -0.0
    with np.errstate(divide="ignore"):  # u = 1: r = 0, the cap applies
        return np.minimum(2.0 * LOGF_ERR / r, np.sqrt(2.0 * LOGF_ERR))


def _spectrum(H, exponent):
    """colored64's spectrum scale s_k and sigma."""
    K = H // 2 + 1
    s = (np.maximum(np.arange(K, dtype=np.float64), 1.0) / H) ** (-exponent / 2.0)
    w = s[1:].copy()
    w[-1] *= (1 + H % 2) / 2.0
    return s, 2.0 * np.sqrt(np.sum(w ** 2)) / H


def icem_noise_slack(n, H, A, seed, offset, exponent):
    """[n, A]: how far the radius slack of its K draws may move every sample of series (sequence, ad).  A radius error
    dr moves zr cos - zi sin by at most dr, and frequency k enters y with weight c_k s_k / (H sigma)."""
    K = H // 2 + 1
    u0 = icem_normals(n, H, A, seed, offset, radii=True)[2]
    s, sigma = _spectrum(H, exponent)
    c = np.full(K, 2.0)
    c[0] = 1.0
    if H % 2 == 0:
        c[-1] = 1.0
    return (radius_slack(u0) * c * s).sum(-1) / H / sigma


def icem_end_slack(keep, A, seed, offset):
    """[keep, A]: the radius slack of the end draws."""
    return radius_slack(icem_end_eps(np.arange(keep), A, seed, offset, radii=True)[1])


# seeds with zero, mixed and all-ones key words; offsets c * 1024 + i of a plan's iterations, and one above 2^32 whose
# counter word is that of 1024 + 2
SEEDS = [0, 0x123456789ABCDEF0, 0xFFFFFFFFFFFFFFFF]
OFFSETS = [1024 + i for i in range(5)] + [7 * 1024 + 4, (1 << 32) + 1024 + 2]


def _edge_rows(per_row, block):
    """One row, and the first two row counts whose rows * per_row elements end one short of, on, or one or two
    past a `block`-thread block edge."""
    out = [1]
    for n in range(1, block + 1):
        if n * per_row >= block - 1 and (n * per_row) % block in (block - 1, 0, 1, 2):
            out.append(n)
            if len(out) == 3:
                break
    return out


def _worst(*errs):
    """The largest error, NaN if any is NaN (Python's max drops a NaN that is not first)."""
    return float(np.max(errs))


def _mu_var(g, H, A):
    return g.uniform(-0.5, 0.5, (H, A)).astype(np.float32), g.uniform(0.2, 2.0, (H, A)).astype(np.float32)


def _noise_error(got, mu, var, sr, si, H, exponent, slack=None):
    """got [n, H, A] against the float64 coloured noise of sr, si [n, A, K], in units of sqrt(var) * max(1, |y|),
    beyond the per-series slack [n, A] of in-kernel draws."""
    y = colored64(sr, si, H, exponent).transpose(0, 2, 1)
    ref = y * np.sqrt(var.astype(np.float64)) + mu
    dev = np.abs(got - ref) / np.sqrt(var) - (0.0 if slack is None else slack[:, None, :])
    return float(np.maximum(dev / np.maximum(1.0, np.abs(y)), 0.0).max())  # NaN (an unwritten element) stays NaN


def _drawn_error(got, mu, var, n, H, A, exponent, seed, offset):
    """In-kernel coloured noise against the restatement, beyond the slack of its draws."""
    return _noise_error(got, mu, var, *icem_normals(n, H, A, seed, offset), H, exponent,
                        icem_noise_slack(n, H, A, seed, offset, exponent))


def _sample_drawn(n, H, A, exponent, mu, var, seed, offset):
    wide = np.full((H, A), 1e30, np.float32)
    return _icem_sample(n, H, A, exponent, mu, var, -wide, wide, seed=seed, offset=offset).astype(np.float64)


def _append_drawn(elite, index, mu, var, seed, offset):
    """b200pets_icem_append_elites with shift 1 and in-kernel end draws: the kept rows [keep, H, A]."""
    from mbrl_lib_b200 import _lib

    lib = _lib.load()
    keep, (_, H, A) = len(index), elite.shape
    dst = torch.full((keep + 1, H, A), -12345.0, device=DEV)  # the row past `keep` must stay untouched
    e_d, i_d, m_d, v_d = _dev(elite, index, mu, var)
    _lib.check(lib.b200pets_icem_append_elites(keep, H, A, _lib.ptr(e_d), _lib.ptr(i_d), 1, _lib.ptr(m_d), _lib.ptr(v_d), None,
                                               seed, offset, _lib.ptr(dst), _lib.stream_ptr()), "icem_append_elites")
    got = dst.cpu().numpy()
    assert (got[keep:] == -12345.0).all()
    assert np.array_equal(got[:keep, :-1].view(np.int32), elite[index][:, 1:].view(np.int32))
    return got[:keep]


def _end_error(got, mu, var, e_ref, slack):
    """The draws recovered from the kept rows' last action against e_ref [keep, A], in units of max(1, |e_ref|), beyond
    the radius slack of the right draws."""
    e = (got[:, -1].astype(np.float64) - mu[-1]) / np.sqrt(var[-1].astype(np.float64))
    return float(np.maximum((np.abs(e - e_ref) - slack) / np.maximum(1.0, np.abs(e_ref)), 0.0).max())  # NaN stays NaN


# ---- known answers of the in-kernel draws --------------------------------------------------------------------------
@pytest.mark.parametrize("H", [2, 3, 8, 41])
def test_icem_sample_draws_follow_the_counter_layout(H):
    """icem_sample_kernel (128-thread blocks) with in-kernel normals equals colored64 of the restated normals."""
    g = np.random.default_rng(H)
    worst, launches = 0.0, 0
    for A in (1, 5, 17):
        mu, var = _mu_var(g, H, A)
        for n in _edge_rows(H * A, 128):
            for seed in SEEDS:
                for offset in OFFSETS:
                    got = _sample_drawn(n, H, A, 2.0, mu, var, seed, offset)
                    worst = _worst(worst, _drawn_error(got, mu, var, n, H, A, 2.0, seed, offset))
                    launches += 1
    _report(f"icem_sample in-kernel normals H {H} ({launches} launches)", worst, NOISE_BAR)


@pytest.mark.parametrize("H", [2, 3, 8, 41])
def test_icem_append_end_draws_follow_the_counter_layout(H):
    """icem_append_kernel (256-thread blocks) with shift 1 and in-kernel end draws: the fresh last action of kept row j
    is drawn at counter j, whatever elite row the permutation puts there."""
    g = np.random.default_rng(100 + H)
    worst, launches = 0.0, 0
    for A in (1, 5, 17):
        mu, var = _mu_var(g, H, A)
        for keep in _edge_rows(H * A, 256):
            elite = g.standard_normal((keep + 3, H, A)).astype(np.float32)
            index = g.permutation(keep + 3)[:keep].astype(np.int64)
            for seed in SEEDS:
                for offset in OFFSETS:
                    got = _append_drawn(elite, index, mu, var, seed, offset)
                    worst = _worst(worst, _end_error(got, mu, var, icem_end_eps(np.arange(keep), A, seed, offset),
                                                  icem_end_slack(keep, A, seed, offset)))
                    launches += 1
    _report(f"icem_append in-kernel end action H {H} ({launches} launches, units of max(1, |e|))", worst, DRAW_BAR)


CONTROL_SEED, CONTROL_OFFSET = 0x123456789ABCDEF0, (3 << 32) + 1024 + 1  # the offset's high word keys the draws
NOISE_CONTROLS = {
    "offset + 1": dict(offset=CONTROL_OFFSET + 1),
    "other stream word": dict(stream=1),
    "sequence off by one": dict(first=1),
    "word k * A + ad": dict(swap_word=True),
    "key without the offset's high word": dict(key=CONTROL_SEED),
    "last element unwritten (NaN)": dict(unwritten=True),
}
END_CONTROLS = {
    "offset + 1": dict(offset=CONTROL_OFFSET + 1),
    "other stream word": dict(stream=0),
    "kept row off by one": dict(rows=1),
    "source elite as the counter": dict(rows="index"),
    "key without the offset's high word": dict(key=CONTROL_SEED),
    "last end action unwritten (NaN)": dict(unwritten=True),
}


def _fails(err, bar):
    """A control's error misses the bar by more than 1 000 times, or is NaN (which no `err <= bar` passes)."""
    return not err <= 1e3 * bar


@pytest.mark.parametrize("kind", list(NOISE_CONTROLS))
def test_noise_negative_controls_fail_the_bar(kind):
    H, A, n = 8, 5, 26  # 1 040 elements: one past the eighth 128-thread block
    g = np.random.default_rng(7)
    mu, var = _mu_var(g, H, A)
    got = _sample_drawn(n, H, A, 2.0, mu, var, CONTROL_SEED, CONTROL_OFFSET)
    slack = icem_noise_slack(n, H, A, CONTROL_SEED, CONTROL_OFFSET, 2.0)
    right = _noise_error(got, mu, var, *icem_normals(n, H, A, CONTROL_SEED, CONTROL_OFFSET), H, 2.0, slack)
    assert right <= NOISE_BAR
    kw = dict(NOISE_CONTROLS[kind])
    offset = kw.pop("offset", CONTROL_OFFSET)
    if kw.pop("unwritten", False):  # an element the kernel never wrote keeps _icem_sample's NaN fill
        got = got.copy()
        got[-1, -1, -1] = np.nan
    # accumulated after a passing launch, as the known-answer tests accumulate
    err = _worst(right, _noise_error(got, mu, var, *icem_normals(n, H, A, CONTROL_SEED, offset, **kw), H, 2.0, slack))
    print(f"coloured noise control '{kind}': {err:.2e} against bar {NOISE_BAR:.0e}")
    assert _fails(err, NOISE_BAR), err


@pytest.mark.parametrize("kind", list(END_CONTROLS))
def test_end_action_negative_controls_fail_the_bar(kind):
    H, A, keep = 8, 5, 30
    g = np.random.default_rng(8)
    mu, var = _mu_var(g, H, A)
    elite = g.standard_normal((50, H, A)).astype(np.float32)
    index = g.permutation(50)[:keep].astype(np.int64)
    got = _append_drawn(elite, index, mu, var, CONTROL_SEED, CONTROL_OFFSET)
    slack = icem_end_slack(keep, A, CONTROL_SEED, CONTROL_OFFSET)
    right = _end_error(got, mu, var, icem_end_eps(np.arange(keep), A, CONTROL_SEED, CONTROL_OFFSET), slack)
    assert right <= DRAW_BAR
    kw = dict(END_CONTROLS[kind])
    offset, rows = kw.pop("offset", CONTROL_OFFSET), kw.pop("rows", 0)
    rows = index if isinstance(rows, str) else np.arange(keep) + rows
    if kw.pop("unwritten", False):
        got = got.copy()
        got[-1, -1, -1] = np.nan
    err = _worst(right, _end_error(got, mu, var, icem_end_eps(rows, A, CONTROL_SEED, offset, **kw), slack))
    print(f"end action control '{kind}': {err:.2e} against bar {DRAW_BAR:.0e}")
    assert _fails(err, DRAW_BAR), err


# ---- long horizons -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [64, 100, 101, 150])
def test_long_horizon_coloured_noise_matches_float64(H):
    """The fp32 sum over up to 76 frequencies (one thread per element) against float64, injected and in-kernel."""
    g = np.random.default_rng(H)
    K = H // 2 + 1
    injected = drawn = 0.0
    for A, n in [(1, 129), (5, 26), (17, 8)]:
        mu, var = _mu_var(g, H, A)
        wide = np.full((H, A), 1e30, np.float32)
        for exponent in (0.0, 1.0, 2.0, 2.5, 4.0):
            sr, si = (g.standard_normal((n, A, K)).astype(np.float32) for _ in range(2))
            got = _icem_sample(n, H, A, exponent, mu, var, -wide, wide, sr, si).astype(np.float64)
            injected = _worst(injected, _noise_error(got, mu, var, sr, si, H, exponent))
        for seed, offset in zip(SEEDS, (1024, 7 * 1024 + 4, OFFSETS[-1])):
            for exponent in (0.0, 2.0):
                got = _sample_drawn(n, H, A, exponent, mu, var, seed, offset)
                drawn = _worst(drawn, _drawn_error(got, mu, var, n, H, A, exponent, seed, offset))
    _report(f"icem_sample H {H}, injected normals", injected, NOISE_BAR)
    _report(f"icem_sample H {H}, in-kernel normals", drawn, NOISE_BAR)


# ---- the fused plan against the loop and the float64 oracle --------------------------------------------------------
def refit_single_cta(opt, H, A):
    """Whether b200pets_icem_plan refits in icem_refit_sample_kernel (api.cu, cem_refit_sample_supported of the workspace's
    largest population: the first population plus the kept elites, or plus the mean's row when none are kept)."""
    rows = max(opt.population_sizes()) + max(min(opt.keep_elite_size, opt.elite_num), 1)
    return rows <= K_SMALL_N and opt.elite_num * H * A * 4 <= ELITE_SMEM_BYTES and opt.elite_num >= 2


def _fused_call(opt, obj, x0):
    """One fused plan under torch.profiler: the solution and the names of the kernels it launched."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        sol = opt.optimize(obj, x0=x0).clone()
        torch.cuda.synchronize()
    return sol, [e.key for e in prof.key_averages()]


def _oracle_noise(opt, H, A, keep_index, carried):
    """The draws of the call the optimiser just made, for icem_optimize: the restated sr / si of iteration i at offset
    c * 1024 + i, the kept elites' permutation the host drew and the restated end draws of the first iteration.  Also
    returns each iteration's coloured noise y [n_i, H, A] and series slack [n_i, A], and the end draws' slack [keep, A]
    (None without carried elites)."""
    f64 = lambda a: torch.from_numpy(np.asarray(a, np.float64))  # noqa: E731
    base, keep, beta = opt._offset * 1024, min(opt.keep_elite_size, opt.elite_num), opt.colored_noise_exponent
    noise, ys, slack, end_slack = [], [], [], None
    for i, n in enumerate(opt.population_sizes()):
        sr, si = icem_normals(n, H, A, opt._seed, base + i)
        d = {"sr": f64(sr), "si": f64(si)}
        ys.append(colored64(sr, si, H, beta).transpose(0, 2, 1))
        slack.append(icem_noise_slack(n, H, A, opt._seed, base + i, beta))
        if carried or i > 0:  # icem_optimize indexes the elites whenever it has any; the last iteration ignores them
            d["keep_perm"] = torch.zeros(0, dtype=torch.int64) if keep_index is None else keep_index[i]
            if i == 0:
                d["end_eps"] = f64(icem_end_eps(np.arange(keep), A, opt._seed, base))
                end_slack = icem_end_slack(keep, A, opt._seed, base)
        noise.append(d)
    return noise, ys, slack, end_slack


def ties_by_index(v):
    """v in float64, each run of equal values made strictly decreasing in index order: the refit kernels rank ties by
    ascending index, torch.topk in no stated order.  Every value moves by less than half the smallest gap between two
    distinct values, so no other order changes."""
    v = np.asarray(v, np.float64)
    u = np.unique(v)
    gap = float(np.diff(u).min()) if u.size > 1 else 1.0
    return v - np.arange(v.size) * (gap / (2.0 * v.size))


class _DrivenDraws(_Driven):
    """_Driven for in-kernel draws.  A population element may differ from the oracle's by the bar plus its allowance:
    a first-order bound, element by element, of how far the draws' slack can move it.
      * a coloured-noise sample mu + sqrt(var) * y: dmu + |y| * dsd plus its series' slack times sqrt(var);
      * a kept elite: its elite's allowance (shifted one step in the first iteration, whose fresh last action adds
        its draw's slack times sqrt(var)); the mean's row: dmu;
      * the refit: mu = alpha mu + (1 - alpha) mean(e) gives dmu' = alpha dmu + (1 - alpha) mean(de), and
        var = alpha var + (1 - alpha) mean((e - m)^2) gives dvar' = alpha dvar + 2 (1 - alpha) mean(|e - m| de),
        dsd = dvar / (2 sqrt(var)), over the oracle's elites e with their allowances de.
    Every call starts from x0 and the initial variance, so dmu = dvar = 0 there; only kept elites bring an allowance
    from the call before.  Clipping to the bounds moves no two values further apart.  Tied values reach the oracle
    broken by index, as the kernels break them."""

    def __init__(self, gpu_obj, var0, alpha, ys, slack, end_slack, keep_perm, prev_allow):
        super().__init__(gpu_obj)
        self.var0, self.alpha, self.ys, self.slack, self.end_slack = var0.numpy(), alpha, ys, slack, end_slack
        self.keep_perm, self.prev_allow, self.otrace = keep_perm, prev_allow, []
        self.dmu = self.dvar = np.zeros_like(self.var0)
        self.allow = self.elite_allow = self.best_allow = None
        self.best, self.largest, self.ties = -np.inf, 0.0, 0

    def absorb(self, i):
        """Iteration i's refit, on the oracle's elites and their allowances."""
        t = self.otrace[i]
        idx = t["elite_idx"].numpy()
        e, de = t["pop"].numpy()[idx], self.allow[idx]
        self.dmu = self.alpha * self.dmu + (1 - self.alpha) * de.mean(0)
        self.dvar = self.alpha * self.dvar + 2 * (1 - self.alpha) * (np.abs(e - e.mean(0)) * de).mean(0)
        self.elite_allow = de
        if float(t["values"][idx[0]]) > self.best:  # the oracle's best solution is this row
            self.best, self.best_allow = float(t["values"][idx[0]]), de[0]

    def oracle(self, pop, i):
        if i > 0:
            self.absorb(i - 1)
        got, ref = self.trace[i][0], pop.numpy()
        var = self.var0 if i == 0 else self.otrace[i - 1]["var"].numpy()
        sd = np.sqrt(var)
        dsd = self.dvar / (2 * sd)
        n = self.slack[i].shape[0]
        allow = np.empty(ref.shape)
        allow[:n] = self.dmu + np.abs(self.ys[i]) * dsd + sd * self.slack[i][:, None, :]
        if ref.shape[0] > n:
            if i == 0:  # the carried elites, shifted, with a fresh last action (dmu = dsd = 0 here)
                kept = self.prev_allow[self.keep_perm[0]]
                allow[n:, :-1] = kept[:, 1:]
                allow[n:, -1] = sd[-1] * self.end_slack
            elif i == len(self.slack) - 1:
                allow[n:] = self.dmu
            else:
                allow[n:] = self.elite_allow[self.keep_perm[i]]
        self.allow = allow
        self.largest = max(self.largest, float(allow.max()))
        self.worst = _worst(self.worst, self.excess(got, ref, allow, f"population {i}"))
        v = self.trace[i][1]
        self.ties += v.size - np.unique(v).size
        return torch.from_numpy(ties_by_index(v))

    def finish(self, return_mean_elites):
        """After the last iteration: the allowances of the elite set, in order, and of the solution."""
        self.absorb(len(self.slack) - 1)
        return self.elite_allow, self.dmu if return_mean_elites else self.best_allow

    @staticmethod
    def excess(got, ref, allow, what):
        """max(|got - ref| - allow) over max(1, max|ref|), held to PLAN_BAR."""
        got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
        assert got.shape == ref.shape, (what, got.shape, ref.shape)
        err = float(np.maximum(np.abs(got - ref) - allow, 0.0).max()) / max(1.0, float(np.abs(ref).max()))  # NaN stays NaN
        assert err <= PLAN_BAR, f"{what}: {err:.3e} > {PLAN_BAR:.0e} beyond its allowance"
        return err


def plan_against_loop_and_oracle(spec, env, fused, loop, P, seed, calls=3):
    """test_gpu_icem_plan.compare_plans over `calls` consecutive calls, plus icem_optimize in float64 on the loop's
    recorded values.  Returns the largest deviation from the oracle beyond its allowance, the largest allowance, the
    number of tied values and the kernels each fused call launched."""
    from mbrl_lib_b200.planning import _FusedObjective
    from oracle import pets_oracle as po

    H, A = fused.lower_bound.shape
    obj = _FusedObjective(env, syn.make_rollout_inputs(spec, with_noise=False)["obs0"], P)
    lb, ub = (torch.from_numpy(b.cpu().numpy().astype(np.float64)) for b in (fused.lower_bound, fused.upper_bound))
    g = np.random.default_rng(seed)
    env._offset = 40
    o_elite, prev_allow, worst, largest, ties, launched = None, None, 0.0, 0.0, 0, []
    for call in range(calls):
        x0 = torch.from_numpy(g.uniform(-0.3, 0.3, (H, A)).astype(np.float32)).to(DEV)
        rng, offset, carried = torch.cuda.get_rng_state(), env._offset, fused.elite is not None
        _, keep_index, _ = fused._fused_draws(env, env._propagation(), H, P)  # the host's draws of this call
        keep_index = None if keep_index is None else keep_index.cpu()
        torch.cuda.set_rng_state(rng)
        sol, kernels = _fused_call(fused, obj, x0)
        launched.append(kernels)
        got_values = [v.clone() for v in fused.last_values]
        after = (torch.cuda.get_rng_state(), env._offset)
        torch.cuda.set_rng_state(rng)
        env._offset = offset
        noise, ys, slack, end_slack = _oracle_noise(fused, H, A, keep_index, carried)
        keep = min(fused.keep_elite_size, fused.elite_num)
        perms = [d["keep_perm"][:keep].numpy() if "keep_perm" in d else None for d in noise]
        drv = _DrivenDraws(lambda seqs: obj(seqs), (ub - lb) ** 2 / 16, fused.alpha, ys, slack, end_slack, perms,
                           prev_allow)  # opaque to the optimiser: the loop
        ref = loop.optimize(drv.gpu, x0=x0).clone()
        torch.cuda.synchronize()
        assert env._offset == after[1] == offset + fused.num_iterations, f"call {call}: environment counter"
        assert fused._offset == loop._offset == call + 1, f"call {call}: optimiser counter"
        assert torch.equal(after[0], torch.cuda.get_rng_state()), f"call {call}: torch generator state"
        assert len(got_values) == len(loop.last_values) == fused.num_iterations
        for i, (v, r) in enumerate(zip(got_values, loop.last_values)):
            assert v.shape == r.shape and torch.equal(v, r), f"call {call}: values of iteration {i} differ"
        assert torch.equal(fused.elite, loop.elite), f"call {call}: elite sets differ"
        assert torch.equal(sol, ref), f"call {call}: solutions differ"
        o_sol, o_elite = po.icem_optimize(
            drv.oracle, torch.from_numpy(x0.cpu().numpy().astype(np.float64)), lb, ub, fused.num_iterations, fused.elite_ratio,
            fused.population_size, fused.population_decay_factor, fused.colored_noise_exponent, fused.keep_elite_frac,
            fused.alpha, noise, prev_elite=o_elite, return_mean_elites=fused.return_mean_elites,
            module=fused.population_size_module, trace=drv.otrace)
        assert len(drv.trace) == len(drv.otrace) == fused.num_iterations
        prev_allow, sol_allow = drv.finish(fused.return_mean_elites)
        largest, ties = max(largest, drv.largest), ties + drv.ties
        worst = _worst(worst, drv.worst,
                       drv.excess(fused.elite.cpu().numpy(), o_elite.numpy(), prev_allow, f"call {call} elite set, in order"),
                       drv.excess(sol.cpu().numpy(), o_sol.numpy(), sol_allow, f"call {call} solution"))
    return worst, largest, ties, launched


def _ran(kernels, name):
    return any(re.search(rf"(^|\W){name}\(", k) for k in kernels)


def run_case(spec, env, H, pop, iters, module, keep_frac, rme, P, seed, single_cta=None):
    fused, loop = (_optimizer(spec, H, pop, iters, module, keep_frac, rme) for _ in range(2))
    fused._seed = loop._seed = OPT_SEED + seed  # torch.initial_seed() differs from process to process
    single = refit_single_cta(fused, H, spec.act_dim)
    if single_cta is not None:
        assert single == single_cta, "the case is off the edge of the single-CTA refit it was chosen for"
    worst, slack, ties, launched = plan_against_loop_and_oracle(spec, env, fused, loop, P, seed)
    for call, kernels in enumerate(launched):
        assert _ran(kernels, "icem_refit_sample_kernel") == single, (call, kernels)
        assert _ran(kernels, "icem_sample_kernel") != single, (call, kernels)
    rows = max(fused.population_sizes()) + max(min(fused.keep_elite_size, fused.elite_num), 1)
    print(f"elite_num {fused.elite_num}, keep {fused.keep_elite_size}, {rows} rows at most, elite set "
          f"{fused.elite_num * H * spec.act_dim * 4} B, {'single-CTA refit' if single else 'chain'}: fused = loop bit for bit, "
          f"max deviation from the float64 oracle {worst:.3e} of scale (bar {PLAN_BAR:.0e}) beyond its allowance "
          f"(at most {slack:.1e}); {ties} tied values")
    assert worst <= PLAN_BAR
    return fused


# name -> (model, precision, H, population, iterations, module, keep_elite_frac, return_mean_elites, particles)
ORACLE_PLANS = {
    "pets_icem_cartpole": ("cartpole", None, 10, 200, 5, 7, 0.3, True, 20),
    "config3_humanoid_trunc_f32": ("humanoid_trunc", "f32", 40, 1000, 5, 5, 0.3, True, 20),
    "config3_humanoid_trunc_tc": ("humanoid_trunc", "bf16_tc", 40, 1000, 5, 5, 0.3, True, 20),
}


@pytest.mark.parametrize("name", list(ORACLE_PLANS))
def test_fused_plan_matches_the_loop_and_float64(name):
    case, precision, H, pop, iters, module, keep_frac, rme, P = ORACLE_PLANS[name]
    if case == "cartpole":
        spec, env = _cartpole_env()
    else:
        spec, _, env = make_env(case, precision, ts1="tile_shuffle")
    run_case(spec, env, H, pop, iters, module, keep_frac, rme, P, seed=len(name))


def _env(spec):
    import mbrl_lib_b200 as bp
    from mbrl_lib_b200 import functions

    model = bp.model_from_arrays(spec, syn.make_model_arrays(spec), DEV)
    return bp.ModelEnv(_Env(spec), model, functions.TERM_FNS[spec.term_fn], None, generator=torch.Generator(device=DEV),
                       precision="f32", ts1="tile_shuffle")


# 24 action dims, learned reward: 40 elites of H 40 fill exactly 150 KB
WIDE = dataclasses.replace(syn.CASES["halfcheetah_small"], name="wide_actions", act_dim=24, learned_rewards=True, reward_fn=None)
# name -> (model, H, population, keep_elite_frac, return_mean_elites, (elite_num, kept elites, largest population),
#          single-CTA refit); 3 iterations, 5 particles, fp32.  The largest population is the first one plus the kept elites.
REFIT_EDGES = {
    "rows_2048": ("halfcheetah_small", 4, 1988, 0.3, True, (199, 60, 2048), True),
    "rows_2049": ("halfcheetah_small", 4, 1989, 0.3, False, (199, 60, 2049), False),
    # the first call evaluates 2 040 rows and the later ones 2 102: every call runs the chain (the module docstring)
    "call_1_above_2048_rows": ("halfcheetah_small", 4, 2040, 0.3, True, (204, 62, 2102), False),
    "elites_153600_B": (WIDE, 40, 400, 0.3, True, (40, 12, 412), True),  # 40 x 40 x 24 floats
    "elites_153600_B_plus_one_elite": (WIDE, 40, 410, 0.3, False, (41, 13, 423), False),  # 157 440 B
    "humanoid_56_elites": ("humanoid_trunc", 40, 560, 0.3, True, (56, 17, 577), True),  # 56 x 2 720 B = 152 320 B
    "humanoid_57_elites": ("humanoid_trunc", 40, 570, 0.3, False, (57, 18, 588), False),  # 155 040 B
    "one_elite": ("halfcheetah_small", 8, 10, 0.3, True, (1, 1, 11), False),
    "two_elites": ("halfcheetah_small", 8, 20, 0.3, False, (2, 1, 21), True),
    "keep_one": ("halfcheetah_small", 8, 200, 0.01, True, (20, 1, 201), True),
    "horizon_2": ("halfcheetah_small", 2, 100, 0.3, True, (10, 3, 103), True),  # DC and Nyquist only
}


@pytest.mark.parametrize("name", list(REFIT_EDGES))
def test_refit_edges_match_the_loop_and_float64(name):
    case, H, pop, keep_frac, rme, (elite_num, keep, rows), single = REFIT_EDGES[name]
    if isinstance(case, syn.CaseSpec):
        spec, env = case, _env(case)
    else:
        spec, _, env = make_env(case, "f32", ts1="tile_shuffle")
    opt = _optimizer(spec, H, pop, 3, None, keep_frac, rme)
    assert (opt.elite_num, opt.keep_elite_size, opt.population_sizes()[0] + opt.keep_elite_size) == (elite_num, keep, rows)
    run_case(spec, env, H, pop, 3, None, keep_frac, rme, 5, seed=len(name), single_cta=single)
