"""The CEM population kernels (csrc/cem.cu) called through the C ABI, against float64 restatements of the reference's
operations and against each other:

1. b200pets_cem_sample / _cem_sample_shard with injected normals against trajectory_opt.py:110-128 in float64, at
   one-block edges, the configurations' shapes and every dims % 4, with the variance, the lower or the upper constraint
   binding, the mean exactly on a bound or outside the bounds; shards at arbitrary first sequences.
2. The Philox draws of the sampler: the law (N(0, 1) truncated to [-2, 2] by redrawing, or plain N(0, 1)), independence
   across lanes, blocks, sequences, iterations, seeds and shards, and a known-answer check against a numpy
   Philox4x32-10 + Box-Muller at the counter layout the kernel documents.
3. The sharded records route (b200pets_cem_local_topk per shard -> concatenate -> b200pets_cem_update_from_records)
   against the float64 refit of the union and against b200pets_cem_update on the whole population, in every kernel
   run_select can pick for either call.
4. b200pets_cem_plan / _cem_plan_batch in both launch structures against the chain b200pets_cem_sample ->
   b200pets_eval_sequences -> b200pets_cem_update with the plan's (seed, offset) arithmetic, bit for bit.

Bars (stated; the measured maxima are printed with -s):
  * sampler, injected normals: |got - ref| <= 1e-6 * max(1, |ref|) (fp32: two subtractions, a square, a sqrt and a
    multiply-add on values of order 1), bit-equal where the restatement is exactly the mean or a bound;
  * Philox known answer: |got - ref| <= 1e-4 * max(1, |ref|) (the kernel's Box-Muller uses the fast log / sincos
    intrinsics, whose absolute error the radius near 0 amplifies; a wrong counter word moves a draw by order 1);
  * laws: KS p-value above 1e-6, correlations below 4 / sqrt(n), tail mass within 4 binomial sigma;
  * records route: mu / dispersion within rtol 1e-4, atol 1e-5 of the float64 refit; everything else exact; bit-equal
    to b200pets_cem_update whenever both land in the same kernel;
  * plans: values of every iteration and the solution bit-equal to the chain.
Measured maxima on an H100 80GB HBM3 (700 W limit), in the units of each bar: sampler 8.4e-8 (truncated) and 5.9e-8
(clipped); Philox known answer 7.9e-6 over 21 007 draws, 929 of them redrawn; smallest KS p-value 0.27 (per lane), 0.85
(pooled), 0.26 (clipped mode, 4.57 % of the draws beyond +-2); tail masses within 0.6 sigma; largest correlation 8.4e-3
(bar 2.8e-2).  The one case whose two routes run in different kernels (4 100 sequences, 2 elites: records in the
single-CTA kernel, whole population in the radix kernel) gave identical mu and dispersion as well.
"""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch
from scipy import stats

from mbrl_lib_b200 import dist as bd
from mbrl_lib_b200 import synthetic as syn
from test_gpu_parity import DEV, make_env

gpu = pytest.mark.gpu
GUARD = -12345.0
CEM_CU = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "mbrl-lib_b200", "csrc", "cem.cu")


def _abi():
    from mbrl_lib_b200 import _lib

    return _lib, _lib.load()


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _dev(*arrays):
    """Device copies of the arrays (None stays None), held by the caller until the kernel that reads them has run."""
    return [None if a is None else _t(a) for a in arrays]


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.int32)


def _report(what, err, bar):
    print(f"{what}: max deviation {err:.3e} of the bar's unit (bar {bar:.0e})")
    assert err <= bar, f"{what}: {err:.3e} > {bar:.0e}"


# ---- float64 restatements --------------------------------------------------------------------------------------------
def cem_sample64(z, mu, disp, lb, ub, clipped):
    """trajectory_opt.py:110-128 in float64: z [n, dims], the rest [dims].  Clipped mode takes the dispersion as a
    standard deviation and clips with the reference's two `where`s; truncated mode takes it as a variance and caps it by
    the squared half-distances to the bounds (squared as they are: a mean outside the bounds still gets a positive cap)."""
    z, mu, disp, lb, ub = (np.asarray(a, np.float64) for a in (z, mu, disp, lb, ub))
    if clipped:
        pop = mu + disp * z
        pop = np.where(pop > lb, pop, lb)
        return np.where(pop < ub, pop, ub)
    mv = np.minimum(((mu - lb) / 2) ** 2, ((ub - mu) / 2) ** 2)
    return z * np.sqrt(np.minimum(mv, disp)) + mu


M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 (Salmon et al. 2011) on arrays of counters; words travel in uint64 so that 32 x 32 products fit."""
    c0, c1, c2, c3 = np.broadcast_arrays(*(np.asarray(c, np.uint64) for c in (c0, c1, c2, c3)))
    k0, k1 = int(k0), int(k1)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c0, np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ np.uint64(k0), p1 & M32, (p0 >> np.uint64(32)) ^ c3 ^ np.uint64(k1), p0 & M32
        k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
    return c0, c1, c2, c3


def philox_normal4(c0, c1, c2, c3, key):
    """common.cuh philox_normal4 in float64: two Box-Muller pairs from the four words of one block."""
    r = philox4x32_10(c0, c1, c2, c3, key & 0xFFFFFFFF, key >> 32)
    u = [((x >> np.uint64(8)).astype(np.float64) + 0.5) / 16777216.0 for x in r]
    r0, r1 = np.sqrt(-2.0 * np.log(u[0])), np.sqrt(-2.0 * np.log(u[2]))
    a0, a1 = 2.0 * np.pi * u[1], 2.0 * np.pi * u[3]
    return np.stack([r0 * np.cos(a0), r0 * np.sin(a0), r1 * np.cos(a1), r1 * np.sin(a1)])


RNG_STREAM_CEM = 0x30000


def cem_draws64(n, dims, seed, offset, first=0, clipped=False):
    """The sampler's N(0, 1) draws as cem.cu documents them: element (sequence, d) is lane d & 3 of the Philox block at
    counter (global sequence, d >> 2, CEM stream | attempt, low word of offset) under key seed ^ (high word of offset);
    unless clipped, a draw outside [-2, 2] is redrawn with the next attempt number.  Also returns the elements one of
    whose attempts fell within 1e-3 of +-2, where fp32 and float64 may disagree on the redraw."""
    key = seed ^ (offset & 0xFFFFFFFF00000000)
    seq = (first + np.arange(n))[:, None]
    blk, lane = (np.arange(dims) >> 2)[None, :], np.broadcast_to(np.arange(dims) & 3, (n, dims))
    draw = lambda attempt: np.take_along_axis(  # noqa: E731
        philox_normal4(seq, blk, RNG_STREAM_CEM | attempt, offset & 0xFFFFFFFF, key), lane[None], axis=0)[0]
    z = draw(0)
    near = np.abs(np.abs(z) - 2.0) < 1e-3
    for attempt in range(1, 65):
        bad = np.abs(z) > 2.0
        if clipped or not bad.any():
            break
        z = np.where(bad, draw(attempt), z)
        near |= bad & (np.abs(np.abs(z) - 2.0) < 1e-3)
    return z, near


def nan_rule(v):
    """trajectory_opt.py:178."""
    return np.where(np.isnan(v), np.float32(-1e-10), v).astype(np.float32)


def topk_order(values, k):
    """Indices of the k largest values by (descending value, ascending index); -0.0 ties with +0.0."""
    key = values + np.float32(0.0)
    return np.lexsort((np.arange(values.size), -key))[:k]


def records64(pop, vals, k, world):
    """What every rank contributes: its shard's top min(k, shard size) sequences as rows [value after the NaN rule,
    sequence] in ascending local index order.  Returns the per-rank records and the global index of every record of the
    rank-ordered union."""
    recs, gidx = [], []
    for r in range(world):
        lo, hi = bd.shard_bounds(vals.size, r, world)
        v = nan_rule(vals[lo:hi])
        sel = np.sort(topk_order(v, bd.records_per_rank(k, hi - lo)))
        recs.append(np.concatenate([v[sel, None], pop[lo:hi][sel]], axis=1))
        gidx.append(lo + sel)
    return recs, np.concatenate(gidx)


def refit_values(N, k, seed):
    """The hazards of tests/test_gpu_scale.py::_refit_values: NaN (-> -1e-10), +inf among the elites, -inf, and the k-th
    value inside a run of k exact zeros of both signs."""
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


def hazard_values(N, k, world, seed):
    """refit_values plus runs of four equal values across every shard boundary: +-0.0 (joining the run the k-th value
    falls in, so the global tie-break by index crosses ranks) at the even boundaries, 2.5 (all elites) at the odd ones."""
    v = refit_values(N, k, seed)
    for r in range(1, world):
        b = bd.shard_bounds(N, r, world)[0]
        v[b - 2:b + 2] = np.float32([0.0, -0.0, -0.0, 0.0]) if r % 2 else np.float32(2.5)
    return v


# run_select's dispatch (cem.cu), restated: which kernel a selection over n values with k elites of `dims` floats runs in
K_SMALL_N = 2048
ELITE_SMEM_BYTES = 150 * 1024
PARTIAL_SMEM_BYTES = 160 * 1024


def select_branch(n, dims, k):
    if n <= K_SMALL_N and k * dims * 4 <= ELITE_SMEM_BYTES:
        return "single_cta"
    return ("counting" if n <= K_SMALL_N else "radix") + ("+global_partials" if 33 * dims * 4 > PARTIAL_SMEM_BYTES else "")


def same_kernel(a, b):
    """single_cta is cem_select_small_kernel; counting and radix are the two rankings of cem_select_kernel, which sums
    the elites the same way after either."""
    return (a == "single_cta") == (b == "single_cta")


# ---- CPU checks of the checkers -----------------------------------------------------------------------------------
def test_philox_restatement_known_answers():
    """Random123's known-answer vectors for philox4x32_10."""
    kat = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
           ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
           ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
            (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
    for ctr, key, want in kat:
        got = philox4x32_10(*[np.array([c]) for c in ctr], *key)
        assert tuple(int(x[0]) for x in got) == want
    z, _ = cem_draws64(4000, 7, 11, 5)
    assert np.abs(z).max() <= 2.0 and stats.kstest(z.ravel(), stats.truncnorm(-2.0, 2.0).cdf).pvalue > 1e-6
    z, _ = cem_draws64(4000, 7, 11, 5, clipped=True)
    assert np.abs(z).max() > 2.0 and stats.kstest(z.ravel(), "norm").pvalue > 1e-6


@pytest.mark.parametrize("tag,clipped", [("trunc_best", False), ("trunc_mean", False), ("clipped_best", True)])
def test_sampler_restatement_reproduces_the_reference_goldens(golden_dir, tag, clipped):
    g = np.load(os.path.join(golden_dir, f"cem_{tag}.npz"))
    N = int(g["N"])
    lb, ub, x0 = (g[k].reshape(-1) for k in ("lb", "ub", "x0"))
    disp0 = np.ones_like(x0) if clipped else (ub - lb) ** 2 / 16
    pop = cem_sample64(g["z"][0].reshape(N, -1), x0, disp0, lb, ub, clipped)
    np.testing.assert_allclose(pop, g["pops"][0].reshape(N, -1), rtol=2e-6, atol=2e-7)


@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_records_restatement_selects_the_unions_elites(world):
    """per-shard top-k -> concatenate -> top-k picks the sequences a plain top-k over the union picks, in that order."""
    for N, k in [(500, 50), (501, 51), (8192, 4096), (4100, 2), (64, 64)]:
        vals = hazard_values(N, k, world, seed=N + world)
        pop = np.arange(N, dtype=np.float32)[:, None] * np.ones((1, 2), np.float32)
        recs, gidx = records64(pop, vals, k, world)
        union = np.concatenate(recs)
        assert union.shape[0] == sum(bd.records_per_rank(k, np.diff(bd.shard_bounds(N, r, world))[0]) for r in range(world))
        assert (np.diff(gidx) > 0).all()  # rank-major, ascending local index: ascending global index
        order = gidx[topk_order(union[:, 0], k)]
        assert np.array_equal(order, topk_order(nan_rule(vals), k))
        assert np.array_equal(union[:, 1], gidx)  # the rows travel with their values


def test_select_branch_restates_run_select():
    """The constants select_branch uses are the ones cem.cu dispatches on; a change there must move the cases below."""
    src = open(CEM_CU).read()
    assert int(re.search(r"constexpr int kSmallN = (\d+);", src).group(1)) == K_SMALL_N
    body = src[src.index("static int run_select("):src.index("int b200pets_cem_update(")]
    assert "n <= kSmallN && (size_t)k * dims * sizeof(float) <= 150 * 1024" in body
    assert "(size_t)33 * dims * sizeof(float) <= 160 * 1024" in body
    for (N, dims, k), worlds, want in RECORD_CASES.values():
        for world in worlds:
            n_loc = [np.diff(bd.shard_bounds(N, r, world))[0] for r in range(world)]
            k_loc = [bd.records_per_rank(k, n) for n in n_loc]
            assert len(set(k_loc)) == 1
            got = ({select_branch(n, dims, kl) for n, kl in zip(n_loc, k_loc)}, select_branch(sum(k_loc), dims, k),
                   select_branch(N, dims, k))
            assert got == ({want[0]}, want[1], want[2]), (N, dims, k, world, got)


def test_sharded_optimizer_refuses_unequal_record_counts():
    """501 sequences over 2 ranks with 301 elites: the ranks would contribute 251 and 250 records."""
    bounds = [[-1.0] * 2] * 3, [[1.0] * 2] * 3
    with pytest.raises(ValueError, match="same number of records"):
        bd.ShardedCEMOptimizer(2, 0.6, 501, *bounds, 0.1, "cpu", rank=0, world=2, gather=lambda rec: rec)


# ---- 1. the sampler with injected normals ------------------------------------------------------------------------------
def _cem_sample(n, dims, mu, disp, lb, ub, z=None, seed=0, offset=0, clipped=0, first=None):
    """b200pets_cem_sample (first None) or b200pets_cem_sample_shard; two guard rows after the population must stay."""
    _lib, lib = _abi()
    pop = torch.full((n + 2, dims), GUARD, device=DEV)
    args = _dev(mu, disp, lb, ub, z)
    ptrs = list(map(_lib.ptr, args))
    if first is None:
        rc = lib.b200pets_cem_sample(n, dims, *ptrs, seed, offset, int(clipped), _lib.ptr(pop), _lib.stream_ptr())
    else:
        rc = lib.b200pets_cem_sample_shard(n, first, dims, *ptrs, seed, offset, int(clipped), _lib.ptr(pop), _lib.stream_ptr())
    _lib.check(rc, "cem_sample")
    got = pop.cpu().numpy()
    assert (got[n:] == GUARD).all(), "rows after the population were written"
    return got[:n]


KINDS = ["variance", "lower", "upper", "mu_at_lb", "mu_at_ub", "mu_outside", "asymmetric"]


def _truncated_problem(g, dims, rot):
    """Per-coordinate bounds, mean and variance; coordinate d is of kind KINDS[(d + rot) % 7]: the variance binds; the
    lower / the upper constraint binds; the mean sits exactly on the lower / upper bound (constraint 0); the mean lies
    outside the bounds; asymmetric bounds with variance and constraints of the same order."""
    kind = (np.arange(dims) + rot) % len(KINDS)
    lb = -g.uniform(0.5, 2.0, dims)
    ub = g.uniform(0.5, 2.0, dims)
    mu = g.uniform(-0.2, 0.2, dims)
    var = g.uniform(0.005, 0.02, dims)
    wide = g.uniform(0.5, 2.0, dims)
    gap = g.uniform(0.1, 0.4, dims)
    mu = np.where(kind == 1, lb + gap, mu)
    mu = np.where(kind == 2, ub - gap, mu)
    var = np.where((kind == 1) | (kind == 2) | (kind == 5), wide, var)
    mu = np.where(kind == 3, lb, mu)
    mu = np.where(kind == 4, ub, mu)
    mu = np.where(kind == 5, np.where(np.arange(dims) % 2 == 0, ub + gap, lb - gap), mu)
    lb = np.where(kind == 6, -g.uniform(0.1, 0.4, dims), lb)
    ub = np.where(kind == 6, g.uniform(1.0, 2.0, dims), ub)
    mu = np.where(kind == 6, g.uniform(-0.05, 0.9, dims), mu)
    var = np.where(kind == 6, g.uniform(0.01, 0.3, dims), var)
    f = lambda a: a.astype(np.float32)  # noqa: E731
    return kind, f(mu), f(var), f(lb), f(ub)


# population x dims at 255 / 256 / 257 and around one 256-thread block for dims 3, 6, 7; several blocks; the shapes of the
# configurations (PETS 500 / 350 x 30 x 6, iCEM 1000 x 40 x 17, the single-CTA limit and one above it, config 5)
SAMPLE_SHAPES = [(255, 1), (256, 1), (257, 1), (85, 3), (86, 3), (42, 6), (43, 6), (36, 7), (37, 7), (1000, 7), (33, 243),
                 (500, 180), (350, 180), (1000, 680), (2048, 180), (2049, 36), (64000, 36)]


@gpu
@pytest.mark.parametrize("n,dims", SAMPLE_SHAPES)
def test_cem_sample_truncated_matches_float64(n, dims):
    g = np.random.default_rng(n * 1000 + dims)
    worst = 0.0
    seen = set()
    for rot in range(0, len(KINDS), min(dims, len(KINDS))):
        kind, mu, var, lb, ub = _truncated_problem(g, dims, rot)
        seen |= set(kind.tolist())
        z = np.clip(g.standard_normal((n, dims)), -2, 2).astype(np.float32)
        got = _cem_sample(n, dims, mu, var, lb, ub, z)
        ref = cem_sample64(z, mu, var, lb, ub, False)
        worst = max(worst, float((np.abs(got - ref) / np.maximum(1.0, np.abs(ref))).max()))
        # which term binds, from the float64 rule: the cases this test is about are all present
        l2, u2 = ((mu.astype(np.float64) - lb) / 2) ** 2, ((ub - mu.astype(np.float64)) / 2) ** 2
        for kd, binds in ((0, var < np.minimum(l2, u2)), (1, l2 < np.minimum(u2, var)), (2, u2 < np.minimum(l2, var))):
            assert binds[kind == kd].all()
        assert ((mu > ub) | (mu < lb))[kind == 5].all() and (np.minimum(l2, u2) > 0)[kind == 5].all()
        pinned = (kind == 3) | (kind == 4)  # constraint 0: every sequence is the mean itself
        assert np.array_equal(_bits(got[:, pinned]), _bits(np.broadcast_to(mu[pinned], (n, int(pinned.sum())))))
    assert seen == set(range(len(KINDS)))
    _report(f"cem_sample truncated {n} x {dims}", worst, 1e-6)


@gpu
@pytest.mark.parametrize("n,dims", SAMPLE_SHAPES)
def test_cem_sample_clipped_matches_float64(n, dims):
    g = np.random.default_rng(n * 1000 + dims + 1)
    mu = g.uniform(-0.5, 0.5, dims).astype(np.float32)
    sd = g.uniform(0.3, 1.5, dims).astype(np.float32)
    lb = (mu - g.uniform(0.4, 0.65, dims) * sd).astype(np.float32)  # about 30 % of N(0, 1) beyond each bound
    ub = (mu + g.uniform(0.4, 0.65, dims) * sd).astype(np.float32)
    z = g.standard_normal((n, dims)).astype(np.float32)
    got = _cem_sample(n, dims, mu, sd, lb, ub, z, clipped=1)
    free = mu.astype(np.float64) + sd.astype(np.float64) * z
    margin = 1e-5 * np.maximum(1.0, np.abs(free))
    below, above = free < lb - margin, free > ub + margin
    if n * dims >= 2000:
        assert 0.2 < below.mean() < 0.4 and 0.2 < above.mean() < 0.4
    assert np.array_equal(got[below], np.broadcast_to(lb, got.shape)[below])
    assert np.array_equal(got[above], np.broadcast_to(ub, got.shape)[above])
    assert (got >= lb).all() and (got <= ub).all()
    ref = cem_sample64(z, mu, sd, lb, ub, True)
    _report(f"cem_sample clipped {n} x {dims}", float((np.abs(got - ref) / np.maximum(1.0, np.abs(ref))).max()), 1e-6)


@gpu
@pytest.mark.parametrize("clipped", [0, 1])
def test_cem_sample_shard_is_a_slice_of_the_population(clipped):
    """Philox draws are keyed by the global sequence index: a shard at any first sequence is that slice of the whole."""
    N, n, dims = 2304, 200, 7
    g = np.random.default_rng(17 + clipped)
    _, mu, disp, lb, ub = _truncated_problem(g, dims, 0)
    seed, offset = 0xC0FFEE12345, 3 * 1024 + 2
    full = _cem_sample(N, dims, mu, disp, lb, ub, None, seed, offset, clipped)
    assert np.unique(full[:, 0]).size > N // 2
    for first in (0, 1, 63, 250, 2047, N - n):
        shard = _cem_sample(n, dims, mu, disp, lb, ub, None, seed, offset, clipped, first=first)
        assert np.array_equal(_bits(shard), _bits(full[first:first + n])), f"shard at {first} differs"
    other = _cem_sample(n, dims, mu, disp, lb, ub, None, seed, offset + 1, clipped, first=63)
    assert not np.array_equal(other, full[63:63 + n])


@gpu
@pytest.mark.parametrize("clipped", [0, 1])
def test_cem_sample_shard_indexes_injected_noise_from_its_own_row_zero(clipped):
    """With injected normals a shard reads z[0 .. n) whatever its first sequence: z is the shard's, not the population's."""
    n, dims = 300, 6
    g = np.random.default_rng(23 + clipped)
    _, mu, disp, lb, ub = _truncated_problem(g, dims, 1)
    z = np.clip(g.standard_normal((n, dims)), -2, 2).astype(np.float32)
    at0 = _cem_sample(n, dims, mu, disp, lb, ub, z, clipped=clipped)
    for first in (1, 250, 5000):
        assert np.array_equal(_bits(_cem_sample(n, dims, mu, disp, lb, ub, z, clipped=clipped, first=first)), _bits(at0))
    ref = cem_sample64(z, mu, disp, lb, ub, clipped)
    assert float((np.abs(at0 - ref) / np.maximum(1.0, np.abs(ref))).max()) <= 1e-6


# ---- 2. the sampler's Philox draws -----------------------------------------------------------------------------------
def _unit_draws(n, dims, seed, offset, clipped=0, first=None):
    """mu 0, dispersion 1, bounds +-1e3: sqrt(min(250 000, 1)) = 1 and 1 * z + 0 = z, so the population is the draws."""
    one, big = np.ones(dims, np.float32), np.full(dims, 1e3, np.float32)
    return _cem_sample(n, dims, 0 * one, one, -big, big, None, seed, offset, clipped, first=first).astype(np.float64)


def _corr(a, b):
    return float(abs(np.corrcoef(a.ravel(), b.ravel())[0, 1]))


@gpu
@pytest.mark.parametrize("clipped", [0, 1])
def test_cem_philox_draws_match_the_documented_counter_layout(clipped):
    """Known answer: lane d & 3 of block (global sequence, d >> 2, stream | attempt, offset) under key seed ^ offset's high
    word, in numpy.  The seed and the offset both use their high words; the shard starts at sequence 123."""
    n, dims, first = 3001, 7, 123
    seed, offset = 0x123456789ABCDEF0, (3 << 32) + 5 * 1024 + 1
    got = _unit_draws(n, dims, seed, offset, clipped, first=first)
    ref, near = cem_draws64(n, dims, seed, offset, first, bool(clipped))
    assert near.mean() < 0.01
    err = (np.abs(got - ref) / np.maximum(1.0, np.abs(ref)))[~near]
    print(f"redrawn elements: {int((np.abs(cem_draws64(n, dims, seed, offset, first, True)[0]) > 2).sum())} of {n * dims}")
    _report(f"cem Philox known answer (clipped {clipped})", float(err.max()), 1e-4)


@gpu
@pytest.mark.parametrize("dims", [8, 7])
def test_cem_philox_draws_are_truncated_normal(dims):
    n, seed, offset = 20000, 4242, 7 * 1024 + 3
    z = _unit_draws(n, dims, seed, offset)
    assert np.abs(z).max() <= 2.0
    tn = stats.truncnorm(-2.0, 2.0)
    ps = {"pooled": stats.kstest(z.ravel(), tn.cdf).pvalue}
    for lane in range(4):
        ps[f"lane {lane}"] = stats.kstest(z[:, lane::4].ravel(), tn.cdf).pvalue
    print(f"cem Philox dims {dims}: KS p-values against N(0,1) truncated to [-2, 2] " + ", ".join(f"{k} {p:.2e}" for k, p in ps.items()))
    assert min(ps.values()) > 1e-6
    # redrawing keeps the density's shape up to +-2; clamping would pile the 4.6 % beyond +-2 onto the last bin
    p_tail = (stats.norm.cdf(2.0) - stats.norm.cdf(1.5)) / (stats.norm.cdf(2.0) - stats.norm.cdf(-2.0))
    sigma = np.sqrt(z.size * p_tail * (1 - p_tail))
    for what, cnt in (("(1.5, 2]", (z > 1.5).sum()), ("[-2, -1.5)", (z < -1.5).sum())):
        dev = (cnt - z.size * p_tail) / sigma
        print(f"  mass in {what}: {cnt} of {z.size}, {dev:+.2f} binomial sigma from the truncated law")
        assert abs(dev) <= 4.0
    bar = 4.0 / np.sqrt(n)
    pairs = {"dims 0, 1 (one block)": (z[:, 0], z[:, 1]), "dims 2, 3 (one block)": (z[:, 2], z[:, 3]),
             "dims 3, 4 (two blocks)": (z[:, 3], z[:, 4]), "dims 0, 4 (same lane)": (z[:, 0], z[:, 4]),
             "neighbouring sequences": (z[:-1], z[1:]),
             "offset, offset + 1": (z, _unit_draws(n, dims, seed, offset + 1)),
             "two seeds": (z, _unit_draws(n, dims, seed + 1, offset)),
             "first sequence 0, 20 000": (z, _unit_draws(n, dims, seed, offset, first=20000))}
    for what, (a, b) in pairs.items():
        c = _corr(a, b)
        assert c < bar, (what, c)
    print(f"  largest correlation {max(_corr(a, b) for a, b in pairs.values()):.2e} (bar {bar:.2e})")


@gpu
def test_cem_philox_draws_clipped_mode_are_plain_normal():
    z = _unit_draws(20000, 7, 4242, 9 * 1024, clipped=1)
    p = stats.kstest(z.ravel(), "norm").pvalue
    beyond = float((np.abs(z) > 2).mean())
    print(f"cem Philox clipped mode: KS p-value against N(0, 1) {p:.2e}, {beyond:.4f} of the draws beyond +-2")
    assert p > 1e-6 and 0.035 < beyond < 0.056  # 2 * (1 - Phi(2)) = 0.0455


# ---- 3. the sharded records route ------------------------------------------------------------------------------------
# (population, dims, k), worlds, (kernel of local_topk, of update_from_records, of the whole-population cem_update)
RECORD_CASES = {
    "pets_500": ((500, 180, 50), (1, 2, 4), ("single_cta", "single_cta", "single_cta")),
    "uneven_501": ((501, 12, 51), (3,), ("single_cta", "single_cta", "single_cta")),
    "counting_icem": ((2000, 680, 200), (2,), ("counting", "counting", "counting")),
    "global_partials": ((3000, 1300, 60), (2,), ("counting+global_partials", "counting+global_partials", "radix+global_partials")),
    "config5": ((64000, 36, 6400), (2, 4, 8), ("radix", "radix", "radix")),
    "every_sequence_a_record": ((8192, 30, 4096), (8,), ("single_cta", "radix", "radix")),
    "two_elites": ((4100, 7, 2), (2,), ("radix", "single_cta", "radix")),
}
# (case, world, unbiased, use_std, elites_out)
RECORD_RUNS = [(c, w, 1, 0, True) for c, (_, worlds, _) in RECORD_CASES.items() for w in worlds] + \
              [(c, 2, u, s, e) for c in ("pets_500", "config5") for u, s, e in ((0, 0, False), (0, 1, True), (1, 1, False))]


def _workspace(lib, n, dims, k):
    nbytes = lib.b200pets_cem_update_workspace_bytes(n, dims, k)
    return torch.empty(nbytes, dtype=torch.uint8, device=DEV), nbytes


def _local_topk(pop, vals, k):
    """b200pets_cem_local_topk on one shard: (records [k, 1 + dims], the shard's values afterwards)."""
    _lib, lib = _abi()
    (n, dims), k = pop.shape, int(k)
    pop_d, v_d = _dev(pop, vals)
    rec = torch.full((k + 2, 1 + dims), GUARD, device=DEV)
    ws, nbytes = _workspace(lib, n, dims, k)
    _lib.check(lib.b200pets_cem_local_topk(n, dims, k, _lib.ptr(pop_d), _lib.ptr(v_d), _lib.ptr(rec), _lib.ptr(ws), nbytes,
                                           _lib.stream_ptr()), "cem_local_topk")
    torch.cuda.synchronize()
    assert bool((rec[k:] == GUARD).all()), "rows after the k records were written"
    return rec[:k].clone(), v_d.cpu().numpy()


def _refit(call, n, dims, k, alpha, unbiased, use_std, data, mu0, disp0, with_elites):
    """b200pets_cem_update (data = (pop, values)) or b200pets_cem_update_from_records (data = (records,)) from (mu0, disp0)
    and a best value of -inf: dict of mu, disp, best_value, best_solution, elites (or None) and the values / records
    tensor the call may have changed in place."""
    _lib, lib = _abi()
    mu, disp = _dev(mu0, disp0)
    best_v = torch.full((1,), float("-inf"), device=DEV)
    best_s = torch.full((dims,), GUARD, device=DEV)
    elites = torch.full((k, dims), float("nan"), device=DEV) if with_elites else None
    ws, nbytes = _workspace(lib, n, dims, k)
    tail = (_lib.ptr(mu), _lib.ptr(disp), _lib.ptr(best_v), _lib.ptr(best_s))
    if call == "update":
        pop_d, v_d = data
        rc = lib.b200pets_cem_update(n, dims, k, alpha, unbiased, use_std, _lib.ptr(pop_d), _lib.ptr(v_d), *tail, None,
                                     _lib.ptr(elites), _lib.ptr(ws), nbytes, _lib.stream_ptr())
    else:
        rc = lib.b200pets_cem_update_from_records(n, dims, k, alpha, unbiased, use_std, _lib.ptr(data[0]), *tail,
                                                  _lib.ptr(elites), _lib.ptr(ws), nbytes, _lib.stream_ptr())
    _lib.check(rc, call)
    torch.cuda.synchronize()
    return {"mu": mu, "disp": disp, "best_value": best_v, "best_solution": best_s, "elites": elites}


def _same(a, b, what):
    for key in ("mu", "disp", "best_value", "best_solution", "elites"):
        if a[key] is not None:
            assert torch.equal(a[key], b[key]), f"{what}: {key} differs, max |diff| {(a[key] - b[key]).abs().max().item():.3e}"


def _deviation(a, b):
    return max(float((a[key] - b[key]).abs().max()) for key in ("mu", "disp"))


@gpu
@pytest.mark.parametrize("case,world,unbiased,use_std,with_elites", RECORD_RUNS)
def test_records_route_equals_the_single_gpu_refit(case, world, unbiased, use_std, with_elites):
    (N, dims, k), _, want = RECORD_CASES[case]
    alpha = 0.1
    vals = hazard_values(N, k, world, seed=N + dims + world)
    g = np.random.default_rng(dims + world)
    pop = g.standard_normal((N, dims)).astype(np.float32)
    mu0 = g.standard_normal(dims).astype(np.float32)
    disp0 = (0.5 + g.random(dims)).astype(np.float32)
    assert np.isnan(vals).any() and np.isposinf(vals).any() and np.isneginf(vals).any()
    ref_recs, gidx = records64(pop, vals, k, world)
    ruled = nan_rule(vals)
    assert ruled[topk_order(ruled, k)[-1]] == 0.0 or case == "two_elites"  # the selection ends inside the run of zeros

    # every rank's records
    recs = []
    for r in range(world):
        lo, hi = bd.shard_bounds(N, r, world)
        k_loc = bd.records_per_rank(k, hi - lo)
        assert select_branch(hi - lo, dims, k_loc) == want[0]
        rec, v_after = _local_topk(pop[lo:hi], vals[lo:hi], k_loc)
        assert np.array_equal(_bits(v_after), _bits(ruled[lo:hi])), f"rank {r}: NaN rule on the shard's values"
        assert np.array_equal(_bits(rec.cpu().numpy()), _bits(ref_recs[r])), f"rank {r}: records differ"
        recs.append(rec)
    union = torch.cat(recs, dim=0).contiguous()  # the all-gather, in rank order
    n_rec = union.shape[0]
    assert select_branch(n_rec, dims, k) == want[1] and select_branch(N, dims, k) == want[2]

    # the records route against float64 over the union population
    before = union.clone()
    got = _refit("records", n_rec, dims, k, alpha, unbiased, use_std, (union,), mu0, disp0, with_elites)
    assert torch.equal(union, before)  # no NaN left in records: nothing to rewrite, and the rows are read-only
    order = topk_order(ruled, k)
    elite = pop[order].astype(np.float64)
    var = elite.var(0, ddof=1 if unbiased else 0)
    nd = np.sqrt(var) if use_std else var
    np.testing.assert_allclose(got["mu"].cpu().numpy(), alpha * mu0 + (1 - alpha) * elite.mean(0), rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(got["disp"].cpu().numpy(), alpha * disp0 + (1 - alpha) * nd, rtol=1e-4, atol=1e-5)
    assert float(got["best_value"]) == float(ruled[order[0]])
    assert np.array_equal(_bits(got["best_solution"].cpu().numpy()), _bits(pop[order[0]]))
    if with_elites:
        assert np.array_equal(_bits(got["elites"].cpu().numpy()), _bits(pop[order]))

    # against b200pets_cem_update on the whole population
    pop_d, v_d = _dev(pop, vals)
    whole = _refit("update", N, dims, k, alpha, unbiased, use_std, (pop_d, v_d), mu0, disp0, with_elites)
    assert np.array_equal(_bits(v_d.cpu().numpy()), _bits(ruled))
    if same_kernel(want[1], want[2]):
        _same(got, whole, f"records route ({want[1]}) against cem_update ({want[2]})")
    else:
        _same({**got, "mu": None, "disp": None}, whole, "records route against cem_update")
        print(f"{case}: records route in {want[1]}, cem_update in {want[2]}: max |mu, dispersion deviation| {_deviation(got, whole):.3e}")

    # the whole population as raw records [value, sequence]: the strided reads of the same kernel, NaN rule included
    raw = torch.cat([_t(vals)[:, None], pop_d], dim=1).contiguous()
    strided = _refit("records", N, dims, k, alpha, unbiased, use_std, (raw,), mu0, disp0, with_elites)
    _same(strided, whole, f"interleaved values and rows ({want[2]}) against contiguous ones")
    assert np.array_equal(_bits(raw[:, 0].cpu().numpy()), _bits(ruled)), "NaN rule on column 0 of the records"
    assert torch.equal(raw[:, 1:], pop_d), "the rows of the records were written"


# ---- 4. plans against the chain of their building blocks ---------------------------------------------------------------
def _chain(env, N, H, P, precision, k, alpha, clipped, iters, call, obs, x0, lb, ub):
    """CEMOptimizer.optimize from the public blocks with b200pets_cem_plan's Philox arithmetic: iteration `it` of the call
    with counter value `call` samples and rolls out with offset call * 1024 + it under the environment's seed."""
    _lib, lib = _abi()
    A = x0.shape[-1]
    dims = H * A
    prop = env._propagation()
    rcfg = _lib.RolloutCfg(N, H, P, _lib.PREC[precision], _lib.PROP[prop], _lib.TS1_TILE_SHUFFLE, env._seed, 0)
    w = (ub - lb).astype(np.float32).reshape(-1)
    mu, disp, lb_d, ub_d, obs_d = _dev(x0.reshape(-1).astype(np.float32), np.ones(dims, np.float32) if clipped else (w * w) / np.float32(16),
                                       lb.reshape(-1), ub.reshape(-1), np.asarray(obs, np.float32))
    pop = torch.empty(N, dims, device=DEV)
    values = torch.empty(N, device=DEV)
    best_v = torch.full((1,), float("-inf"), device=DEV)
    best_s = torch.zeros(dims, device=DEV)
    ws, nbytes = _workspace(lib, N, dims, k)
    ebytes = lib.b200pets_eval_workspace_bytes(env.staged.handle, C.byref(rcfg))
    ews = torch.empty(max(ebytes, 1), dtype=torch.uint8, device=DEV)
    out = torch.empty(iters, N, device=DEV)
    stream = _lib.stream_ptr()
    for it in range(iters):
        off = call * 1024 + it
        _lib.check(lib.b200pets_cem_sample(N, dims, _lib.ptr(mu), _lib.ptr(disp), _lib.ptr(lb_d), _lib.ptr(ub_d), None, env._seed, off,
                                           int(clipped), _lib.ptr(pop), stream), "cem_sample")
        rcfg.offset = off
        _lib.check(lib.b200pets_eval_sequences(env.staged.handle, C.byref(rcfg), _lib.ptr(obs_d), _lib.ptr(pop), None, None,
                                               _lib.ptr(values), None, _lib.ptr(ews), ews.numel(), stream), "eval_sequences")
        _lib.check(lib.b200pets_cem_update(N, dims, k, alpha, 1, int(clipped), _lib.ptr(pop), _lib.ptr(values), _lib.ptr(mu),
                                           _lib.ptr(disp), _lib.ptr(best_v), _lib.ptr(best_s), None, None, _lib.ptr(ws), nbytes,
                                           stream), "cem_update")
        out[it].copy_(values)  # after the in-place NaN rule, like the plan's values_out
    torch.cuda.synchronize()
    return out, mu.view(H, A), best_s.view(H, A)


def _plan_env(name, precision):
    spec, _, env = make_env(name, precision, ts1="tile_shuffle")
    env._few_groups = lambda *a: False  # the model's own tile-shuffle draws at every population size
    obs0 = syn.make_rollout_inputs(spec, with_noise=False)["obs0"]
    return spec, env, obs0


def _check_plan(spec, env, obs0, precision, N, iters, clipped, rme, elite_ratio=0.1, horizon=None, merged=True, x0=None,
                call=50, K=None):
    """One plan (or a batch of K) against the chain; returns the plan's solution and values."""
    import mbrl_lib_b200 as bp
    from mbrl_lib_b200.planning import _FusedBatchObjective, _FusedObjective

    H, A, P, alpha = horizon or spec.horizon, spec.act_dim, spec.particles, 0.1
    lb, ub = np.full((H, A), spec.action_lb, np.float32), np.full((H, A), spec.action_ub, np.float32)
    opt = bp.CEMOptimizer(iters, elite_ratio, N, lb.tolist(), ub.tolist(), alpha, DEV, return_mean_elites=rme, clipped_normal=clipped)
    opt.record_values = True
    k = opt.elite_num
    assert (select_branch(N, H * A, k) == "single_cta") == merged, "the plan would take the other launch structure"
    g = np.random.default_rng(N + iters)
    if x0 is None:
        x0 = g.uniform(-0.3, 0.3, (K or 1, H, A)).astype(np.float32) * (ub - lb) / 2
    obs = np.stack([obs0 + 0.1 * j * g.standard_normal(obs0.shape) for j in range(K or 1)])
    env._offset = call - 1
    if K is None:
        sol = opt.optimize(_FusedObjective(env, obs[0], P), x0=_t(x0[0]))[None]
        vals = opt.last_values[None]
    else:
        sol = opt.optimize_batch(_FusedBatchObjective(env, obs, P), x0=_t(x0))
        vals = opt.last_values
    torch.cuda.synchronize()
    assert env._offset == call - 1 + (K or 1)
    what = f"{spec.name} {precision} pop {N} iters {iters} clipped {clipped} mean {rme}"
    for j in range(K or 1):
        c_vals, c_mu, c_best = _chain(env, N, H, P, env.precision_for(env._propagation()), k, alpha, clipped, iters, call + j,
                                      obs[j], x0[j], lb, ub)
        assert bool(torch.isfinite(c_vals).all())
        for it in range(iters):
            assert torch.equal(vals[j, it], c_vals[it]), \
                f"{what}: problem {j} iteration {it}: {(vals[j, it] != c_vals[it]).sum().item()} of {N} values differ from the chain"
        assert torch.equal(sol[j], c_mu if rme else c_best), f"{what}: problem {j}: solution differs from the chain"
        if iters > 1:
            assert not torch.equal(c_vals[0], c_vals[1])
    return sol, vals


# (clipped_normal, return_mean_elites, iterations)
PLAN_MODES = [(False, True, 5), (True, False, 2), (False, False, 1), (True, True, 5)]


@gpu
@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
@pytest.mark.parametrize("N", [64, 500, 2048])
@pytest.mark.parametrize("name", ["halfcheetah_small", "cartpole"])
def test_merged_plan_equals_the_chain(name, N, precision):
    """Rollout + one refit-and-sample kernel per iteration: sampling grids of 1 to 64 CTAs (64 x 15 elements to 2 048 x 72,
    where every CTA strides), the refit flag handed from CTA 0 to the rest."""
    spec, env, obs0 = _plan_env(name, precision)
    for clipped, rme, iters in PLAN_MODES:
        _check_plan(spec, env, obs0, precision, N, iters, clipped, rme)


@gpu
@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
@pytest.mark.parametrize("N", [2049, 4000])
def test_three_launch_plan_above_the_single_cta_refit_equals_the_chain(N, precision):
    """Sample, rollout, particle mean + radix refit as separate launches."""
    spec, env, obs0 = _plan_env("halfcheetah_small", precision)
    for clipped, rme, iters in PLAN_MODES[:2]:
        _check_plan(spec, env, obs0, precision, N, iters, clipped, rme, merged=False)


@gpu
@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
def test_three_launch_plan_with_a_large_elite_set_equals_the_chain(precision):
    """humanoid_trunc (A 17) at H 40, pop 1 000, elite ratio 0.25: 250 x 680 floats of elite rows exceed the single-CTA
    refit's shared memory, so a population below 2 048 takes the counting refit behind separate sample launches."""
    spec, env, obs0 = _plan_env("humanoid_trunc", precision)
    _check_plan(spec, env, obs0, precision, 1000, 3, False, True, elite_ratio=0.25, horizon=40, merged=False)
    _check_plan(spec, env, obs0, precision, 1000, 2, True, False, elite_ratio=0.25, horizon=40, merged=False)


@gpu
@pytest.mark.parametrize("rme", [True, False])
@pytest.mark.parametrize("N", [500, 2049])
def test_plan_from_a_mean_on_the_bound_equals_the_chain(N, rme):
    """x0 exactly at the upper bound in every other coordinate: the variance cap is 0 there from the first population on,
    all sequences agree in those coordinates and every refit averages equal numbers, in either launch structure."""
    spec, env, obs0 = _plan_env("halfcheetah_small", "f32")
    H, A = spec.horizon, spec.act_dim
    x0 = np.random.default_rng(5).uniform(-0.3, 0.3, (1, H, A)).astype(np.float32)
    at_ub = (np.arange(H * A) % 2 == 0).reshape(H, A)
    x0[0][at_ub] = spec.action_ub
    sol, _ = _check_plan(spec, env, obs0, "f32", N, 5, False, rme, merged=N <= 2048, x0=x0)
    assert bool((sol[0][_t(at_ub)] == spec.action_ub).all()), "a coordinate whose population never left the bound moved"
    assert bool((sol[0][_t(~at_ub)].abs() <= spec.action_ub).all())


@gpu
@pytest.mark.parametrize("N,merged", [(500, True), (2049, False)])
def test_batched_plan_equals_the_chain_per_problem(N, merged):
    """Problem j of a batch of 3 is the chain at counter value first + j."""
    spec, env, obs0 = _plan_env("halfcheetah_small", "bf16_tc")
    _check_plan(spec, env, obs0, "bf16_tc", N, 3, False, True, merged=merged, K=3)
    _check_plan(spec, env, obs0, "bf16_tc", N, 2, True, False, merged=merged, K=3)
