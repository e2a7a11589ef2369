"""The iCEM and MPPI kernels (b200pets_icem_sample / icem_append_elites / mppi_sample / mppi_update) called through the
C ABI at the shapes their configurations run, against float64 restatements of the reference's operations; the
optimisers over three consecutive calls against the oracle driven by the GPU's own objective values; the in-kernel
Philox draws against the laws the reference samples from.

Bars (stated; the measured maxima are printed with -s):
  * coloured noise, injected normals: |got - ref| <= 1e-5 * sqrt(var) * max(1, |y|) before clipping (fp32 DFT of at most
    21 bins and powf spectrum against float64), clipped elements exactly at the bound;
  * kept elites: copies bit-equal; the fresh last action within 2 units of (1 ulp of the result + 1 ulp of sqrt(var)
    times |e|): one rounding of the sqrt and one of the fused multiply-add, or two if the compiler does not fuse;
  * MPPI sample: |got - ref| <= 1e-5 * max(1, |ref|) (fp32 recurrence of at most 64 steps), clipped elements exactly at
    the bound;  MPPI update: NaN rule bit-exact, mean within 1e-5 * max(1, max|pop|) of float64;
  * optimisers: populations, elites (in order), means and solutions within 2e-5 * max(1, max|ref|) of the oracle in
    float64 (fp32 refits compound over the iterations).
Measured maxima on an H100 80GB HBM3 (700 W limit), in the units of each bar: coloured noise 8.6e-7 (wide bounds) and
6.8e-7 (clipping bounds); end action 0.49; MPPI sample 2.2e-7; MPPI update 1.6e-7; iCEM chains 9.5e-7, MPPI chain
5.7e-7; humanoid values 1.5e-7 (fp32) and, on the tensor-core kernel, a median of 3e-6 with at most one sequence per
population beyond 5e-3 (a termination flip, up to 8.6e-2).
"""
import numpy as np
import pytest
import torch
from scipy import stats

from mbrl_lib_b200 import synthetic as syn
from test_gpu_parity import DEV, make_env

pytestmark = pytest.mark.gpu


def _abi():
    from mbrl_lib_b200 import _lib

    return _lib, _lib.load()


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _dev(*arrays):
    """Device copies of the arrays (None stays None), held by the caller until the kernel that reads them has run: a
    temporary whose only use is ``_lib.ptr(_t(a))`` is freed before the launch and its memory handed to the next copy."""
    return [None if a is None else _t(a) for a in arrays]


def _report(what, err, bar):
    print(f"{what}: max deviation {err:.3e} of the bar's unit (bar {bar:.0e})")
    assert err <= bar, f"{what}: {err:.3e} > {bar:.0e}"


# ---- float64 restatements ------------------------------------------------------------------------------------------
def colored64(sr, si, H, exponent):
    """util/math.py:318-396 in float64 from unit normals sr, si [..., H//2+1] -> [..., H]."""
    K = H // 2 + 1
    s = (np.maximum(np.arange(K, dtype=np.float64), 1.0) / H) ** (-exponent / 2.0)  # f_0 := f_1 (cut-off 1/H)
    w = s[1:].copy()
    w[-1] *= (1 + H % 2) / 2.0
    sigma = 2.0 * np.sqrt(np.sum(w ** 2)) / H
    re = sr.astype(np.float64) * s
    im = si.astype(np.float64) * s
    im[..., 0] = 0.0
    if H % 2 == 0:
        im[..., -1] = 0.0
    return np.fft.irfft(re + 1j * im, n=H, axis=-1) / sigma


def mppi_pop64(z, mean, past, beta):
    """trajectory_opt.py:262-287 in float64, before clipping: the recurrence runs on the unclipped values."""
    N, H, A = z.shape
    v = np.empty((N, H, A))
    prev = np.broadcast_to(past.astype(np.float64), (N, A))
    for t in range(H):
        prev = beta * (mean[t].astype(np.float64) + z[:, t].astype(np.float64)) + (1.0 - beta) * prev
        v[:, t] = prev
    return v


def _icem_inputs(g, n, H, A):
    K = H // 2 + 1
    sr = g.standard_normal((n, A, K)).astype(np.float32)
    si = g.standard_normal((n, A, K)).astype(np.float32)
    mu = g.uniform(-0.5, 0.5, (H, A)).astype(np.float32)
    var = g.uniform(0.2, 2.0, (H, A)).astype(np.float32)
    return sr, si, mu, var


def _icem_sample(n, H, A, exponent, mu, var, lb, ub, sr=None, si=None, seed=0, offset=0):
    _lib, lib = _abi()
    pop = torch.full((n, H, A), float("nan"), device=DEV)
    args = _dev(mu, var, lb, ub, sr, si)
    _lib.check(lib.b200pets_icem_sample(n, H, A, float(exponent), *map(_lib.ptr, args), seed, offset, _lib.ptr(pop),
                                        _lib.stream_ptr()), "icem_sample")
    return pop.cpu().numpy()


# ---- icem_sample, injected normals -----------------------------------------------------------------------------------
# (A, n): n * A at 127 / 128 / 129 and either side of one 128-thread block for every A, plus several blocks
ICEM_AN = [(1, 127), (1, 128), (1, 129), (6, 21), (6, 22), (17, 7), (17, 8), (17, 61)]


@pytest.mark.parametrize("exponent", [0.0, 1.0, 2.0, 2.5, 4.0])
@pytest.mark.parametrize("H", [2, 3, 7, 8, 10, 30, 40, 41])
def test_icem_sample_matches_float64(H, exponent):
    g = np.random.default_rng(H * 10 + int(exponent * 2))
    worst_free = worst_clip = 0.0
    for A, n in ICEM_AN:
        sr, si, mu, var = _icem_inputs(g, n, H, A)
        y = colored64(sr, si, H, exponent).transpose(0, 2, 1)  # [n, H, A]
        ref = y * np.sqrt(var.astype(np.float64)) + mu
        wide = np.full((H, A), 1e30, np.float32)
        got = _icem_sample(n, H, A, exponent, mu, var, -wide, wide, sr, si)
        err = np.abs(got - ref) / (np.sqrt(var) * np.maximum(1.0, np.abs(y)))
        worst_free = max(worst_free, float(err.max()))
        # bounds that clip at both ends: ~30 % of the elements on each side
        lb = (mu - g.uniform(0.3, 0.7, (H, A)) * np.sqrt(var)).astype(np.float32)
        ub = (mu + g.uniform(0.3, 0.7, (H, A)) * np.sqrt(var)).astype(np.float32)
        got = _icem_sample(n, H, A, exponent, mu, var, lb, ub, sr, si)
        margin = 1e-4 * np.sqrt(var) * np.maximum(1.0, np.abs(y))
        below, above = ref < lb - margin, ref > ub + margin
        assert below.any() and above.any()
        assert np.array_equal(got[below], np.broadcast_to(lb, got.shape)[below])
        assert np.array_equal(got[above], np.broadcast_to(ub, got.shape)[above])
        assert (got >= lb).all() and (got <= ub).all()
        inside = ~(below | above)
        clipped_ref = np.clip(ref, lb, ub)
        worst_clip = max(worst_clip, float((np.abs(got - clipped_ref) / (np.sqrt(var) * np.maximum(1.0, np.abs(y))))[inside].max()))
    _report(f"icem_sample H {H} exponent {exponent} (wide bounds)", worst_free, 1e-5)
    _report(f"icem_sample H {H} exponent {exponent} (clipping bounds, unclipped elements)", worst_clip, 1e-5)


# ---- icem_append_elites ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,A,elite_num", [(10, 1, 20), (40, 17, 100), (7, 6, 47)])
@pytest.mark.parametrize("shift", [0, 1])
def test_icem_append_elites_matches_float64(H, A, elite_num, shift):
    _lib, lib = _abi()
    g = np.random.default_rng(H + A + shift)
    elite = g.standard_normal((elite_num, H, A)).astype(np.float32)
    mu = g.uniform(-0.5, 0.5, (H, A)).astype(np.float32)
    var = g.uniform(0.2, 2.0, (H, A)).astype(np.float32)
    worst = 0.0
    for keep in sorted({1, min(30, elite_num), elite_num}):
        index = g.integers(0, elite_num, keep).astype(np.int64)  # arbitrary rows, repeats allowed
        end_eps = g.standard_normal((keep, A)).astype(np.float32)
        dst = torch.full((keep + 2, H, A), -12345.0, device=DEV)  # two rows past `keep` must stay untouched
        e_d, i_d, m_d, v_d, x_d = _dev(elite, index, mu, var, end_eps)
        _lib.check(lib.b200pets_icem_append_elites(keep, H, A, _lib.ptr(e_d), _lib.ptr(i_d), shift, _lib.ptr(m_d), _lib.ptr(v_d),
                                                   _lib.ptr(x_d), 0, 0, _lib.ptr(dst), _lib.stream_ptr()), "icem_append_elites")
        got = dst.cpu().numpy()
        assert (got[keep:] == -12345.0).all()
        got = got[:keep]
        rows = elite[index]
        if not shift:
            assert np.array_equal(got.view(np.int32), rows.view(np.int32))
            continue
        assert np.array_equal(got[:, :-1].view(np.int32), rows[:, 1:].view(np.int32))
        sd = np.sqrt(var[-1].astype(np.float64))
        ref = mu[-1].astype(np.float64) + sd * end_eps
        ulp = np.spacing(np.abs(ref).astype(np.float32)) + np.spacing(sd.astype(np.float32)) * np.abs(end_eps)
        worst = max(worst, float((np.abs(got[:, -1] - ref) / ulp).max()))
    if shift:
        _report(f"icem_append end action H {H} A {A} (units: 1 ulp of the result + 1 ulp of sqrt(var) x |e|)", worst, 2.0)


# ---- mppi_sample ---------------------------------------------------------------------------------------------------
def _mppi_sample(N, H, A, beta, mean, past, lb, ub, z=None, seed=0, offset=0):
    _lib, lib = _abi()
    pop = torch.full((N, H, A), float("nan"), device=DEV)
    args = _dev(mean, past, lb, ub, z)
    _lib.check(lib.b200pets_mppi_sample(N, H, A, float(beta), *map(_lib.ptr, args), seed, offset, _lib.ptr(pop),
                                        _lib.stream_ptr()), "mppi_sample")
    return pop.cpu().numpy()


@pytest.mark.parametrize("H", [1, 2, 30, 64])
@pytest.mark.parametrize("N", [1, 127, 128, 129, 350, 5000])
def test_mppi_sample_matches_float64(N, H):
    g = np.random.default_rng(N * 100 + H)
    worst = 0.0
    for A in (1, 6, 17):
        z = np.clip(g.standard_normal((N, H, A)), -2, 2).astype(np.float32)
        mean = g.uniform(-0.5, 0.5, (H, A)).astype(np.float32)
        past = g.uniform(-1.5, 1.5, A).astype(np.float32)  # nonzero past action
        lb = (-g.uniform(0.1, 0.8, (H, A))).astype(np.float32)  # asymmetric per-(t, a) bounds that clip heavily
        ub = g.uniform(0.2, 1.2, (H, A)).astype(np.float32)
        for beta in (0.0, 0.5, 0.9, 1.0):
            v = mppi_pop64(z, mean, past, beta)
            got = _mppi_sample(N, H, A, beta, mean, past, lb, ub, z)
            tol = 1e-5 * np.maximum(1.0, np.abs(v))
            below, above = v < lb - tol, v > ub + tol
            assert np.array_equal(got[below], np.broadcast_to(lb, got.shape)[below])
            assert np.array_equal(got[above], np.broadcast_to(ub, got.shape)[above])
            worst = max(worst, float((np.abs(got - np.clip(v, lb, ub)) / np.maximum(1.0, np.abs(v))).max()))
        if N * H >= 128 * 30:
            assert below.mean() > 0.1 and above.mean() > 0.1  # the clipping is heavy at beta = 1
    _report(f"mppi_sample N {N} H {H}", worst, 1e-5)


# ---- mppi_update ---------------------------------------------------------------------------------------------------
def _mppi_values(kind, N, g):
    v = (3.0 * g.standard_normal(N)).astype(np.float32)
    if kind == "nan_neginf":
        v[g.permutation(N)[:max(1, N // 50)]] = np.nan
        v[g.permutation(N)[:max(1, N // 100)]] = -np.inf
    elif kind == "dominant":
        v[g.integers(N)] = 60.0
    elif kind == "equal":
        v[:] = np.float32(-0.75)
    elif kind == "underflow":
        v = g.uniform(-1e4, 0.0, N).astype(np.float32)
    elif kind == "posinf":
        v[g.integers(N)] = np.inf
    return v


def _mppi_update(N, dims, gamma, pop_d, vals):
    _lib, lib = _abi()
    v_d = _t(vals)
    out = torch.full((dims,), -777.0, device=DEV)
    nbytes = lib.b200pets_mppi_update_workspace_bytes(N, dims)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    _lib.check(lib.b200pets_mppi_update(N, dims, float(gamma), _lib.ptr(pop_d), _lib.ptr(v_d), _lib.ptr(out), _lib.ptr(ws),
                                        nbytes, _lib.stream_ptr()), "mppi_update")
    return v_d.cpu().numpy(), out.cpu().numpy()


KINDS = ["normal", "nan_neginf", "dominant", "equal", "underflow", "posinf"]


@pytest.mark.parametrize("dims", [1, 32, 33, 180, 1025, 2000])
@pytest.mark.parametrize("N", [1, 33, 350, 1024, 1025, 5000, 20000])
def test_mppi_update_matches_float64(N, dims):
    g = np.random.default_rng(N + 7 * dims)
    gen = torch.Generator(device=DEV).manual_seed(N * 31 + dims)
    pop_d = torch.randn(N, dims, device=DEV, generator=gen) * 1.5
    pop = pop_d.cpu().numpy().astype(np.float64)
    scale = max(1.0, float(np.abs(pop).max()))
    runs = [(k, gm) for k in KINDS for gm in (0.0, 0.9, 10.0)]
    if N * dims > 2_000_000:  # one CTA reads the whole population: keep the largest shapes to a few calls
        runs = [("nan_neginf", 0.9), ("underflow", 10.0), ("posinf", 0.9)]
    worst = 0.0
    for kind, gamma in runs:
        vals = _mppi_values(kind, N, g)
        v_after, mean = _mppi_update(N, dims, gamma, pop_d, vals)
        ref_v = np.where(np.isnan(vals), np.float32(-1e-10), vals)
        assert np.array_equal(v_after.view(np.int32), ref_v.view(np.int32)), kind  # NaN rule in place, bit-exact
        v64 = ref_v.astype(np.float64)
        with np.errstate(invalid="ignore", over="ignore"):
            w = np.exp(gamma * (v64 - v64.max()))
            ref = (w @ pop) / (w.sum() + 1e-10)
        if kind == "posinf":  # +inf - max is NaN: the reference's mean is NaN, ours must not be a finite number
            assert np.isnan(ref).all()
        # 0 * (-inf - max) is NaN as well: with gamma 0 a -inf value makes the reference's mean NaN too
        assert np.array_equal(np.isnan(mean), np.isnan(ref)), (kind, gamma, mean[:4], ref[:4])
        if np.isnan(ref).any():
            continue
        assert np.isfinite(mean).all(), (kind, gamma)
        worst = max(worst, float(np.abs(mean - ref).max()) / scale)
    _report(f"mppi_update N {N} dims {dims}", worst, 1e-5)


# ---- optimisers against the oracle -------------------------------------------------------------------------------
def _quad(target):
    return lambda pop: -((pop - target) ** 2).sum(dim=(1, 2)) + 0.3 * torch.sin(3.0 * pop).sum(dim=(1, 2))


def _close(got, ref, what, bar=2e-5):
    got = np.asarray(got, np.float64)
    ref = np.asarray(ref, np.float64)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    err = float(np.abs(got - ref).max()) / max(1.0, float(np.abs(ref).max())) if ref.size else 0.0
    assert err <= bar, f"{what}: {err:.3e} > {bar:.0e}"
    return err


class _Driven:
    """Objective pair for the GPU optimiser and the oracle: the GPU's objective records (pop, values) of every
    iteration; the oracle's asserts its population i equals the GPU's and returns the GPU's values for iteration i, so
    that both chains rank the same numbers and no elite can flip on rounding."""

    def __init__(self, gpu_obj):
        self.gpu_obj, self.trace, self.worst = gpu_obj, [], 0.0

    def gpu(self, pop):
        v = self.gpu_obj(pop)
        self.trace.append((pop.detach().cpu().numpy().copy(), v.detach().cpu().numpy().copy()))
        return v

    def oracle(self, pop, i):
        self.worst = max(self.worst, _close(self.trace[i][0], pop.numpy(), f"population {i}"))
        return torch.from_numpy(self.trace[i][1].astype(np.float64))


def _icem_noise(g, sizes, A, H, elite_num, keep, has_elite):
    """Injected draws of one call: per iteration sr / si [n_i, A, K]; a permutation of the elites whenever elites are
    kept; end_eps for the shifted kept elites of iteration 0."""
    K = H // 2 + 1
    noise = []
    for i, n in enumerate(sizes):
        d = {"sr": g.standard_normal((n, A, K)).astype(np.float32), "si": g.standard_normal((n, A, K)).astype(np.float32)}
        if has_elite or i > 0:
            d["keep_perm"] = g.permutation(elite_num).astype(np.int64)
            if i == 0:
                d["end_eps"] = g.standard_normal((min(keep, elite_num), A)).astype(np.float32)
        noise.append(d)
    return noise


def run_icem_against_oracle(H, A, pop0, elite_ratio, decay, exponent, keep_frac, iters, module, ret_mean, gpu_obj,
                            seed=0, calls=3, pop_bar=2e-5):
    import mbrl_lib_b200 as bp
    from oracle import pets_oracle as po

    g = np.random.default_rng(seed)
    lb = np.tile(g.uniform(-1.2, -0.6, A), (H, 1)).astype(np.float32)
    ub = np.tile(g.uniform(0.6, 1.2, A), (H, 1)).astype(np.float32)
    opt = bp.ICEMOptimizer(iters, elite_ratio, pop0, decay, exponent, lb.tolist(), ub.tolist(), keep_frac, 0.1, DEV,
                           return_mean_elites=ret_mean, population_size_module=module)
    sizes = opt.population_sizes()
    assert sizes == po.icem_population_sizes(iters, pop0, decay, opt.elite_num, module)
    f64 = lambda a: torch.from_numpy(np.asarray(a, np.float64))  # noqa: E731
    o_elite = None
    worst = 0.0
    for call in range(calls):
        x0 = g.uniform(-0.3, 0.3, (H, A)).astype(np.float32)
        noise = _icem_noise(g, sizes, A, H, opt.elite_num, opt.keep_elite_size, call > 0)
        drv = _Driven(gpu_obj)
        gpu_noise = [{k: _t(v) for k, v in d.items()} for d in noise]
        sol = opt.optimize(drv.gpu, x0=_t(x0), _noise=gpu_noise).cpu().numpy()
        assert len(drv.trace) == iters
        otrace = []
        o_noise = [{k: (f64(v) if v.dtype == np.float32 else torch.from_numpy(v)) for k, v in d.items()} for d in noise]
        o_sol, o_elite = po.icem_optimize(drv.oracle, f64(x0), f64(lb), f64(ub), iters, elite_ratio, pop0, decay, exponent,
                                          keep_frac, 0.1, o_noise, prev_elite=o_elite, return_mean_elites=ret_mean,
                                          module=module, trace=otrace)
        # every population pins the previous iteration's mu / var and, through keep_perm, the order of its elite set;
        # the last iteration's elite set (by descending value) and mu (the solution when return_mean_elites) directly
        assert len(otrace) == iters
        worst = max(worst, drv.worst, _close(opt.elite.cpu().numpy(), o_elite.numpy(), f"call {call} elite set, in order"),
                    _close(sol, o_sol.numpy(), f"call {call} solution"))
    print(f"iCEM H {H} A {A} pop {pop0} iters {iters}: max deviation from the float64 oracle {worst:.3e} of scale")
    assert worst <= pop_bar
    return opt


def _target(H, A, seed):
    return _t(np.random.default_rng(seed).uniform(-0.4, 0.4, (H, A)).astype(np.float32))


# (H, A, pop, elite_ratio, decay, exponent, keep_frac, iterations, module, return_mean_elites)
ICEM_CASES = {
    "pets_icem_cartpole": (10, 1, 200, 0.1, 1.3, 2.0, 0.3, 5, 7, True),
    "bench_config3": (40, 17, 1000, 0.1, 1.3, 2.0, 0.3, 5, 5, True),
    "odd_horizon": (7, 3, 120, 0.1, 1.3, 2.5, 0.3, 4, None, False),
    "one_iteration": (10, 2, 100, 0.1, 1.3, 2.0, 0.3, 1, None, False),
    "two_iterations": (10, 2, 100, 0.1, 1.3, 2.0, 0.3, 2, 5, True),
    "keep_none": (8, 2, 100, 0.1, 1.3, 1.0, 0.0, 3, None, False),
    "keep_above_elite_num": (8, 2, 30, 0.1, 1.3, 2.0, 0.5, 3, 7, False),  # elite_num 3, keep rounded up to 7
    "population_floor": (8, 2, 100, 0.1, 4.0, 2.0, 0.3, 4, None, True),  # sizes 100, 25, 20, 20: floor 2 * elite_num
}


@pytest.mark.parametrize("case", list(ICEM_CASES))
def test_icem_optimizer_matches_oracle(case):
    H, A, pop0, er, decay, beta, kf, iters, module, ret_mean = ICEM_CASES[case]
    opt = run_icem_against_oracle(H, A, pop0, er, decay, beta, kf, iters, module, ret_mean, _quad(_target(H, A, 3)),
                                  seed=list(ICEM_CASES).index(case))
    if case == "keep_above_elite_num":
        assert opt.elite_num == 3 and opt.keep_elite_size == 7
    if case == "population_floor":
        assert opt.population_sizes()[2:] == [2 * opt.elite_num] * (iters - 2)


def test_mppi_optimizer_matches_oracle():
    """pets_mppi_halfcheetah: N 350, H 30, A 6, 5 refinements, gamma 0.9, sigma 1, beta 0.9; three calls, so that the
    shifted mean and the past action are exercised."""
    import mbrl_lib_b200 as bp
    from oracle import pets_oracle as po

    N, H, A, iters, gamma, beta = 350, 30, 6, 5, 0.9, 0.9
    g = np.random.default_rng(30)
    lb = np.tile(-np.ones(A), (H, 1)).astype(np.float32)
    ub = np.tile(np.ones(A), (H, 1)).astype(np.float32)
    opt = bp.MPPIOptimizer(iters, N, gamma, 1.0, beta, lb.tolist(), ub.tolist(), DEV)
    obj = _quad(_target(H, A, 4))
    mean = torch.zeros(H, A, dtype=torch.float64)
    worst = 0.0
    for call in range(3):
        z = np.clip(g.standard_normal((iters, N, H, A)), -2, 2).astype(np.float32)
        drv = _Driven(obj)
        sol = opt.optimize(drv.gpu, _noise=_t(z)).cpu().numpy()
        otrace = []
        mean = po.mppi_optimize(drv.oracle, mean, torch.from_numpy(lb.astype(np.float64)), torch.from_numpy(ub.astype(np.float64)),
                                iters, N, gamma, beta, torch.from_numpy(z.astype(np.float64)), trace=otrace)
        assert len(drv.trace) == iters
        worst = max(worst, drv.worst, _close(sol, mean.numpy(), f"call {call} mean"))
    print(f"MPPI: max deviation from the float64 oracle {worst:.3e} of scale")


# ---- in-kernel draws against the reference's laws -------------------------------------------------------------------
def _corr(a, b):
    return float(abs(np.corrcoef(a.ravel(), b.ravel())[0, 1]))


@pytest.mark.parametrize("exponent", [0.0, 2.0])
@pytest.mark.parametrize("H", [8, 30, 41])
def test_icem_philox_spectrum_is_unit_normal(H, exponent):
    """X = rfft(y * sigma) recovers the kernel's scaled spectrum: X_k / s_k must be N(0, 1) in Re and Im for every
    frequency (Im 0 at DC and, for even H, at Nyquist), independent across parts, frequencies, action dims and
    sequences."""
    n, A = 20000, 2
    K = H // 2 + 1
    big = np.full((H, A), 1e6, np.float32)
    y = _icem_sample(n, H, A, exponent, np.zeros((H, A), np.float32), np.ones((H, A), np.float32), -big, big,
                     seed=1234, offset=77).astype(np.float64)
    s = (np.maximum(np.arange(K), 1.0) / H) ** (-exponent / 2.0)
    w = s[1:].copy()
    w[-1] *= (1 + H % 2) / 2.0
    sigma = 2.0 * np.sqrt(np.sum(w ** 2)) / H
    X = np.fft.rfft(y.transpose(0, 2, 1) * sigma, axis=-1) / s  # [n, A, K]
    bar = 4.0 / np.sqrt(n)
    pmin = 1.0
    for k in range(K):
        real_only = k == 0 or (H % 2 == 0 and k == K - 1)
        parts = [X[..., k].real] + ([] if real_only else [X[..., k].imag])
        if real_only:
            assert np.abs(X[..., k].imag).max() <= 1e-3, (k, np.abs(X[..., k].imag).max())
        for p in parts:
            pmin = min(pmin, stats.kstest(p.ravel(), "norm").pvalue)
        if not real_only:
            assert _corr(X[..., k].real, X[..., k].imag) < bar
        if k + 1 < K:
            assert _corr(X[..., k].real, X[..., k + 1].real) < bar
        assert _corr(X[:, 0, k].real, X[:, 1, k].real) < bar  # action dims
        assert _corr(X[:-1, 0, k].real, X[1:, 0, k].real) < bar  # neighbouring sequences
    print(f"icem Philox H {H} exponent {exponent}: smallest KS p-value over {2 * K} (frequency, part) pairs {pmin:.2e}")
    assert pmin > 1e-6


def test_mppi_philox_draws_are_truncated_normal():
    N, H, A, beta = 20000, 8, 4, 0.9
    g = np.random.default_rng(8)
    mean = g.uniform(-0.5, 0.5, (H, A)).astype(np.float32)
    past = g.uniform(-1, 1, A).astype(np.float32)
    big = np.full((H, A), 1e6, np.float32)
    pop = _mppi_sample(N, H, A, beta, mean, past, -big, big, seed=99, offset=5).astype(np.float64)
    prev = np.concatenate([np.broadcast_to(past, (N, 1, A)), pop[:, :-1]], axis=1)
    z = (pop - (1 - beta) * prev) / beta - mean
    assert np.abs(z).max() <= 2.0 + 1e-4
    tn = stats.truncnorm(-2.0, 2.0)
    p = stats.kstest(z.ravel(), tn.cdf).pvalue
    print(f"mppi Philox: KS p-value against N(0,1) truncated to [-2, 2] {p:.2e}")
    assert p > 1e-6
    bar = 4.0 / np.sqrt(N)
    for t in range(H - 1):
        assert _corr(z[:, t], z[:, t + 1]) < bar
    for a in range(A - 1):
        assert _corr(z[:, :, a], z[:, :, a + 1]) < bar


def test_icem_append_philox_end_action_is_normal():
    _lib, lib = _abi()
    keep, H, A = 5000, 6, 4
    g = np.random.default_rng(9)
    elite = g.standard_normal((keep, H, A)).astype(np.float32)
    mu = g.uniform(-0.5, 0.5, (H, A)).astype(np.float32)
    var = g.uniform(0.2, 2.0, (H, A)).astype(np.float32)
    dst = torch.empty(keep, H, A, device=DEV)
    e_d, m_d, v_d = _dev(elite, mu, var)
    _lib.check(lib.b200pets_icem_append_elites(keep, H, A, _lib.ptr(e_d), None, 1, _lib.ptr(m_d), _lib.ptr(v_d), None, 4321, 3,
                                               _lib.ptr(dst), _lib.stream_ptr()), "icem_append_elites")
    got = dst.cpu().numpy()
    assert np.array_equal(got[:, :-1], elite[:, 1:])  # no index vector: row j is elite j
    e = (got[:, -1].astype(np.float64) - mu[-1]) / np.sqrt(var[-1].astype(np.float64))
    p = stats.kstest(e.ravel(), "norm").pvalue
    print(f"icem_append Philox: KS p-value against N(0, 1) {p:.2e}")
    assert p > 1e-6
    for a in range(A - 1):
        assert _corr(e[:, a], e[:, a + 1]) < 4.0 / np.sqrt(keep)


# ---- iCEM over the model ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision,tol", [("f32", 2e-4), ("bf16_tc", 5e-3)])
def test_icem_over_model_matches_oracle(precision, tol):
    """bench config 3's iCEM settings (pop 1000 decaying by 1.3, 5 iterations, H 40, coloured noise exponent 2, keep 0.3,
    module 5) over the humanoid_trunc model with few particles, model draws injected through the objective: every
    iteration's values against the oracle rollout of the GPU's population, and the optimiser chain against the oracle
    driven by those values.  Its refits run cem_update's counting branch with iCEM's flags (elite set 100 x 680 floats).

    Humanoid's termination (height outside [1, 2]) makes the returns discrete: over 40 steps the tensor-core kernel's
    bf16 trajectories can cross the threshold one step away from the oracle's and zero a particle's remaining rewards.
    The fp32 kernel is held to its bar on every sequence; the tensor-core kernel to test_gpu_parity's rule for
    termination cases (at most 2 % of the sequences beyond the bar, mean deviation within 1e-2 x max(1, mean |return|))."""
    from oracle import pets_oracle as po
    from test_gpu_parity import assert_close_discrete

    spec, arrays, env = make_env("humanoid_trunc", precision, ts1="perms")
    H, P = 40, 5
    obs0 = syn.make_rollout_inputs(spec, with_noise=False)["obs0"]
    oracle = po.OracleModel(spec, arrays)
    oracle.emulate_bf16 = precision == "bf16_tc"
    g = np.random.default_rng(40)
    worst = [0.0]

    def gpu_obj(pop):
        B = pop.shape[0] * P
        perms = np.stack([g.permutation(B) for _ in range(H)]).astype(np.int64)
        eps = g.standard_normal((H, B, spec.out_size), dtype=np.float32)
        v = env.evaluate_action_sequences(pop, obs0, P, _perms=_t(perms), _eps=_t(eps))
        ref = oracle.evaluate_action_sequences(pop.cpu(), obs0, P, torch.from_numpy(perms), torch.from_numpy(eps)).numpy()
        got = v.cpu().numpy()
        diff = np.abs(got - ref) / max(1.0, float(np.abs(ref).max()))
        worst[0] = max(worst[0], float(diff.max()))
        print(f"  population {pop.shape[0]}: max {diff.max():.3e}, median {np.median(diff):.3e}, "
              f"{int((diff > tol).sum())} sequences beyond {tol:.0e}")
        if precision == "f32":
            assert diff.max() <= tol, f"values of a population of {pop.shape[0]}: {diff.max():.3e} > {tol:.0e}"
        else:
            assert_close_discrete(got, ref, P, tol=tol)
        return v

    run_icem_against_oracle(H, spec.act_dim, 1000, 0.1, 1.3, 2.0, 0.3, 5, 5, True, gpu_obj, seed=41, calls=2)
    print(f"iCEM over humanoid_trunc ({precision}): values within {worst[0]:.3e} of scale of the oracle rollout")
