"""PlaNet's three latent kernels at every rows-per-CTA tile they launch: ``latent_rollout_kernel<R>`` through
b200pets_latent_step (csrc/latent.cu), ``rssm_seq_forward_kernel<R>`` and ``rssm_seq_backward_kernel<R>`` (csrc/
latent_train.cu), R in {1, 2, 4, 8, 16, 32}.

A tile holds R rows; R is the smallest power of two >= ceil(B / SMs), at most 32, halved while R rows do not fit in the
opt-in shared memory (latent_tile).  Only R > 1 has rows past B in its last tile, splits the elementwise loops into
(row, column) and reads several rows per weight load, so every case here picks its batch from the plan queries
(b200pets_latent_plan_info, b200pets_latent_train_plan_info) on the device it runs on: for each reachable (kernel, size,
R) the smallest batch that lands on R (a nearly empty last tile) and the largest one minus 1 (a last tile one row
short), searched up to 32 x SMs, past which the rule never changes.  Sizes: PlaNet's (A 6, L 30, Hb = Hf = 200, E 1024),
an odd one (A 1, L 7, Hb 37, Hf 45, E 13) and the largest Hb = Hf each kernel family accepts at A 6, L 30 (found from
the support queries: 788 for training and 1203 for the rollout on an H100).  T is 3 except one case of PlaNet's 49 steps.

* Coverage: each kernel reaches all six tiles across the cases; the halved plans (the backward at PlaNet's size above
  16 x SMs rows, both training kernels at 788) are halved because twice their tile exceeds the opt-in shared memory.
* Training against float64 (oracle/planet_train_f64.py) with injected draws, through the ReLU masks the fp32 forward
  chose (see tests/test_gpu_latent_train.py): the five outputs (bar 1e-4 of max(1, |x|)), dP and the 13 recurrence
  gradients through random upstream gradients (bar 1e-4 relative norm).  The rollout step, sampled and deterministic,
  per column against oracle/latent_f64.py (bar 3e-5 of max(1, |column|)).  Every deviation prints as ``DEVIATION``.
  Measured on an H100 80GB HBM3 (132 SMs, 700 W power limit): states at most 1.1e-6, gradients at most 1.4e-6, the
  step at most 1.1e-6, each worst at Hb = Hf = 788 or 1203 on 8-row tiles.
* A row's bits do not depend on its tile: every sum runs in a fixed k order per column in one thread and every other
  operation is per element, so the first row of the first tile, the last row of a full tile and every row of the
  partial last tile equal, bit for bit, the same rows run alone at R = 1 (outputs, all 12 tape fields, dP; the step's
  outputs).
* Rows past B are never written: outputs, tape and dP with R spare rows of a NaN-payload sentinel stay bit-unchanged
  there, and no NaN reaches rows < B.
* In-kernel draws on multi-row tiles equal the numpy Philox of the counter layout, for every (b, t, j).
* Softplus at its threshold: the std halves of b_q2 / b_p2 spread over {-100, -30, -5, 0, 5, 25, 100}, min_std 0.1 and
  0, against float64 (torch's threshold of 20 in both) at the bars above, per column; softplus(100) would be inf in fp32
  without the threshold, and its gradient NaN.  Measured: states 1.2e-5 (beliefs, where the posterior's std reaches
  100), gradients 2.0e-6, the step 8.0e-7.
* The ABI paths Python never takes: a forward without a tape is bit-equal to the taped one, a NULL upstream gradient is
  bit-equal to a zero tensor, and ``latent_train.eval_score`` on a multi-row tile matches the float64 loss terms per
  (b, t) (1e-4 of max(1, |x|); measured 1.5e-7).

The file runs in about 25 seconds on the H100 above.
"""
import contextlib
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from mbrl_lib_b200 import _lib, latent, latent_train, models
from oracle import latent_f64 as lo
from oracle import planet_train_f64 as po
from test_gpu_latent import latent_draws64
from test_gpu_latent_train import DEC, ENC, ODD, OUTS, PLANET, _batch, _largest, _rel, train_draws64

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TILES = (1, 2, 4, 8, 16, 32)
STATE_BAR, GRAD_BAR, STEP_BAR = 1e-4, 1e-4, 3e-5
SENTINEL = 0x7FC0BEEF  # a quiet NaN with a payload no kernel produces
GRADS = ["dP", "W_e", "b_e", "W_ih", "W_hh", "b_ih", "b_hh", "W_q1", "W_q2", "b_q2", "W_p1", "b_p1", "W_p2", "b_p2"]
FWD_TAPE, BWD_TAPE = latent_train._TAPE_FWD, latent_train._TAPE_BWD
SOFTPLUS_EDGES = (-100.0, -30.0, -5.0, 0.0, 5.0, 25.0, 100.0)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _max_smem():
    return torch.cuda.get_device_properties(0).shared_memory_per_block_optin


# ---- sizes and plans -------------------------------------------------------------------------------------------------
def _train_size(name):
    if name == "largest":
        H = _largest()
        return (6, 30, H, H, 1024)
    return {"planet": PLANET, "odd": ODD}[name]


@functools.lru_cache(None)
def _rollout_largest():
    """The largest Hb = Hf that b200pets_latent_model_create accepts at A 6, L 30 (its refusal comes before it reads a
    weight; an accepted size is staged from one zero buffer)."""
    lib = _lib.load()
    hi_ = 2048
    buf = torch.zeros(3 * hi_ * (hi_ + 32), device=DEV)
    ptrs = (C.c_void_p * 16)(*[buf.data_ptr()] * 16)
    d = _lib.LatentDesc(6, 30, 0, 0, 0.1)
    lo_, hi = 1, hi_
    while lo_ < hi:
        mid = (lo_ + hi + 1) // 2
        d.belief_size = d.hidden_size = mid
        h = C.c_void_p()
        ok = lib.b200pets_latent_model_create(C.byref(d), ptrs, _lib.stream_ptr(), C.byref(h)) == 0
        if ok:
            lib.b200pets_latent_model_destroy(h)
        lo_, hi = (mid, hi) if ok else (lo_, mid - 1)
    torch.cuda.synchronize()
    assert lo_ < hi_
    return lo_


def _rollout_size(name):
    if name == "largest":
        H = _rollout_largest()
        return (6, 30, H, H)
    return {"planet": PLANET[:4], "odd": ODD[:4]}[name]


def _desc(size, min_std=0.1):
    return _lib.LatentTrainDesc(*size, min_std)


def _train_plan(size, B, backward):
    info = (C.c_int32 * 4)()
    _lib.check(_lib.load().b200pets_latent_train_plan_info(C.byref(_desc(size)), B, int(backward), info))
    return {"rows": info[0], "ctas": info[1], "smem": info[2], "row_bytes": info[3]}


@functools.lru_cache(None)
def _staged(size):
    """The rollout's staged model at ``size`` (its source is ``.src``), shared by the tests and the plan queries."""
    return latent.StagedLatentModel(_rollout_model(size))


def _rollout_plan(size, B):
    p = _staged(size).plan_info(B)
    return {"rows": p["rows_per_cta"], "ctas": p["ctas"], "smem": p["smem"], "row_bytes": p["row_bytes"]}


def _plan(kernel, size, B):
    return _rollout_plan(size, B) if kernel == "rollout" else _train_plan(size, B, kernel == "backward")


@functools.lru_cache(None)
def _tile_of_batch(kernel, size):
    """R for every batch 1 .. 32 x SMs: past 32 x SMs the tile never changes."""
    return [_plan(kernel, size, B)["rows"] for B in range(1, 32 * _sms() + 1)]


def _batches(kernel, size, R):
    """The smallest batch that lands on tile R and the largest (up to 32 x SMs) minus 1; [] when R is never launched."""
    Bs = [B for B, r in enumerate(_tile_of_batch(kernel, size), start=1) if r == R]
    if not Bs:
        return []
    return sorted({Bs[0], max(Bs[-1] - 1, 1)})


def _train_batches(size, R):
    return sorted(set(_batches("forward", size, R)) | set(_batches("backward", size, R)))


def _wanted(B):
    R = 1
    while R < -(-B // _sms()) and R < 32:
        R *= 2
    return R


def _rows_to_check(B, tiles):
    """The first row of the first tile, the last row of a full tile and every row of the partial last tile, per tile."""
    rows = {0}
    for R in tiles:
        if B >= R:
            rows.add(R - 1)
        rows |= set(range(B - B % R, B))
    return sorted(rows)


# ---- models and calls ------------------------------------------------------------------------------------------------
def _train_model(size, seed=0, min_std=0.1, rng_seed=None):
    A, L, Hb, Hf, E = size
    torch.manual_seed(seed)
    rng = None
    if rng_seed is not None:
        rng = torch.Generator(device=DEV)
        rng.manual_seed(rng_seed)
    return models.PlaNetModel(A, L, Hb, Hf, device=DEV, obs_shape=(3, 16, 16), obs_encoding_size=E, encoder_config=ENC,
                              decoder_config=DEC, min_std=min_std, rng=rng)


def _rollout_model(size, seed=0, min_std=0.1):
    A, L, Hb, Hf = size
    torch.manual_seed(seed)
    return models.PlaNetModel(A, L, Hb, Hf, device=DEV, min_std=min_std)


def _inputs(size, B, T, seed):
    A, L, _, Hf, _ = size
    g = np.random.default_rng(seed)
    P = torch.from_numpy(0.5 * g.standard_normal((B, T, Hf))).float()
    act = torch.from_numpy(np.clip(g.standard_normal((B, T, A)), -1, 1)).float()
    eq, ep = (torch.from_numpy(g.standard_normal((T, B, L))).float() for _ in range(2))
    return P, act, eq, ep


def _ups(size, B, T, seed):
    _, L, Hb, _, _ = size
    g = np.random.default_rng(seed)
    return [torch.from_numpy(g.standard_normal((B, T, w))).float() for w in (Hb, 2 * L, L, 2 * L, L)]


def _buf(shape, fill):
    if fill is None:
        return torch.empty(shape, device=DEV)
    return torch.full(shape, fill, dtype=torch.int32, device=DEV).view(torch.float32)


def _widths(desc):
    L, Hb, Hf = desc.latent_size, desc.belief_size, desc.hidden_size
    return dict(e=Hb, gates=4 * Hb, q1=Hf, p1=Hf, pre_std=2 * L, eps=2 * L, de=Hb, dgi=3 * Hb, dghn=Hb, dq=2 * L, dv=Hf,
                dp=2 * L)


def _forward(model, P, act, eps, *, seed=0, offset=0, spare=0, fill=None, tape=True):
    """b200pets_latent_seq_forward for the B rows of P: the five outputs and the 12 tape fields, each [B + spare, T, w]
    (the spare rows filled with ``fill``'s bits)."""
    lib = _lib.load()
    d = latent_train.train_desc(model)
    B, T = P.shape[:2]
    L, Hb = d.latent_size, d.belief_size
    params = latent_train.recurrence_params(model)
    ptrs = (C.c_void_p * len(params))(*[p.data_ptr() for p in params])
    out = [_buf((B + spare, T, w), fill) for w in (Hb, 2 * L, L, 2 * L, L)]
    tp = {k: _buf((B + spare, T, w), fill) for k, w in _widths(d).items()}
    t = _lib.LatentTape(*[tp[k].data_ptr() for k in FWD_TAPE + BWD_TAPE])
    ws = torch.empty(lib.b200pets_latent_train_workspace_bytes(C.byref(d), B, T), dtype=torch.uint8, device=DEV)
    eq, ep = eps if eps is not None else (None, None)
    _lib.check(lib.b200pets_latent_seq_forward(C.byref(d), ptrs, B, T, _lib.ptr(P), _lib.ptr(act), _lib.ptr(eq),
                                               _lib.ptr(ep), seed, offset, *[_lib.ptr(o) for o in out],
                                               C.byref(t) if tape else None, _lib.ptr(ws), ws.numel(),
                                               _lib.stream_ptr()))
    torch.cuda.synchronize()
    return out, tp


def _backward(model, B, out, tp, ups, *, spare=0, fill=None):
    """b200pets_latent_seq_backward for B rows after :func:`_forward`: dP [B + spare, T, Hf] (the tape's backward
    fields are written in place)."""
    lib = _lib.load()
    d = latent_train.train_desc(model)
    T = out[0].shape[1]
    params = latent_train.recurrence_params(model)
    ptrs = (C.c_void_p * len(params))(*[p.data_ptr() for p in params])
    t = _lib.LatentTape(*[tp[k].data_ptr() for k in FWD_TAPE + BWD_TAPE])
    dP = _buf((B + spare, T, d.hidden_size), fill)
    _lib.check(lib.b200pets_latent_seq_backward(C.byref(d), ptrs, B, T, _lib.ptr(out[0]), *[_lib.ptr(u) for u in ups],
                                                C.byref(t), _lib.ptr(dP), _lib.stream_ptr()))
    torch.cuda.synchronize()
    return dP


def _dev(*xs):
    return [None if x is None else x.to(DEV) for x in xs]


def _step(staged, B, s, h, a, eps, sample, *, seed=0, offset=0, spare=0, fill=None):
    """b200pets_latent_step for B rows: (next_latent [B + spare, L], next_belief [B + spare, Hb], reward [B + spare])."""
    d = staged.desc
    outs = [_buf((B + spare, d.latent_size), fill), _buf((B + spare, d.belief_size), fill), _buf((B + spare,), fill)]
    _lib.check(staged.lib.b200pets_latent_step(staged.handle, B, _lib.ptr(s), _lib.ptr(h), _lib.ptr(a), _lib.ptr(eps),
                                               seed, offset, int(sample), *[_lib.ptr(o) for o in outs],
                                               _lib.stream_ptr()))
    torch.cuda.synchronize()
    return outs


def _step_inputs(size, B, seed):
    A, L, Hb, _ = size
    g = np.random.default_rng(seed)
    return (g.standard_normal((B, L)).astype(np.float32), np.tanh(g.standard_normal((B, Hb))).astype(np.float32),
            np.clip(g.standard_normal((B, A)), -1, 1).astype(np.float32), g.standard_normal((B, L)).astype(np.float32))


@contextlib.contextmanager
def _no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _col_err(got, want):
    """Worst column of max |got - want| / max(1, max |want column|) over the last axis."""
    got = got.detach().double().cpu().reshape(-1, want.shape[-1] if want.dim() > 1 else 1)
    want = want.detach().double().cpu().reshape(got.shape)
    return float(((got - want).abs().amax(0) / want.abs().amax(0).clamp(min=1.0)).max())


def _bits(x):
    return x.contiguous().view(torch.int32)


# ---- a: coverage -----------------------------------------------------------------------------------------------------
def test_every_tile_is_covered():
    """Every kernel reaches all six tiles across the cases below, and each plan below its wanted tile is halved for
    shared memory: twice its tile would not fit in the opt-in shared memory of a CTA."""
    sms, max_smem = _sms(), _max_smem()
    reached = {"forward": set(), "backward": set(), "rollout": set()}
    halved = set()
    print(f"\n{sms} SMs, {max_smem} bytes of opt-in shared memory per CTA")
    print(f"{'kernel':9s} {'size':8s} {'B':>6s} {'R':>3s} {'CTAs':>5s} {'row bytes':>9s} halved")
    for kernel in ("forward", "backward", "rollout"):
        for name in ("planet", "odd", "largest"):
            size = _rollout_size(name) if kernel == "rollout" else _train_size(name)
            Bs = sorted({B for R in TILES for B in (_batches(kernel, size, R) if kernel == "rollout"
                                                     else _train_batches(size, R))})
            for B in Bs:
                p = _plan(kernel, size, B)
                R = p["rows"]
                reached[kernel].add(R)
                assert p["ctas"] == -(-B // R) and p["smem"] >= R * p["row_bytes"], (kernel, name, B, p)
                cut = R < _wanted(B)
                if cut:
                    assert 2 * R * p["row_bytes"] > max_smem, (kernel, name, B, p)
                    halved.add((kernel, name, B))
                else:
                    assert R == _wanted(B), (kernel, name, B, p)
                print(f"{kernel:9s} {name:8s} {B:6d} {R:3d} {p['ctas']:5d} {p['row_bytes']:9d} {'halved' if cut else ''}")
    for kernel, tiles in reached.items():
        assert tiles == set(TILES), (kernel, sorted(tiles))
    for B in range(16 * sms + 1, 32 * sms + 1, 97):
        assert _train_plan(PLANET, B, True)["rows"] == 16 and _train_plan(PLANET, B, False)["rows"] == 32, B
    big = _train_size("largest")
    for backward in (False, True):
        assert _train_plan(big, 32 * sms, backward)["rows"] == 8, backward
    assert any(k == "backward" and n == "planet" for k, n, _ in halved)
    assert {k for k, n, _ in halved if n == "largest"} >= {"forward", "backward"}


def test_train_plan_info_refusals():
    lib = _lib.load()
    info = (C.c_int32 * 4)()
    d = _desc(PLANET)
    assert lib.b200pets_latent_train_plan_info(C.byref(d), 1, 0, info) == 0 and info[0] == 1 and info[1] == 1
    assert lib.b200pets_latent_train_plan_info(C.byref(d), 0, 0, info) == -1
    assert lib.b200pets_latent_train_plan_info(None, 5, 0, info) == -1
    assert lib.b200pets_latent_train_plan_info(C.byref(d), 5, 1, None) == -1
    H = _largest()
    d.belief_size = d.hidden_size = H + 1
    assert lib.b200pets_latent_train_plan_info(C.byref(d), 5, 1, info) == -2
    d.belief_size = 0
    assert lib.b200pets_latent_train_plan_info(C.byref(d), 5, 0, info) == -1


# ---- b: against float64 ----------------------------------------------------------------------------------------------
def _check_train_f64(tag, model, size, B, T, seed):
    P, act, eq, ep = _inputs(size, B, T, seed)
    ups = _ups(size, B, T, seed + 1)
    Pd, actd = _dev(P, act)
    out, tp = _forward(model, Pd, actd, _dev(eq, ep))
    dP = _backward(model, B, out, tp, _dev(*ups))
    params = latent_train.recurrence_params(model)
    with _no_tf32():
        got_g = [dP] + latent_train.weight_grads(tp, dP, actd, out[0], out[2], params[6])
    masks = {k: (tp[k] > 0).double().cpu() for k in ("e", "q1", "p1")}
    m64 = po.as_f64(model)
    P64 = P.double().requires_grad_()
    want = po.forward(m64, None, act.double(), eq.double(), ep.double(), P=P64, masks=masks)
    for k, got in zip(OUTS, out):
        err = _col_err(got, want[k])
        print(f"DEVIATION {tag} {k} {err:.2e}")
        assert err <= STATE_BAR, f"{tag} {k}: {err:.2e}"
    want_g = torch.autograd.grad(sum((want[k] * u.double()).sum() for k, u in zip(OUTS, ups)),
                                 [P64] + latent_train.recurrence_params(m64))
    for n, a, b in zip(GRADS, got_g, want_g):
        rel = _rel(a, b)
        print(f"DEVIATION {tag} grad_{n} {rel:.2e}")
        assert rel <= GRAD_BAR, f"{tag} grad {n}: {rel:.2e}"


@pytest.mark.parametrize("R", TILES)
@pytest.mark.parametrize("name", ["planet", "odd", "largest"])
def test_training_kernels_match_float64(name, R):
    size = _train_size(name)
    Bs = _train_batches(size, R)
    if not Bs:
        pytest.skip(f"neither training kernel launches {R}-row tiles at Hb = Hf = {size[2]}")
    model = _train_model(size)
    for B in Bs:
        tiles = (_train_plan(size, B, False)["rows"], _train_plan(size, B, True)["rows"])
        assert R in tiles
        _check_train_f64(f"{name}_B{B}_R{tiles[0]}/{tiles[1]}_T3", model, size, B, 3, seed=B)


def test_training_kernels_match_float64_over_49_steps():
    """PlaNet's sequence length on a multi-row tile of both kernels."""
    B = 2 * _sms() + 36
    assert _train_plan(PLANET, B, False)["rows"] == 4 and _train_plan(PLANET, B, True)["rows"] == 4
    _check_train_f64(f"planet_B{B}_R4_T49", _train_model(PLANET), PLANET, B, 49, seed=49)


@pytest.mark.parametrize("R", TILES)
@pytest.mark.parametrize("name", ["planet", "odd", "largest"])
def test_step_matches_float64(name, R):
    size = _rollout_size(name)
    Bs = _batches("rollout", size, R)
    if not Bs:
        pytest.skip(f"the rollout never launches {R}-row tiles at Hb = Hf = {size[2]}")
    staged = _staged(size)
    p = lo.params_of(staged.src)
    for B in Bs:
        assert _rollout_plan(size, B)["rows"] == R
        s, h, a, e = _step_inputs(size, B, seed=B)
        for sample in (False, True):
            got = _step(staged, B, *_dev(*(torch.from_numpy(x) for x in (s, h, a, e))), sample)
            want = lo.step(p, s, h, a, e if sample else None)
            for what, g, w in zip(("latent", "belief", "reward"), got, want):
                err = _col_err(g, torch.from_numpy(np.asarray(w)))
                print(f"DEVIATION step_{name}_B{B}_R{R}_{'sampled' if sample else 'mean'} {what} {err:.2e}")
                assert err <= STEP_BAR, (name, B, R, sample, what, err)


# ---- c: a row's bits do not depend on its tile -----------------------------------------------------------------------
@pytest.mark.parametrize("R", TILES[1:])
@pytest.mark.parametrize("name", ["planet", "odd", "largest"])
def test_training_rows_are_bit_equal_across_tiles(name, R):
    size = _train_size(name)
    Bs = _train_batches(size, R)
    if not Bs:
        pytest.skip(f"neither training kernel launches {R}-row tiles at Hb = Hf = {size[2]}")
    model = _train_model(size)
    T = 3
    for B in Bs:
        tiles = (_train_plan(size, B, False)["rows"], _train_plan(size, B, True)["rows"])
        rows = _rows_to_check(B, tiles)
        k = len(rows)
        assert _train_plan(size, k, False)["rows"] == 1 and _train_plan(size, k, True)["rows"] == 1
        P, act, eq, ep = _inputs(size, B, T, seed=B)
        ups = _ups(size, B, T, seed=B + 1)
        out, tp = _forward(model, *_dev(P, act), _dev(eq, ep))
        dP = _backward(model, B, out, tp, _dev(*ups))
        idx = torch.tensor(rows)
        out1, tp1 = _forward(model, *_dev(P[idx], act[idx]), _dev(eq[:, idx].contiguous(), ep[:, idx].contiguous()))
        dP1 = _backward(model, k, out1, tp1, _dev(*(u[idx] for u in ups)))
        sel = idx.to(DEV)
        for what, a, b in [*zip(OUTS, out, out1), *((f, tp[f], tp1[f]) for f in FWD_TAPE + BWD_TAPE), ("dP", dP, dP1)]:
            assert torch.equal(_bits(a[sel]), _bits(b)), f"{name} B={B} tiles {tiles}: {what} of rows {rows} differs " \
                                                         f"from the same rows at R = 1"


@pytest.mark.parametrize("R", TILES[1:])
@pytest.mark.parametrize("name", ["planet", "odd", "largest"])
def test_step_rows_are_bit_equal_across_tiles(name, R):
    size = _rollout_size(name)
    Bs = _batches("rollout", size, R)
    if not Bs:
        pytest.skip(f"the rollout never launches {R}-row tiles at Hb = Hf = {size[2]}")
    staged = _staged(size)
    for B in Bs:
        rows = _rows_to_check(B, (R,))
        assert _rollout_plan(size, len(rows))["rows"] == 1
        idx = torch.tensor(rows)
        xs = [torch.from_numpy(x) for x in _step_inputs(size, B, seed=B)]
        for sample in (False, True):
            full = _step(staged, B, *_dev(*xs), sample)
            alone = _step(staged, len(rows), *_dev(*(x[idx] for x in xs)), sample)
            for what, a, b in zip(("latent", "belief", "reward"), full, alone):
                assert torch.equal(_bits(a[idx.to(DEV)]), _bits(b)), (name, B, R, sample, what, rows)


# ---- d: rows past B are never written --------------------------------------------------------------------------------
def _spare_ok(what, x, B):
    bad = x[B:].contiguous().view(torch.int32) != SENTINEL
    assert not bad.any(), f"{what}: {int(bad.sum())} words past row {B} were written"
    assert not torch.isnan(x[:B]).any(), f"{what}: NaN in rows < {B} (a row not written, or a sentinel read)"


@pytest.mark.parametrize("name", ["planet", "odd", "largest"])
def test_training_kernels_write_no_row_past_the_batch(name):
    size = _train_size(name)
    model = _train_model(size)
    T = 2
    for R in TILES[1:]:
        for B in _train_batches(size, R):
            spare = _train_plan(size, B, False)["rows"]
            P, act, _, _ = _inputs(size, B, T, seed=B)
            ups = _ups(size, B, T, seed=B + 1)
            out, tp = _forward(model, *_dev(P, act), None, seed=99, offset=B, spare=spare, fill=SENTINEL)
            dP = _backward(model, B, out, tp, _dev(*ups), spare=spare, fill=SENTINEL)
            for what, x in [*zip(OUTS, out), *tp.items(), ("dP", dP)]:
                _spare_ok(f"{name} B={B} {what}", x, B)


@pytest.mark.parametrize("name", ["planet", "odd", "largest"])
def test_step_writes_no_row_past_the_batch(name):
    size = _rollout_size(name)
    staged = _staged(size)
    for R in TILES[1:]:
        for B in _batches("rollout", size, R):
            s, h, a, _ = (torch.from_numpy(x) for x in _step_inputs(size, B, seed=B))
            for sample in (False, True):
                outs = _step(staged, B, *_dev(s, h, a), None, sample, seed=7, offset=B, spare=R, fill=SENTINEL)
                for what, x in zip(("latent", "belief", "reward"), outs):
                    _spare_ok(f"{name} B={B} sample={sample} {what}", x, B)


# ---- e: in-kernel draws on multi-row tiles ---------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["planet", "odd"])
def test_training_draws_on_multi_row_tiles(name):
    size = _train_size(name)
    model = _train_model(size)
    L, T = size[1], 3
    seed, offset = 0x0123_4567_89AB_CDEF, (5 << 32) + 12
    for R in TILES[1:]:
        B = _batches("forward", size, R)[0]  # a last tile of one row
        P, act, _, _ = _inputs(size, B, T, seed=B)
        _, tp = _forward(model, *_dev(P, act), None, seed=seed, offset=offset)
        eps = tp["eps"].double().cpu().numpy()
        for kind in (0, 1):
            want = train_draws64(B, T, L, kind, seed, offset)
            err = float(np.abs(eps[..., kind * L:(kind + 1) * L] - want).max())
            assert err <= 2e-5 * max(1.0, float(np.abs(want).max())), (name, B, R, kind, err)


@pytest.mark.parametrize("name", ["planet", "odd"])
def test_step_draws_on_multi_row_tiles(name):
    size = _rollout_size(name)
    staged = _staged(size)
    p = lo.params_of(staged.src)
    seed, offset = 0x0FED_CBA9_8765_4321, (9 << 32) + 1024 * 3
    for R in TILES[1:]:
        for B in _batches("rollout", size, R):
            s, h, a, _ = _step_inputs(size, B, seed=B)
            got = _step(staged, B, *_dev(*(torch.from_numpy(x) for x in (s, h, a))), None, True, seed=seed,
                        offset=offset)
            want = lo.step(p, s, h, a, latent_draws64(B, size[1], 0, seed, offset))
            for what, g, w in zip(("latent", "belief", "reward"), got, want):
                err = _col_err(g, torch.from_numpy(np.asarray(w)))
                assert err <= STEP_BAR, (name, B, R, what, err)


# ---- f: softplus at its threshold ------------------------------------------------------------------------------------
def _spread_std_bias(bias, L):
    with torch.no_grad():
        for j in range(L):
            bias[L + j] = SOFTPLUS_EDGES[j % len(SOFTPLUS_EDGES)]


@pytest.mark.parametrize("min_std", [0.1, 0.0])
def test_training_softplus_edges(min_std):
    model = _train_model(PLANET, seed=2, min_std=min_std)
    L = PLANET[1]
    _spread_std_bias(model.posterior_transition_model[2].bias, L)
    _spread_std_bias(model.prior_transition_model[2].bias, L)
    B = _batches("forward", PLANET, 2)[0]
    _check_train_f64(f"softplus_min_std{min_std}_B{B}", model, PLANET, B, 3, seed=5)


@pytest.mark.parametrize("min_std", [0.1, 0.0])
def test_step_softplus_edges(min_std):
    size = PLANET[:4]
    model = _rollout_model(size, seed=2, min_std=min_std)
    _spread_std_bias(model.prior_transition_model[2].bias, size[1])
    staged = latent.StagedLatentModel(model)
    p = lo.params_of(model)
    B = _batches("rollout", size, 2)[0]
    s, h, a, e = _step_inputs(size, B, seed=3)
    got = _step(staged, B, *_dev(*(torch.from_numpy(x) for x in (s, h, a, e))), True)
    want = lo.step(p, s, h, a, e)
    for what, g, w in zip(("latent", "belief", "reward"), got, want):
        err = _col_err(g, torch.from_numpy(np.asarray(w)))
        print(f"DEVIATION step_softplus_min_std{min_std} {what} {err:.2e}")
        assert err <= STEP_BAR, (what, err)


# ---- g: the ABI paths Python never takes -----------------------------------------------------------------------------
@pytest.mark.parametrize("R", [1, 8])
def test_forward_without_a_tape_equals_the_taped_forward(R):
    B = _batches("forward", PLANET, R)[-1]
    model = _train_model(PLANET)
    P, act, eq, ep = _inputs(PLANET, B, 3, seed=R)
    for eps in (_dev(eq, ep), None):
        taped, _ = _forward(model, *_dev(P, act), eps, seed=3, offset=8)
        bare, _ = _forward(model, *_dev(P, act), eps, seed=3, offset=8, tape=False)
        for what, a, b in zip(OUTS, taped, bare):
            assert torch.equal(_bits(a), _bits(b)), (R, eps is None, what)


@pytest.mark.parametrize("R", [1, 4])
def test_null_upstream_gradients_equal_zeros(R):
    B = _batches("backward", ODD, R)[0]
    model = _train_model(ODD)
    P, act, eq, ep = _inputs(ODD, B, 3, seed=R)
    ups = _dev(*_ups(ODD, B, 3, seed=R + 1))
    out, tp = _forward(model, *_dev(P, act), _dev(eq, ep))
    for i, what in enumerate(OUTS):
        with_zero = list(ups)
        with_zero[i] = torch.zeros_like(ups[i])
        with_null = list(ups)
        with_null[i] = None
        dP0 = _backward(model, B, out, tp, with_zero)
        t0 = {k: tp[k].clone() for k in BWD_TAPE}
        dPn = _backward(model, B, out, tp, with_null)
        assert torch.equal(_bits(dP0), _bits(dPn)), (R, what, "dP")
        for k in BWD_TAPE:
            assert torch.equal(_bits(t0[k]), _bits(tp[k])), (R, what, k)


def test_eval_score_on_a_multi_row_tile_matches_float64():
    """latent_train.eval_score runs the forward kernel without a tape and with in-kernel draws: the draws come from
    the numpy Philox at the model rng's (seed, offset), the convolutions in float64 on the oracle's side."""
    S = 3
    B = _batches("forward", PLANET, 2)[0]
    model = _train_model(PLANET, seed=6, rng_seed=21)
    batch = _batch(model, B, S, seed=8)
    seed, offset = int(model.rng.initial_seed()), int(model.rng.get_offset())
    with _no_tf32():
        score, _ = latent_train.eval_score(model, batch)
    L = PLANET[1]
    eq, ep = (torch.from_numpy(train_draws64(B, S - 1, L, k, seed, offset)).permute(1, 0, 2) for k in (0, 1))
    m64 = po.as_f64(model)
    with torch.no_grad():
        obs = torch.from_numpy(batch.obs).double() / 256.0 - 0.5
        o, r, k, _ = po.loss_terms(m64, obs, torch.from_numpy(batch.act).double(),
                                   torch.from_numpy(batch.rewards).double(), eq, ep)
        want = o + r + m64.kl_scale * k
    got = score.double().cpu()
    assert got.shape == want.shape == (B, S - 1)
    err = float(((got - want).abs() / want.abs().clamp(min=1.0)).max())
    print(f"DEVIATION eval_score_B{B} loss {err:.2e}")
    assert err <= 1e-4, err
