"""Training PlaNet's latent model on the device (csrc/latent_train.cu, mbrl_lib_b200/latent_train.py) against the float64
restatement of the reference's per-step loop (oracle/planet_train_f64.py).

* Forward (b200pets_latent_seq_forward) with injected draws: the five outputs of every step against float64 at PlaNet's
  sizes (A 6, L 30, Hb = Hf = 200, encoding 1024), an odd size (A 1, L 7, Hb 37, Hf 45, encoding 13) and the largest
  Hb = Hf the row limit accepts at A 6, L 30 (788), with (B, T) in {(1, 1), (3, 2), (50, 49)}.  Measured at most
  6.1e-7; bar: 1e-4 of max(1, |x|).
* Backward: dP and every recurrence parameter's gradient through random upstream gradients, against float64 autograd
  through the ReLU masks the fp32 forward chose.  Bar: 1e-4 relative norm per tensor.  Where no mask differs from
  float64's own, the plain float64 gradient is held to the same bar.  Where one does, the plain comparison is not held to
  it: a pre-activation within rounding of 0 that fp32 and float64 place on opposite sides passes or blocks that
  element's whole gradient, so its dP entry differs by its full size (the largest size at B 50, T 49 has such elements
  and a plain dP deviation of 2.3e-4), which says nothing about the kernels' arithmetic.
* One full ``update`` (the convolutions in float64 on the oracle's side, TF32 off on ours) against the float64 oracle:
  the loss terms, every parameter's clipped gradient (1e-4 relative norm) and the parameters after the Adam step.
* In-kernel draws equal a numpy Philox of the RNG_STREAM_LATENT_TRAIN counter layout (common.cuh).
* Both kernels are bit-identical across two runs.
* Drop-in: ``ModelTrainer.train(dataset, num_epochs=1, batch_callback=cb, evaluate=False)`` as
  mbrl/algorithms/planet.py:144-146 calls it, over the container with a list of sequence batches and over the
  reference's PlaNetModel with its replay buffer's sequence sampler (skipped without oracle/_ref); ``LatentModelEnv``
  plans with the new weights afterwards.  A model the kernels refuse trains through the reference's own ``update``.
* 100 updates against the reference's own fp32 ``PlaNetModel.update`` on cuda (TF32 off), same weights and draws, at
  A 6, L 30, Hb = Hf = 200: the parameters' distance relative to the reference's parameter movement, over all
  parameters and per tensor.  Measured 9.4e-7 to 9.5e-7 overall and 1.2e-6 to 2.4e-6 on the worst tensor.  The control
  is the reference's fp32 run against the float64 oracle over the same updates: 0.083 to 0.25 overall and 0.25 to 0.39
  on the worst tensor (cuDNN's fp32 convolutions are not bit-identical from run to run).  Adam
  moves a parameter whose gradient hovers near 0 by a full step in the direction of its sign, so rounding alone can
  carry such a tensor a long way; another draw set moved that bias 0.41 between the device path and the reference.
  Bar: twice the control, so the device path may not drift from the reference further than fp32 rounding carries the
  reference from float64.
"""
import ctypes as C
import importlib
import types

import numpy as np
import pytest
import torch

import mbrl_lib_b200 as bp
from baseline import reference_arm as ra
from mbrl_lib_b200 import _lib, functions, latent_train, models
from oracle import planet_train_f64 as po

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
mbrl, REF_SRC = ra.import_reference()
needs_ref = pytest.mark.skipif(mbrl is None, reason=f"reference not importable here: {REF_SRC}")

STATE_BAR, GRAD_BAR = 1e-4, 1e-4
RNG_STREAM_LATENT_TRAIN = 0x80000
ENC = ((3, 8, 4, 2), (8, 16, 4, 2))  # 3 x 16 x 16 frames -> 16 x 2 x 2
DEC = ((32, 1, 1), ((32, 16, 5, 2), (16, 8, 5, 2), (8, 3, 4, 1)))  # -> 3 x 16 x 16
PLANET, ODD = (6, 30, 200, 200, 1024), (1, 7, 37, 45, 13)


def _largest():
    """The largest Hb = Hf that b200pets_latent_train_supported accepts at A 6, L 30."""
    lib = _lib.load()
    d = _lib.LatentTrainDesc(6, 30, 0, 0, 1024, 0.1)
    lo_, hi = 1, 4096
    while lo_ < hi:
        mid = (lo_ + hi + 1) // 2
        d.belief_size = d.hidden_size = mid
        lo_, hi = (mid, hi) if lib.b200pets_latent_train_supported(C.byref(d)) == 0 else (lo_, mid - 1)
    return lo_


def _model(size, seed=0, rng_seed=None):
    A, L, Hb, Hf, E = size
    torch.manual_seed(seed)
    rng = None
    if rng_seed is not None:
        rng = torch.Generator(device=DEV)
        rng.manual_seed(rng_seed)
    return models.PlaNetModel(A, L, Hb, Hf, device=DEV, obs_shape=(3, 16, 16), obs_encoding_size=E, encoder_config=ENC,
                              decoder_config=DEC, rng=rng)


def _inputs(model, B, T, seed):
    g = np.random.default_rng(seed)
    A, L, Hf = model.action_size, model.latent_state_size, model.prior_transition_model[0].out_features
    P = torch.from_numpy(0.5 * g.standard_normal((B, T, Hf))).float()
    act = torch.from_numpy(np.clip(g.standard_normal((B, T, A)), -1, 1)).float()
    eq, ep = (torch.from_numpy(g.standard_normal((T, B, L))).float() for _ in range(2))
    return P, act, eq, ep


def _err(got, want):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    return float((got - want).abs().max() / max(1.0, float(want.abs().max())))


def _rel(got, want):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    return float((got - want).norm() / max(float(want.norm()), 1e-30))


OUTS = ("beliefs", "post_params", "post_samples", "prior_params", "prior_samples")
CASES = [(s, B, T) for s in ("planet", "odd", "largest") for (B, T) in ((1, 1), (3, 2), (50, 49))]


def _size(name):
    if name == "largest":
        H = _largest()
        return (6, 30, H, H, 1024)
    return {"planet": PLANET, "odd": ODD}[name]


@pytest.mark.parametrize("name,B,T", CASES)
def test_forward_and_backward_match_float64(name, B, T):
    model = _model(_size(name))
    P, act, eq, ep = _inputs(model, B, T, seed=B * 100 + T)
    Pd = P.to(DEV).requires_grad_()
    out = latent_train.recurrence(model, Pd, act.to(DEV), eps=(eq, ep))
    m64 = po.as_f64(model)
    P64 = P.double().requires_grad_()
    pre = {}
    want = po.forward(m64, None, act.double(), eq.double(), ep.double(), P=P64, pre=pre)
    for k, got in zip(OUTS, out):
        err = _err(got, want[k])
        print(f"{name} B={B} T={T} {k}: {err:.2e}")
        assert err <= STATE_BAR, f"{name} B={B} T={T} {k}: {err:.2e}"
    g = np.random.default_rng(7)
    ups = [torch.from_numpy(g.standard_normal(tuple(o.shape))) for o in out]
    params = latent_train.recurrence_params(model)
    got = torch.autograd.grad(sum((o * u.float().to(DEV)).sum() for o, u in zip(out, ups)), [Pd] + params)
    # the ReLU masks the kernel's fp32 forward chose (the forward is bit-deterministic, so a second call chooses the same)
    _, tape, _ = _raw(model, P.to(DEV), act.to(DEV), (eq.to(DEV), ep.to(DEV)), 0, 0, [None] * 5)
    masks = {k: (tape[k] > 0).double().cpu() for k in ("e", "q1", "p1")}
    flips = {k: int(((pre[k] > 0).double() != masks[k]).sum()) for k in masks}
    print(f"{name} B={B} T={T} ReLU masks that differ from float64's: {flips}")
    P64m = P.double().requires_grad_()
    m64m = po.as_f64(model)
    wm = po.forward(m64m, None, act.double(), eq.double(), ep.double(), P=P64m, masks=masks)
    want_m = torch.autograd.grad(sum((wm[k] * u).sum() for k, u in zip(OUTS, ups)),
                                 [P64m] + latent_train.recurrence_params(m64m))
    want_g = torch.autograd.grad(sum((want[k] * u).sum() for k, u in zip(OUTS, ups)),
                                 [P64] + latent_train.recurrence_params(m64))
    names = ["dP", "W_e", "b_e", "W_ih", "W_hh", "b_ih", "b_hh", "W_q1", "W_q2", "b_q2", "W_p1", "b_p1", "W_p2", "b_p2"]
    for n, a, b, c in zip(names, got, want_m, want_g):
        rel, rel_plain = _rel(a, b), _rel(a, c)
        print(f"{name} B={B} T={T} grad {n}: {rel:.2e} (through float64's own masks {rel_plain:.2e})")
        assert rel <= GRAD_BAR, f"{name} B={B} T={T} grad {n}: {rel:.2e}"
        if not any(flips.values()):
            assert rel_plain <= GRAD_BAR, f"{name} B={B} T={T} grad {n} with identical masks: {rel_plain:.2e}"


def _batch(model, B, S, seed):
    g = np.random.default_rng(seed)
    return types.SimpleNamespace(obs=g.integers(0, 256, (B, S, 3, 16, 16)).astype(np.float32),
                                 act=np.clip(g.standard_normal((B, S, model.action_size)), -1, 1).astype(np.float32),
                                 rewards=g.standard_normal((B, S)).astype(np.float32), next_obs=None, terminateds=None,
                                 truncateds=None)


@pytest.fixture
def no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


@pytest.mark.parametrize("size,B,S", [((2, 4, 16, 16, 32), 3, 6), (PLANET, 4, 8)])
def test_update_matches_float64(no_tf32, size, B, S):
    model = _model(size, seed=3)
    m64 = po.as_f64(model)
    batch = _batch(model, B, S, seed=11)
    g = np.random.default_rng(12)
    L = model.latent_state_size
    eq, ep = (torch.from_numpy(g.standard_normal((S - 1, B, L))) for _ in range(2))
    opt = torch.optim.Adam(model.parameters(), lr=1e-3, eps=1e-4)
    opt64 = torch.optim.Adam(m64.parameters(), lr=1e-3, eps=1e-4)
    lv, meta = latent_train.update(model, batch, opt, eps=(eq.float(), ep.float()))
    obs = torch.from_numpy(batch.obs).double() / 256.0 - 0.5
    want = po.update(m64, obs, torch.from_numpy(batch.act).double(), torch.from_numpy(batch.rewards).double(),
                     eq, ep, opt64)
    got = (lv, meta["observations_loss"], meta["reward_loss"], meta["kl_loss"], meta["grad_norm"])
    for what, a, b in zip(("loss", "observations_loss", "reward_loss", "kl_loss", "grad_norm"), got, want):
        print(f"update {size}: {what} {abs(a - b) / max(1.0, abs(b)):.2e}")
        assert abs(a - b) <= 1e-4 * max(1.0, abs(b)), (what, a, b)
    assert meta["reconstruction"].shape == (B, S - 1, 3, 16, 16)
    for (n, p), p64 in zip(model.named_parameters(), m64.parameters()):
        rel = _rel(p.grad, p64.grad)
        print(f"update {size}: grad {n} {rel:.2e}")
        assert rel <= GRAD_BAR, (n, rel)
        assert _err(p, p64) <= 1e-6, n


def _raw(model, P, act, eps, seed, offset, ups):
    """One forward and one backward call through the C ABI: outputs, the tape and dP."""
    lib = _lib.load()
    d = latent_train.train_desc(model)
    B, T = P.shape[:2]
    L, Hb, Hf = d.latent_size, d.belief_size, d.hidden_size
    params = latent_train.recurrence_params(model)
    ptrs = (C.c_void_p * len(params))(*[p.data_ptr() for p in params])
    out = [torch.empty(B, T, w, device=DEV) for w in (Hb, 2 * L, L, 2 * L, L)]
    widths = dict(e=Hb, gates=4 * Hb, q1=Hf, p1=Hf, pre_std=2 * L, eps=2 * L, de=Hb, dgi=3 * Hb, dghn=Hb, dq=2 * L, dv=Hf,
                  dp=2 * L)
    tape = {k: torch.empty(B, T, w, device=DEV) for k, w in widths.items()}
    t = _lib.LatentTape(*[tape[k].data_ptr() for k in widths])
    ws = torch.empty(lib.b200pets_latent_train_workspace_bytes(C.byref(d), B, T), dtype=torch.uint8, device=DEV)
    eq, ep = eps if eps is not None else (None, None)
    _lib.check(lib.b200pets_latent_seq_forward(C.byref(d), ptrs, B, T, _lib.ptr(P), _lib.ptr(act), _lib.ptr(eq),
                                               _lib.ptr(ep), seed, offset, *[_lib.ptr(o) for o in out], C.byref(t),
                                               _lib.ptr(ws), ws.numel(), _lib.stream_ptr()))
    dP = torch.empty(B, T, Hf, device=DEV)
    _lib.check(lib.b200pets_latent_seq_backward(C.byref(d), ptrs, B, T, _lib.ptr(out[0]), *[_lib.ptr(u) for u in ups],
                                                C.byref(t), _lib.ptr(dP), _lib.stream_ptr()))
    torch.cuda.synchronize()
    return out, tape, dP


M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    c0, c1, c2, c3 = np.broadcast_arrays(*(np.asarray(c, np.uint64) for c in (c0, c1, c2, c3)))
    k0, k1 = int(k0), int(k1)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c0, np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ np.uint64(k0), p1 & M32, (p0 >> np.uint64(32)) ^ c3 ^ np.uint64(k1), p0 & M32
        k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
    return c0, c1, c2, c3


def train_draws64(B, T, L, kind, seed, offset):
    """[B, T, L]: lane j & 3 of the Box-Muller block at counter (b, t, RNG_STREAM_LATENT_TRAIN | kind << 15 | j >> 2,
    low word of offset) under key seed ^ (high word of offset)."""
    key = (seed ^ (offset & 0xFFFFFFFF00000000)) & 0xFFFFFFFFFFFFFFFF
    b, t, j = np.arange(B)[:, None, None], np.arange(T)[None, :, None], np.arange(L)[None, None, :]
    r = philox4x32_10(b, t, RNG_STREAM_LATENT_TRAIN | (kind << 15) | (j >> 2), offset & 0xFFFFFFFF, key & 0xFFFFFFFF,
                      key >> 32)
    u = [((x >> np.uint64(8)).astype(np.float64) + 0.5) / 16777216.0 for x in r]
    lane = np.broadcast_to(j & 3, (B, T, L))
    ur, ua = np.where(lane < 2, u[0], u[2]), np.where(lane < 2, u[1], u[3])
    rad, ang = np.sqrt(-2.0 * np.log(ur)), 2.0 * np.pi * ua
    return np.where(lane & 1, rad * np.sin(ang), rad * np.cos(ang))


def test_in_kernel_draws_match_numpy_philox_and_kernels_are_deterministic():
    model = _model(ODD)
    B, T = 5, 6
    P, act, _, _ = _inputs(model, B, T, seed=1)
    P, act = P.to(DEV), act.to(DEV)
    g = np.random.default_rng(2)
    L = model.latent_state_size
    ups = [torch.from_numpy(g.standard_normal((B, T, w))).float().to(DEV) for w in (37, 2 * L, L, 2 * L, L)]
    seed, offset = 0x1234_5678_9ABC_DEF0, (3 << 32) + 8
    out1, tape1, dP1 = _raw(model, P, act, None, seed, offset, ups)
    eps = tape1["eps"].double().cpu().numpy()
    for kind in (0, 1):
        want = train_draws64(B, T, L, kind, seed, offset)
        err = np.abs(eps[..., kind * L:(kind + 1) * L] - want).max()
        assert err <= 2e-5 * max(1.0, np.abs(want).max()), (kind, err)
    out2, tape2, dP2 = _raw(model, P, act, None, seed, offset, ups)
    assert all(torch.equal(a, b) for a, b in zip(out1, out2))
    assert all(torch.equal(tape1[k], tape2[k]) for k in tape1)
    assert torch.equal(dP1, dP2)
    out3, tape3, _ = _raw(model, P, act, None, seed, offset + 4, ups)
    assert not torch.equal(tape1["eps"], tape3["eps"])


def test_refusals():
    lib = _lib.load()
    d = _lib.LatentTrainDesc(6, 30, 200, 200, 1024, 0.1)
    assert lib.b200pets_latent_train_supported(C.byref(d)) == 0
    H = _largest()
    d.belief_size = d.hidden_size = H + 1
    assert lib.b200pets_latent_train_supported(C.byref(d)) == -2
    d.belief_size = 0
    assert lib.b200pets_latent_train_supported(C.byref(d)) == -1


def _sequences(model, n, B, S, seed):
    return [_batch(model, B, S, seed + i) for i in range(n)]


def test_trainer_drop_in_over_the_container():
    model = _model(PLANET, seed=4, rng_seed=9)
    model.set_posterior(np.zeros(30), np.zeros(200))
    seen = []

    def cb(epoch, loss, meta, mode):
        seen.append((epoch, loss, dict(meta), mode))

    env = bp.ModelEnv(_EnvStub(6), model, functions.no_termination, generator=torch.Generator(device=DEV))
    actions = torch.rand(16, 5, 6, device=DEV) * 2 - 1
    eps = torch.randn(5, 16, 30, device=DEV)
    before = env.evaluate_action_sequences(actions, np.zeros((3, 16, 16)), 1, _eps=eps).clone()
    trainer = bp.ModelTrainer(model, optim_lr=1e-3, optim_eps=1e-4)
    assert trainer._latent_supported()
    losses, scores = trainer.train(_sequences(model, 3, 5, 8, 20), num_epochs=1, batch_callback=cb, evaluate=False)
    assert len(losses) == 1 and scores == [] and len(seen) == 3
    for epoch, loss, meta, mode in seen:
        assert epoch == 0 and mode == "train" and np.isfinite(loss)
        assert {"reconstruction", "observations_loss", "reward_loss", "kl_loss", "grad_norm"} <= set(meta)
    st = trainer.optimizer.state_dict()["state"]
    assert len(st) == len(list(model.parameters())) and all(float(s["step"]) == 3 for s in st.values())
    after = env.evaluate_action_sequences(actions, np.zeros((3, 16, 16)), 1, _eps=eps)
    fresh = bp.ModelEnv(_EnvStub(6), model, functions.no_termination, generator=torch.Generator(device=DEV))
    assert not torch.equal(before, after)
    assert torch.equal(after, fresh.evaluate_action_sequences(actions, np.zeros((3, 16, 16)), 1, _eps=eps))
    score = trainer.evaluate(_sequences(model, 2, 5, 8, 40))  # loss(reduce=False) per (b, t), averaged over time
    assert score.shape == (10,) and torch.isfinite(score).all()


class _Box:
    def __init__(self, lo_, hi, shape):
        self.low, self.high, self.shape = np.full(shape, lo_, np.float32), np.full(shape, hi, np.float32), shape


class _EnvStub:
    def __init__(self, A):
        self.observation_space = _Box(0, 255, (3, 16, 16))
        self.action_space = _Box(-1.0, 1.0, (A,))


def _ref_model(Hb=200, Hf=200):
    return mbrl.models.PlaNetModel(obs_shape=(3, 16, 16), obs_encoding_size=32, encoder_config=ENC, decoder_config=DEC,
                                   latent_state_size=30, action_size=6, belief_size=Hb, hidden_size_fcs=Hf, device=DEV)


def _ref_dataset(batch_size=4, sequence_length=8, batches=3):
    g = np.random.default_rng(0)
    replay_buffer, common = (importlib.import_module(f"mbrl.util.{n}") for n in ("replay_buffer", "common"))
    buf = replay_buffer.ReplayBuffer(400, (3, 16, 16), (6,), obs_type=np.uint8, rng=g,
                                               max_trajectory_length=50)
    for _ in range(4):
        for t in range(50):
            buf.add(g.integers(0, 256, (3, 16, 16), dtype=np.uint8), g.uniform(-1, 1, 6).astype(np.float32),
                    g.integers(0, 256, (3, 16, 16), dtype=np.uint8), float(g.standard_normal()), False, t == 49)
    ds, _ = common.get_sequence_buffer_iterator(buf, batch_size, 0, sequence_length,
                                                          max_batches_per_loop_train=batches, use_simple_sampler=True)
    return ds


@needs_ref
def test_trainer_drop_in_over_the_reference_model():
    model = _ref_model()
    trainer = bp.ModelTrainer(model, optim_lr=1e-3, optim_eps=1e-4)
    assert trainer._latent_supported()
    seen = []
    trainer.train(_ref_dataset(), num_epochs=1, batch_callback=lambda *a: seen.append(a), evaluate=False)
    assert len(seen) == 3 and all("grad_norm" in a[2] for a in seen)
    assert all(float(s["step"]) == 3 for s in trainer.optimizer.state_dict()["state"].values())


@needs_ref
def test_refused_sizes_train_through_the_reference_update():
    H = _largest() + 4
    model = _ref_model(Hb=H, Hf=H)
    trainer = bp.ModelTrainer(model, optim_lr=1e-3, optim_eps=1e-4)
    assert not trainer._latent_supported()
    calls = []
    orig = model.update
    model.update = lambda *a, **k: (calls.append(1), orig(*a, **k))[1]
    trainer.train(_ref_dataset(batch_size=2, sequence_length=3, batches=1), num_epochs=1,
                  batch_callback=lambda *a: None, evaluate=False)
    assert calls == [1]


def _inject(model, queue):
    """The reference's _sample_state_from_params reading its draws from ``queue`` (posterior, prior, posterior, ...)."""
    L = model.latent_state_size

    def sample(params, generator, deterministic=False):
        return params[:, :L] if deterministic else params[:, :L] + params[:, L:] * queue.pop(0)

    model._sample_state_from_params = sample


def _drift(mine, ref, p0):
    """(worst per-tensor distance relative to the reference's movement, its name, the same over all parameters)."""
    per = [(float((p.detach().cpu().double() - q.detach().cpu().double()).norm() /
                  (q.detach().cpu().double() - z).norm()), k)
           for (k, p), q, z in zip(mine.named_parameters(), ref.parameters(), p0)]
    d = sum(float((p.detach().cpu().double() - q.detach().cpu().double()).norm()) ** 2
            for p, q in zip(mine.parameters(), ref.parameters()))
    m = sum(float((q.detach().cpu().double() - z).norm()) ** 2 for q, z in zip(ref.parameters(), p0))
    worst, where = max(per)
    return worst, where, (d / m) ** 0.5


@needs_ref
def test_drift_against_the_reference_over_100_updates(no_tf32):
    """100 updates of latent_train.update and of the reference's own PlaNetModel.update on cuda, fp32, from the same
    weights with the same draws.  The control is the reference's fp32 against the float64 oracle over the same updates:
    how far fp32 rounding alone carries a run."""
    B, S, n = 8, 12, 100
    models_ = []
    for _ in range(2):
        torch.manual_seed(5)  # dreamer_init draws from the global generator: both start from the same weights
        models_.append(_ref_model())
    mine, ref = models_
    m64 = po.as_f64(ref)
    p0 = [p.detach().cpu().double().clone() for p in ref.parameters()]
    opt_m = torch.optim.Adam(mine.parameters(), lr=1e-3, eps=1e-4)
    opt_r = torch.optim.Adam(ref.parameters(), lr=1e-3, eps=1e-4)
    opt_64 = torch.optim.Adam(m64.parameters(), lr=1e-3, eps=1e-4)
    queue = []
    _inject(ref, queue)
    g = torch.Generator().manual_seed(3)
    for u in range(n):
        batch = _batch(ref, B, S, seed=1000 + u)
        eq, ep = (torch.randn(S - 1, B, 30, generator=g, dtype=torch.float64) for _ in range(2))
        lm, _ = latent_train.update(mine, batch, opt_m, eps=(eq.float().to(DEV), ep.float().to(DEV)))
        queue.extend(x.float().to(DEV) for t in range(S - 1) for x in (eq[t], ep[t]))
        lr_, _ = ref.update(batch, opt_r)
        assert not queue
        obs = torch.from_numpy(batch.obs).double() / 256.0 - 0.5
        po.update(m64, obs, torch.from_numpy(batch.act).double(), torch.from_numpy(batch.rewards).double(), eq, ep, opt_64)
        if u + 1 in (1, 10, 100):
            w, where, tot = _drift(mine, ref, p0)
            cw, cwhere, ctot = _drift(ref, m64, p0)
            print(f"drift after {u + 1} updates: all parameters {tot:.3e}, worst tensor {w:.3e} [{where}]; control "
                  f"(reference fp32 vs float64): all {ctot:.3e}, worst {cw:.3e} [{cwhere}]; loss {lm:.6g} vs {lr_:.6g}")
    # no farther from the reference than fp32 rounding carries the reference itself from float64 (see the docstring)
    assert tot <= max(2 * ctot, 1e-5), (tot, ctot)
    assert w <= max(2 * cw, 1e-5), (w, where, cw)
