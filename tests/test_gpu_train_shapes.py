"""Device training (csrc/train.cu, ``mbrl_lib_b200.ModelTrainer``) at the shapes mbrl-lib's configs train, with the
partial last minibatch every real epoch ends with.

Every device-training test here runs a last step of ``last_batch < Bm`` rows, as a replay buffer that does not divide
evenly into minibatches makes on every epoch.  Stated tolerances (the deviations the tests print as
``DEVIATION <name> <value>``; worst measured on an H100 80GB HBM3, 700 W power limit, in brackets):
  A. one launch over a short epoch against float64 autograd + ``torch.optim.Adam``, Adam state pre-filled (step 2):
       per-step loss          |l32 - l64| <= 1e-6 * max(1, |l64|)                               (3.3e-7)
       parameter movement     |dp32 - dp64| <= 2e-4 * max |dp64| + S half fp32 ulps of p        (3.3e-6)
                              (dp = p_end - p_start over the S steps; each fp32 step rounds the stored p once, which
                              only matters for the logvar bounds, |p| ~ 4 against a movement ~ 1e-3)
       exp_avg / exp_avg_sq   max |x32 - x64| <= 1e-5 * max |x64|                              (2.0e-7 / 3.2e-7)
     negative controls, float64 checkers with one deliberate error; each must miss a bar by 10x or more:
       the partial step normalised by Bm with the padding rows included            (7.3e3 x)
       Adam bias correction at t + 1 / t - 1                                       (3.2e2 x)
       layer 0's bias gradient dropped                                             (67 x)
     (the worst ratio deviation / bar over the four metrics, the smallest over all shapes)
  B. ~200 steps from a fresh optimizer against the PyTorch fp32 trainer on the same minibatches:
       max |p_dev - p_torch| <= 3e-5 * max |p_torch - p_0|                          (3.9e-6)
       per-step losses within 1e-5 * max(1, |l|): the NLL crosses zero as the logvar falls (from ~1.6 to
       -15), where a plain relative error means nothing                              (3.6e-7)
     Models the kernels refuse (8 hidden layers, hid_size 1024) run the reference loop: equal under torch.equal.
  C. train() end to end against the reference loop, iterators built as get_basic_buffer_iterators builds them over
     float64 stores with a float64 normaliser: identical epoch counts, elite sets and next generator draw; loss and
     score histories within 1e-5 relative                                            (1.0e-6 / 2.5e-7)
  D. bit for bit (torch.equal): S steps in one launch == S launches of one step; NaN-filled workspaces; padded index
     entries pointing at other rows; a repeated run; eval_score over a NaN-filled or reused workspace
  E. eval_score against a float64 forward at 1, 31, 32, 33 and 4097 rows: 1e-6 relative        (1.6e-7)
  F. preprocessing against OneDTransitionRewardModel._process_batch on float64 CPU tensors (D = 45, A = 17): float32
     stores within 1e-6 * max(1, |x|) (1.2e-7); float64 stores: the double result rounded once, targets equal,
     inputs within one fp32 ulp (sin / cos of two libraries)                          (all equal)
"""
import copy
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from mbrl_lib_b200 import _lib, functions, models, replay, trainer as tr  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LR, WD = 2.8e-4, 1e-4
BARS = {"loss": 1e-6, "update": 2e-4, "exp_avg": 1e-5, "exp_avg_sq": 1e-5}


def _report(name, value):
    print(f"DEVIATION {name} {value:.3e}")


# name: in, out (incl. reward), hid, hidden layers, E, Bm, rows of the epoch, activation, deterministic, learned bounds
CASES = {
    "pets_cartpole": (5, 4, 200, 4, 7, 256, 257, "silu", False, False),
    "pets_cartpole_paper": (6, 4, 200, 4, 7, 256, 300, "silu", False, False),
    "pets_hopper": (14, 12, 200, 4, 7, 32, 97, "silu", False, False),
    "pets_halfcheetah": (24, 18, 200, 4, 7, 32, 72, "silu", False, False),
    "pets_reacher": (26, 20, 200, 4, 5, 32, 95, "silu", False, False),
    "pets_pusher": (27, 21, 200, 4, 5, 32, 95, "silu", False, False),
    "mbpo_ant": (35, 28, 200, 4, 7, 256, 545, "silu", False, False),
    "mbpo_humanoid": (62, 46, 200, 4, 7, 256, 656, "silu", False, False),
    "one_hidden_deterministic": (23, 17, 64, 1, 5, 33, 70, "silu", True, False),
    "seven_hidden_relu": (23, 18, 33, 7, 3, 32, 65, "relu", False, False),
    "hid32_leaky_relu": (23, 18, 32, 4, 7, 32, 40, "leaky_relu", False, False),
    "hid512": (40, 21, 512, 2, 2, 64, 100, "silu", False, False),
    "learned_bounds": (24, 18, 200, 3, 7, 32, 75, "silu", False, True),
}


def _model(E, in_size, out_size, hid, act, det, seed, num_layers=4, learn_bounds=False, **wrapper_kw):
    torch.manual_seed(seed)
    mlp = models.GaussianMLP(in_size, out_size, DEV, num_layers=num_layers, ensemble_size=E, hid_size=hid,
                             deterministic=det, activation=act)
    with torch.no_grad():
        for layer in [s[0] for s in mlp.hidden_layers] + [mlp.mean_and_logvar]:
            layer.weight.normal_(0.0, 1.0 / (2.0 * np.sqrt(layer.weight.shape[1])))
            layer.bias.normal_(0.0, 0.05)
        if not det:
            mlp.min_logvar.fill_(-4.0)
            mlp.max_logvar.fill_(0.3)
            mlp.min_logvar.requires_grad_(learn_bounds)
            mlp.max_logvar.requires_grad_(learn_bounds)
    return models.OneDTransitionRewardModel(mlp, **wrapper_kw)


def _case_model(name, seed=0):
    i, o, hid, L, E, _, _, act, det, bounds = CASES[name]
    return _model(E, i, o, hid, act, det, seed=seed, num_layers=L, learn_bounds=bounds)


def _prefill_state(opt, params, seed, step=9.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    for p in params:
        if not p.requires_grad:
            continue
        opt.state[p] = {"step": torch.tensor(step),
                        "exp_avg": (torch.randn(p.shape, generator=g) * 1e-2).to(p.device, p.dtype),
                        "exp_avg_sq": (torch.rand(p.shape, generator=g) * 1e-4 + 1e-6).to(p.device, p.dtype)}


def _data(name, rows, seed):
    i, o = CASES[name][:2]
    g = torch.Generator(device="cpu").manual_seed(seed)
    X = torch.randn(rows, i, generator=g)
    Y = torch.randn(rows, o, generator=g) * 0.5
    return X.to(DEV), Y.to(DEV)


def _epoch(E, rows, Bm, seed):
    """One bootstrapped epoch as ``epoch_indices`` lays it out: a permutation of the rows per member, cut into steps of
    Bm, the last step's entries past ``last_batch`` zero."""
    rng = np.random.default_rng(seed)
    steps = (rows - 1) // Bm + 1
    idx = np.zeros((E, steps * Bm), np.int32)
    idx[:, :rows] = np.stack([rng.permutation(rows) for _ in range(E)])
    return idx.reshape(E, steps, Bm), rows - (steps - 1) * Bm


# ---- A. a short epoch against float64 autograd and Adam ---------------------------------------------------------------
# Adam steps taken before the epoch.  Non-zero moments make the first update smooth; a small count makes the bias
# corrections differ enough between t and t +- 1 (at t = 10 the two corrections' changes nearly cancel) for an off-by-one
# step count to show.
A_STEP = 2.0


def _float64_epoch(model, X, Y, idx, last_batch, error=None):
    """The epoch's steps through a float64 copy of the model and torch.optim.Adam, optionally with one deliberate error:
    "bm_norm" (the partial step over all Bm entries, padding included), "t+1" / "t-1" (bias correction one step off),
    "no_b0_grad" (layer 0's bias gradient dropped)."""
    m64 = copy.deepcopy(model.model).double()
    opt = torch.optim.Adam(m64.parameters(), lr=LR, weight_decay=WD, eps=1e-8)
    _prefill_state(opt, list(m64.parameters()), seed=7, step=A_STEP + {"t+1": 1.0, "t-1": -1.0}.get(error, 0.0))
    X64, Y64 = X.double(), Y.double()
    steps, Bm = idx.shape[1], idx.shape[2]
    losses = []
    for s in range(steps):
        B = last_batch if s == steps - 1 and error != "bm_norm" else Bm
        rows = torch.from_numpy(idx[:, s, :B].astype(np.int64)).to(DEV)
        opt.zero_grad()
        loss, _ = m64.loss(X64[rows], Y64[rows])
        loss.backward()
        if error == "no_b0_grad":
            m64.hidden_layers[0][0].bias.grad.zero_()
        opt.step()
        losses.append(float(loss))
    return m64, opt, np.array(losses)


def _deviations(model, opt32, p0, losses32, m64, opt64, losses64, steps):
    dev = {"loss": float(np.max(np.abs(losses32 - losses64) / np.maximum(1.0, np.abs(losses64)))),
           "update": 0.0, "exp_avg": 0.0, "exp_avg_sq": 0.0}
    for p, a, q in zip(model.parameters(), p0, m64.parameters()):
        if not p.requires_grad:
            assert torch.equal(p.detach().double(), a)
            continue
        du, du64 = p.detach().double() - a, q.detach() - a
        ulps = steps * torch.from_numpy(np.spacing(np.abs(p.detach().cpu().numpy()))).to(DEV).double() / 2
        dev["update"] = max(dev["update"], float(((du - du64).abs() - ulps).clamp_min(0).max() / du64.abs().max()))
        st, st64 = opt32.state[p], opt64.state[q]
        for k in ("exp_avg", "exp_avg_sq"):
            dev[k] = max(dev[k], float((st[k].double() - st64[k]).abs().max() / st64[k].abs().max()))
    return dev


@pytest.mark.parametrize("name", list(CASES))
def test_short_epoch_matches_float64(name):
    E, Bm, rows = CASES[name][4:7]
    model = _case_model(name, seed=len(name))
    trainer = tr.ModelTrainer(model, optim_lr=LR, weight_decay=WD, optim_eps=1e-8)
    _prefill_state(trainer.optimizer, list(model.parameters()), seed=7, step=A_STEP)
    p0 = [p.detach().double().clone() for p in model.parameters()]
    ref = copy.deepcopy(model)  # the checkers start from the same weights
    X, Y = _data(name, rows, seed=rows)
    idx, last_batch = _epoch(E, rows, Bm, seed=E + Bm)
    assert last_batch < Bm
    steps = idx.shape[1]
    dm = tr._DeviceModel(model, trainer.optimizer)
    losses32 = dm.run_steps(X, Y, idx, last_batch).astype(np.float64)
    dm.close()
    assert float(trainer.optimizer.state[model.model.mean_and_logvar.weight]["step"]) == A_STEP + steps

    m64, opt64, losses64 = _float64_epoch(ref, X, Y, idx, last_batch)
    dev = _deviations(model, trainer.optimizer, p0, losses32, m64, opt64, losses64, steps)
    for k, v in dev.items():
        _report(f"epoch_{k}[{name}]", v)
    assert all(dev[k] <= BARS[k] for k in BARS), dev

    for error in ("bm_norm", "t+1", "t-1", "no_b0_grad"):
        m64, opt64, losses64 = _float64_epoch(ref, X, Y, idx, last_batch, error=error)
        cdev = _deviations(model, trainer.optimizer, p0, losses32, m64, opt64, losses64, steps)
        miss = max(cdev[k] / BARS[k] for k in BARS)
        _report(f"control_{error}[{name}]", miss)
        assert miss >= 10.0, (error, cdev)


# ---- B. a fresh optimizer against the PyTorch fp32 trainer -----------------------------------------------------------
@pytest.mark.parametrize("name", ["pets_halfcheetah", "mbpo_humanoid"])
def test_fresh_optimizer_follows_the_pytorch_trainer(name):
    i, o, E, Bm, rows = CASES[name][0], CASES[name][1], *CASES[name][4:7]
    model = _case_model(name, seed=3)
    ref = copy.deepcopy(model)
    trainer = tr.ModelTrainer(model, optim_lr=LR, weight_decay=WD)
    opt = torch.optim.Adam(ref.parameters(), lr=LR, weight_decay=WD, eps=1e-8)
    p0 = [p.detach().clone() for p in model.parameters()]
    g = torch.Generator(device="cpu").manual_seed(5)
    X = torch.randn(rows, i, generator=g).to(DEV)
    Y = (torch.tanh(X[:, :o] * 0.7) + 0.05 * torch.randn(rows, o, generator=g).to(DEV)).contiguous()
    dm = tr._DeviceModel(model, trainer.optimizer)
    losses, ref_losses = [], []
    epoch = 0
    while len(losses) < 200:
        idx, last_batch = _epoch(E, rows, Bm, seed=100 + epoch)
        assert last_batch < Bm
        losses += list(dm.run_steps(X, Y, idx, last_batch))
        for s in range(idx.shape[1]):
            B = last_batch if s == idx.shape[1] - 1 else Bm
            r = torch.from_numpy(idx[:, s, :B].astype(np.int64)).to(DEV)
            ref_losses.append(ref.model.update(X[r], opt, target=Y[r])[0])
        epoch += 1
    dm.close()
    assert float(trainer.optimizer.state[model.model.mean_and_logvar.weight]["step"]) == len(losses)
    worst = max(float((p - q).abs().max() / (q - a).abs().max())
                for p, q, a in zip(model.parameters(), ref.parameters(), p0) if p.requires_grad)
    # the NLL passes near zero as the logvar falls: losses are compared relative to max(1, |l|)
    lerr = float(np.max(np.abs(np.array(losses) - ref_losses) / np.maximum(1.0, np.abs(ref_losses))))
    _report(f"fresh_params[{name}]", worst)
    _report(f"fresh_losses[{name}]", lerr)
    assert worst <= 3e-5 and lerr <= 1e-5


# ---- C. train() end to end against the reference loop -----------------------------------------------------------------
def _transitions(n, D, A, seed):
    """float64 transitions, as the PETS / MBPO replay buffers hold them."""
    rng = np.random.default_rng(seed)
    obs = rng.standard_normal((n, D))
    act = rng.uniform(-1, 1, (n, A))
    M = rng.standard_normal((D + A, D)) * 0.5
    nxt = obs + np.tanh(np.concatenate([obs, act], 1) @ M) + 0.1 * rng.standard_normal((n, D))
    rew = np.sin(obs[:, 0]) + act.sum(1) + 0.1 * rng.standard_normal(n)
    return replay.TransitionBatch(obs, act, nxt, rew, np.zeros(n, bool), np.zeros(n, bool))


def _train_model(E, store, seed, num_layers=3, hid=64):
    """ReLU, float64 normaliser from the store; at E = 5, 3 elites and members 3 and 4 with a dead first layer, so the
    elite set is clear-cut."""
    D, A = store.obs.shape[1], store.act.shape[1]
    model = _model(E, D + A, D + 1, hid, "relu", False, seed=seed, num_layers=num_layers, num_elites=min(3, E),
                   normalize=True, normalize_double_precision=True)
    x = np.concatenate([store.obs, store.act], 1)
    model.input_normalizer.mean = torch.tensor(x.mean(0, keepdims=True), device=DEV)
    model.input_normalizer.std = torch.tensor(x.std(0, ddof=1, keepdims=True), device=DEV)
    if E == 5:
        with torch.no_grad():
            first = model.model.hidden_layers[0][0]
            first.weight[3:].zero_()
            first.bias[3:].fill_(-1.0)
    return model


def _iterators(store, layout, E, batch, seed):
    """get_basic_buffer_iterators: a shuffled store, the bootstrap training iterator drawing with replacement, a
    validation TransitionIterator without shuffling, one generator for all of it."""
    rng = np.random.default_rng(seed)
    data = store[rng.permutation(len(store))]
    val_size = int(len(store) * (0.0 if layout in ("pets", "bootstrap_e1") else 0.2))
    n = len(store) - val_size
    train = data[:n]
    val = replay.TransitionIterator(data[n:], batch, shuffle_each_epoch=False, rng=rng) if val_size else None
    if layout == "transition_iterator":
        ds = replay.TransitionIterator(train, batch, shuffle_each_epoch=True, rng=rng)
    elif layout == "member_slices":  # a plain iterable of [E, B, ...] bootstrap batches, the last one short
        members = np.stack([rng.permutation(n) for _ in range(E)])
        ds = [replay.TransitionBatch(*(np.stack(c) for c in zip(*(train[m[i:i + batch]].astuple() for m in members))))
              for i in range(0, n, batch)]
        assert len(ds[-1].obs[0]) < batch
    else:
        ds = replay.BootstrapIterator(train, batch, E, shuffle_each_epoch=True, permute_indices=False, rng=rng)
    if not isinstance(ds, list):
        last_batch, Bm = ds.num_stored - (len(ds) - 1) * batch, batch
        assert last_batch < Bm
    if val is not None:
        assert val.num_stored % batch != 0  # a partial last validation batch
    return ds, val, rng


def _train_run(model, layout, E, store, device, **kw):
    """device: True (asserts the kernels take the model), False (the reference loop), None (as a user calls it)."""
    ds, val, rng = _iterators(store, layout, E, 32, seed=31)
    trainer = tr.ModelTrainer(model, optim_lr=1e-3, weight_decay=1e-4)
    if device:
        assert trainer._device_supported()
    elif device is not None:
        trainer._device_supported = lambda: False
    seen = []
    cb = lambda m, it, ep, loss, score, best: seen.append((score.cpu().numpy(), best.cpu().numpy()))
    out = trainer.train(ds, val, callback=cb, **kw)
    return out, seen, int(rng.integers(1 << 62))


@pytest.mark.parametrize("layout,E", [("pets", 5), ("mbpo", 5), ("transition_iterator", 5), ("bootstrap_e1", 1),
                                      ("member_slices", 5)])
def test_train_matches_the_reference_loop(layout, E):
    store = _transitions(330, 4, 2, seed=E + len(layout))
    model = _train_model(E, store, seed=2)
    ref_model = copy.deepcopy(model)
    kw = dict(num_epochs=20, patience=3, improvement_threshold=0.1)
    (l_dev, s_dev), _, draw_dev = _train_run(model, layout, E, store, True, **kw)
    (l_ref, s_ref), seen_ref, draw_ref = _train_run(ref_model, layout, E, store, False, **kw)
    assert len(l_dev) == len(l_ref) and len(s_dev) == len(s_ref) == len(l_ref)
    lerr = float(np.max(np.abs(np.array(l_dev) - l_ref) / np.abs(l_ref)))
    serr = float(np.max(np.abs(np.array(s_dev) - s_ref) / np.abs(s_ref)))
    _report(f"train_loss_history[{layout}]", lerr)
    _report(f"train_score_history[{layout}]", serr)
    assert lerr <= 1e-5 and serr <= 1e-5
    assert draw_dev == draw_ref  # the shared generator advanced alike
    # the decisions are clear-cut: every epoch's best relative improvement is far from the threshold, measured against
    # the two runs' deviation
    best = None
    for score, b in seen_ref:
        if best is not None:
            margin = float(np.max((best - score) / np.abs(best))) - kw["improvement_threshold"]
            assert abs(margin) > max(1e-4, 100 * serr), margin
        best = b
    if E > 1:
        assert set(model.model.elite_models) == set(ref_model.model.elite_models)
        ranked = np.sort(seen_ref[-1][1])
        assert (ranked[3] - ranked[2]) / ranked[2] > 100 * max(serr, 1e-6), ranked
    else:
        assert model.model.elite_models is None and ref_model.model.elite_models is None


# ---- models the kernels refuse ---------------------------------------------------------------------------------------
def test_eight_hidden_layers_run_the_reference_loop():
    store = _transitions(210, 4, 2, seed=41)
    model = _train_model(5, store, seed=3, num_layers=8, hid=32)
    ref_model = copy.deepcopy(model)
    trainer = tr.ModelTrainer(model, optim_lr=3e-3, weight_decay=1e-4)
    assert not trainer._device_supported()
    lib = _lib.load()
    assert lib.b200pets_trainer_supported(C.byref(tr.train_desc(model.model, trainer.optimizer.param_groups[0]))) == -2
    assert b"hidden layers" in lib.b200pets_last_error()
    results = []
    for m, device in ((model, None), (ref_model, False)):
        out, _, draw = _train_run(m, "mbpo", 5, store, device, num_epochs=3)
        results.append((out, draw))
    assert results[0] == results[1]
    for p, q in zip(model.parameters(), ref_model.parameters()):
        assert torch.equal(p, q)
    assert model.model.elite_models == ref_model.model.elite_models
    val = replay.TransitionIterator(store, 32)
    ev = tr.ModelTrainer(model).evaluate(val)
    fallback = tr.ModelTrainer(model)
    fallback._device_supported = lambda: False
    assert torch.equal(ev, fallback.evaluate(val))


def test_layers_too_wide_for_evaluation_run_the_reference_loop():
    store = _transitions(210, 4, 2, seed=43)
    model = _train_model(5, store, seed=4, num_layers=2, hid=1024)
    ref_model = copy.deepcopy(model)
    trainer = tr.ModelTrainer(model)
    assert not trainer._device_supported()
    assert b"shared memory" in _lib.load().b200pets_last_error()
    (l_dev, s_dev), _, draw_dev = _train_run(model, "mbpo", 5, store, None, num_epochs=3)
    (l_ref, s_ref), _, draw_ref = _train_run(ref_model, "mbpo", 5, store, False, num_epochs=3)
    assert len(l_dev) == len(l_ref) == 3 and draw_dev == draw_ref
    assert float(np.max(np.abs(np.array(l_dev) - l_ref) / np.abs(l_ref))) <= 1e-5
    assert float(np.max(np.abs(np.array(s_dev) - s_ref) / np.abs(s_ref))) <= 1e-5
    assert set(model.model.elite_models) == set(ref_model.model.elite_models)
    val = replay.TransitionIterator(store, 32)
    assert torch.allclose(tr.ModelTrainer(model).evaluate(val), tr.ModelTrainer(ref_model).evaluate(val), rtol=1e-5)


# ---- D. invariants that hold bit for bit -----------------------------------------------------------------------------
def _c_epoch(name, X, Y, idx, last_batch, launches, ws_fill):
    """The epoch through the C ABI with a workspace this test owns: ``launches`` [(first step, end step)], each one
    train_epoch call with batch = Bm and the Adam step count it starts from.  Returns parameters, both moments, losses."""
    E, Bm = idx.shape[0], idx.shape[2]
    steps = idx.shape[1]
    model = _case_model(name, seed=11)
    opt = torch.optim.Adam(model.parameters(), lr=LR, weight_decay=WD, eps=1e-8)
    _prefill_state(opt, list(model.parameters()), seed=7)
    dm = tr._DeviceModel(model, opt)
    nbytes = dm.lib.b200pets_train_workspace_bytes(dm.handle, Bm)
    ws = torch.full((nbytes // 4,), ws_fill, device=DEV)
    losses = torch.full((steps,), float("nan"), device=DEV)
    for s0, s1 in launches:
        sub = torch.from_numpy(np.ascontiguousarray(idx[:, s0:s1])).to(DEV)
        lb = last_batch if s1 == steps else Bm
        _lib.check(dm.lib.b200pets_train_epoch(dm.handle, int(X.shape[0]), _lib.ptr(X), _lib.ptr(Y), _lib.ptr(sub),
                                               s1 - s0, Bm, lb, 9 + s0, _lib.ptr(losses[s0:]), _lib.ptr(ws), nbytes,
                                               dm.stream()), "train_epoch")
    torch.cuda.synchronize()
    dm.close()
    trained = [p for p in model.parameters() if p.requires_grad]
    return ([p.detach().clone() for p in model.parameters()] + [opt.state[p]["exp_avg"].clone() for p in trained] +
            [opt.state[p]["exp_avg_sq"].clone() for p in trained] + [losses])


def _same(a, b):
    return len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("name", ["mbpo_humanoid", "learned_bounds", "seven_hidden_relu"])
def test_epoch_invariants_bit_for_bit(name):
    E, Bm, rows = CASES[name][4:7]
    X, Y = _data(name, rows, seed=17)
    idx, last_batch = _epoch(E, rows, Bm, seed=19)
    assert last_batch < Bm
    steps = idx.shape[1]
    whole = [(0, steps)]
    base = _c_epoch(name, X, Y, idx, last_batch, whole, float("nan"))
    assert all(bool(torch.isfinite(t).all()) for t in base)
    assert _same(base, _c_epoch(name, X, Y, idx, last_batch, whole, 0.0))  # the workspace's contents are never read
    assert _same(base, _c_epoch(name, X, Y, idx, last_batch, [(s, s + 1) for s in range(steps)], float("nan")))
    padded = idx.copy()
    padded[:, -1, last_batch:] = (np.arange(Bm - last_batch) * 7 + 3) % rows  # other rows, all in range
    assert not np.array_equal(padded, idx)
    assert _same(base, _c_epoch(name, X, Y, padded, last_batch, whole, float("nan")))
    assert _same(base, _c_epoch(name, X, Y, idx, last_batch, whole, float("nan")))  # reproducible


@pytest.mark.parametrize("name", ["mbpo_humanoid", "learned_bounds"])
def test_eval_score_workspace_invariants(name):
    model = _case_model(name, seed=13)
    trainer = tr.ModelTrainer(model)
    dm = tr._DeviceModel(model, trainer.optimizer)
    X, Y = _data(name, 4097, seed=23)
    rows = int(X.shape[0])
    nbytes = dm.lib.b200pets_eval_score_workspace_bytes(dm.handle, rows)

    def score(ws):
        out = torch.full((dm.E,), float("nan"), device=DEV)
        _lib.check(dm.lib.b200pets_eval_score(dm.handle, rows, _lib.ptr(X), _lib.ptr(Y), _lib.ptr(out), _lib.ptr(ws),
                                              nbytes, dm.stream()), "eval_score")
        return out.clone()

    zero = score(torch.zeros(nbytes // 4, device=DEV))
    nan_ws = torch.full((nbytes // 4,), float("nan"), device=DEV)
    first = score(nan_ws)
    second = score(nan_ws)  # the same workspace again, as left by the first call
    dm.close()
    assert bool(torch.isfinite(zero).all())
    assert torch.equal(zero, first) and torch.equal(first, second)


# ---- E. eval_score against a float64 forward -------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CASES))
def test_eval_score_matches_float64(name):
    model = _case_model(name, seed=29)
    trainer = tr.ModelTrainer(model)
    dm = tr._DeviceModel(model, trainer.optimizer)
    m64 = copy.deepcopy(model.model).double()
    worst = 0.0
    for rows in (1, 31, 32, 33, 4097):
        X, Y = _data(name, rows, seed=rows)
        got = dm.eval_score(X, Y).double()
        with torch.no_grad():
            mean64, _ = m64.forward(X.double())
            want = ((mean64 - Y.double()) ** 2).mean((1, 2))
        worst = max(worst, float(((got - want).abs() / want).max()))
    dm.close()
    _report(f"eval_score[{name}]", worst)
    assert worst <= 1e-6


# ---- F. preprocessing against the float64 mirror ---------------------------------------------------------------------
@pytest.mark.parametrize("store_dtype", ["float32", "float64"])
@pytest.mark.parametrize("proc", [None, "halfcheetah", "cartpole"])
@pytest.mark.parametrize("delta,learned", [(True, True), (False, True), (True, False)])
def test_preprocess_matches_the_float64_mirror(store_dtype, proc, delta, learned):
    """D = 45 observation columns, so the no_delta bitmask needs its second word (columns 33 and 44, and -1 = 44)."""
    D, A, n = 45, 17, 1000
    Dp = D + (1 if proc == "cartpole" else 0)
    rng = np.random.default_rng(D + A + int(delta) + 2 * int(learned))
    cols = [rng.standard_normal((n, D)), rng.uniform(-1, 1, (n, A)), rng.standard_normal((n, D)) * 2,
            rng.standard_normal(n)]
    dt = np.float64 if store_dtype == "float64" else np.float32
    store = replay.TransitionBatch(*(c.astype(dt) for c in cols), np.zeros(n, bool), np.zeros(n, bool))
    kw = dict(target_is_delta=delta, learned_rewards=learned, normalize=True,
              normalize_double_precision=store_dtype == "float64", obs_process_fn=functions.OBS_PROCESS_FNS[proc],
              no_delta_list=[0, 33, 44, -1])
    model = _model(2, Dp + A, D + int(learned), 32, "silu", False, seed=1, num_layers=1, **kw)
    norm_dt = torch.float64 if store_dtype == "float64" else torch.float32
    mean, std = rng.standard_normal((1, Dp + A)), rng.uniform(0.5, 2.0, (1, Dp + A))
    model.input_normalizer.mean = torch.tensor(mean, dtype=norm_dt, device=DEV)
    model.input_normalizer.std = torch.tensor(std, dtype=norm_dt, device=DEV)
    trainer = tr.ModelTrainer(model)
    dm = tr._DeviceModel(model, trainer.optimizer)
    X, Y, _ = dm.stage(store)
    dm.close()
    X, Y = X.cpu().numpy(), Y.cpu().numpy()

    # the reference's _process_batch over float64 CPU tensors (the float32 statistics promoted): the double computation,
    # rounded to float32 once at the end
    mirror = models.OneDTransitionRewardModel(models.GaussianMLP(Dp + A, D + int(learned), "cpu", num_layers=1, hid_size=4),
                                              **kw)
    mirror.input_normalizer.mean = model.input_normalizer.mean.cpu().double()
    mirror.input_normalizer.std = model.input_normalizer.std.cpu().double()
    b64 = replay.TransitionBatch(*(c.astype(np.float64) for c in store.astuple()[:4]), store.terminateds, store.truncateds)
    x_ref, y_ref = (t.numpy() for t in mirror._process_batch(b64))
    assert X.shape == x_ref.shape and Y.shape == y_ref.shape
    xe = float(np.max(np.abs(X.astype(np.float64) - x_ref) / np.maximum(1.0, np.abs(x_ref))))
    ye = float(np.max(np.abs(Y.astype(np.float64) - y_ref) / np.maximum(1.0, np.abs(y_ref))))
    tag = f"{store_dtype},{proc},{delta},{learned}"
    _report(f"preprocess_inputs[{tag}]", xe)
    _report(f"preprocess_targets[{tag}]", ye)
    if store_dtype == "float32":
        assert xe <= 1e-6 and ye <= 1e-6
    else:
        np.testing.assert_array_equal(Y, y_ref)
        assert np.all(np.abs(X - x_ref) <= np.spacing(np.abs(x_ref)))
