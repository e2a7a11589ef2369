"""Device training (``mbrl_lib_b200.ModelTrainer``, csrc/train.cu) against PyTorch.

Stated tolerances (from the deviations these tests print as ``DEVIATION <name> <value>``, measured on an H100):
  * one Adam step against torch autograd + torch.optim.Adam in float64, Adam state pre-filled (step 9, non-zero
    moments) so that the update is a smooth function of the gradient:
      loss                   |l32 - l64| <= 1e-6 * max(1, |l64|)                          (measured 8e-8)
      parameter update       |du32 - du64| <= 2e-4 * max |du64| + half an fp32 ulp of p   (measured 4e-5 of max |du64|;
                             du = p_new - p_old; the ulp term is the fp32 storage of p itself, which dominates for the
                             logvar bounds: |p| ~ 4 against updates ~ 3e-4)
      exp_avg / exp_avg_sq   max |x32 - x64| <= 1e-5 * max |x64|                        (measured 9e-7 / 1.5e-6)
  * 500 steps against the PyTorch fp32 trainer on the same minibatches: max |p_dev - p_torch| <= 3e-5 * max |p_torch - p_0|
    (measured 3e-6: fp32 rounding of two summation orders, compounded), per-step losses within 1e-5 relative (1.5e-6)
  * train() against the reference loop: identical epoch count, early-stop epoch and elite set; loss and score histories
    within 1e-5 relative (measured 1e-7)
  * preprocessing against float64: 1e-6 * max(1, |x|) (measured 1.5e-7); eval_score against a float64 forward: 1e-6
    relative (measured 4e-8)
  * ModelEnv after train(): bit-identical to a freshly staged copy of the trained model
"""
import copy
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from mbrl_lib_b200 import functions, models, replay, synthetic as syn, trainer as tr  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _report(name, value):
    print(f"DEVIATION {name} {value:.3e}")


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


def _prefill_state(opt, params, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    for p in params:
        if not p.requires_grad:
            continue
        opt.state[p] = {"step": torch.tensor(9.0),
                        "exp_avg": (torch.randn(p.shape, generator=g) * 1e-2).to(p.device, p.dtype),
                        "exp_avg_sq": (torch.rand(p.shape, generator=g) * 1e-4 + 1e-6).to(p.device, p.dtype)}


STEP_CASES = [  # activation, deterministic, learned reward, E, Bm, hid, learned bounds
    ("silu", False, True, 7, 32, 200, False),
    ("relu", False, False, 5, 256, 143, False),
    ("leaky_relu", False, True, 1, 1, 143, True),
    ("silu", True, True, 5, 1, 64, False),
    ("relu", True, False, 7, 32, 143, False),
    ("leaky_relu", True, True, 1, 256, 200, False),
    ("silu", False, False, 1, 32, 143, True),
    ("relu", False, True, 7, 1, 64, False),
    ("leaky_relu", False, False, 5, 32, 143, False),
]


@pytest.mark.parametrize("act,det,learned,E,Bm,hid,bounds", STEP_CASES)
def test_one_adam_step_matches_float64(act, det, learned, E, Bm, hid, bounds):
    D, A = 17, 6
    out = D + int(learned)
    model = _model(E, D + A, out, hid, act, det, seed=E * 1000 + Bm + hid, learn_bounds=bounds, learned_rewards=learned)
    trainer = tr.ModelTrainer(model, optim_lr=2.8e-4, weight_decay=1e-4, optim_eps=1e-8)
    params = list(model.parameters())
    _prefill_state(trainer.optimizer, params, seed=7)
    m64 = copy.deepcopy(model.model).double()
    opt64 = torch.optim.Adam(m64.parameters(), lr=2.8e-4, weight_decay=1e-4, eps=1e-8)
    _prefill_state(opt64, list(m64.parameters()), seed=7)
    old = [p.detach().double().clone() for p in params]

    n = 300
    g = torch.Generator(device="cpu").manual_seed(E + Bm)
    X = torch.randn(n, D + A, generator=g).to(DEV)
    Y = (torch.randn(n, out, generator=g) * 0.5).to(DEV)
    idx = torch.randint(0, n, (E, 1, Bm), generator=g).numpy().astype(np.int32)
    dm = tr._DeviceModel(model, trainer.optimizer)
    loss32 = float(dm.run_steps(X, Y, idx, Bm)[0])
    dm.close()

    rows = torch.from_numpy(idx[:, 0].astype(np.int64)).to(DEV)
    x64, y64 = X.double()[rows], Y.double()[rows]
    opt64.zero_grad()
    loss64, _ = m64.loss(x64, y64)
    loss64.backward()
    opt64.step()
    _report(f"step_loss[{act},{det},{learned},{E},{Bm},{hid}]", abs(loss32 - float(loss64)) / max(1.0, abs(float(loss64))))
    assert abs(loss32 - float(loss64)) <= 1e-6 * max(1.0, abs(float(loss64)))

    for p, p0, q in zip(params, old, m64.parameters()):
        if not p.requires_grad:
            assert torch.equal(p.detach().double(), p0)
            continue
        du, du64 = p.detach().double() - p0, q.detach() - p0
        half_ulp = torch.from_numpy(np.spacing(np.abs(p.detach().cpu().numpy()))).to(DEV).double() / 2
        err = float(((du - du64).abs() - half_ulp).clamp_min(0).max() / du64.abs().max())
        st, st64 = trainer.optimizer.state[p], opt64.state[q]
        em = float((st["exp_avg"].double() - st64["exp_avg"]).abs().max() / st64["exp_avg"].abs().max())
        ev = float((st["exp_avg_sq"].double() - st64["exp_avg_sq"]).abs().max() / st64["exp_avg_sq"].abs().max())
        _report(f"step_update[{act},{det},{E},{Bm},{tuple(p.shape)}]", err)
        _report(f"step_exp_avg[{act},{det},{E},{Bm},{tuple(p.shape)}]", em)
        _report(f"step_exp_avg_sq[{act},{det},{E},{Bm},{tuple(p.shape)}]", ev)
        assert err <= 2e-4 and em <= 1e-5 and ev <= 1e-5, (tuple(p.shape), err, em, ev)
        assert float(st["step"]) == 10.0


def test_500_steps_follow_the_pytorch_trainer():
    E, D, A, Bm, steps = 7, 18, 6, 32, 500
    model = _model(E, D + A, D + 1, 200, "silu", False, seed=3)
    ref = copy.deepcopy(model)
    trainer = tr.ModelTrainer(model, optim_lr=2.8e-4, weight_decay=1e-4)
    opt = torch.optim.Adam(ref.parameters(), lr=2.8e-4, weight_decay=1e-4, eps=1e-8)
    p0 = [p.detach().clone() for p in model.parameters()]
    n = 4000
    g = torch.Generator(device="cpu").manual_seed(5)
    X = torch.randn(n, D + A, generator=g).to(DEV)
    Y = (torch.tanh(X[:, :D + 1] * 0.7) + 0.05 * torch.randn(n, D + 1, generator=g).to(DEV)).contiguous()
    idx = torch.randint(0, n, (E, steps, Bm), generator=g).numpy().astype(np.int32)
    dm = tr._DeviceModel(model, trainer.optimizer)
    losses = dm.run_steps(X, Y, idx, Bm)
    dm.close()
    ref_losses = []
    for s in range(steps):
        rows = torch.from_numpy(idx[:, s].astype(np.int64)).to(DEV)
        loss, _ = ref.model.update(X[rows], opt, target=Y[rows])
        ref_losses.append(loss)
    worst = 0.0
    for p, q, a in zip(model.parameters(), ref.parameters(), p0):
        if p.requires_grad:
            worst = max(worst, float((p - q).abs().max() / (q - a).abs().max()))
    lerr = float(np.max(np.abs(losses - np.array(ref_losses)) / np.abs(ref_losses)))
    _report("trajectory_params", worst)
    _report("trajectory_losses", lerr)
    assert worst <= 3e-5 and lerr <= 1e-5


# ---- train() end to end ----------------------------------------------------------------------------------------------
def _transitions(n, D, A, seed):
    rng = np.random.default_rng(seed)
    obs = rng.standard_normal((n, D)).astype(np.float32)
    act = rng.uniform(-1, 1, (n, A)).astype(np.float32)
    M = rng.standard_normal((D + A, D)).astype(np.float32) * 0.5
    nxt = (obs + np.tanh(np.concatenate([obs, act], 1) @ M) + 0.1 * rng.standard_normal((n, D))).astype(np.float32)
    rew = (np.sin(obs[:, 0]) + act.sum(1) + 0.1 * rng.standard_normal(n)).astype(np.float32)
    return replay.TransitionBatch(obs, act, nxt, rew, np.zeros(n, bool), np.zeros(n, bool))


def _fixture(seed=0):
    """E = 5, ReLU, 3 elites, members 3 and 4 with a dead first layer (zero weights, bias -1: they only learn their output
    bias).  The test checks that the fixture's decisions are clear-cut in the reference run: every epoch's improvement is
    far from the threshold, and the elite set's boundary far from the runs' deviation."""
    D, A = 4, 2
    model = _model(5, D + A, D + 1, 64, "relu", False, seed=seed, num_layers=3, num_elites=3)
    with torch.no_grad():
        first = model.model.hidden_layers[0][0]
        first.weight[3:].zero_()
        first.bias[3:].fill_(-1.0)
    return model, _transitions(1024, D, A, seed + 1), _transitions(512, D, A, seed + 2)


def _run(model, train_store, val_store, device, **kw):
    trainer = tr.ModelTrainer(model, optim_lr=3e-3, weight_decay=1e-4)
    if not device:
        trainer._device_supported = lambda: False
    ds = replay.BootstrapIterator(train_store, 32, 5, shuffle_each_epoch=True, rng=np.random.default_rng(11))
    val = replay.TransitionIterator(val_store, 64) if val_store is not None else None
    seen = []
    cb = lambda m, it, ep, loss, score, best: seen.append((None if score is None else score.cpu().numpy(),
                                                          None if best is None else best.cpu().numpy()))
    out = trainer.train(ds, val, callback=cb, **kw)
    return trainer, out, seen


def test_train_end_to_end_matches_the_reference_loop():
    model, train_store, val_store = _fixture()
    ref_model = copy.deepcopy(model)
    kw = dict(num_epochs=40, patience=3, improvement_threshold=0.1)
    _, (l_dev, s_dev), seen_dev = _run(model, train_store, val_store, True, **kw)
    _, (l_ref, s_ref), seen_ref = _run(ref_model, train_store, val_store, False, **kw)
    # the fixture is clear-cut: in the reference run every epoch's best relative improvement is far from the threshold
    best = None
    for score, b in seen_ref:
        if best is not None:
            margin = float(np.max((best - score) / np.abs(best))) - kw["improvement_threshold"]
            assert abs(margin) > 0.01, margin
        best = b
    assert len(l_dev) == len(l_ref) < kw["num_epochs"], (len(l_dev), len(l_ref))  # same early stop
    assert len(s_dev) == len(s_ref)
    lerr = float(np.max(np.abs(np.array(l_dev) - l_ref) / np.abs(l_ref)))
    serr = float(np.max(np.abs(np.array(s_dev) - s_ref) / np.abs(s_ref)))
    _report("train_loss_history", lerr)
    _report("train_score_history", serr)
    assert lerr <= 1e-5 and serr <= 1e-5
    assert set(model.model.elite_models) == set(ref_model.model.elite_models)
    # the elite set is clear-cut too: the 3rd and 4th best scores are apart by far more than the two runs' deviation
    ranked = np.sort(seen_ref[-1][1])
    assert (ranked[3] - ranked[2]) / ranked[2] > 100 * max(serr, 1e-6), ranked


def test_train_on_a_float64_store_matches_the_reference_loop():
    """pets.train / mbpo.train build float64 replay buffers (normalize_double_precision): the per-epoch path must read
    them as double, computing as the reference does, and follow the reference loop as closely as on float32 data."""
    model, train_store, val_store = _fixture(seed=8)
    model.input_normalizer = models.Normalizer(model.model.in_size, DEV, dtype=torch.float64)
    x = np.concatenate([train_store.obs, train_store.act], 1).astype(np.float64)
    model.input_normalizer.mean = torch.tensor(x.mean(0, keepdims=True), device=DEV)
    model.input_normalizer.std = torch.tensor(x.std(0, ddof=1, keepdims=True), device=DEV)
    rng = np.random.default_rng(23)
    f64 = lambda st: replay.TransitionBatch(*(v.astype(np.float64) + 1e-9 * rng.standard_normal(v.shape)
                                              for v in st.astuple()[:4]), st.terminateds, st.truncateds)
    train_store, val_store = f64(train_store), f64(val_store)
    ref_model = copy.deepcopy(model)
    trainer, (l_dev, s_dev), _ = _run(model, train_store, val_store, True, num_epochs=4)
    assert trainer._store_supported(replay.TransitionIterator(train_store, 32))  # the per-epoch path, not a fallback
    _, (l_ref, s_ref), _ = _run(ref_model, train_store, val_store, False, num_epochs=4)
    lerr = float(np.max(np.abs(np.array(l_dev) - l_ref) / np.abs(l_ref)))
    serr = float(np.max(np.abs(np.array(s_dev) - s_ref) / np.abs(s_ref)))
    _report("train_f64_loss_history", lerr)
    _report("train_f64_score_history", serr)
    assert len(l_dev) == len(l_ref) == 4 and lerr <= 1e-5 and serr <= 1e-5
    for p, q in zip(model.parameters(), ref_model.parameters()):
        assert float((p - q).abs().max()) <= 1e-4 * max(1e-3, float(q.abs().max()))


def test_train_batch_callback_runs_the_reference_loop():
    model, train_store, _ = _fixture(seed=4)
    ref_model = copy.deepcopy(model)
    calls = []
    trainer = tr.ModelTrainer(model, optim_lr=3e-3, weight_decay=1e-4)
    ds = replay.BootstrapIterator(train_store, 32, 5, shuffle_each_epoch=True, rng=np.random.default_rng(11))
    out = trainer.train(ds, num_epochs=2, batch_callback=lambda ep, loss, meta, mode: calls.append((ep, mode)))
    _, out_ref, _ = _run(ref_model, train_store, None, False, num_epochs=2)
    assert calls.count((0, "train")) == calls.count((1, "train")) == 32 and calls.count((1, "eval")) == 32
    assert out == out_ref  # the same PyTorch loop on the same minibatches
    for p, q in zip(model.parameters(), ref_model.parameters()):
        assert torch.equal(p, q)


def test_train_without_evaluation():
    model, train_store, _ = _fixture(seed=5)
    ref_model = copy.deepcopy(model)
    elites_before = model.model.elite_models
    _, (l_dev, s_dev), _ = _run(model, train_store, None, True, num_epochs=3, evaluate=False)
    _, (l_ref, s_ref), _ = _run(ref_model, train_store, None, False, num_epochs=3, evaluate=False)
    assert s_dev == s_ref == [] and len(l_dev) == 3 and model.model.elite_models == elites_before
    assert float(np.max(np.abs(np.array(l_dev) - l_ref) / np.abs(l_ref))) <= 1e-5


def test_plain_iterable_takes_one_fused_step_per_batch():
    model, train_store, _ = _fixture(seed=6)
    ref_model = copy.deepcopy(model)
    batches = [train_store[i:i + 32] for i in range(0, 256, 32)]
    tm = tr.ModelTrainer(model, optim_lr=3e-3, weight_decay=1e-4)
    l_dev, _ = tm.train(batches, num_epochs=2, evaluate=False)
    tr_ref = tr.ModelTrainer(ref_model, optim_lr=3e-3, weight_decay=1e-4)
    tr_ref._device_supported = lambda: False
    l_ref, _ = tr_ref.train(batches, num_epochs=2, evaluate=False)
    assert float(np.max(np.abs(np.array(l_dev) - l_ref) / np.abs(l_ref))) <= 1e-5
    assert float(tm.optimizer.state[model.model.mean_and_logvar.weight]["step"]) == 16


# ---- preprocessing and evaluation ------------------------------------------------------------------------------------
@pytest.mark.parametrize("proc,norm,store_dtype", [("halfcheetah", "float64", "float32"), ("cartpole", "float64", "float32"),
                                                   ("halfcheetah", "float32", "float32"), (None, None, "float32"),
                                                   ("halfcheetah", "float64", "float64"), ("cartpole", "float32", "float64"),
                                                   (None, None, "float64")])
def test_preprocess_and_eval_score_match_float64(proc, norm, store_dtype):
    """Float32 stores: the reference computes in float32 (float64 statistics promote the normalisation), so the float64
    restatement bounds the rounding.  Float64 stores (mbrl-lib's PETS / MBPO replay buffers): the reference computes in
    double and rounds at the end, so the inputs and targets must be that double result rounded to float32."""
    D, A = (18, 6) if proc != "cartpole" else (4, 1)
    Dp = D + (1 if proc == "cartpole" else 0)
    store = _transitions(3001, D, A, seed=9)
    if store_dtype == "float64":  # values that float32 cannot hold: a float32 reading of the store would show
        rng = np.random.default_rng(17)
        store = replay.TransitionBatch(*(x.astype(np.float64) + 1e-9 * rng.standard_normal(x.shape) for x in store.astuple()[:4]),
                                       store.terminateds, store.truncateds)
    model = _model(7, Dp + A, D + 1, 200, "silu", False, seed=2, normalize=norm is not None,
                   normalize_double_precision=norm == "float64", obs_process_fn=functions.OBS_PROCESS_FNS[proc],
                   no_delta_list=[0, 2])
    o64, a64 = store.obs.astype(np.float64), store.act.astype(np.float64)
    if proc == "halfcheetah":
        po = np.concatenate([o64[:, 1:2], np.sin(o64[:, 2:3]), np.cos(o64[:, 2:3]), o64[:, 3:]], 1)
    elif proc == "cartpole":
        po = np.concatenate([np.sin(o64[:, 1:2]), np.cos(o64[:, 1:2]), o64[:, :1], o64[:, 2:]], 1)
    else:
        po = o64
    x64 = np.concatenate([po, a64], 1)
    if norm is not None:
        rng = np.random.default_rng(3)
        mean, std = rng.standard_normal((1, Dp + A)), rng.uniform(0.5, 2.0, (1, Dp + A))
        dt = torch.float64 if norm == "float64" else torch.float32
        model.input_normalizer.mean = torch.tensor(mean, dtype=dt, device=DEV)
        model.input_normalizer.std = torch.tensor(std, dtype=dt, device=DEV)
        x64 = (x64 - mean) / std
    y64 = store.next_obs.astype(np.float64) - o64
    y64[:, [0, 2]] = store.next_obs[:, [0, 2]]
    y64 = np.concatenate([y64, store.rewards[:, None].astype(np.float64)], 1)

    trainer = tr.ModelTrainer(model)
    dm = tr._DeviceModel(model, trainer.optimizer)
    X, Y, _ = dm.stage(store)
    xe = float(np.max(np.abs(X.cpu().numpy() - x64) / np.maximum(1.0, np.abs(x64))))
    ye = float(np.max(np.abs(Y.cpu().numpy() - y64) / np.maximum(1.0, np.abs(y64))))
    _report(f"preprocess_inputs[{proc},{norm},{store_dtype}]", xe)
    _report(f"preprocess_targets[{proc},{norm},{store_dtype}]", ye)
    assert xe <= 1e-6 and ye <= 1e-6
    if store_dtype == "float64":  # the double computation rounded once: equal up to sin / cos / division rounding
        assert np.max(np.abs(Y.cpu().numpy() - y64.astype(np.float32))) <= 1e-7 * max(1.0, np.abs(y64).max())
        np.testing.assert_array_equal(Y.cpu().numpy()[:, -1], store.rewards.astype(np.float32))
    scores = dm.eval_score(X, Y).cpu().numpy().astype(np.float64)
    dm.close()
    m64 = copy.deepcopy(model.model).double()
    with torch.no_grad():
        mean64, _ = m64.forward(X.double())
        want = ((mean64 - Y.double()) ** 2).mean((1, 2)).cpu().numpy()
    se = float(np.max(np.abs(scores - want) / want))
    _report(f"eval_score[{proc},{norm},{store_dtype}]", se)
    assert se <= 1e-6
    # evaluate() on an iterator is the same kernel over the iterator's store, per member
    ev = trainer.evaluate(replay.BootstrapIterator(store, 32, 7)).cpu().numpy()
    assert np.array_equal(ev, scores.astype(np.float32))


# ---- the planner sees the trained weights ----------------------------------------------------------------------------
class _Box:
    def __init__(self, lo, hi, n):
        self.low, self.high, self.shape = np.full(n, lo, np.float32), np.full(n, hi, np.float32), (n,)


@pytest.mark.parametrize("hand_off", [False, True])
def test_model_env_sees_the_trained_weights(hand_off):
    import mbrl_lib_b200 as bp

    spec = syn.CASES["halfcheetah_small"]
    arrays = syn.make_model_arrays(spec)
    inp = syn.make_rollout_inputs(spec)
    model = bp.model_from_arrays(spec, arrays, DEV)

    class _Env:
        observation_space = _Box(-np.inf, np.inf, spec.obs_dim)
        action_space = _Box(spec.action_lb, spec.action_ub, spec.act_dim)

    def evaluate(env):
        out = env.evaluate_action_sequences(torch.from_numpy(inp["actions"]).to(DEV), inp["obs0"], spec.particles,
                                            _perms=torch.from_numpy(inp["perms"]).to(DEV),
                                            _eps=torch.from_numpy(inp["eps"]).to(DEV))
        return out.cpu().numpy()

    env = bp.ModelEnv(_Env(), model, functions.no_termination, functions.reward_halfcheetah,
                      generator=torch.Generator(device=DEV), precision="f32", ts1="perms")
    before = evaluate(env)
    trainer = tr.ModelTrainer(model, optim_lr=1e-3, weight_decay=1e-5)
    if hand_off:
        env.hand_off_from(trainer)
    store = _transitions(640, spec.obs_dim, spec.act_dim, seed=13)
    trainer.train(replay.BootstrapIterator(store, 32, spec.ensemble_size, rng=np.random.default_rng(0)), num_epochs=2,
                  evaluate=False)
    after = evaluate(env)
    fresh = bp.ModelEnv(_Env(), copy.deepcopy(model), functions.no_termination, functions.reward_halfcheetah,
                        generator=torch.Generator(device=DEV), precision="f32", ts1="perms")
    assert not np.array_equal(before, after)
    assert np.array_equal(after, evaluate(fresh))


# ---- the reference's own objects -------------------------------------------------------------------------------------
def test_trains_real_reference_objects():
    from baseline import reference_arm as ra

    mbrl, src = ra.import_reference()
    if mbrl is None:
        pytest.skip(f"reference not importable here: {src}")
    from mbrl.types import TransitionBatch
    from mbrl.util.replay_buffer import BootstrapIterator

    spec = syn.CASES["halfcheetah_small"]
    env = ra.build_model_env(mbrl, spec, syn.make_model_arrays(spec))
    wrapper = env.dynamics_model.to(DEV)
    wrapper.device = wrapper.model.device = torch.device(DEV)
    nz = wrapper.input_normalizer
    if nz is not None:
        nz.mean, nz.std, nz.device = nz.mean.to(DEV), nz.std.to(DEV), torch.device(DEV)
    assert wrapper.obs_process_fn is None
    ref = copy.deepcopy(wrapper)
    s = _transitions(640, spec.obs_dim, spec.act_dim, seed=21)
    store = TransitionBatch(s.obs, s.act, s.next_obs, s.rewards, s.terminateds, s.truncateds)
    results = []
    for m, device in ((wrapper, True), (ref, False)):
        trainer = tr.ModelTrainer(m, optim_lr=1e-3, weight_decay=1e-5)
        assert trainer._device_supported()
        if not device:
            trainer._device_supported = lambda: False
        ds = BootstrapIterator(store, 32, spec.ensemble_size, shuffle_each_epoch=True, rng=np.random.default_rng(2))
        assert tr._iterator_kind(ds) == "bootstrap"
        results.append(trainer.train(ds, num_epochs=2))
    (l_dev, s_dev), (l_ref, s_ref) = results
    assert float(np.max(np.abs(np.array(l_dev) - l_ref) / np.abs(l_ref))) <= 1e-5
    assert float(np.max(np.abs(np.array(s_dev) - s_ref) / np.abs(s_ref))) <= 1e-5
