"""CPU checks of the training path's host side: the C ABI's refusals, the minibatch rows read from the iterators, which
datasets / models take the device path, and the reference PyTorch loop ``ModelTrainer`` falls back to."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from mbrl_lib_b200 import _lib, models, replay, trainer as tr  # noqa: E402


def _desc(**kw):
    d = _lib.TrainDesc()
    vals = dict(ensemble_size=2, in_size=4, out_size=3, hid_size=8, num_hidden=2, activation=_lib.ACT["silu"],
                deterministic=0, learn_logvar_bounds=0, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0)
    vals.update(kw)
    for k, v in vals.items():
        setattr(d, k, v)
    return d


def _ptrs(n, null_at=None):
    return (C.c_void_p * n)(*[None if i == null_at else 0x1000 + 256 * i for i in range(n)])


def _create(d, P, M, V):
    h = C.c_void_p()
    rc = _lib.load().b200pets_trainer_create(C.byref(d), P, M, V, C.byref(h))
    return rc, h


def test_trainer_create_refusals():
    lib = _lib.load()
    n = 2 * 3 + 2
    rc, h = _create(_desc(), _ptrs(n), _ptrs(n), _ptrs(n))
    assert rc == 0 and h.value
    lib.b200pets_trainer_destroy(h)
    assert _create(_desc(), _ptrs(n, null_at=3), _ptrs(n), _ptrs(n))[0] == -1  # a NULL bias
    assert _create(_desc(), _ptrs(n), _ptrs(n), _ptrs(n, null_at=0))[0] == -1  # a NULL moment
    assert _create(_desc(), _ptrs(n, null_at=7), _ptrs(n), _ptrs(n))[0] == -1  # a NULL logvar bound
    assert lib.b200pets_trainer_create(None, _ptrs(n), _ptrs(n), _ptrs(n), C.byref(C.c_void_p())) == -1
    assert lib.b200pets_trainer_create(C.byref(_desc()), _ptrs(n), _ptrs(n), _ptrs(n), None) == -1
    # fixed bounds need no moments; learned bounds do
    rc, h = _create(_desc(), _ptrs(n), _ptrs(n, null_at=6), _ptrs(n, null_at=7))
    assert rc == 0
    lib.b200pets_trainer_destroy(h)
    assert _create(_desc(learn_logvar_bounds=1), _ptrs(n), _ptrs(n, null_at=6), _ptrs(n))[0] == -1
    # 8 layers (7 hidden + output) is the limit
    assert _create(_desc(num_hidden=7), _ptrs(16 + 2), _ptrs(18), _ptrs(18))[0] == 0
    rc = _create(_desc(num_hidden=8), _ptrs(18 + 2), _ptrs(20), _ptrs(20))[0]
    assert rc == -2 and b"hidden layers" in lib.b200pets_last_error()
    rc = _create(_desc(activation=7), _ptrs(n), _ptrs(n), _ptrs(n))[0]
    assert rc == -2 and b"activation" in lib.b200pets_last_error()
    assert _create(_desc(hid_size=0), _ptrs(n), _ptrs(n), _ptrs(n))[0] == -1


def test_epoch_and_eval_refusals():
    lib = _lib.load()
    n = 2 * 3 + 2
    rc, h = _create(_desc(), _ptrs(n), _ptrs(n), _ptrs(n))
    assert rc == 0
    try:
        need = lib.b200pets_train_workspace_bytes(h, 32)
        assert need > 0 and lib.b200pets_train_workspace_bytes(h, 64) > need
        p = C.c_void_p(0x1000)
        args = lambda **kw: dict(dict(rows=100, X=p, Y=p, idx=p, steps=4, batch=32, last=4, step=0, losses=p, ws=p,
                                      nbytes=need), **kw)

        def epoch(**kw):
            a = args(**kw)
            return lib.b200pets_train_epoch(h, a["rows"], a["X"], a["Y"], a["idx"], a["steps"], a["batch"], a["last"],
                                            a["step"], a["losses"], a["ws"], a["nbytes"], None)

        for null in ("X", "Y", "idx", "losses", "ws"):
            assert epoch(**{null: None}) == -1
        assert epoch(nbytes=need - 1) == -1 and b"workspace" in lib.b200pets_last_error()
        assert epoch(last=33) == -1 and epoch(last=0) == -1 and epoch(steps=0) == -1 and epoch(rows=0) == -1
        assert lib.b200pets_train_epoch(None, 100, p, p, p, 4, 32, 4, 0, p, p, need, None) == -1
        eneed = lib.b200pets_eval_score_workspace_bytes(h, 1000)
        assert eneed > 0
        assert lib.b200pets_eval_score(h, 1000, p, p, p, p, eneed - 1, None) == -1
        assert lib.b200pets_eval_score(h, 1000, None, p, p, p, eneed, None) == -1
        assert lib.b200pets_eval_score(h, 1000, p, p, None, p, eneed, None) == -1
        assert lib.b200pets_eval_score(h, 0, p, p, p, p, eneed, None) == -1
    finally:
        lib.b200pets_trainer_destroy(h)


def test_preprocess_refusals():
    lib = _lib.load()
    d = _lib.PrepDesc()
    d.obs_dim, d.act_dim, d.obs_process, d.norm_mode, d.target_is_delta, d.learned_rewards = 4, 2, 0, 0, 1, 1
    p = C.c_void_p(0x1000)
    nd = (C.c_int32 * 1)(5)
    assert lib.b200pets_train_preprocess(C.byref(d), 10, p, p, p, p, None, None, nd, 1, p, p, None) == -1  # column 5 of 4
    assert lib.b200pets_train_preprocess(C.byref(d), 10, p, p, p, None, None, None, nd, 0, p, p, None) == -1  # no reward
    d.norm_mode = 2
    assert lib.b200pets_train_preprocess(C.byref(d), 10, p, p, p, p, None, None, nd, 0, p, p, None) == -1  # no statistics
    d.norm_mode, d.obs_process = 0, 9
    assert lib.b200pets_train_preprocess(C.byref(d), 10, p, p, p, p, None, None, nd, 0, p, p, None) == -2
    d.obs_process, d.dtype = 0, 2  # neither float32 nor float64
    assert lib.b200pets_train_preprocess(C.byref(d), 10, p, p, p, p, None, None, nd, 0, p, p, None) == -2
    assert b"dtype" in lib.b200pets_last_error()


def test_transition_dtype_is_the_references_compute_precision():
    f32 = _store()
    f64 = replay.TransitionBatch(*(x.astype(np.float64) if x.dtype == np.float32 else x for x in f32.astuple()))
    assert tr.transition_dtype(f32) == torch.float32
    assert tr.transition_dtype(f64) == torch.float64
    mixed = replay.TransitionBatch(f32.obs, f64.act, f32.next_obs, f32.rewards, f32.terminateds, f32.truncateds)
    assert tr.transition_dtype(mixed) == torch.float64  # numpy / torch promote the float32 columns against it
    # the reward column alone does not change the precision: it is rounded to float32 at the end either way
    assert tr.transition_dtype(replay.TransitionBatch(*f32.astuple()[:3], f64.rewards, *f32.astuple()[4:])) == torch.float32
    half = replay.TransitionBatch(f32.obs.astype(np.float16), *f32.astuple()[1:])
    assert tr.transition_dtype(half) is None
    ds = replay.TransitionIterator(half, 8)
    assert not tr.ModelTrainer._store_supported(ds) and tr.ModelTrainer._store_supported(replay.TransitionIterator(f64, 8))


# ---- minibatches ---------------------------------------------------------------------------------------------------
def _store(n=103, D=3, A=2, seed=0):
    rng = np.random.default_rng(seed)
    f = lambda *s: rng.standard_normal(s).astype(np.float32)
    return replay.TransitionBatch(f(n, D), f(n, A), f(n, D), f(n), np.zeros(n, bool), np.zeros(n, bool))


@pytest.mark.parametrize("kind", ["plain", "plain_shuffle", "boot_perm", "boot_replace", "boot_one"])
def test_epoch_indices_are_the_iterators_minibatches(kind):
    import copy

    store = _store()
    E = 1 if kind == "boot_one" else 4
    if kind.startswith("plain"):
        ds = replay.TransitionIterator(store, 16, shuffle_each_epoch=kind == "plain_shuffle", rng=np.random.default_rng(1))
    else:
        ds = replay.BootstrapIterator(store, 16, E, shuffle_each_epoch=True, permute_indices=kind != "boot_replace",
                                      rng=np.random.default_rng(1))
    twin = copy.deepcopy(ds)
    for epoch in range(3):
        idx, last = tr.epoch_indices(ds, tr._iterator_kind(ds), E)
        batches = list(twin)
        assert idx.shape == (E, len(batches), 16) and last == len(batches[-1].obs if batches[-1].obs.ndim == 2
                                                                      else batches[-1].obs[0])
        for s, b in enumerate(batches):
            rows = idx[:, s, :last if s == len(batches) - 1 else 16]
            if b.obs.ndim == 3:
                np.testing.assert_array_equal(b.obs, store.obs[rows])
            else:
                for e in range(E):
                    np.testing.assert_array_equal(b.obs, store.obs[rows[e]])
        assert ds._current_batch == twin._current_batch
    # the generators advanced alike
    assert ds._rng.integers(1 << 30) == twin._rng.integers(1 << 30)


def test_iterator_recognition():
    store = _store()
    assert tr._iterator_kind(replay.TransitionIterator(store, 8)) == "plain"
    assert tr._iterator_kind(replay.BootstrapIterator(store, 8, 3)) == "bootstrap"

    class Windows(replay.BootstrapIterator):  # forms its batches differently: not the fast path
        def __getitem__(self, item):
            return self.transitions[item]

    assert tr._iterator_kind(Windows(store, 8, 3)) is None
    assert tr._iterator_kind([store[:8], store[8:16]]) is None


def _small_model(device="cpu", E=3, deterministic=False, seed=0):
    torch.manual_seed(seed)
    mlp = models.GaussianMLP(5, 4, device, num_layers=2, ensemble_size=E, hid_size=16, deterministic=deterministic,
                             activation="silu")
    with torch.no_grad():
        for p in mlp.parameters():
            if p.requires_grad:
                p.normal_(0.0, 0.3)
    return models.OneDTransitionRewardModel(mlp, num_elites=2)


def test_cpu_model_runs_the_reference_loop():
    """No CUDA parameters -> the reference's PyTorch loop: losses per epoch, scores, elites, callbacks."""
    model = _small_model()
    store = _store(n=64, D=3, A=2)
    ds = replay.BootstrapIterator(store, 16, 3, shuffle_each_epoch=True, rng=np.random.default_rng(0))
    trainer = tr.ModelTrainer(model, optim_lr=1e-2, weight_decay=1e-4)
    assert not trainer._device_supported()
    seen = []
    losses, scores = trainer.train(ds, num_epochs=3, batch_callback=lambda *a: seen.append(a[-1]))
    assert len(losses) == 3 and len(scores) == 3 and all(np.isfinite(losses))
    assert seen.count("train") == 3 * 4 and seen.count("eval") == 3 * 4
    assert model.model.elite_models is not None and len(model.model.elite_models) == 2
    assert all(float(trainer.optimizer.state[p]["step"]) == 12 for p in model.parameters() if p.requires_grad)
    losses2, scores2 = trainer.train(ds, num_epochs=2, evaluate=False)
    assert len(losses2) == 2 and scores2 == []


def test_container_loss_is_the_reference_formula():
    """GaussianMLP.loss restated by hand in float64: NLL through the soft bounds, plus the bound penalty."""
    model = _small_model().model.double()
    x = torch.randn(3, 7, 5, dtype=torch.float64)
    y = torch.randn(3, 7, 4, dtype=torch.float64)
    h = x
    for layer in model.hidden_layers:
        z = h @ layer[0].weight + layer[0].bias
        h = z * torch.sigmoid(z)
    o = h @ model.mean_and_logvar.weight + model.mean_and_logvar.bias
    mean, lv = o[..., :4], o[..., 4:]
    sp = lambda t: torch.log1p(torch.exp(t))
    lv = model.max_logvar - sp(model.max_logvar - lv)
    lv = model.min_logvar + sp(lv - model.min_logvar)
    want = (((mean - y) ** 2 * torch.exp(-lv) + lv).mean((1, 2)).sum()
            + 0.01 * (model.max_logvar.sum() - model.min_logvar.sum()))
    got, _ = model.loss(x, y)
    assert abs(got.item() - want.item()) < 1e-10


def test_stage_refuses_a_model_the_transitions_do_not_fit():
    """pets_cartpole_paper_version without dynamics_model.in_size=6: the cartpole obs_process_fn makes 4 + 1 observation
    columns and the action one more, so a model of in_size 5 would have the preprocessing kernel write past its staged
    inputs.  The check runs on the host, before anything is copied or launched."""
    from mbrl_lib_b200 import functions

    mlp = models.GaussianMLP(5, 5, "cpu", num_layers=2, ensemble_size=2, hid_size=8)
    model = models.OneDTransitionRewardModel(mlp, obs_process_fn=functions.OBS_PROCESS_FNS["cartpole"])
    store = _store(n=16, D=4, A=1)
    with pytest.raises(ValueError, match="in_size 5"):
        tr.check_model_sizes(model, 4, 1)
    dm = tr._DeviceModel(model, tr.ModelTrainer(model).optimizer)  # a handle only: nothing runs on a CPU model
    try:
        with pytest.raises(ValueError, match="in_size 5"):
            dm.stage(store)
    finally:
        dm.close()
    # the sizes that do fit, and the reward column
    tr.check_model_sizes(models.OneDTransitionRewardModel(models.GaussianMLP(6, 5, "cpu", num_layers=1, hid_size=8),
                                                          obs_process_fn=functions.OBS_PROCESS_FNS["cartpole"]), 4, 1)
    with pytest.raises(ValueError, match="out_size 5"):
        tr.check_model_sizes(models.OneDTransitionRewardModel(models.GaussianMLP(5, 5, "cpu", num_layers=1, hid_size=8),
                                                              learned_rewards=False), 4, 1)


def test_trainer_supported_refuses_what_trainer_create_refuses():
    lib = _lib.load()
    assert lib.b200pets_trainer_supported(None) == -1
    assert lib.b200pets_trainer_supported(C.byref(_desc(num_hidden=8))) == -2
    assert b"trainer_supported" in lib.b200pets_last_error() and b"hidden layers" in lib.b200pets_last_error()
    assert lib.b200pets_trainer_supported(C.byref(_desc(activation=7))) == -2
    assert lib.b200pets_trainer_supported(C.byref(_desc(hid_size=0))) == -1
