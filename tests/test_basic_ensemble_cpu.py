"""BasicEnsemble on the host: what the staging reads from the model object, when it re-stages, what it refuses, and
the member draws ``ModelEnv`` and the fused plans make (no device needed)."""
import numpy as np
import pytest
import torch

import mbrl_lib_b200 as bp
from mbrl_lib_b200 import synthetic as syn
from mbrl_lib_b200.models import basic_ensemble_from_arrays
from mbrl_lib_b200.staging import StagedModel


def _spec(prop="random_model"):
    import dataclasses

    s = syn.CASES["halfcheetah_small"]
    return dataclasses.replace(s, propagation=prop, elites=None)


def _model(prop="random_model"):
    spec = _spec(prop)
    return spec, basic_ensemble_from_arrays(spec, syn.make_model_arrays(spec), "cpu")


def test_staging_reads_the_container():
    from mbrl_lib_b200 import functions

    spec, model = _model()
    st = StagedModel(model, functions.REWARD_FNS[spec.reward_fn], None, stage=False)
    d = st._describe()
    assert st.member_rule == "rows"
    assert d.member_rule == 1 and d.ensemble_size == spec.ensemble_size == d.num_members
    assert st.members() == list(range(spec.ensemble_size))
    assert (d.in_size, d.out_size, d.hid_size, d.num_hidden) == (spec.in_size, spec.out_size, spec.hid_size, spec.num_layers)


def test_staging_reads_mbrl_basic_ensemble():
    from baseline import reference_arm as ra

    mbrl, src = ra.import_reference()
    if mbrl is None:
        pytest.skip(f"reference not importable here: {src}")
    from mbrl.models import BasicEnsemble, OneDTransitionRewardModel
    cfg = {"_target_": "mbrl.models.GaussianMLP", "device": "cpu", "num_layers": 4, "in_size": 23, "out_size": 18,
           "ensemble_size": 1, "hid_size": 200, "deterministic": False, "activation_fn_cfg": {"_target_": "torch.nn.SiLU"}}
    ens = BasicEnsemble(5, "cpu", cfg, propagation_method="fixed_model")
    model = OneDTransitionRewardModel(ens, target_is_delta=True, normalize=True, learned_rewards=True)
    st = StagedModel(model, None, None, stage=False)
    d = st._describe()
    assert st.member_rule == "rows" and d.ensemble_size == 5 and d.num_members == 5 and d.in_size == 23


def test_signature_follows_every_member():
    _, model = _model()
    st = StagedModel(model, None, None, stage=False)
    sig = st._signature()
    with torch.no_grad():
        model.model.members[3].mean_and_logvar.weight.add_(1.0)
    assert st._signature() != sig
    sig = st._signature()
    from mbrl_lib_b200 import staging

    staging.mark_trained(model.model.members[1])
    assert st._signature() != sig


def test_refusals():
    _, model = _model()
    members = model.model.members
    # unequal log-variance bounds
    with torch.no_grad():
        members[2].max_logvar.add_(0.25)
    with pytest.raises(NotImplementedError, match="learn_logvar_bounds"):
        StagedModel(model, None, None, stage=False)
    # a member of another shape
    _, model = _model()
    model.model.members[1] = bp.GaussianMLP(model.model.in_size, model.model.out_size, "cpu", num_layers=2, hid_size=16,
                                            activation="silu")
    with pytest.raises(NotImplementedError, match="differs"):
        StagedModel(model, None, None, stage=False)
    # a member that is itself an ensemble
    _, model = _model()
    m0 = model.model.members[0]
    model.model.members[0] = bp.GaussianMLP(m0.in_size, m0.out_size, "cpu", num_layers=4, ensemble_size=2,
                                            hid_size=200, activation="silu")
    with pytest.raises(NotImplementedError, match="ensemble_size"):
        StagedModel(model, None, None, stage=False)


def _env(prop):
    """A ModelEnv's host logic over a BasicEnsemble, without a device."""
    _, model = _model(prop)
    env = bp.ModelEnv.__new__(bp.ModelEnv)
    env.staged = StagedModel(model, None, None, stage=False)
    env.device = torch.device("cpu")
    env._rng = torch.Generator().manual_seed(5)
    env.ts1 = "perms"
    return env


@pytest.mark.parametrize("prop", ["random_model", "fixed_model", "expectation"])
def test_evaluation_draws(prop):
    env = _env(prop)
    N, H, P, M = 13, 4, 3, 7
    got = env._eval_perms(prop, N, H, P)
    if prop == "expectation":
        assert got is None
        return
    ref = torch.Generator().manual_seed(5)
    n = H if prop == "random_model" else 1
    want = torch.stack([torch.randint(M, (N * P,), generator=ref) for _ in range(n)])
    assert got.shape == (n, N * P) and torch.equal(got, want)


@pytest.mark.parametrize("prop", ["random_model", "fixed_model"])
def test_fused_cem_draws_in_loop_order(prop):
    env = _env(prop)
    opt = bp.CEMOptimizer(3, 0.1, 11, [[-1.0]] * 4, [[1.0]] * 4, 0.1, "cpu", return_mean_elites=True)
    got = opt._plan_perms(env, prop, 4, 2)
    ref = torch.Generator().manual_seed(5)
    n = 4 if prop == "random_model" else 1
    want = torch.stack([torch.stack([torch.randint(7, (22,), generator=ref) for _ in range(n)]) for _ in range(3)])
    assert torch.equal(got, want)


def test_reset_and_step_draws():
    """reset draws fixed_model's indices, step draws random_model's: one randint(M, (B,)) each, on the env's generator."""
    env = _env("fixed_model")
    env._fresh = lambda: None
    state = env.reset(np.zeros((9, 17), np.float32))
    ref = torch.Generator().manual_seed(5)
    assert torch.equal(state["propagation_indices"], torch.randint(7, (9,), generator=ref))
    # step under random_model, with the library call and the device plumbing stubbed: the indices it passes
    env = _env("random_model")
    calls = []
    env.lib = type("L", (), {"b200pets_step": lambda self, *a: calls.append(a) or 0})()
    env.staged.handle = None
    env.staged.desc = type("D", (), {"reward_fn": -1, "term_fn": -1})()  # known reward / termination functions
    env._fresh = lambda: None
    env._return_as_np = False
    env._seed = 0
    env.precision_for = lambda prop: "f32"
    env._call_offset = lambda: 0
    import mbrl_lib_b200._lib as L
    real_ptr = L.ptr
    seen = []
    L.ptr = lambda t: seen.append(t) or 0
    L.stream_ptr, real_stream = (lambda: 0), L.stream_ptr
    try:
        import contextlib
        torch_cuda_device = torch.cuda.device
        torch.cuda.device = lambda d: contextlib.nullcontext()
        env.step(np.zeros((9, 6), np.float32), {"obs": torch.zeros(9, 17)})
    finally:
        L.ptr, L.stream_ptr = real_ptr, real_stream
        torch.cuda.device = torch_cuda_device
    ref = torch.Generator().manual_seed(5)
    assert len(calls) == 1 and torch.equal(seen[2], torch.randint(7, (9,), generator=ref))


@pytest.mark.parametrize("prop", ["random_model", "fixed_model"])
def test_fused_icem_draws_in_loop_order(prop):
    """Per iteration: the kept elites' permutation (default generator) and then that evaluation's member indices."""
    env = _env(prop)
    opt = bp.ICEMOptimizer(3, 0.1, 40, 1.3, 2.0, [[-1.0]] * 4, [[1.0]] * 4, 0.3, 0.1, "cpu", return_mean_elites=True)
    rows, _, perms = opt._fused_draws(env, prop, 4, 2)
    ref = torch.Generator().manual_seed(5)
    n = 4 if prop == "random_model" else 1
    assert len(perms) == 3
    for r, p in zip(rows, perms):
        want = torch.stack([torch.randint(7, (r * 2,), generator=ref) for _ in range(n)])
        assert torch.equal(p, want)


@pytest.mark.parametrize("prop", ["random_model", "fixed_model"])
def test_batched_evaluation_draws_problem_by_problem(prop):
    """evaluate_action_sequences_batch (and the batched MPPI and CEM plans through _eval_perms) draw problem k's
    indices after problem k-1's, as K single calls do."""
    env = _env(prop)
    per = [env._eval_perms(prop, 5, 3, 2) for _ in range(4)]
    ref = torch.Generator().manual_seed(5)
    n = 3 if prop == "random_model" else 1
    for p in per:
        assert torch.equal(p, torch.stack([torch.randint(7, (10,), generator=ref) for _ in range(n)]))


def test_more_refusals():
    # a member that differs only in activation
    _, model = _model()
    m = model.model.members[1]
    for seq in m.hidden_layers:
        seq[1] = torch.nn.ReLU()
    with pytest.raises(NotImplementedError, match="differs"):
        StagedModel(model, None, None, stage=False)
    # a member that differs only in deterministic
    spec, model = _model()
    m0 = model.model.members[0]
    model.model.members[0] = bp.GaussianMLP(m0.in_size, m0.out_size, "cpu", num_layers=spec.num_layers, ensemble_size=1,
                                            hid_size=spec.hid_size, deterministic=True, activation=spec.activation)
    with pytest.raises(NotImplementedError, match="differs"):
        StagedModel(model, None, None, stage=False)
    # propagation_method None with more than one member
    env = _env("random_model")
    env.staged.mlp.propagation_method = None
    with pytest.raises(ValueError, match="propagation_method"):
        env._propagation()
