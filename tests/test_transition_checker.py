"""The float64 model step (oracle/transition_f64.py) pinned on the CPU before the GPU tests trust it.

* against ``OracleModel.step`` (fp32, itself pinned to the reference's goldens) on every propagation, a deterministic
  model, both observation preprocessors, fp32 / fp64 / no normaliser and a learned reward: measured <= 7.3e-7 of
  max(1, |ref|), the oracle's fp32 rounding (torch's softplus threshold on plan_logvar_extreme);
* against the reference's own goldens ``tests/golden/step_*.npz``;
* in bf16 mode against ``OracleModel(emulate_bf16=True)``: measured <= 4.3e-5 (an activation within an fp32 ulp of a
  bf16 rounding boundary rounds the other way).
"""
import os

import numpy as np
import pytest
import torch

from mbrl_lib_b200 import synthetic as syn
from oracle import pets_oracle as po
from oracle.transition_f64 import TransitionF64, assignment_from_perm, bf16_round, known_done, known_reward

CASES = ["halfcheetah_small", "hopper_tsinf", "silu_expectation", "relu_expectation", "pusher_det", "pets_halfcheetah_small",
         "cartpole_pets", "cartpole", "tc_shallow", "humanoid_trunc", "ant_learned_fn", "plan_logvar_extreme",
         "plan_hid14_deep"]


def _rel(got, ref):
    return float((np.abs(np.asarray(got, np.float64) - ref) / np.maximum(1.0, np.abs(ref))).max())


def _compare(name, bf16):
    spec = syn.CASES[name]
    arrays = syn.make_model_arrays(spec)
    M = spec.num_models
    inp = syn.make_step_inputs(spec, 60 * M)
    om = po.OracleModel(spec, arrays)
    om.emulate_bf16 = bf16
    on, orw, od = om.step(torch.from_numpy(inp["obs"]), torch.from_numpy(inp["act"]), torch.from_numpy(inp["perm"]),
                          torch.from_numpy(inp["eps"]))
    members = None if spec.propagation == "expectation" else assignment_from_perm(inp["perm"], M)
    nobs, rew = TransitionF64(spec, arrays).step(inp["obs"], inp["act"], members, inp["eps"], bf16=bf16)
    out = {"next_obs": _rel(on.numpy(), nobs)}
    if spec.reward_fn is None:
        out["reward"] = _rel(orw.numpy()[:, 0], rew)
    else:  # the oracle's known reward and done, restated on its own next_obs
        out["reward"] = _rel(orw.numpy()[:, 0], known_reward(spec.reward_fn, inp["act"], on.numpy()))
        assert np.array_equal(known_done(spec.term_fn, inp["act"], on.numpy()), od.numpy()[:, 0])
    return out


@pytest.mark.parametrize("name", CASES)
def test_checker_matches_fp32_oracle(name):
    err = _compare(name, bf16=False)
    assert max(err.values()) <= 2e-6, err


@pytest.mark.parametrize("name", CASES)
def test_checker_bf16_mode_matches_bf16_oracle(name):
    err = _compare(name, bf16=True)
    assert max(err.values()) <= 2e-4, err


@pytest.mark.parametrize("name,batch", [("mbpo_halfcheetah_small", 1000), ("cartpole", 500)])
def test_checker_matches_reference_goldens(golden_dir, name, batch):
    spec = syn.CASES[name]
    arrays = syn.make_model_arrays(spec)
    inp = syn.make_step_inputs(spec, batch)
    g = np.load(os.path.join(golden_dir, f"step_{name}.npz"))
    assert str(g["input_sum"]) == syn.checksum(inp)
    members = assignment_from_perm(inp["perm"], spec.num_models)
    nobs, rew = TransitionF64(spec, arrays).step(inp["obs"], inp["act"], members, inp["eps"])
    assert _rel(g["next_obs"], nobs) <= 2e-6
    if spec.reward_fn is None:
        assert _rel(g["reward"][:, 0], rew) <= 2e-6
    else:
        assert np.array_equal(known_reward(spec.reward_fn, inp["act"], g["next_obs"]), g["reward"][:, 0])
    assert np.array_equal(known_done(spec.term_fn, inp["act"], g["next_obs"]), g["done"][:, 0])


def test_bf16_round_matches_torch():
    """bf16_round is round-to-nearest-even to 8 significant bits (torch's fp32 -> bf16 conversion on fp32 inputs)."""
    g = np.random.default_rng(0)
    x = np.concatenate([g.standard_normal(10000) * 10.0 ** g.integers(-6, 6, 10000), [0.0, -0.0, 1.0, 1.00390625,
                                                                                       1.01171875, -3.0e-30]])
    x32 = x.astype(np.float32)
    want = torch.from_numpy(x32).to(torch.bfloat16).double().numpy()
    assert np.array_equal(bf16_round(x32.astype(np.float64)), want)


def test_checker_reads_options_from_the_model():
    """from_model takes the activation slope, delta options, elite order and normaliser from the model object."""
    import dataclasses

    import mbrl_lib_b200 as bp

    spec = dataclasses.replace(syn.CASES["cartpole"], learned_rewards=True, reward_fn=None, no_delta_list=(1, 3),
                               elites=(4, 1, 2, 0))
    arrays = syn.make_model_arrays(spec)
    model = bp.model_from_arrays(spec, arrays, "cpu")
    model.model.hidden_layers[0][1].negative_slope = 0.2
    ck = TransitionF64.from_model(spec, model)
    assert ck.slope == 0.2 and ck.no_delta == [1, 3] and ck.members == [4, 1, 2, 0]
    assert ck.norm_mean.dtype == np.float32
    ref = TransitionF64(spec, arrays, slope=0.2)
    inp = syn.make_step_inputs(spec, 50)
    mem = np.arange(50) % 4
    a = ck.step(inp["obs"], inp["act"], mem, inp["eps"])
    b = ref.step(inp["obs"], inp["act"], mem, inp["eps"])
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert not np.array_equal(a[0], TransitionF64(spec, arrays).step(inp["obs"], inp["act"], mem, inp["eps"])[0])

