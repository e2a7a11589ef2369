"""CPU checks of PlaNet's latent path: the float64 oracle against the reference's goldens, staging against real reference
and local PlaNet objects (read only, stage=False), and the latent kernels' resource use."""
import importlib.util
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from baseline import reference_arm as ra
from mbrl_lib_b200 import latent, models
from oracle import latent_f64 as lo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
mbrl, REF_SRC = ra.import_reference()
needs_ref = pytest.mark.skipif(mbrl is None, reason=f"reference not importable here: {REF_SRC}")
WEIGHT_SEED = 7  # oracle/gen_golden_planet.py
TOL = 2e-5       # the goldens are the reference's fp32 on the CPU


def _golden_params():
    s = lo.GOLDEN_SIZES
    m = models.PlaNetModel(s["action_size"], s["latent_state_size"], s["belief_size"], s["hidden_size_fcs"],
                           min_std=s["min_std"])
    lo.fill_params(m, WEIGHT_SEED)
    return lo.params_of(m)


def _close(got, want, what):
    err = float(np.max(np.abs(np.asarray(got, np.float64) - want) / (1.0 + np.abs(want))))
    assert err <= TOL, f"{what}: {err:.3e} > {TOL}"


def test_oracle_step_reproduces_the_reference(golden_dir):
    g = np.load(os.path.join(golden_dir, "planet_step.npz"))
    p, inp = _golden_params(), lo.golden_inputs("step")
    for tag, eps in (("det", None), ("smp", inp["eps"])):
        s, h, r = lo.step(p, inp["latent"], inp["belief"], inp["act"], eps)
        _close(s, g[f"{tag}_latent"], f"{tag} latent")
        _close(h, g[f"{tag}_belief"], f"{tag} belief")
        _close(r, g[f"{tag}_reward"][:, 0], f"{tag} reward")


def test_oracle_returns_reproduce_the_reference(golden_dir):
    g = np.load(os.path.join(golden_dir, "planet_eval.npz"))
    p, inp = _golden_params(), lo.golden_inputs("eval")
    ret, rows = lo.evaluate(p, inp["latent0"], inp["belief0"], inp["actions"], inp["particles"], inp["eps"])
    _close(ret, g["returns"], "returns")
    assert rows.shape == (inp["actions"].shape[0] * inp["particles"],)


def test_oracle_cem_plan_reproduces_the_reference(golden_dir):
    g = np.load(os.path.join(golden_dir, "planet_cem.npz"))
    p, inp = _golden_params(), lo.golden_inputs("cem")
    H, A = inp["horizon"], lo.GOLDEN_SIZES["action_size"]
    trace = []
    sol = lo.cem_plan(p, inp["latent0"], inp["belief0"], np.zeros((H, A)), -np.ones((H, A)), np.ones((H, A)),
                      inp["iterations"], inp["elite_ratio"], inp["population"], inp["alpha"], inp["z"], inp["eps"],
                      particles=inp["particles"], trace=trace)
    _close(np.stack([t["values"].numpy() for t in trace]), g["values"], "values")
    _close(sol, g["solution"], "solution")


def _check_staged(staged, model):
    d = staged.desc
    assert (d.action_size, d.latent_size, d.belief_size, d.hidden_size) == \
        (model.action_size, model.latent_state_size, model.belief_size, model.prior_transition_model[0].out_features)
    assert d.min_std == pytest.approx(model.min_std)
    params = staged.params()
    assert len(params) == 16
    assert params[2] is model.belief_model.rnn.weight_ih and params[14] is model.reward_model[4].weight
    sig = staged.signature()
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    loss = sum((p ** 2).sum() for p in latent.latent_params(model))
    loss.backward()
    opt.step()
    assert staged.signature() != sig  # an optimizer step bumps the version counters: the next call re-stages


@needs_ref
def test_staging_reads_a_real_reference_planet_model():
    model = mbrl.models.PlaNetModel(
        obs_shape=(3, 64, 64), obs_encoding_size=1024,
        encoder_config=((3, 32, 4, 2), (32, 64, 4, 2), (64, 128, 4, 2), (128, 256, 4, 2)),
        decoder_config=((1024, 1, 1), ((1024, 128, 5, 2), (128, 64, 5, 2), (64, 32, 6, 2), (32, 3, 6, 2))),
        latent_state_size=30, action_size=6, belief_size=200, hidden_size_fcs=200, device="cpu")
    staged = latent.StagedLatentModel(model, stage=False)
    assert sum(p.numel() for p in staged.params()) == 387_461  # the planning path's parameters at PlaNet's sizes
    _check_staged(staged, model)


def test_staging_reads_the_local_container():
    model = models.PlaNetModel(6, 30, 200, 200, seed=1)
    _check_staged(latent.StagedLatentModel(model, stage=False), model)


def test_staging_refuses_other_activations():
    model = models.PlaNetModel(2, 3, 8, 8)
    model.reward_model[1] = torch.nn.SiLU()
    with pytest.raises(NotImplementedError, match="reward_model"):
        latent.StagedLatentModel(model, stage=False)


def test_latent_kernels_have_no_stack_frame():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cuobjdump = shutil.which("cuobjdump") or os.path.join(os.path.dirname(nvcc), "cuobjdump")
    if not (os.path.exists(nvcc) and os.path.exists(cuobjdump)):
        pytest.skip("needs nvcc and cuobjdump")
    spec = importlib.util.spec_from_file_location("b200pets_build_latent", os.path.join(ROOT, "mbrl-lib_b200", "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    out = subprocess.run([cuobjdump, "-res-usage", mod.build()], capture_output=True, text=True, check=True).stdout
    res, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+)", line)
        if m and name:
            res[name] = (int(m.group(1)), int(m.group(2)))
            name = None
    rollout = {n: r for n, r in res.items() if "latent_rollout_kernel" in n}
    assert sorted(int(re.search(r"ILi(\d+)E", n).group(1)) for n in rollout) == [1, 2, 4, 8, 16, 32], sorted(rollout)
    for n, (regs, stack) in rollout.items():
        assert stack == 0, f"{n}: {stack} B stack frame"
        assert regs <= 255, n  # one 256-thread CTA per SM at least (__launch_bounds__(256, 1))
    packing = {n: r for n, r in res.items() if "latent_pack_kernel" in n or "latent_bias_kernel" in n}
    assert len(packing) == 2 and all(r[1] == 0 for r in packing.values()), packing
