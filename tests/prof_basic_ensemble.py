"""Time ``agent.act`` with CEM over a BasicEnsemble at pets_halfcheetah shapes, on cuda:0.

Model: ``conf/dynamics_model/basic_ensemble.yaml``'s, 5 one-member GaussianMLPs of 4 x 200 SiLU on HalfCheetah's dims
(synthetic weights).  Agent: CEM, population 500, H 30, 20 particles, 5 iterations, under ``fixed_model`` and
``random_model``.  Compared with:
* the same shapes on a GaussianMLP ensemble of 5 (the project's GaussianMLP path, in-kernel member draw);
* the reference's own ``ModelEnv`` and ``mbrl.planning`` agent over the reference's ``BasicEnsemble`` with the same
  weights, on cuda, when the reference is importable (``oracle/_ref``).

The project's paths alternate for 3 rounds of REPS actions each, every action ending in the agent's device-to-host
copy; the script prints the median ms per action of each and the card's name, power limit and max SM clock.

    python tests/prof_basic_ensemble.py [REPS]
"""
import dataclasses
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import mbrl_lib_b200 as bp  # noqa: E402
from mbrl_lib_b200 import functions, synthetic as syn  # noqa: E402
from mbrl_lib_b200.models import basic_ensemble_from_arrays  # noqa: E402

DEV = "cuda:0"
POP, H, P, ITERS = 500, 30, 20, 5


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as exc:  # pragma: no cover - depends on the box
        out = f"nvidia-smi unavailable ({type(exc).__name__})"
    return f"{name}, power limit / max SM clock: {out}"


class _Box:
    def __init__(self, lo, hi, n):
        self.low, self.high, self.shape = np.full(n, lo, np.float32), np.full(n, hi, np.float32), (n,)


def spec_for(prop):
    return dataclasses.replace(syn.CASES["halfcheetah"], ensemble_size=5, elites=None, propagation=prop)


def agent_cfg(spec):
    return {"_target_": "mbrl.planning.TrajectoryOptimizerAgent", "action_lb": [spec.action_lb] * spec.act_dim,
            "action_ub": [spec.action_ub] * spec.act_dim, "planning_horizon": H, "replan_freq": 1, "verbose": False,
            "optimizer_cfg": {"_target_": "mbrl.planning.CEMOptimizer", "num_iterations": ITERS, "elite_ratio": 0.1,
                              "population_size": POP, "alpha": 0.1, "device": DEV, "lower_bound": "???",
                              "upper_bound": "???", "return_mean_elites": True, "clipped_normal": False}}


def our_agent(spec, arrays, basic):
    build = basic_ensemble_from_arrays if basic else bp.model_from_arrays
    model = build(spec, arrays, DEV)

    class _Env:
        observation_space = _Box(-np.inf, np.inf, spec.obs_dim)
        action_space = _Box(spec.action_lb, spec.action_ub, spec.act_dim)

    env = bp.ModelEnv(_Env(), model, functions.TERM_FNS[spec.term_fn], functions.REWARD_FNS[spec.reward_fn],
                      generator=torch.Generator(device=DEV).manual_seed(0))
    return env, bp.create_trajectory_optim_agent_for_model(env, agent_cfg(spec), num_particles=P)


def ref_agent(spec, arrays):
    """The reference's BasicEnsemble with the same weights, its ModelEnv and its agent (None, reason without it)."""
    from baseline import reference_arm as ra

    mbrl, src = ra.import_reference()
    if mbrl is None:
        return None, src
    import mbrl.env.reward_fns as rf
    import mbrl.env.termination_fns as tf
    import mbrl.models as mm
    import mbrl.planning as mp

    member_cfg = {"_target_": "mbrl.models.GaussianMLP", "device": DEV, "num_layers": spec.num_layers, "in_size": spec.in_size,
                  "out_size": spec.out_size, "ensemble_size": 1, "hid_size": spec.hid_size, "deterministic": False,
                  "activation_fn_cfg": {"_target_": "torch.nn.SiLU"}}
    ens = mm.BasicEnsemble(spec.ensemble_size, DEV, member_cfg, propagation_method=spec.propagation)
    with torch.no_grad():
        for e, m in enumerate(ens.members):
            layers = [seq[0] for seq in m.hidden_layers] + [m.mean_and_logvar]
            for li, lin in enumerate(layers):
                lin.weight.copy_(torch.from_numpy(arrays["weights"][li][e:e + 1]))
                lin.bias.copy_(torch.from_numpy(arrays["biases"][li][e:e + 1]))
            m.min_logvar.copy_(torch.from_numpy(arrays["min_logvar"]))
            m.max_logvar.copy_(torch.from_numpy(arrays["max_logvar"]))
    model = mm.OneDTransitionRewardModel(ens, target_is_delta=spec.target_is_delta, normalize=False,
                                         learned_rewards=spec.learned_rewards)

    class _Env:
        observation_space = _Box(-np.inf, np.inf, spec.obs_dim)
        action_space = _Box(spec.action_lb, spec.action_ub, spec.act_dim)

    env = mm.ModelEnv(_Env(), model, getattr(tf, spec.term_fn), getattr(rf, spec.reward_fn),
                      generator=torch.Generator(device=DEV).manual_seed(0))
    from omegaconf import OmegaConf

    agent = mp.create_trajectory_optim_agent_for_model(env, OmegaConf.create(agent_cfg(spec)), num_particles=P)
    return agent, src


def ms_per_act(agent, obs, reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        agent.act(obs)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / reps


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    print(card())
    print(f"agent.act, CEM pop {POP}, H {H}, {P} particles, {ITERS} iterations; ensemble of 5 x 4x200 SiLU, HalfCheetah dims")
    for prop in ("fixed_model", "random_model"):
        spec = spec_for(prop)
        arrays = syn.make_model_arrays(spec)
        obs = np.random.default_rng(0).standard_normal(spec.obs_dim)
        paths = {}
        for label, basic in (("BasicEnsemble", True), ("GaussianMLP ensemble", False)):
            env, agent = our_agent(spec, arrays, basic)
            paths[f"{label} ({env.precision_for(prop)})"] = agent
        for agent in paths.values():  # warm-up: module load, plans, workspaces
            ms_per_act(agent, obs, 2)
        times = {k: [] for k in paths}
        for _ in range(3):
            for k, agent in paths.items():
                times[k].append(ms_per_act(agent, obs, reps))
        for k, v in times.items():
            print(f"  {prop:12s} {k:32s} {np.median(v):9.3f} ms per act  (rounds {', '.join(f'{x:.3f}' for x in v)})")
        try:
            agent, src = ref_agent(spec, arrays)
        except Exception as exc:  # pragma: no cover - depends on the reference's dependencies here
            agent, src = None, f"{type(exc).__name__}: {exc}"
        if agent is None:
            print(f"  {prop:12s} reference: not measured ({src})")
            continue
        ms_per_act(agent, obs, 1)
        r = max(1, reps // 5)
        print(f"  {prop:12s} {'reference ModelEnv + agent (cuda)':32s} {np.median([ms_per_act(agent, obs, r) for _ in range(3)]):9.3f} ms per act")


if __name__ == "__main__":
    main()
