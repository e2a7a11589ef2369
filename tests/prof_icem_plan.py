"""Time ``agent.act`` with iCEM over the model: the fused plan (one ``b200pets_icem_plan`` call per action) against the
per-iteration loop (the same agent with the objective passed as an opaque closure), on cuda:0.

Shapes:
* pets_icem_cartpole: an ensemble of 7 with 5 elites, 4 x 200 SiLU on CartPole's dims; population 200 decaying by 1.3,
  H 10, 5 iterations, 20 particles, population_size_module 7;
* bench config 3: humanoid_trunc and humanoid_v4, population 1000 decaying by 1.3, H 40, 5 iterations, 20 particles,
  module 5.

The two paths alternate for 3 rounds of REPS actions each, every action ending in the agent's device-to-host copy; the
script prints the median ms per action of each path and the card's name, power limit and max SM clock.

    python tests/prof_icem_plan.py [REPS]
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

DEV = "cuda:0"


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


def make_env(spec):
    model = bp.model_from_arrays(spec, syn.make_model_arrays(spec), DEV)

    class _Env:
        observation_space = _Box(-np.inf, np.inf, spec.obs_dim)
        action_space = _Box(spec.action_lb, spec.action_ub, spec.act_dim)

    rew = functions.REWARD_FNS[spec.reward_fn] if spec.reward_fn else None
    return bp.ModelEnv(_Env(), model, functions.TERM_FNS[spec.term_fn], rew, generator=torch.Generator(device=DEV).manual_seed(0))


# name -> (model spec, population, H, particles, module)
SHAPES = {
    "pets_icem_cartpole": (dataclasses.replace(syn.CASES["cartpole_pets"], ensemble_size=7, elites=(0, 2, 3, 5, 6), hid_size=200,
                                               num_layers=4), 200, 10, 20, 7),
    "config3_humanoid_trunc": (syn.CASES["humanoid_trunc"], 1000, 40, 20, 5),
    "config3_humanoid_v4": (syn.CASES["humanoid_v4"], 1000, 40, 20, 5),
}


def agent_for(env, pop, H, P, module):
    cfg = {"_target_": "mbrl.planning.TrajectoryOptimizerAgent", "action_lb": "???", "action_ub": "???", "planning_horizon": H,
           "replan_freq": 1, "verbose": False,
           "optimizer_cfg": {"_target_": "mbrl.planning.ICEMOptimizer", "num_iterations": 5, "elite_ratio": 0.1,
                             "population_size": pop, "population_decay_factor": 1.3, "colored_noise_exponent": 2.0,
                             "keep_elite_frac": 0.3, "alpha": 0.1, "device": DEV, "return_mean_elites": True,
                             "population_size_module": module}}
    return bp.create_trajectory_optim_agent_for_model(env, cfg, num_particles=P)


def ms_per_act(agent, obs, reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        agent.act(obs)  # ends in the plan's device-to-host copy and a stream synchronise
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps * 1e3


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    print(card())
    for name, (spec, pop, H, P, module) in SHAPES.items():
        env = make_env(spec)
        fused, loop = agent_for(env, pop, H, P, module), agent_for(env, pop, H, P, module)
        loop.set_trajectory_eval_fn(lambda o, seqs: env.evaluate_action_sequences(seqs, o, P))  # opaque: the loop
        obs = syn.make_rollout_inputs(spec, with_noise=False)["obs0"]
        for agent in (fused, loop):  # warm-up: modules, workspaces, the carried elites
            for _ in range(3):
                agent.act(obs)
        times = {"fused": [], "loop": []}
        for _ in range(3):
            times["fused"].append(ms_per_act(fused, obs, reps))
            times["loop"].append(ms_per_act(loop, obs, reps))
        f, lp = float(np.median(times["fused"])), float(np.median(times["loop"]))
        print(f"{name} ({env.precision}, pop {pop}, H {H}, {P} particles, 5 iterations): fused {f:.3f} ms/act, loop {lp:.3f} "
              f"ms/act, loop / fused {lp / f:.2f}  (rounds: fused {[round(t, 3) for t in times['fused']]}, "
              f"loop {[round(t, 3) for t in times['loop']]})", flush=True)


if __name__ == "__main__":
    main()
