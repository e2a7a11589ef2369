"""Time ``agent.act`` at the planet_cheetah_run planner config (CEM: population 1000, horizon 12, 10 iterations, elite
ratio 0.1, alpha 0, clipped normal, 1 particle) over a PlaNetModel on cuda:0:

* device: this project's ``ModelEnv`` + agent, one ``b200pets_latent_cem_plan`` call per action;
* reference: oracle/_ref's ``mbrl.models.ModelEnv`` + ``mbrl.planning`` agent over the same model object (skipped when
  oracle/_ref is absent).

The two alternate for 3 rounds of REPS actions each; the script prints the median ms per action of each, the card's
name, power limit and max SM clock, and the plan's FLOP (from the shapes) over its time as a share of the 67 TFLOP/s
FP32 data-sheet rate of an H100 SXM.

    python tests/prof_latent_plan.py [REPS]
"""
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import mbrl_lib_b200 as bp  # noqa: E402
from baseline import reference_arm as ra  # noqa: E402
from mbrl_lib_b200 import functions, models  # noqa: E402

A, L, HB, HF = 6, 30, 200, 200
POP, H, ITERS = 1000, 12, 10
FP32_PEAK = 67e12


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as exc:  # pragma: no cover - depends on the box
        out = f"nvidia-smi unavailable ({type(exc).__name__})"
    return f"{name}, power limit / max SM clock: {out}"


def plan_flop():
    """2 x multiply-adds per row-step (embedding, GRU, prior, reward) x rows x steps x iterations."""
    mac = (L + A) * HB + 2 * 3 * HB * HB + HB * HF + HF * 2 * L + (HB + L) * HF + HF * HF + HF
    return 2.0 * mac * POP * H * ITERS


class _Box:
    def __init__(self, lo, hi, shape):
        self.low, self.high, self.shape = np.full(shape, lo, np.float32), np.full(shape, hi, np.float32), shape


class _Env:
    observation_space = _Box(0, 255, (3, 64, 64))
    action_space = _Box(-1.0, 1.0, (A,))


def agent_cfg():
    return {"_target_": "mbrl.planning.TrajectoryOptimizerAgent", "action_lb": [-1.0] * A, "action_ub": [1.0] * A,
            "planning_horizon": H, "replan_freq": 1, "keep_last_solution": False, "verbose": False,
            "optimizer_cfg": {"_target_": "mbrl.planning.CEMOptimizer", "num_iterations": ITERS, "elite_ratio": 0.1,
                              "population_size": POP, "alpha": 0.0, "lower_bound": "???", "upper_bound": "???",
                              "return_mean_elites": True, "device": "cuda:0", "clipped_normal": True}}


def time_act(agent, obs, reps):
    agent.act(obs)  # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        agent.act(obs)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / reps


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    mbrl, src = ra.import_reference()
    obs = np.random.default_rng(0).integers(0, 255, (3, 64, 64), dtype=np.uint8)
    if mbrl is not None:
        model = mbrl.models.PlaNetModel(
            obs_shape=(3, 64, 64), obs_encoding_size=1024,
            encoder_config=((3, 32, 4, 2), (32, 64, 4, 2), (64, 128, 4, 2), (128, 256, 4, 2)),
            decoder_config=((1024, 1, 1), ((1024, 128, 5, 2), (128, 64, 5, 2), (64, 32, 6, 2), (32, 3, 6, 2))),
            latent_state_size=L, action_size=A, belief_size=HB, hidden_size_fcs=HF, device="cuda:0")
        rng = torch.Generator(device="cuda:0")
        model.update_posterior(obs, rng=rng)
        term = mbrl.env.termination_fns.no_termination
    else:
        print(f"reference not importable ({src}): timing the device plan alone over the local container")
        model = models.PlaNetModel(A, L, HB, HF, device="cuda:0", seed=0)
        model.set_posterior(np.zeros(L), np.zeros(HB))
        rng, term = torch.Generator(device="cuda:0"), functions.no_termination
    env = bp.ModelEnv(_Env(), model, term, generator=rng)
    ours = bp.create_trajectory_optim_agent_for_model(env, agent_cfg())
    ref = None
    if mbrl is not None:
        import omegaconf

        ref_env = mbrl.models.ModelEnv(_Env(), model, term, generator=rng)
        ref = mbrl.planning.create_trajectory_optim_agent_for_model(ref_env, omegaconf.OmegaConf.create(agent_cfg()))
    t_ours, t_ref = [], []
    for _ in range(3):
        t_ours.append(time_act(ours, obs, reps))
        if ref is not None:
            t_ref.append(time_act(ref, obs, max(1, reps // 10)))
    print(card())
    m = float(np.median(t_ours))
    print(f"device plan  : {m:.3f} ms per act (rounds {['%.3f' % t for t in t_ours]}); "
          f"{plan_flop() / 1e9:.1f} GFLOP -> {plan_flop() / (m * 1e-3) / 1e12:.2f} TFLOP/s = "
          f"{100 * plan_flop() / (m * 1e-3) / FP32_PEAK:.1f} % of 67 TFLOP/s FP32")
    if t_ref:
        r = float(np.median(t_ref))
        print(f"reference    : {r:.3f} ms per act (rounds {['%.3f' % t for t in t_ref]}); speed-up {r / m:.1f}x")


if __name__ == "__main__":
    main()
