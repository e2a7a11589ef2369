"""Cost of a reward callable the kernels do not know, at the PETS HalfCheetah config (bench.py's build_problem: pop 500 x
20 particles x H 30, ensemble 7 / 5 elites, 4 x 200 SiLU, tile shuffle, precision "auto").

Times, with CUDA events, evaluate_action_sequences and agent.act (5-iteration CEM plan) twice: with the in-kernel
halfcheetah reward, and with the same torch function wrapped in a lambda (windowed rollout + one callable call per
window + masking kernel; agent.act then runs CEM's per-iteration loop instead of the one-call plan).

    python tests/prof_callables.py [--reps N]
"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from mbrl_lib_b200 import synthetic as syn  # noqa: E402


def gpu_description():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as exc:  # pragma: no cover - depends on the box
        out = f"nvidia-smi unavailable ({type(exc).__name__})"
    return f"{name}, power limit / max SM clock: {out}"


def time_ms(fn, reps):
    """Mean ms per call over `reps` calls between two CUDA events (3 untimed warm-up calls first)."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def main():
    import mbrl_lib_b200 as bp
    from mbrl_lib_b200 import functions

    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    dev = "cuda:0"
    torch.manual_seed(0)
    spec, arrays, env_known = bench.build_problem(dev)
    env_lambda = bp.ModelEnv(env_known, bp.model_from_arrays(spec, arrays, dev), functions.TERM_FNS[spec.term_fn],
                             lambda act, next_obs: functions.reward_halfcheetah(act, next_obs),
                             generator=torch.Generator(device=dev).manual_seed(0), precision="auto", ts1="tile_shuffle")
    assert not env_known.has_external_callables() and env_lambda.has_external_callables()
    inp = syn.make_rollout_inputs(spec, with_noise=False)
    acts = torch.from_numpy(inp["actions"]).to(dev)
    obs0 = inp["obs0"]
    H, A, N, P = spec.horizon, spec.act_dim, spec.population, spec.particles
    print(gpu_description())
    print(f"PETS HalfCheetah: pop {N} x {P} particles x H {H}, precision {env_known.precision}, {args.reps} timed calls each")
    rows = {}
    for label, env in (("in-kernel reward", env_known), ("lambda reward", env_lambda)):
        ev = time_ms(lambda: env.evaluate_action_sequences(acts, obs0, P), args.reps)
        cfg = {"_target_": "mbrl.planning.TrajectoryOptimizerAgent", "planning_horizon": H, "replan_freq": 1, "verbose": False,
               "optimizer_cfg": {"_target_": "mbrl.planning.CEMOptimizer", "num_iterations": bench.CEM_ITERS,
                                 "elite_ratio": bench.ELITE_RATIO, "population_size": N, "alpha": bench.ALPHA, "device": dev,
                                 "return_mean_elites": True}}
        agent = bp.create_trajectory_optim_agent_for_model(env, cfg, num_particles=P)
        act_ms = time_ms(lambda: agent.act(obs0), args.reps)
        rows[label] = (ev, act_ms)
        print(f"{label:17s} evaluate_action_sequences {ev:8.3f} ms ({N / (ev * 1e-3):.3e} sequences/s)   "
              f"agent.act {act_ms:8.3f} ms ({bench.CEM_ITERS * N / (act_ms * 1e-3):.3e} sequences/s)")
    (e0, a0), (e1, a1) = rows["in-kernel reward"], rows["lambda reward"]
    print(f"lambda / in-kernel: evaluate x{e1 / e0:.2f}, agent.act x{a1 / a0:.2f}")
    r0 = env_known.evaluate_action_sequences(acts, obs0, P, _offset=99 * 1024)
    r1 = env_lambda.evaluate_action_sequences(acts, obs0, P, _offset=99 * 1024)
    scale = max(1.0, float(r0.abs().max()))
    print(f"same draws, lambda vs in-kernel returns: max |diff| {float((r1 - r0).abs().max()) / scale:.2e} of scale {scale:.3g}")
    assert np.isfinite(r1.cpu().numpy()).all()


if __name__ == "__main__":
    main()
