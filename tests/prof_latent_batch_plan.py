"""One ``agent.act_batch`` over K PlaNet posteriors (one ``b200pets_latent_cem_plan_batch``) against K single
``agent.act`` calls (K ``b200pets_latent_cem_plan``), at the planet_cheetah_run planner config (CEM: population 1000,
horizon 12, 10 iterations, elite ratio 0.1, alpha 0, clipped normal, 1 particle; A 6, L 30, belief = hidden = 200) over
the local PlaNetModel container on cuda:0.

For each K the two alternate for --rounds rounds of --reps calls each, after a warm-up of both; the script prints the
medians as ms per batch and per problem, the rollout's rows per CTA and CTAs, and the plan's FLOP (prof_latent_plan.py's
plan_flop, times K) over its time as TFLOP/s and as a share of the 67 TFLOP/s FP32 data-sheet rate of an H100 SXM, with
the card's name, power limit and max SM clock read in the same run.

    python tests/prof_latent_batch_plan.py [--ks 1,2,4,8,16] [--reps 10] [--rounds 3]
"""
import argparse
import math
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import mbrl_lib_b200 as bp  # noqa: E402
from mbrl_lib_b200 import functions, models  # noqa: E402
from prof_latent_plan import A, FP32_PEAK, HB, HF, L, POP, _Env, agent_cfg, card, plan_flop  # noqa: E402


def timed(fn, reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1,2,4,8,16")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    dev = "cuda:0"
    model = models.PlaNetModel(A, L, HB, HF, device=dev, seed=0)
    model.set_posterior(np.zeros(L), np.zeros(HB))
    rng = torch.Generator(device=dev)
    env = bp.ModelEnv(_Env(), model, functions.no_termination, generator=rng)
    agent = bp.create_trajectory_optim_agent_for_model(env, agent_cfg())
    print(card())
    print(f"planet_cheetah_run planner: CEM pop {POP} x H 12 x 10 iterations; {args.rounds} alternated rounds of "
          f"{args.reps} timed calls per K and mode")
    print(f"{'K':>3} {'batch ms':>9} {'ms/problem':>11} {'K singles ms':>13} {'ms/problem':>11} {'speed-up':>9} "
          f"{'rows/CTA':>9} {'CTAs':>5} {'batch TFLOP/s':>14} {'of FP32':>8} {'singles TFLOP/s':>16} {'of FP32':>8}")
    g = np.random.default_rng(0)
    for K in [int(k) for k in args.ks.split(",")]:
        latent = torch.from_numpy(g.standard_normal((K, L)).astype(np.float32)).to(dev)
        belief = torch.from_numpy(np.tanh(g.standard_normal((K, HB))).astype(np.float32)).to(dev)
        obs = np.zeros((K, 3, 64, 64), np.uint8)
        env.set_posterior_batch(latent, belief)

        def batched():
            return agent.act_batch(obs)

        def singles():
            for k in range(K):
                model.set_posterior(latent[k], belief[k])
                agent.act(obs[k])

        for _ in range(2):
            batched()
            singles()
        tb, ts = [], []
        for _ in range(args.rounds):
            tb.append(timed(batched, args.reps))
            ts.append(timed(singles, args.reps))
        b, s = float(np.median(tb)), float(np.median(ts))
        info = env.staged.plan_info(K * POP)
        ctas = K * math.ceil(POP / info["rows_per_cta"])
        flop = K * plan_flop()
        rb, rs = flop / (b * 1e-3) / 1e12, flop / (s * 1e-3) / 1e12
        print(f"{K:>3} {b:>9.3f} {b / K:>11.3f} {s:>13.3f} {s / K:>11.3f} {s / b:>8.2f}x {info['rows_per_cta']:>9} "
              f"{ctas:>5} {rb:>14.2f} {100 * rb * 1e12 / FP32_PEAK:>7.1f}% {rs:>16.2f} {100 * rs * 1e12 / FP32_PEAK:>7.1f}%")


if __name__ == "__main__":
    main()
