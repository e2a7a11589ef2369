"""Batched CEM plan against K single plans, at the PETS HalfCheetah config (bench.py's build_problem: pop 500 x 20
particles x H 30, ensemble 7 / 5 elites, 4 x 200 SiLU, tile shuffle, precision "auto"), 5 CEM iterations.

For each K, times with CUDA events one CEMOptimizer.optimize_batch over K observations (one b200pets_cem_plan_batch)
and K CEMOptimizer.optimize calls (K b200pets_cem_plan), alternating the two over --rounds rounds of --reps calls each
after a warm-up of both.  Prints ms per call and sequences/s (K x 5 x 500 / time) for both, with the card's name,
power limit and SM clocks read in the same run, and checks that the batched solutions equal the single ones.

    python tests/prof_batch_plan.py [--ks 1,2,4,8,16] [--reps 10] [--rounds 3]
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from prof_callables import gpu_description  # noqa: E402


def main():
    import mbrl_lib_b200 as bp
    from mbrl_lib_b200.planning import _FusedBatchObjective, _FusedObjective

    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1,2,4,8,16")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    dev = "cuda:0"
    torch.manual_seed(0)
    spec, _, env = bench.build_problem(dev)
    H, A, N, P = spec.horizon, spec.act_dim, spec.population, spec.particles
    iters = bench.CEM_ITERS
    lb, ub = np.full((H, A), spec.action_lb).tolist(), np.full((H, A), spec.action_ub).tolist()
    opt = bp.CEMOptimizer(iters, bench.ELITE_RATIO, N, lb, ub, bench.ALPHA, dev, return_mean_elites=True)
    print(gpu_description())
    print(f"PETS HalfCheetah: pop {N} x {P} particles x H {H}, {iters} CEM iterations, precision {env.precision}; "
          f"{args.rounds} alternated rounds of {args.reps} timed calls per K and mode")
    g = np.random.default_rng(0)
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    print(f"{'K':>3} {'batched ms':>11} {'K singles ms':>13} {'batched seq/s':>14} {'singles seq/s':>14} {'speed-up':>9}")
    for K in [int(k) for k in args.ks.split(",")]:
        obs = g.standard_normal((K, spec.obs_dim))
        x0 = torch.zeros(K, H, A, device=dev)
        batch_obj = _FusedBatchObjective(env, obs, P)
        single_objs = [_FusedObjective(env, obs[k], P) for k in range(K)]

        def batched():
            return opt.optimize_batch(batch_obj, x0=x0)

        def singles():
            return [opt.optimize(single_objs[k], x0=x0[k]) for k in range(K)]

        for _ in range(3):
            batched()
            singles()
        # same counter values for both: the batched solutions equal the single ones
        env._offset = 1000
        sb = batched().clone()
        env._offset = 1000
        ss = torch.stack(singles())
        torch.cuda.synchronize()
        assert torch.equal(sb, ss), "batched plan differs from the single plans"
        times = {"batched": [], "singles": []}
        for _ in range(args.rounds):
            for label, fn in (("batched", batched), ("singles", singles)):
                torch.cuda.synchronize()
                s.record()
                for _ in range(args.reps):
                    fn()
                e.record()
                torch.cuda.synchronize()
                times[label].append(s.elapsed_time(e) / args.reps)
        tb, ts = float(np.median(times["batched"])), float(np.median(times["singles"]))
        seqs = K * iters * N
        print(f"{K:>3} {tb:>11.3f} {ts:>13.3f} {seqs / (tb * 1e-3):>14.3e} {seqs / (ts * 1e-3):>14.3e} {ts / tb:>8.2f}x"
              f"   (batched rounds {', '.join(f'{t:.3f}' for t in times['batched'])}; "
              f"singles {', '.join(f'{t:.3f}' for t in times['singles'])})")


if __name__ == "__main__":
    main()
