"""Batched MPPI plan against K single plans, at the pets_mppi_halfcheetah config (bench.py's model, pop 350 x 20 particles x
H 30, ensemble 7 / 5 elites, 4 x 200 SiLU, tile shuffle, precision "auto"), 5 refinements, gamma 0.9, beta 0.9.

For each K, times with CUDA events one MPPIOptimizer.optimize_batch over K observations (one b200pets_mppi_plan_batch)
and K MPPIOptimizer.optimize calls (per refinement: sample kernel, evaluate_action_sequences, update kernel), alternating
the two over --rounds rounds of --reps calls each after a warm-up of both.  Prints ms per call and sequences/s
(K x 5 x 350 / time) for both, with the card's name, power limit and SM clocks read in the same run, and checks that the
batched plans equal the single ones at the same counter values.

    python tests/prof_batch_mppi.py [--ks 1,2,4,8,16] [--reps 10] [--rounds 3]
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from prof_callables import gpu_description  # noqa: E402

POPULATION, REFINEMENTS, GAMMA, SIGMA, BETA = 350, 5, 0.9, 1.0, 0.9  # conf/overrides/pets_mppi_halfcheetah.yaml


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
    spec, _, env = bench.build_problem_variant(dev, bench.WORKLOAD, population=POPULATION)
    H, A, N, P = spec.horizon, spec.act_dim, spec.population, spec.particles
    lb, ub = np.full((H, A), spec.action_lb).tolist(), np.full((H, A), spec.action_ub).tolist()
    opt = bp.MPPIOptimizer(REFINEMENTS, N, GAMMA, SIGMA, BETA, lb, ub, dev)
    print(gpu_description())
    print(f"pets_mppi_halfcheetah: pop {N} x {P} particles x H {H}, {REFINEMENTS} MPPI refinements, precision {env.precision}; "
          f"{args.rounds} alternated rounds of {args.reps} timed calls per K and mode")
    g = np.random.default_rng(0)
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    print(f"{'K':>3} {'batched ms':>11} {'K singles ms':>13} {'batched seq/s':>14} {'singles seq/s':>14} {'speed-up':>9}")
    for K in [int(k) for k in args.ks.split(",")]:
        obs = g.standard_normal((K, spec.obs_dim))
        batch_obj = _FusedBatchObjective(env, obs, P)
        single_objs = [_FusedObjective(env, obs[k], P) for k in range(K)]

        def batched():
            return opt.optimize_batch(batch_obj)

        def singles():
            return [opt.optimize(single_objs[k]) for k in range(K)]

        for _ in range(3):
            batched()
            singles()
        # same counter values and carried means for both: the batched plans equal the single ones
        means = opt.batch_mean.clone()
        env._offset, opt._offset = 1000, 500
        pb = batched().clone()
        ps = []
        for k in range(K):
            env._offset, opt._offset = 1000 + k * REFINEMENTS, 500 + k
            opt.mean = means[k].clone()
            ps.append(opt.optimize(single_objs[k]))
        torch.cuda.synchronize()
        assert torch.equal(pb, torch.stack(ps)), "batched plan differs from the single plans"
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
        seqs = K * REFINEMENTS * N
        print(f"{K:>3} {tb:>11.3f} {ts:>13.3f} {seqs / (tb * 1e-3):>14.3e} {seqs / (ts * 1e-3):>14.3e} {ts / tb:>8.2f}x"
              f"   (batched rounds {', '.join(f'{t:.3f}' for t in times['batched'])}; "
              f"singles {', '.join(f'{t:.3f}' for t in times['singles'])})")


if __name__ == "__main__":
    main()
