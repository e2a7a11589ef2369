"""Time SAC.update_parameters: mbrl_lib_b200.SAC (one launch) against the reference's pytorch_sac_pranz24.SAC on the same
GPU, at the shipped mbpo_* configurations, alternated over 3 rounds (medians reported).

    python tests/prof_sac_update.py [--updates 200] [--out RESULTS.json]

Per configuration it prints ms per update of both agents, the kernel time from CUDA events, the achieved FLOP/s (FLOPs
counted from the shapes below) and ms per MBPO environment step (num_sac_updates_per_step x ms per update).  The card's
name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from baseline import reference_arm as ra  # noqa: E402
from mbrl_lib_b200 import replay, sac as bsac  # noqa: E402

CONFIGS = [  # name, obs, act, hidden, target_update_interval, automatic_entropy_tuning, lr, num_sac_updates_per_step
    ("mbpo_cartpole", 4, 1, 256, 4, True, 3e-4, 20),
    ("mbpo_hopper", 11, 3, 512, 4, False, 3e-4, 40),
    ("mbpo_halfcheetah", 17, 6, 512, 1, True, 3e-4, 10),
    ("mbpo_ant", 27, 8, 1024, 4, False, 1e-4, 20),
    ("mbpo_humanoid", 45, 17, 1024, 4, False, 1e-4, 20),
]
B = 256


def flops(D, A, H, Bn=B):
    """Multiply-adds x 2 of one update as the kernel computes it."""
    lin = lambda rows, k, n: 2 * rows * k * n  # noqa: E731
    fwd_pol = lin(2 * Bn, D, H) + lin(2 * Bn, H, H) + 2 * lin(2 * Bn, H, A)
    fwd_q = 2 * (lin(Bn, D + A, H) + lin(Bn, H, H) + lin(Bn, H, 1))  # both nets, one input
    critic_bwd = 2 * (lin(Bn, H, H) + lin(Bn, H, 1) + lin(Bn, H, H) + lin(Bn, D + A, H))  # data grad of layer 2, wgrads
    pol_bwd = 2 * (lin(Bn, H, H) + lin(Bn, H, A)) + 2 * lin(Bn, H, A) + lin(Bn, H, H) + 2 * lin(Bn, H, A) \
        + lin(Bn, H, H) + lin(Bn, D, H)
    return fwd_pol + 3 * fwd_q + critic_bwd + pol_bwd


class Memory:
    def __init__(self, batches):
        self.batches, self.i = batches, 0

    def sample(self, n):
        b = self.batches[self.i % len(self.batches)]
        self.i += 1
        return b


class Box:
    def __init__(self, A):
        self.low, self.high, self.shape = -np.ones(A, np.float32), np.ones(A, np.float32), (A,)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--updates", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the card and the rows as JSON to this path")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "prof_sac_update.py measures on a GPU"
    mbrl, src = ra.import_reference()
    assert mbrl is not None, f"the reference is not importable: {src}"
    from mbrl.third_party.pytorch_sac_pranz24.sac import SAC as RefSAC

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card)
    rows = []
    for name, D, A, H, interval, tuning, lr, per_step in CONFIGS:
        cfg = types.SimpleNamespace(gamma=0.99, tau=0.005, alpha=0.2, policy="Gaussian", target_update_interval=interval,
                                    automatic_entropy_tuning=tuning, target_entropy=None, hidden_size=H, device="cuda:0",
                                    lr=lr)
        rng = np.random.default_rng(0)
        batches = [replay.TransitionBatch(rng.standard_normal((B, D)).astype(np.float32),
                                          rng.uniform(-1, 1, (B, A)).astype(np.float32),
                                          rng.standard_normal((B, D)).astype(np.float32),
                                          rng.standard_normal(B).astype(np.float32), rng.random(B) < 0.05,
                                          np.zeros(B, bool)) for _ in range(16)]
        torch.manual_seed(0)
        agents = {"device": bsac.SAC(D, Box(A), cfg), "reference": RefSAC(D, Box(A), cfg)}
        mems = {k: Memory(batches) for k in agents}
        times = {k: [] for k in agents}
        counter = {k: 0 for k in agents}

        def run(k, n):
            a, m = agents[k], mems[k]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(n):
                a.update_parameters(m, B, counter[k], reverse_mask=True)
                counter[k] += 1
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) / n * 1e3

        for k in agents:
            run(k, 20)  # warm-up
        for _ in range(args.rounds):
            for k in agents:
                times[k].append(run(k, args.updates))
        # kernel time: CUDA events around the launch alone, on the staged batch of the last update
        dev = agents["device"]
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        import ctypes as C
        from mbrl_lib_b200 import _lib

        lib = _lib.load()
        h = dev._handle
        steps = (C.c_int64 * 3)(counter["device"], counter["device"], counter["device"] if tuning else 0)
        n_k = 200
        ev0.record()
        for i in range(n_k):
            _lib.check(lib.b200pets_sac_update(h, B, 1, 1, steps, _lib.ptr(dev._stage_dev), None, dev._seed, 10_000 + i,
                                               _lib.ptr(dev._alpha_dev), _lib.ptr(dev._stats_dev), _lib.ptr(dev._ws),
                                               dev._ws.numel(), _lib.stream_ptr()), "sac_update")
        ev1.record()
        torch.cuda.synchronize()
        k_ms = ev0.elapsed_time(ev1) / n_k
        f = flops(D, A, H)
        row = dict(config=name, obs=D, act=A, hidden=H, interval=interval, tuning=tuning,
                   device_ms=float(np.median(times["device"])), reference_ms=float(np.median(times["reference"])),
                   kernel_ms=k_ms, gflop=f / 1e9, kernel_tflops=f / k_ms / 1e9, updates_per_step=per_step)
        row["speedup"] = row["reference_ms"] / row["device_ms"]
        row["device_ms_per_env_step"] = per_step * row["device_ms"]
        row["reference_ms_per_env_step"] = per_step * row["reference_ms"]
        rows.append(row)
        print(json.dumps(row), flush=True)
    print("| config | obs/act/hidden | reference ms/update | device ms/update | speed-up | kernel ms | kernel TFLOP/s "
          "| updates/env step | reference ms/env step | device ms/env step |")
    print("|---|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['config']} | {r['obs']}/{r['act']}/{r['hidden']} | {r['reference_ms']:.3f} | {r['device_ms']:.3f} | "
              f"{r['speedup']:.1f}x | {r['kernel_ms']:.3f} | {r['kernel_tflops']:.2f} | {r['updates_per_step']} | "
              f"{r['reference_ms_per_env_step']:.1f} | {r['device_ms_per_env_step']:.1f} |")
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(dict(card=card, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
