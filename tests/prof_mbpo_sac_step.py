"""Time one MBPO environment step's SAC updates (num_sac_updates_per_step of them, batch 256) at the shipped mbpo_*
configurations, three ways, in the same process and alternated over 3 rounds (medians reported):

  host      today's drop-in: mbrl_lib_b200.SAC.update_parameters per update on an unmirrored ReplayBuffer (sample,
            pack into pinned memory, copy, launch, copy the statistics back, synchronise)
  mirror    update_parameters per update on a buffer mirrored with replay.mirror_transitions_to_device (indices drawn on
            the host, copied, rows gathered on the device)
  many      mbpo.update_agent on the mirrored buffer: all of the step's updates as one update_many call

    python tests/prof_mbpo_sac_step.py [--rows 1000000] [--steps 10] [--out RESULTS.json]

Each buffer holds --rows transitions (float32, as the rollouts store them).  It also prints the kernel alone (CUDA
events over back-to-back b200pets_sac_update launches) and reads the card's name, power limit and clock in the same run.
"""
import argparse
import ctypes as C
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
from mbrl_lib_b200 import _lib, mbpo, replay, sac as bsac  # noqa: E402

CONFIGS = [  # name, obs, act, hidden, target_update_interval, automatic_entropy_tuning, lr, num_sac_updates_per_step
    ("mbpo_cartpole", 4, 1, 256, 4, True, 3e-4, 20),
    ("mbpo_hopper", 11, 3, 512, 4, False, 3e-4, 40),
    ("mbpo_halfcheetah", 17, 6, 512, 1, True, 3e-4, 10),
    ("mbpo_ant", 27, 8, 1024, 4, False, 1e-4, 20),
    ("mbpo_humanoid", 45, 17, 1024, 4, False, 1e-4, 20),
]
B = 256
VARIANTS = ("host", "mirror", "many")


class Box:
    def __init__(self, A):
        self.low, self.high, self.shape = -np.ones(A, np.float32), np.ones(A, np.float32), (A,)


def _buffer(ReplayBuffer, rows, D, A, data):
    buf = ReplayBuffer(rows, (D,), (A,), rng=np.random.default_rng(1))
    buf.add_batch(*data)
    return buf


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=10, help="environment steps per timed window")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the card and the rows as JSON to this path")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "prof_mbpo_sac_step.py measures on a GPU"
    mbrl, src = ra.import_reference()
    assert mbrl is not None, f"the reference is not importable: {src}"
    from mbrl.util.replay_buffer import ReplayBuffer

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    rows = []
    for name, D, A, H, interval, tuning, lr, per_step in CONFIGS:
        cfg = types.SimpleNamespace(gamma=0.99, tau=0.005, alpha=0.2, policy="Gaussian", target_update_interval=interval,
                                    automatic_entropy_tuning=tuning, target_entropy=None, hidden_size=H, device="cuda:0",
                                    lr=lr)
        g = np.random.default_rng(0)
        n = args.rows
        data = (g.standard_normal((n, D), dtype=np.float32), g.uniform(-1, 1, (n, A)).astype(np.float32),
                g.standard_normal((n, D), dtype=np.float32), g.standard_normal(n, dtype=np.float32), g.random(n) < 0.05,
                np.zeros(n, bool))
        host_buf = _buffer(ReplayBuffer, n, D, A, data)
        dev_buf = _buffer(ReplayBuffer, n, D, A, data)
        del data
        mirror = replay.mirror_transitions_to_device(dev_buf, "cuda:0")
        mirror.flush()
        agents, made, rngs = {}, {}, {}
        for k in VARIANTS:
            torch.manual_seed(0)
            agents[k] = types.SimpleNamespace(sac_agent=bsac.SAC(D, Box(A), cfg))
            made[k], rngs[k] = 0, np.random.default_rng(2)
        bufs = {"host": host_buf, "mirror": dev_buf, "many": dev_buf}

        def env_step(k):
            a, buf = agents[k].sac_agent, bufs[k]
            if k == "many":
                made[k] = mbpo.update_agent(agents[k], None, buf, rngs[k], per_step, 0.0, B, True, made[k])
                return
            for _ in range(per_step):  # mbpo.py:258-275 with real_data_ratio 0
                rngs[k].random()
                a.update_parameters(buf, B, made[k], reverse_mask=True)
                made[k] += 1

        def window(k):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                env_step(k)
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) / args.steps * 1e3

        for k in VARIANTS:
            window(k)  # warm-up: every shape and buffer of the timed window
        times = {k: [] for k in VARIANTS}
        for _ in range(args.rounds):
            for k in VARIANTS:
                times[k].append(window(k))
        # the kernel alone: CUDA events around back-to-back launches on the last staged batch
        a = agents["host"].sac_agent
        lib = _lib.load()
        steps = (C.c_int64 * 3)(made["host"], made["host"], made["host"] if tuning else 0)
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n_k = 100
        ev0.record()
        for i in range(n_k):
            _lib.check(lib.b200pets_sac_update(a._handle, B, 1, 1, steps, _lib.ptr(a._stage_dev), None, a._seed, 10_000 + i,
                                               _lib.ptr(a._alpha_dev), _lib.ptr(a._stats_dev), _lib.ptr(a._ws),
                                               a._ws.numel(), _lib.stream_ptr()), "sac_update")
        ev1.record()
        torch.cuda.synchronize()
        k_ms = ev0.elapsed_time(ev1) / n_k
        row = dict(config=name, obs=D, act=A, hidden=H, updates_per_step=per_step, buffer_rows=n, kernel_ms=k_ms,
                   kernel_ms_per_env_step=k_ms * per_step)
        for k in VARIANTS:
            row[f"{k}_ms_per_env_step"] = float(np.median(times[k]))
            row[f"{k}_ms_per_update"] = row[f"{k}_ms_per_env_step"] / per_step
            row[f"{k}_all_rounds"] = times[k]
        row["saving_mirror"] = 1 - row["mirror_ms_per_env_step"] / row["host_ms_per_env_step"]
        row["saving_many"] = 1 - row["many_ms_per_env_step"] / row["host_ms_per_env_step"]
        rows.append(row)
        print(json.dumps(row), flush=True)
        mirror.close()
        del host_buf, dev_buf, agents
    print(f"card: {card}")
    print("| config | updates/env step | host ms/env step (ms/update) | mirror | mirror + update_agent | kernel alone "
          "ms/env step (ms/update) | saved by update_agent |")
    print("|---|---|---|---|---|---|---|")
    for r in rows:
        cell = lambda k: f"{r[k + '_ms_per_env_step']:.2f} ({r[k + '_ms_per_update']:.3f})"  # noqa: E731
        print(f"| {r['config']} | {r['updates_per_step']} | {cell('host')} | {cell('mirror')} | {cell('many')} | "
              f"{r['kernel_ms_per_env_step']:.2f} ({r['kernel_ms']:.3f}) | {100 * r['saving_many']:.1f} % |")
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(dict(card=card, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
