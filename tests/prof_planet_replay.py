"""Time PlaNet's model training from the replay buffer at planet_cheetah_run shapes, with and without the device mirror:
one ``train()`` of 100 updates, each on 50 sequences of 50 3 x 64 x 64 frames (A 6, L 30, Hb = Hf = 200, encoding
1024), drawn by the reference's own ``SequenceTransitionSampler`` from the reference's own ``ReplayBuffer`` with float32
frames (``create_replay_buffer``'s type for PlaNet), filled through ``add`` with dmc2gym-style frames (5-bit values
plus uniform noise below the quantum) for 5 and for 100 trajectories of 250 steps.

Arms, alternated round by round from the same weights and the same buffer rng state (medians reported):
  host    mbrl_lib_b200.ModelTrainer on an unmirrored buffer: the sampler forms each batch on the host and it is copied;
  mirror  the same with ``replay.mirror_to_device(buffer)``: each batch is gathered on the device (the mirror is
          flushed before the timed call, so the time is the updates').
Also: one episode's flush (250 rows, host clock around a synchronised flush), the ``sequence_gather_kernel`` time from
CUDA events over many launches with its bytes over time against 3.35 TB/s, for float32 frames and for uint8 frames (a
second buffer of 10 trajectories), whether the two arms' first-update losses
are equal, and the card's name, power limit and max SM clock, read in the same run.

    python tests/prof_planet_replay.py [--rounds 3] [--updates 100] [--out result.json]
"""
import argparse
import copy
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import mbrl_lib_b200 as bp  # noqa: E402
from baseline import reference_arm as ra  # noqa: E402
from mbrl_lib_b200 import replay  # noqa: E402

DEV = "cuda:0"
B, S, A, L, H, E = 50, 50, 6, 30, 200, 1024
EP = 250
FRAME = (3, 64, 64)
ENC = ((3, 32, 4, 2), (32, 64, 4, 2), (64, 128, 4, 2), (128, 256, 4, 2))
DEC = ((1024, 1, 1), ((1024, 128, 5, 2), (128, 64, 5, 2), (64, 32, 6, 2), (32, 3, 6, 2)))
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def episode(buf, g):
    """One trajectory of EP steps through ``add``, as planet.py's rollout stores it (next_obs = the next frame)."""
    frames = (g.integers(0, 32, (EP + 1, *FRAME)) * 8 + g.uniform(0, 8, (EP + 1, *FRAME))).astype(np.float32)
    for t in range(EP):
        buf.add(frames[t], g.uniform(-1, 1, A).astype(np.float32), frames[t + 1], float(g.standard_normal()), False,
                t == EP - 1)


def gather_time(mirror, starts, reps=200):
    """ms per ``b200pets_sequence_gather`` of one batch, CUDA events around ``reps`` launches, and the bytes it moves."""
    F = int(np.prod(FRAME))
    outs = (torch.empty(B, S - 1, *FRAME, device=DEV), torch.empty(B, S - 1, A, device=DEV),
            torch.empty(B, S - 1, device=DEV))
    for _ in range(10):
        mirror.gather(starts, S, *outs)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(reps):
        mirror.gather(starts, S, *outs)
    ev[1].record()
    torch.cuda.synchronize()
    k_ms = ev[0].elapsed_time(ev[1]) / reps
    frames = B * (S - 1)
    itemsize = 1 if mirror.storage == torch.uint8 else 4
    nbytes = frames * (F * (itemsize + 4) + A * 8 + 8) + B * 8  # frames read and written, act, rew, starts
    return {"ms": k_ms, "bytes": nbytes, "bytes_per_s": nbytes / (k_ms * 1e-3),
            "share_of_3.35TB_per_s": nbytes / (k_ms * 1e-3) / HBM_BYTES_PER_S}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--updates", type=int, default=100)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    mbrl, src = ra.import_reference()
    if mbrl is None:
        raise SystemExit(f"the reference is not importable: {src}")
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from mbrl.util import common
    from mbrl.util.replay_buffer import ReplayBuffer

    torch.manual_seed(0)
    base = mbrl.models.PlaNetModel(obs_shape=FRAME, obs_encoding_size=E, encoder_config=ENC, decoder_config=DEC,
                                   latent_state_size=L, action_size=A, belief_size=H, hidden_size_fcs=H, device=DEV)
    g = np.random.default_rng(0)
    buf = ReplayBuffer(100 * EP + EP, FRAME, (A,), obs_type=np.float32, rng=np.random.default_rng(1),
                       max_trajectory_length=EP)
    res = {"card": card(), "updates_per_train": args.updates, "rounds": args.rounds, "batch": B, "sequence_length": S,
           "frame": list(FRAME), "obs_dtype": "float32", "by_trajectories": {}}

    def run(arm, updates, losses=None):
        m = copy.deepcopy(base)
        trainer = bp.ModelTrainer(m, optim_lr=1e-3, optim_eps=1e-4)
        buf.rng.bit_generator.state = rng_state
        ds, _ = common.get_sequence_buffer_iterator(buf, B, 0, S, max_batches_per_loop_train=updates,
                                                    use_simple_sampler=True)
        mirror = None
        if arm == "mirror":
            mirror = replay.mirror_to_device(buf, DEV)
            mirror.flush()
        cb = (lambda *a: losses.append(a[1]) if len(losses) == 0 else None) if losses is not None else (lambda *a: None)
        try:
            return timed(lambda: trainer.train(ds, num_epochs=1, batch_callback=cb, evaluate=False))
        finally:
            if mirror is not None:
                mirror.close()

    for trajectories in (5, 100):
        while len(buf.trajectory_indices) < trajectories:
            episode(buf, g)
        rng_state = copy.deepcopy(buf.rng.bit_generator.state)
        first = {"host": [], "mirror": []}
        for arm in ("host", "mirror"):  # warm-up: module loads, cuDNN algorithm choice
            run(arm, 3, first[arm])
        times = {"host": [], "mirror": []}
        for _ in range(args.rounds):
            for arm in times:
                times[arm].append(run(arm, args.updates) / args.updates * 1e3)
        med = {k: float(np.median(v)) for k, v in times.items()}
        res["by_trajectories"][trajectories] = {
            "rows_stored": int(buf.num_stored), "ms_per_update": med, "ms_per_update_all": times,
            "speedup": med["host"] / med["mirror"], "first_update_losses": first,
            "first_update_losses_equal": first["host"] == first["mirror"]}

    # one episode's flush, on the 100-trajectory buffer
    mirror = replay.mirror_to_device(buf, DEV)
    full_rows = int(buf.num_stored)
    t_full = timed(mirror.flush)
    t_ep = []
    for _ in range(3):
        episode(buf, g)
        t_ep.append(timed(mirror.flush))
    res["flush"] = {"full_rows": full_rows, "full_ms": t_full * 1e3,
                    "episode_rows": EP, "episode_ms": float(np.median(t_ep) * 1e3), "episode_ms_all": [x * 1e3 for x in t_ep]}

    # the gather kernel alone, float32 frames (this buffer) and uint8 frames (a buffer of its own)
    from mbrl_lib_b200 import trainer as tr

    ds, _ = common.get_sequence_buffer_iterator(buf, B, 0, S, max_batches_per_loop_train=1, use_simple_sampler=True)
    starts = torch.from_numpy(next(tr.sequence_starts(ds, "sampler"))).to(DEV)
    res["sequence_gather_kernel"] = {"float32": gather_time(mirror, starts)}
    mirror.close()
    buf8 = ReplayBuffer(10 * EP, FRAME, (A,), obs_type=np.uint8, rng=np.random.default_rng(2), max_trajectory_length=EP)
    for _ in range(10):
        frames8 = g.integers(0, 256, (EP + 1, *FRAME), dtype=np.uint8)
        for t in range(EP):
            buf8.add(frames8[t], g.uniform(-1, 1, A).astype(np.float32), frames8[t + 1], 0.0, False, t == EP - 1)
    mirror8 = replay.mirror_to_device(buf8, DEV)
    mirror8.flush()
    ds8, _ = common.get_sequence_buffer_iterator(buf8, B, 0, S, max_batches_per_loop_train=1, use_simple_sampler=True)
    starts8 = torch.from_numpy(next(tr.sequence_starts(ds8, "sampler"))).to(DEV)
    res["sequence_gather_kernel"]["uint8"] = gather_time(mirror8, starts8)
    mirror8.close()
    print(json.dumps(res, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
