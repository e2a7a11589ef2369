"""Time PlaNet's model training at planet_cheetah_run shapes: one ``train()`` of 100 updates, each on 50 sequences of 50
3 x 64 x 64 frames (A 6, L 30, Hb = Hf = 200, encoding 1024), on synthetic pixel sequences.

Arms, alternated round by round (medians reported):
  reference  the reference's ModelTrainer and PlaNetModel.update (oracle/_ref);
  batched    this project's batched structure with the recurrence as a per-step PyTorch loop (an ablation that lives in
             this script only: it shows what the kernels themselves buy);
  device     mbrl_lib_b200.ModelTrainer: the batched structure with the recurrence kernels.
Then one device update is split: host batch formation and the host-to-device copy (host clock), the update's wall
time given a formed batch, device time per kernel family and per recurrence kernel (torch.profiler kernel durations),
and the weight-gradient matmuls alone (CUDA events).  The card's name and power limit are read in the same run.

    python tests/prof_planet_train.py [--rounds 3] [--updates 100] [--out result.json]
"""
import argparse
import copy
import json
import os
import subprocess
import sys
import time
import types

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import mbrl_lib_b200 as bp  # noqa: E402
from baseline import reference_arm as ra  # noqa: E402
from mbrl_lib_b200 import latent_train  # noqa: E402

DEV = "cuda:0"
B, S, A, L, H, E = 50, 50, 6, 30, 200, 1024
ENC = ((3, 32, 4, 2), (32, 64, 4, 2), (64, 128, 4, 2), (128, 256, 4, 2))
DEC = ((1024, 1, 1), ((1024, 128, 5, 2), (128, 64, 5, 2), (64, 32, 6, 2), (32, 3, 6, 2)))


class Sequences:
    """``updates`` batches of B random sequences of S frames gathered from a uint8 pool into float32 arrays on the
    host, as mbrl-lib's sequence sampler hands them over."""

    def __init__(self, updates, seed=0):
        g = np.random.default_rng(seed)
        self.frames = g.integers(0, 256, (4000, 3, 64, 64), dtype=np.uint8)
        self.acts = g.uniform(-1, 1, (4000, A)).astype(np.float32)
        self.rews = g.standard_normal(4000).astype(np.float32)
        self.updates, self.g = updates, g
        self.num_stored = 4000

    def __iter__(self):
        for _ in range(self.updates):
            start = self.g.integers(0, 4000 - S, B)[:, None] + np.arange(S)[None]
            yield types.SimpleNamespace(obs=self.frames[start].astype(np.float32), act=self.acts[start],
                                        rewards=self.rews[start], next_obs=None, terminateds=None, truncateds=None)


def per_step_recurrence(model, P, act, eps=None):
    """The recurrence as the reference computes it, one step at a time in PyTorch, on the batched structure's P."""
    Bn, T = P.shape[:2]
    Hb = model.belief_size
    q1, q2 = model.posterior_transition_model[0], model.posterior_transition_model[2]
    s = torch.zeros(Bn, L, device=P.device)
    h = torch.zeros(Bn, Hb, device=P.device)
    outs = [[] for _ in range(5)]
    for t in range(T):
        h = model.belief_model(s, act[:, t], h)
        q = model.posterior_transition_model[3](q2(F.relu(F.linear(h, q1.weight[:, :Hb]) + P[:, t])))
        s = q[:, :L] + q[:, L:] * torch.randn(Bn, L, device=P.device, generator=model.rng)
        p = model.prior_transition_model(h)
        sp = p[:, :L] + p[:, L:] * torch.randn(Bn, L, device=P.device, generator=model.rng)
        for o, v in zip(outs, (h, q, s, p, sp)):
            o.append(v)
    return tuple(torch.stack(o, 1) for o in outs)


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--updates", type=int, default=100)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    mbrl, src = ra.import_reference()
    if mbrl is None:
        raise SystemExit(f"the reference is not importable: {src}")
    torch.manual_seed(0)
    base = mbrl.models.PlaNetModel(obs_shape=(3, 64, 64), obs_encoding_size=E, encoder_config=ENC, decoder_config=DEC,
                                   latent_state_size=L, action_size=A, belief_size=H, hidden_size_fcs=H, device=DEV)
    cb = lambda *a: None  # noqa: E731  (mbrl/algorithms/planet.py always passes one)
    arms = {
        "reference": lambda m: mbrl.models.ModelTrainer(m, optim_lr=1e-3, optim_eps=1e-4),
        "batched": lambda m: mbrl.models.ModelTrainer(m, optim_lr=1e-3, optim_eps=1e-4),
        "device": lambda m: bp.ModelTrainer(m, optim_lr=1e-3, optim_eps=1e-4),
    }
    kernel_recurrence = latent_train.recurrence

    def run(name, updates):
        m = copy.deepcopy(base)
        trainer = arms[name](m)
        if name == "batched":  # the batched loss and update with the per-step recurrence in place of the kernels
            latent_train.recurrence = per_step_recurrence
            m.update = lambda batch, opt, target=None: latent_train.update(m, batch, opt)
        try:
            return timed(lambda: trainer.train(Sequences(updates), num_epochs=1, batch_callback=cb, evaluate=False))
        finally:
            latent_train.recurrence = kernel_recurrence

    for name in arms:  # warm-up: module loads, cuDNN algorithm choice
        run(name, 3)
    times = {k: [] for k in arms}
    for _ in range(args.rounds):
        for name in arms:
            times[name].append(run(name, args.updates) / args.updates * 1e3)
    med = {k: float(np.median(v)) for k, v in times.items()}

    # one device update, split: host batch formation, the host-to-device copy, the rest of the update's wall time, and
    # the device time by kernel family (torch.profiler kernel durations)
    m = copy.deepcopy(base)
    trainer = bp.ModelTrainer(m, optim_lr=1e-3, optim_eps=1e-4)
    trainer.train(Sequences(3), num_epochs=1, batch_callback=cb, evaluate=False)
    seqs, batches, t_form = iter(Sequences(10)), [], []
    for _ in range(10):
        t0 = time.perf_counter()
        batches.append(next(seqs))
        t_form.append(time.perf_counter() - t0)
    t_copy = [timed(lambda b=b: [torch.as_tensor(x).to(DEV) for x in (b.obs, b.act, b.rewards)]) for b in batches]
    t_update = [timed(lambda b=b: latent_train.update(m, b, trainer.optimizer)) for b in batches]
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for b in batches:
            latent_train.update(m, b, trainer.optimizer)
        torch.cuda.synchronize()
    fam = {"recurrence kernels (forward, backward, re-pack)": 0.0, "convolutions (encoder, decoder)": 0.0,
           "clip + Adam": 0.0, "H2D copy": 0.0, "other": 0.0}
    kern = {"rssm_seq_forward_kernel": 0.0, "rssm_seq_backward_kernel": 0.0, "re-pack (latent_pack, latent_bias)": 0.0}
    for ev in prof.key_averages():
        t = ev.device_time_total / 1e3 / len(batches)  # ms per update
        n = ev.key.lower()
        if "rssm_seq" in n or "latent_pack" in n or "latent_bias" in n:
            fam["recurrence kernels (forward, backward, re-pack)"] += t
            key = next((k for k in kern if k in n), "re-pack (latent_pack, latent_bias)")
            kern[key] += t
        elif "conv" in n or "cudnn" in n or "dgrad" in n or "wgrad" in n or "fprop" in n or "xmma" in n:
            fam["convolutions (encoder, decoder)"] += t
        elif "adam" in n or "foreach" in n or "multi_tensor" in n or "norm" in n:
            fam["clip + Adam"] += t
        elif "memcpy htod" in n:
            fam["H2D copy"] += t
        elif ev.device_time_total > 0 and not n.startswith("profilerstep"):
            fam["other"] += t

    # the weight-gradient products (torch matmuls over all B x T rows) alone, with CUDA events, on tensors of the
    # shapes the backward pass hands them
    T = S - 1
    shapes = {"e": H, "gates": 4 * H, "q1": H, "p1": H, "pre_std": 2 * L, "eps": 2 * L, "de": H, "dgi": 3 * H,
              "dghn": H, "dq": 2 * L, "dv": H, "dp": 2 * L}
    tape = {k: torch.randn(B, T, w, device=DEV) for k, w in shapes.items()}
    dP, act = torch.randn(B, T, H, device=DEV), torch.rand(B, T, A, device=DEV) * 2 - 1
    bel, smp = torch.randn(B, T, H, device=DEV), torch.randn(B, T, L, device=DEV)
    W_q1 = m.posterior_transition_model[0].weight.detach()
    for _ in range(5):
        latent_train.weight_grads(tape, dP, act, bel, smp, W_q1)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    reps = 100
    ev[0].record()
    for _ in range(reps):
        latent_train.weight_grads(tape, dP, act, bel, smp, W_q1)
    ev[1].record()
    torch.cuda.synchronize()
    t_wgrad = ev[0].elapsed_time(ev[1]) / reps

    rows = B * T
    fwd_flop = 2 * rows * (H * (L + A) + 6 * H * H + 2 * H * H + 2 * (2 * L * H))
    bwd_flop = 2 * rows * (2 * (2 * L * H) + 2 * H * H + 6 * H * H + H * L)
    wgrad_flop = 2 * rows * (H * (L + A) + 6 * H * H + H * H + 2 * L * H + H * H + 2 * L * H)
    fk, bk = kern["rssm_seq_forward_kernel"], kern["rssm_seq_backward_kernel"]
    res = {"card": card(), "updates_per_train": args.updates, "rounds": args.rounds, "ms_per_update": med,
           "ms_per_update_all": times, "speedup_vs_reference": med["reference"] / med["device"],
           "speedup_vs_batched": med["batched"] / med["device"],
           "host_batch_formation_ms": float(np.median(t_form) * 1e3), "h2d_copy_wall_ms": float(np.median(t_copy) * 1e3),
           "update_wall_ms_given_a_formed_batch": float(np.median(t_update) * 1e3),
           "device_ms_per_update_by_family": fam, "recurrence_kernel_ms": kern,
           "forward_kernel_tflops": fwd_flop / fk / 1e9, "backward_kernel_tflops": bwd_flop / bk / 1e9,
           "weight_grad_matmuls_ms": t_wgrad, "weight_grad_matmuls_tflops": wgrad_flop / t_wgrad / 1e9}
    print(json.dumps(res, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
