"""Writes tests/golden/sac_*.npz: three consecutive SAC.update_parameters of the reference's own pytorch_sac_pranz24 agent
on CPU, with Normal.rsample patched to consume recorded draws, for tests/test_sac_cpu.py to check oracle/sac_f64.py
against.  Each file holds the initial networks and optimizer states, every update's batch and draws, and the networks,
Adam moments, log_alpha and returned statistics after each update.

    python oracle/gen_golden_sac.py     (needs the reference in oracle/_ref; see oracle/install_ref.py)
"""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from baseline import reference_arm as ra  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
CASES = {  # name: obs, act, hidden, batch, automatic_entropy_tuning, target_update_interval, reverse_mask
    "sac_tuning": (5, 2, 16, 12, True, 1, True),
    "sac_interval2": (7, 3, 24, 9, False, 2, False),
}


class Box:
    def __init__(self, A):
        self.low = -np.linspace(1.0, 2.0, A).astype(np.float32)
        self.high = np.linspace(1.0, 3.0, A).astype(np.float32)
        self.shape = (A,)


class Memory:
    def __init__(self, batches):
        self.batches = batches

    def sample(self, n):
        return self.batches.pop(0)


def generate(name, D, A, H, B, tuning, interval, reverse):
    mbrl, src = ra.import_reference()
    assert mbrl is not None, f"the reference is not importable: {src}"
    from mbrl.third_party.pytorch_sac_pranz24.sac import SAC
    from mbrl.types import TransitionBatch

    torch.manual_seed(len(name))
    args = types.SimpleNamespace(gamma=0.99, tau=0.05, alpha=0.2, policy="Gaussian", target_update_interval=interval,
                                 automatic_entropy_tuning=tuning, target_entropy=None, hidden_size=H, device="cpu", lr=1e-2)
    agent = SAC(D, Box(A), args)
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for p in list(agent.critic.parameters()) + list(agent.policy.parameters()):
            if p.dim() == 1:
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)
    out = {"cfg": np.array([D, A, H, B, int(tuning), interval, int(reverse)]),
           "hyper": np.array([args.gamma, args.tau, args.alpha, args.lr]),
           "scale": agent.policy.action_scale.numpy(), "bias": agent.policy.action_bias.numpy()}
    for prefix, mod in (("critic", agent.critic), ("target", agent.critic_target), ("policy", agent.policy)):
        for k, v in mod.state_dict().items():
            out[f"init/{prefix}/{k}"] = v.numpy().copy()
    rng = np.random.default_rng(2)
    queue = []
    torch.distributions.Normal.rsample = lambda d, sample_shape=torch.Size(): d.loc + queue.pop(0) * d.scale
    for u in range(3):
        b = TransitionBatch(rng.standard_normal((B, D)).astype(np.float32), rng.uniform(-1, 1, (B, A)).astype(np.float32),
                            rng.standard_normal((B, D)).astype(np.float32), rng.standard_normal(B).astype(np.float32),
                            rng.random(B) < 0.4, np.zeros(B, bool))
        eps = rng.standard_normal((2, B, A)).astype(np.float32)
        queue.extend([torch.from_numpy(eps[0]), torch.from_numpy(eps[1])])
        stats = agent.update_parameters(Memory([b]), B, u, reverse_mask=reverse)
        for k, v in zip(("obs", "act", "next_obs", "rewards", "terminateds"), b.astuple()):
            out[f"u{u}/batch/{k}"] = v
        out[f"u{u}/eps"] = eps
        out[f"u{u}/stats"] = np.array(stats, np.float64)
        for prefix, mod, opt in (("critic", agent.critic, agent.critic_optim), ("target", agent.critic_target, None),
                                 ("policy", agent.policy, agent.policy_optim)):
            for (k, p) in mod.named_parameters():
                out[f"u{u}/{prefix}/{k}"] = p.detach().numpy().copy()
                if opt is not None:
                    out[f"u{u}/{prefix}_m/{k}"] = opt.state[p]["exp_avg"].numpy().copy()
                    out[f"u{u}/{prefix}_v/{k}"] = opt.state[p]["exp_avg_sq"].numpy().copy()
        if tuning:
            out[f"u{u}/log_alpha"] = agent.log_alpha.detach().numpy().copy()
            st = agent.alpha_optim.state[agent.log_alpha]
            out[f"u{u}/log_alpha_m"], out[f"u{u}/log_alpha_v"] = st["exp_avg"].numpy().copy(), st["exp_avg_sq"].numpy().copy()
    path = os.path.join(OUT, f"{name}.npz")
    np.savez_compressed(path, **out)
    return path


if __name__ == "__main__":
    for name, case in CASES.items():
        print(generate(name, *case))
