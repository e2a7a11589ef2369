"""Generate tests/golden/planet_train.npz from the *imported reference*: one ``PlaNetModel.update`` (planet.py:484-519) of
mbrl-lib's own model on the CPU, copied into oracle/_ref by oracle/install_ref.py:

    PYTHONPATH=oracle/ref_shims:oracle/_ref python oracle/gen_golden_planet_train.py

Small configuration: 3 x 16 x 16 frames, A 2, L 4, Hb = Hf = 16, encoding 32, B 3, sequence length 6 (T 5), free nats
0.1 (about the median KL per (b, t) here, so the maximum against it passes the gradient for some steps and not others;
at the default 3 the prior would get no gradient).  The
weights are the reference's own initialisation under ``torch.manual_seed``; the batch and the draws come from a numpy
seed, and the reference's ``_sample_state_from_params`` is fed those draws (posterior, then prior, per step).  The file
holds the parameters before the update (``param/<name>``), the batch (frames as uint8), the draws, the loss terms, every parameter's
clipped gradient (``grad/<name>``) and the parameters after one torch.optim.Adam step (lr 1e-3, eps 1e-4, the
arguments mbrl/algorithms/planet.py:92 gives ModelTrainer; ``after/<name>``).  TEST INFRASTRUCTURE.
"""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import mbrl.models  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
SIZES = dict(obs_shape=(3, 16, 16), obs_encoding_size=32, encoder_config=((3, 8, 4, 2), (8, 16, 4, 2)),
             decoder_config=((32, 1, 1), ((32, 16, 5, 2), (16, 8, 5, 2), (8, 3, 4, 1))), latent_state_size=4,
             action_size=2, belief_size=16, hidden_size_fcs=16, free_nats=0.1)
B, S = 3, 6
TORCH_SEED, DATA_SEED = 0, 1


def inputs():
    """The batch (pixel values 0..255 as float32) and the draws eps_q, eps_p [T, B, L] (float64)."""
    g = np.random.default_rng(DATA_SEED)
    obs = g.integers(0, 256, (B, S, 3, 16, 16)).astype(np.float32)
    act = g.uniform(-1, 1, (B, S, 2)).astype(np.float32)
    rew = g.standard_normal((B, S)).astype(np.float32)
    eq, ep = (g.standard_normal((S - 1, B, 4)) for _ in range(2))
    return obs, act, rew, eq, ep


def main():
    torch.manual_seed(TORCH_SEED)
    model = mbrl.models.PlaNetModel(device="cpu", **SIZES)
    obs, act, rew, eq, ep = inputs()
    draws = [torch.from_numpy(e).float() for t in range(S - 1) for e in (eq[t], ep[t])]
    L = model.latent_state_size
    model._sample_state_from_params = lambda params, generator, deterministic=False: \
        params[:, :L] if deterministic else params[:, :L] + params[:, L:] * draws.pop(0)
    out = {f"param/{k}": v.detach().numpy().copy() for k, v in model.named_parameters()}
    opt = torch.optim.Adam(model.parameters(), lr=1e-3, eps=1e-4)
    batch = types.SimpleNamespace(obs=obs, act=act, rewards=rew, next_obs=None, terminateds=None, truncateds=None)
    loss, meta = model.update(batch, opt)
    assert not draws
    out.update({f"grad/{k}": v.grad.numpy().copy() for k, v in model.named_parameters()})
    out.update({f"after/{k}": v.detach().numpy().copy() for k, v in model.named_parameters()})
    out.update(obs=obs.astype(np.uint8), act=act, rewards=rew, eps_q=eq, eps_p=ep,
               loss=np.float64(loss), observations_loss=np.float64(meta["observations_loss"]),
               reward_loss=np.float64(meta["reward_loss"]), kl_loss=np.float64(meta["kl_loss"]),
               grad_norm=np.float64(meta["grad_norm"]))
    path = os.path.join(GOLD, "planet_train.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
