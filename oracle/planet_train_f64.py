"""PlaNetModel.forward / loss / update (mbrl/models/planet.py:354-519) restated per step, as the reference runs them, for
a float64 copy of a model on the CPU, with the draws injected: ``eps_q[t]`` / ``eps_p[t]`` (``[B, L]`` each) stand for
the posterior's and the prior's ``torch.randn`` of step t, in the order the reference draws them.

The model is read by attribute (mbrl-lib's ``PlaNetModel`` or the container of ``mbrl_lib_b200.models``); use
:func:`as_f64` for a float64 CPU copy."""
from __future__ import annotations

import copy

import torch
import torch.nn.functional as F


def as_f64(model):
    m = copy.deepcopy(model).double().cpu()
    m.free_nats = m.free_nats.double().cpu()
    return m


def _split(params, L, min_std):
    return params[:, :L], F.softplus(params[:, L:]) + min_std


def forward(m, next_obs, action, eps_q, eps_p, P=None, masks=None, pre=None):
    """The five stacked outputs of PlaNetModel.forward.  ``P [B, T, Hf]`` (the posterior's encoding half) replaces the
    encoder when given.  ``masks`` (``{"e": [B, T, Hb], "q1": [B, T, Hf], "p1": [B, T, Hf]}``, 0 / 1) replaces the
    three ReLUs of the recurrence by those fixed masks: the float64 function an fp32 run computes where its ReLUs chose
    as it did, for separating rounding from a pre-activation that lies on the other side of 0 in fp32.  ``pre``, a dict,
    receives those three layers' pre-activations ``[B, T, .]``."""
    B, T = next_obs.shape[:2] if next_obs is not None else P.shape[:2]
    L, Hb = m.latent_state_size, m.belief_size
    s = torch.zeros(B, L, dtype=torch.float64)
    h = torch.zeros(B, Hb, dtype=torch.float64)
    emb = m.belief_model.embedding_layer[0]
    q1, q2 = m.posterior_transition_model[0], m.posterior_transition_model[2]
    p1, p2 = m.prior_transition_model[0], m.prior_transition_model[2]
    seen = {"e": [], "q1": [], "p1": []}

    def relu(x, k, t):
        seen[k].append(x.detach())
        return F.relu(x) if masks is None else x * masks[k][:, t]

    out = {k: [] for k in ("beliefs", "post_params", "post_samples", "prior_params", "prior_samples")}
    for t in range(T):
        e = relu(emb(torch.cat([s, action[:, t]], 1)), "e", t)
        h = m.belief_model.rnn(e, h)
        if P is None:
            enc = m.encoder(next_obs[:, t])
            u = q1(torch.cat([h, enc], 1))
        else:
            u = F.linear(h, q1.weight[:, :Hb]) + P[:, t]
        mq, sq = _split(q2(relu(u, "q1", t)), L, m.min_std)
        s = mq + sq * eps_q[t]
        mp, sp = _split(p2(relu(p1(h), "p1", t)), L, m.min_std)
        out["beliefs"].append(h)
        out["post_params"].append(torch.cat([mq, sq], 1))
        out["post_samples"].append(s)
        out["prior_params"].append(torch.cat([mp, sp], 1))
        out["prior_samples"].append(mp + sp * eps_p[t])
    if pre is not None:
        pre.update({k: torch.stack(v, 1) for k, v in seen.items()})
    return {k: torch.stack(v, 1) for k, v in out.items()}


def loss_terms(m, obs, action, rewards, eps_q, eps_p):
    """planet.py:429-462 on processed tensors (obs already ``/ 256 - 0.5``): per-(b, t) losses and the reconstruction."""
    next_obs, act, rew = obs[:, 1:], action[:, :-1], rewards[:, :-1]
    L = m.latent_state_size
    o = forward(m, next_obs, act, eps_q, eps_p)
    B, T = next_obs.shape[:2]
    pred_obs = torch.stack([m.decoder(torch.cat([o["post_samples"][:, t], o["beliefs"][:, t]], -1)) for t in range(T)], 1)
    pred_rew = torch.stack([m.reward_model(torch.cat([o["beliefs"][:, t], o["post_samples"][:, t]], 1))[:, 0]
                            for t in range(T)], 1)
    obs_loss = F.mse_loss(pred_obs, next_obs, reduction="none").sum((2, 3, 4))
    reward_loss = F.mse_loss(pred_rew, rew, reduction="none")
    qp, pp = o["post_params"], o["prior_params"]
    kl = torch.distributions.kl_divergence(torch.distributions.Normal(qp[..., :L], qp[..., L:]),
                                           torch.distributions.Normal(pp[..., :L], pp[..., L:])).sum(2).max(m.free_nats)
    return obs_loss, reward_loss, kl, pred_obs


def update(m, obs, action, rewards, eps_q, eps_p, optimizer):
    """planet.py:484-519: one clipped optimizer step; returns (loss, observations_loss, reward_loss, kl_loss,
    grad_norm)."""
    m.train()
    optimizer.zero_grad()
    o, r, k, _ = loss_terms(m, obs, action, rewards, eps_q, eps_p)
    o, r, k = o.mean(), r.mean(), k.mean()
    total = o + r + m.kl_scale * k
    total.backward()
    torch.nn.utils.clip_grad_norm_(m.parameters(), m.grad_clip_norm, norm_type=2)
    gn = sum(float(p.grad.norm(2)) for p in m.parameters() if p.grad is not None)
    optimizer.step()
    return float(total.detach()), float(o.detach()), float(r.detach()), float(k.detach()), gn
