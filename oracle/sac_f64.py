"""One SAC.update_parameters of mbrl-lib's pytorch_sac_pranz24 agent (sac.py:76-173) restated in float64: torch autograd and
torch.optim.Adam on CPU, with the reparameterisation draws injected.

Networks are dicts of tensors keyed as the reference's state_dicts (QNetwork: linear1 .. linear6; GaussianPolicy:
linear1, linear2, mean_linear, log_std_linear).  Adam state is a dict {key: (step, exp_avg, exp_avg_sq)}.
"""
import torch
import torch.nn.functional as F
from torch.distributions import Normal

CRITIC_KEYS = [f"linear{i}.{w}" for i in range(1, 7) for w in ("weight", "bias")]
POLICY_KEYS = [f"{n}.{w}" for n in ("linear1", "linear2", "mean_linear", "log_std_linear") for w in ("weight", "bias")]


def q_values(P, s, a):
    xu = torch.cat([s, a], 1)
    out = []
    for first in (1, 4):
        h = F.relu(F.linear(xu, P[f"linear{first}.weight"], P[f"linear{first}.bias"]))
        h = F.relu(F.linear(h, P[f"linear{first + 1}.weight"], P[f"linear{first + 1}.bias"]))
        out.append(F.linear(h, P[f"linear{first + 2}.weight"], P[f"linear{first + 2}.bias"]))
    return out


def policy_sample(P, s, eps, scale, bias):
    """GaussianPolicy.sample with Normal.rsample's draw replaced by `eps`: (action, log_prob [B][1], log_std before the
    clamp)."""
    h = F.relu(F.linear(s, P["linear1.weight"], P["linear1.bias"]))
    h = F.relu(F.linear(h, P["linear2.weight"], P["linear2.bias"]))
    mean = F.linear(h, P["mean_linear.weight"], P["mean_linear.bias"])
    lsr = F.linear(h, P["log_std_linear.weight"], P["log_std_linear.bias"])
    std = torch.clamp(lsr, min=-20, max=2).exp()
    normal = Normal(mean, std)
    x = mean + eps * std
    y = torch.tanh(x)
    logp = normal.log_prob(x) - torch.log(scale * (1 - y.pow(2)) + 1e-6)
    return y * scale + bias, logp.sum(1, keepdim=True), lsr


def _adam(params, state, lr):
    keys = list(params)
    opt = torch.optim.Adam([params[k] for k in keys], lr=lr, foreach=False)
    for k in keys:
        step, m, v = state[k]
        opt.state[params[k]] = {"step": torch.tensor(float(step)), "exp_avg": m.clone(), "exp_avg_sq": v.clone()}
    return opt


def _state_out(opt, params):
    return {k: (int(opt.state[p]["step"]), opt.state[p]["exp_avg"].detach().clone(),
                opt.state[p]["exp_avg_sq"].detach().clone()) for k, p in params.items()}


def sac_update(critic, target, policy, critic_state, policy_state, batch, eps, cfg, log_alpha=None, alpha_state=None):
    """One update.  batch = (s, a, s', r, terminated) as float64 tensors ([B][..], r and terminated [B]); eps [2][B][A] (on
    s', then on s); cfg: gamma, tau, lr, alpha (the temperature this update uses), tuning, target_entropy,
    target_update_interval, updates, reverse_mask, scale, bias.  Returns a dict with the new critic, target, policy,
    their Adam states, log_alpha and its state, alpha, and the statistics [qf1, qf2, policy, alpha loss, alpha, reward mean,
    -mean(log pi)]."""
    f64 = lambda t: torch.as_tensor(t, dtype=torch.float64)
    s, a, s2, r, term = (f64(x) for x in batch)
    eps = f64(eps)
    scale, bias = f64(cfg["scale"]), f64(cfg["bias"])
    C = {k: f64(v).clone().requires_grad_(True) for k, v in critic.items()}
    T = {k: f64(v).clone() for k, v in target.items()}
    P = {k: f64(v).clone().requires_grad_(True) for k, v in policy.items()}
    copt = _adam(C, critic_state, cfg["lr"])
    popt = _adam(P, policy_state, cfg["lr"])
    alpha = float(cfg["alpha"])
    r, term = r.reshape(-1, 1), term.reshape(-1, 1)
    mask = (1.0 - term) if cfg["reverse_mask"] else term

    with torch.no_grad():
        a2, logp2, _ = policy_sample(P, s2, eps[0], scale, bias)
        qt1, qt2 = q_values(T, s2, a2)
        y = r + mask * cfg["gamma"] * (torch.min(qt1, qt2) - alpha * logp2)
    q1, q2 = q_values(C, s, a)
    qf1_loss, qf2_loss = F.mse_loss(q1, y), F.mse_loss(q2, y)
    copt.zero_grad()
    (qf1_loss + qf2_loss).backward()
    copt.step()

    pi, logp, _ = policy_sample(P, s, eps[1], scale, bias)
    qp1, qp2 = q_values(C, s, pi)
    policy_loss = (alpha * logp - torch.min(qp1, qp2)).mean()
    popt.zero_grad()
    policy_loss.backward()
    popt.step()

    out = {}
    alpha_loss, new_alpha = 0.0, alpha
    if cfg["tuning"]:
        la = f64(log_alpha).clone().requires_grad_(True)
        aopt = _adam({"log_alpha": la}, {"log_alpha": alpha_state}, cfg["lr"])
        loss = -(la * (logp + cfg["target_entropy"]).detach()).mean()
        aopt.zero_grad()
        loss.backward()
        aopt.step()
        alpha_loss, new_alpha = float(loss.detach()), float(la.detach().exp())
        out["log_alpha"] = la.detach().clone()
        out["alpha_state"] = _state_out(aopt, {"log_alpha": la})["log_alpha"]
    if cfg["updates"] % cfg["target_update_interval"] == 0:
        T = {k: T[k] * (1.0 - cfg["tau"]) + C[k].detach() * cfg["tau"] for k in T}
    out.update(critic={k: v.detach().clone() for k, v in C.items()}, target=T,
               policy={k: v.detach().clone() for k, v in P.items()},
               critic_state=_state_out(copt, C), policy_state=_state_out(popt, P), alpha=new_alpha,
               stats=[qf1_loss.item(), qf2_loss.item(), policy_loss.item(), alpha_loss, new_alpha, float(r.mean()),
                      -logp.mean().item()])
    return out
