"""Float64 restatement of PlaNet's latent model as the planner uses it (mbrl/models/planet.py:82-114, 231-264, 531-581;
mbrl/models/model_env.py:145-191), with injected draws.  TEST INFRASTRUCTURE; nothing shipped uses it.

``params`` is a dict of float64 numpy arrays in torch's layout (``[out, in]`` weights), read from any object with
PlaNet's attribute layout by :func:`params_of`.
"""
import numpy as np
import torch

from oracle import pets_oracle as po


def params_of(model) -> dict:
    emb, rnn = model.belief_model.embedding_layer[0], model.belief_model.rnn
    p1, p2 = model.prior_transition_model[0], model.prior_transition_model[2]
    r1, r2, r3 = model.reward_model[0], model.reward_model[2], model.reward_model[4]

    def f(t):
        return t.detach().cpu().double().numpy()

    return {"We": f(emb.weight), "be": f(emb.bias), "Wih": f(rnn.weight_ih), "Whh": f(rnn.weight_hh),
            "bih": f(rnn.bias_ih), "bhh": f(rnn.bias_hh), "Wp1": f(p1.weight), "bp1": f(p1.bias), "Wp2": f(p2.weight),
            "bp2": f(p2.bias), "Wr1": f(r1.weight), "br1": f(r1.bias), "Wr2": f(r2.weight), "br2": f(r2.bias),
            "Wr3": f(r3.weight), "br3": f(r3.bias), "min_std": float(model.min_std)}


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def _softplus(x):  # torch F.softplus: beta 1, threshold 20
    return np.where(x > 20.0, x, np.log1p(np.exp(np.minimum(x, 20.0))))


def step(p, latent, belief, act, eps=None):
    """PlaNetModel.sample for a batch: ``(next_latent [B, L], next_belief [B, Hb], reward [B])``; ``eps [B, L]`` are the
    draws (``None``: deterministic, the prior's mean)."""
    latent, belief, act = (np.asarray(x, np.float64) for x in (latent, belief, act))
    Hb, L = belief.shape[1], latent.shape[1]
    e = np.maximum(np.concatenate([latent, act], 1) @ p["We"].T + p["be"], 0.0)
    gi = e @ p["Wih"].T + p["bih"]
    gh = belief @ p["Whh"].T + p["bhh"]
    r = _sigmoid(gi[:, :Hb] + gh[:, :Hb])
    z = _sigmoid(gi[:, Hb:2 * Hb] + gh[:, Hb:2 * Hb])
    n = np.tanh(gi[:, 2 * Hb:] + r * gh[:, 2 * Hb:])
    h = (1.0 - z) * n + z * belief
    q = np.maximum(h @ p["Wp1"].T + p["bp1"], 0.0) @ p["Wp2"].T + p["bp2"]
    mean = q[:, :L]
    s = mean if eps is None else mean + (_softplus(q[:, L:]) + p["min_std"]) * np.asarray(eps, np.float64)
    x = np.maximum(np.concatenate([h, s], 1) @ p["Wr1"].T + p["br1"], 0.0)
    x = np.maximum(x @ p["Wr2"].T + p["br2"], 0.0)
    rew = (x @ p["Wr3"].T + p["br3"])[:, 0]
    return s, h, rew


def evaluate(p, latent0, belief0, actions, particles, eps):
    """ModelEnv.evaluate_action_sequences from the posterior with no_termination: ``(returns [N], row_returns [B])``;
    ``eps [H, B, L]`` the draws of every step (sample=True), rows ``n * P + p``."""
    actions = np.asarray(actions, np.float64)
    N, H, _ = actions.shape
    B = N * particles
    s = np.tile(np.asarray(latent0, np.float64).reshape(1, -1), (B, 1))
    h = np.tile(np.asarray(belief0, np.float64).reshape(1, -1), (B, 1))
    total = np.zeros(B)
    for t in range(H):
        s, h, rew = step(p, s, h, np.repeat(actions[:, t], particles, axis=0), eps[t])
        total += rew
    return total.reshape(N, particles).mean(1), total


def cem_plan(p, latent0, belief0, x0, lb, ub, num_iterations, elite_ratio, population_size, alpha, z, eps,
             particles=1, return_mean_elites=True, clipped_normal=True, trace=None):
    """CEMOptimizer.optimize over :func:`evaluate` in float64: ``z [it, N, H, A]`` the population draws, ``eps [it, H,
    B, L]`` the model draws of every iteration's evaluation.  Returns the solution ``[H, A]``."""
    t64 = lambda a: torch.as_tensor(np.asarray(a, np.float64))  # noqa: E731

    def obj(pop, i):
        return t64(evaluate(p, latent0, belief0, pop.numpy(), particles, eps[i])[0])

    sol = po.cem_optimize(obj, t64(x0), t64(lb), t64(ub), num_iterations, elite_ratio, population_size, alpha,
                          [t64(zi) for zi in z], return_mean_elites=return_mean_elites, clipped_normal=clipped_normal,
                          trace=trace)
    return sol.numpy()


# ---- seeded inputs of the goldens (tests/golden/planet_*.npz), regenerated anywhere from numpy seeds -------------
GOLDEN_SIZES = {"action_size": 3, "latent_state_size": 5, "belief_size": 16, "hidden_size_fcs": 12, "min_std": 0.1}


def fill_params(model, seed, scale=0.3):
    """Overwrite every planning parameter of ``model`` (PlaNet's layout) with N(0, scale^2) draws from numpy ``seed``,
    in the order of ``b200pets_latent_model_create``."""
    from mbrl_lib_b200.latent import latent_params

    rng = np.random.default_rng(seed)
    with torch.no_grad():
        for t in latent_params(model):
            t.copy_(torch.from_numpy(rng.normal(0.0, scale, tuple(t.shape)).astype(np.float32)))


def golden_inputs(kind, seed=0):
    """Inputs of one golden: "step" (B 6), "eval" (N 5, H 4, P 2) or "cem" (N 20, H 3, 3 iterations, P 2), float32."""
    A, L, Hb = GOLDEN_SIZES["action_size"], GOLDEN_SIZES["latent_state_size"], GOLDEN_SIZES["belief_size"]
    rng = np.random.default_rng(100 + seed)
    f = lambda *s: rng.standard_normal(s).astype(np.float32)  # noqa: E731
    if kind == "step":
        B = 6
        return {"latent": f(B, L), "belief": np.tanh(f(B, Hb)), "act": np.clip(f(B, A), -1, 1), "eps": f(B, L)}
    post = {"latent0": f(L), "belief0": np.tanh(f(Hb))}
    if kind == "eval":
        N, H, P = 5, 4, 2
        return {**post, "actions": np.clip(f(N, H, A), -1, 1), "eps": f(H, N * P, L), "particles": P}
    N, H, P, it = 20, 3, 2, 3
    return {**post, "z": f(it, N, H, A), "eps": f(it, H, N * P, L), "particles": P, "population": N, "horizon": H,
            "iterations": it, "elite_ratio": 0.2, "alpha": 0.1}
