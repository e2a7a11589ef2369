"""Generate the PlaNet goldens (tests/golden/planet_{step,eval,cem}.npz) from the *imported reference*: mbrl-lib's own
``PlaNetModel``, ``ModelEnv`` and ``CEMOptimizer`` on the CPU, copied into oracle/_ref by oracle/install_ref.py:

    PYTHONPATH=oracle/ref_shims:oracle/_ref python oracle/gen_golden_planet.py

The weights and every input come from numpy seeds (oracle.latent_f64.fill_params / golden_inputs); the reference's
``torch.randn`` (the prior's draw, planet.py:289-306) and ``torch.randn_like`` (CEM's clipped-normal population,
trajectory_opt.py:110-118) are monkey-fed those draws, so the files hold outputs only.  TEST INFRASTRUCTURE.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import mbrl.env.termination_fns as ref_term  # noqa: E402
import mbrl.models  # noqa: E402
import mbrl.planning  # noqa: E402

from oracle import latent_f64 as lo  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
WEIGHT_SEED = 7


def build_reference():
    """The reference's PlaNetModel at the golden sizes (the encoder / decoder of planet.yaml, unused here)."""
    s = lo.GOLDEN_SIZES
    model = mbrl.models.PlaNetModel(
        obs_shape=(3, 64, 64), obs_encoding_size=1024,
        encoder_config=((3, 32, 4, 2), (32, 64, 4, 2), (64, 128, 4, 2), (128, 256, 4, 2)),
        decoder_config=((1024, 1, 1), ((1024, 128, 5, 2), (128, 64, 5, 2), (64, 32, 6, 2), (32, 3, 6, 2))),
        latent_state_size=s["latent_state_size"], action_size=s["action_size"], belief_size=s["belief_size"],
        hidden_size_fcs=s["hidden_size_fcs"], device="cpu", min_std=s["min_std"])
    lo.fill_params(model, WEIGHT_SEED)
    return model


class _Env:
    def __init__(self, A):
        import gymnasium

        self.observation_space = gymnasium.spaces.Box(0, 255, (3, 64, 64))
        self.action_space = gymnasium.spaces.Box(-1.0, 1.0, (A,))


class FeedRandn:
    """torch.randn / torch.randn_like return the queued draws in call order."""

    def __init__(self, randn=(), randn_like=()):
        self.randn, self.randn_like = [torch.from_numpy(np.ascontiguousarray(x)) for x in randn], \
            [torch.from_numpy(np.ascontiguousarray(x)) for x in randn_like]

    def __enter__(self):
        self._r, self._rl = torch.randn, torch.randn_like

        def randn(*size, **kw):
            z = self.randn.pop(0)
            assert tuple(z.shape) == tuple(size[0] if len(size) == 1 else size), (z.shape, size)
            return z.to(kw.get("dtype") or torch.float32)

        def randn_like(t, **kw):
            z = self.randn_like.pop(0)
            assert z.shape == t.shape, (z.shape, t.shape)
            return z.to(t.dtype)

        torch.randn, torch.randn_like = randn, randn_like
        return self

    def __exit__(self, *a):
        torch.randn, torch.randn_like = self._r, self._rl
        assert not self.randn and not self.randn_like, "unused injected draws"


def _set_posterior(model, inp):
    model._current_posterior_sample = torch.from_numpy(inp["latent0"]).view(1, -1)
    model._current_belief = torch.from_numpy(inp["belief0"]).view(1, -1)


def main():
    model = build_reference()
    A = lo.GOLDEN_SIZES["action_size"]
    env = mbrl.models.ModelEnv(_Env(A), model, ref_term.no_termination, generator=torch.Generator())
    obs = np.zeros((3, 64, 64), np.uint8)

    inp = lo.golden_inputs("step")
    state = {"latent": torch.from_numpy(inp["latent"]), "belief": torch.from_numpy(inp["belief"])}
    env._return_as_np = False  # what reset(..., return_as_np=False) sets; the step states are given directly
    det = env.step(torch.from_numpy(inp["act"]), state, sample=False)
    with FeedRandn(randn=[inp["eps"]]):
        smp = env.step(torch.from_numpy(inp["act"]), state, sample=True)
    np.savez(os.path.join(GOLD, "planet_step.npz"),
             det_latent=det[0].numpy(), det_belief=det[3]["belief"].numpy(), det_reward=det[1].numpy(),
             smp_latent=smp[0].numpy(), smp_belief=smp[3]["belief"].numpy(), smp_reward=smp[1].numpy())

    inp = lo.golden_inputs("eval")
    _set_posterior(model, inp)
    with FeedRandn(randn=list(inp["eps"])):
        ret = env.evaluate_action_sequences(torch.from_numpy(inp["actions"]), obs, inp["particles"])
    np.savez(os.path.join(GOLD, "planet_eval.npz"), returns=ret.numpy())

    inp = lo.golden_inputs("cem")
    _set_posterior(model, inp)
    H, N, it = inp["horizon"], inp["population"], inp["iterations"]
    lower, upper = [[-1.0] * A] * H, [[1.0] * A] * H
    opt = mbrl.planning.CEMOptimizer(num_iterations=it, elite_ratio=inp["elite_ratio"], population_size=N,
                                     lower_bound=lower, upper_bound=upper, alpha=inp["alpha"], device="cpu",
                                     return_mean_elites=True, clipped_normal=True)
    values = []
    draws = [e for i in range(it) for e in inp["eps"][i]]
    with FeedRandn(randn=draws, randn_like=list(inp["z"])):
        sol = opt.optimize(lambda pop: env.evaluate_action_sequences(pop, obs, inp["particles"]), torch.zeros(H, A),
                           callback=lambda pop, v, i: values.append(v.clone().numpy()))
    np.savez(os.path.join(GOLD, "planet_cem.npz"), solution=sol.numpy(), values=np.stack(values))
    print("planet goldens written; cem solution", sol.numpy().round(4).tolist())


if __name__ == "__main__":
    main()
