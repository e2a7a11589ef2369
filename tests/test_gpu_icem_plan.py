"""The fused iCEM plan (``ICEMOptimizer.optimize`` over the model's objective: one ``b200pets_icem_plan`` call) against
the per-iteration loop it replaces, which the same optimiser runs when the objective is wrapped in a plain lambda.

Both paths start from the same torch CUDA generator state, environment counter and optimiser state, and are compared
bit for bit (``torch.equal``) over three consecutive calls (carried, shifted elites): the solution, the elite set, every
iteration's values, both counters and the generator state afterwards.  The cases cover both rollout kernels, the three
propagation modes with tile shuffle and with permutations, a population whose permutation decision flips mid-plan,
1, 2 and 5 iterations, ``population_size_module`` None / 5 / 7 (kept elites rounded above ``elite_num`` included),
``return_mean_elites`` both ways, and populations beyond the single-CTA refit, which run the optimiser's own kernels.
"""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

from mbrl_lib_b200 import synthetic as syn
from test_gpu_parity import DEV, _Env, make_env

pytestmark = pytest.mark.gpu

# name -> (model case, precision, ts1, H, population, iterations, module, keep_elite_frac, return_mean_elites, particles)
PLANS = {
    "few_groups_flip": ("halfcheetah_small", "f32", "tile_shuffle", 10, 200, 5, 7, 0.3, True, 5),  # perms from iteration 2
    "tile_shuffle_tc": ("halfcheetah_small", "bf16_tc", "tile_shuffle", 10, 200, 5, 7, 0.3, False, 20),
    "ts1_perms": ("halfcheetah_small", "bf16_tc", "perms", 12, 100, 2, 5, 0.3, True, 5),
    "humanoid_trunc_f32": ("humanoid_trunc", "f32", "tile_shuffle", 10, 300, 5, 5, 0.3, True, 10),
    "humanoid_trunc_tc": ("humanoid_trunc", "bf16_tc", "tile_shuffle", 10, 300, 5, 5, 0.3, False, 10),
    "humanoid_v4_f32": ("humanoid_v4", "f32", "tile_shuffle", 6, 200, 5, None, 0.3, True, 10),
    "fixed_model": ("hopper_tsinf", "f32", "tile_shuffle", 9, 150, 5, None, 0.3, False, 6),
    "fixed_model_perms": ("hopper_tsinf", "f32", "perms", 9, 64, 2, 7, 0.3, True, 6),
    "expectation": ("silu_expectation", "f32", "tile_shuffle", 6, 120, 5, 5, 0.3, True, 5),
    "one_iteration": ("halfcheetah_small", "f32", "tile_shuffle", 8, 100, 1, None, 0.3, False, 5),
    "keep_above_elite_num": ("halfcheetah_small", "f32", "tile_shuffle", 8, 30, 3, 7, 0.5, False, 5),  # 3 elites, keep 7
    "keep_none": ("halfcheetah_small", "f32", "tile_shuffle", 8, 100, 3, None, 0.0, True, 5),
    "rows_above_refit": ("halfcheetah_small", "f32", "tile_shuffle", 4, 2100, 2, None, 0.3, True, 5),  # 2 100 rows > 2 048
    "elites_above_refit": ("humanoid_trunc", "f32", "tile_shuffle", 40, 1000, 5, 5, 0.3, True, 5),  # elite set 272 KB
}


def _optimizer(spec, H, pop, iters, module, keep_frac, rme):
    import mbrl_lib_b200 as bp

    lb, ub = np.full((H, spec.act_dim), spec.action_lb).tolist(), np.full((H, spec.act_dim), spec.action_ub).tolist()
    opt = bp.ICEMOptimizer(iters, 0.1, pop, 1.3, 2.0, lb, ub, keep_frac, 0.1, DEV, return_mean_elites=rme,
                           population_size_module=module)
    opt.record_values = True
    return opt


def _plan(opt, obj, x0):
    sol = opt.optimize(obj, x0=x0).clone()
    torch.cuda.synchronize()
    return sol, opt.elite.clone(), [v.clone() for v in opt.last_values]


def compare_plans(env, fused, loop, obs, P, x0s):
    """Run each warm start of x0s through both optimisers, the loop from the state the fused plan started from."""
    from mbrl_lib_b200.planning import _FusedObjective

    obj = _FusedObjective(env, obs, P)
    for call, x0 in enumerate(x0s):
        rng, offset = torch.cuda.get_rng_state(), env._offset
        got = _plan(fused, obj, x0)
        after = (torch.cuda.get_rng_state(), env._offset, fused._offset)
        torch.cuda.set_rng_state(rng)
        env._offset = offset
        ref = _plan(loop, lambda seqs: obj(seqs), x0)
        assert env._offset == offset + loop.num_iterations == after[1], f"call {call}: environment counter"
        assert fused._offset == loop._offset == call + 1, f"call {call}: optimiser counter"
        assert torch.equal(after[0], torch.cuda.get_rng_state()), f"call {call}: torch generator state"
        assert len(got[2]) == len(ref[2]) == loop.num_iterations
        for i, (v, r) in enumerate(zip(got[2], ref[2])):
            assert v.shape == r.shape and torch.equal(v, r), f"call {call}: values of iteration {i} differ"
        assert torch.equal(got[1], ref[1]), f"call {call}: elite sets differ"
        assert torch.equal(got[0], ref[0]), f"call {call}: solutions differ"
        assert torch.isfinite(got[0]).all()


@pytest.mark.parametrize("name", list(PLANS))
def test_fused_plan_equals_the_loop(name):
    case, precision, ts1, H, pop, iters, module, keep_frac, rme, P = PLANS[name]
    spec, _, env = make_env(case, precision, ts1=ts1)
    fused, loop = (_optimizer(spec, H, pop, iters, module, keep_frac, rme) for _ in range(2))
    if name == "few_groups_flip":
        flips = [env._few_groups(n + fused.keep_elite_size, P) for n in fused.population_sizes()]
        assert not flips[0] and flips[-1], flips
    if name == "keep_above_elite_num":
        assert fused.elite_num == 3 and fused.keep_elite_size == 7
    rows =max(fused.population_sizes()) + min(fused.keep_elite_size, fused.elite_num)
    refit_cta = rows <= 2048 and fused.elite_num * H * spec.act_dim * 4 <= 150 * 1024
    assert refit_cta == (name not in ("rows_above_refit", "elites_above_refit")), (name, rows)
    obs = syn.make_rollout_inputs(spec, with_noise=False)["obs0"]
    g = np.random.default_rng(len(name))
    x0s = [torch.from_numpy(g.uniform(-0.3, 0.3, (H, spec.act_dim)).astype(np.float32)).to(DEV) for _ in range(3)]
    env._offset = 40
    compare_plans(env, fused, loop, obs, P, x0s)


def _cartpole_env():
    """pets_icem_cartpole's model: an ensemble of 7 with 5 elites, 4 x 200 SiLU, on CartPole's dims."""
    import mbrl_lib_b200 as bp
    from mbrl_lib_b200 import functions

    spec = dataclasses.replace(syn.CASES["cartpole_pets"], ensemble_size=7, elites=(0, 2, 3, 5, 6), hid_size=200, num_layers=4)
    model = bp.model_from_arrays(spec, syn.make_model_arrays(spec), DEV)
    env = bp.ModelEnv(_Env(spec), model, functions.TERM_FNS[spec.term_fn], functions.REWARD_FNS[spec.reward_fn],
                      generator=torch.Generator(device=DEV))
    return spec, env


ICEM_CARTPOLE = {"_target_": "mbrl.planning.ICEMOptimizer", "num_iterations": 5, "elite_ratio": 0.1, "population_size": 200,
                 "population_decay_factor": 1.3, "colored_noise_exponent": 2.0, "keep_elite_frac": 0.3, "alpha": 0.1,
                 "device": DEV, "return_mean_elites": True, "population_size_module": 7}


def cartpole_agent(env, H=10, P=20):
    import mbrl_lib_b200 as bp

    cfg = {"_target_": "mbrl.planning.TrajectoryOptimizerAgent", "action_lb": "???", "action_ub": "???", "planning_horizon": H,
           "optimizer_cfg": dict(ICEM_CARTPOLE), "replan_freq": 1, "verbose": False}
    return bp.create_trajectory_optim_agent_for_model(env, cfg, num_particles=P)


def test_agent_act_takes_the_fused_plan(monkeypatch):
    """agent.act with icem.yaml at pets_icem_cartpole's shapes never reaches evaluate_action_sequences, and its actions
    are the loop's."""
    spec, env = _cartpole_env()
    agent, ref = cartpole_agent(env), cartpole_agent(env)
    ref.set_trajectory_eval_fn(lambda o, seqs: env.evaluate_action_sequences(seqs, o, 20))  # opaque: the loop
    obs = syn.make_rollout_inputs(spec, with_noise=False)["obs0"]
    real = env.evaluate_action_sequences
    for step in range(3):
        rng, offset = torch.cuda.get_rng_state(), env._offset
        monkeypatch.setattr(env, "evaluate_action_sequences", lambda *a, **k: pytest.fail("the fused plan evaluated"))
        got = agent.act(obs)
        monkeypatch.setattr(env, "evaluate_action_sequences", real)
        assert env._offset == offset + 5
        torch.cuda.set_rng_state(rng)
        env._offset = offset
        want = ref.act(obs)
        assert np.array_equal(got, want), f"step {step}: {got} != {want}"
        assert torch.equal(agent.optimizer.optimizer.elite, ref.optimizer.optimizer.elite)


def test_plan_refusals():
    """Every refusal of b200pets_icem_plan happens before its first launch, with b200pets_last_error text; the optimiser
    raises the loop's ValueError for a fixed_model batch the members do not divide before any launch."""
    from mbrl_lib_b200 import _lib
    from mbrl_lib_b200.planning import _FusedObjective

    spec, _, env = make_env("halfcheetah_small", "f32", ts1="tile_shuffle")
    lib = _lib.load()
    H, A, P = 8, spec.act_dim, 5
    sizes = (C.c_int32 * 3)(100, 77, 60)
    t = lambda n: torch.zeros(n, device=DEV)  # noqa: E731
    obs0, x0, lb, ub, sol, elite = t(spec.obs_dim), t(H * A), t(H * A) - 1, t(H * A) + 1, t(H * A), t(10 * H * A)

    def rcfg(**over):
        r = _lib.RolloutCfg(0, H, P, _lib.PREC["f32"], _lib.PROP["random_model"], _lib.TS1_TILE_SHUFFLE, 1, 2, 0, 0)
        for k, v in over.items():
            setattr(r, k, v)
        return r

    def icfg(**over):
        c = _lib.IcemCfg(3, 10, 3, 0.1, 2.0, 1, 7, 1)
        for k, v in over.items():
            setattr(c, k, v)
        return c

    ws = torch.empty(lib.b200pets_icem_plan_workspace_bytes(env.staged.handle, C.byref(rcfg()), C.byref(icfg()), sizes),
                     dtype=torch.uint8, device=DEV)

    def plan(r=None, c=None, s=sizes, nbytes=None, **ptrs):
        p = dict(obs0=obs0, x0=x0, lb=lb, ub=ub, sol=sol, elite=elite, ws=ws)
        p.update(ptrs)
        return lib.b200pets_icem_plan(env.staged.handle, C.byref(r or rcfg()), C.byref(c or icfg()), s, _lib.ptr(p["obs0"]),
                                      _lib.ptr(p["x0"]), _lib.ptr(p["lb"]), _lib.ptr(p["ub"]), None, None, None, _lib.ptr(p["sol"]),
                                      _lib.ptr(p["elite"]), None, _lib.ptr(p["ws"]), ws.numel() if nbytes is None else nbytes,
                                      _lib.stream_ptr())

    def refused(rc, text, code=-1):
        assert rc == code, (rc, lib.b200pets_last_error().decode())
        assert text in lib.b200pets_last_error().decode()

    for name in ("obs0", "x0", "lb", "ub", "sol", "elite", "ws"):
        refused(plan(**{name: None}), "null argument")
    refused(plan(s=None), "null argument")
    refused(plan(c=icfg(num_iterations=0)), "num_iterations")
    refused(plan(r=rcfg(horizon=1)), "horizon of at least 2")
    refused(plan(c=icfg(keep=11)), "kept elites")
    # rows per iteration: 100, 77 + 3 kept elites, 60 + the mean
    refused(plan(c=icfg(elite_num=0, keep=0)), "elites of a smallest population of 61")
    refused(plan(c=icfg(elite_num=62)), "elites of a smallest population of 61")
    refused(plan(s=(C.c_int32 * 3)(100, 77, 0)), "population 0 of iteration 2")
    refused(plan(r=rcfg(particles=1)), "multiple of the number of models")  # 61 rows of the last iteration, 5 members
    refused(plan(r=rcfg(first_sequence=10)), "sharded", -2)
    refused(plan(r=rcfg(global_population=200)), "sharded", -2)
    refused(plan(nbytes=ws.numel() - 1), "workspace too small")
    torch.cuda.synchronize()

    # fixed_model: a batch the members do not divide raises before any launch, with the loop's message
    _, _, tsinf = make_env("hopper_tsinf", "f32", ts1="tile_shuffle")
    opt = _optimizer(syn.CASES["hopper_tsinf"], 9, 101, 2, None, 0.3, True)
    offset = tsinf._offset
    with pytest.raises(ValueError, match="multiple of the number of models"):
        opt.optimize(_FusedObjective(tsinf, syn.make_rollout_inputs(syn.CASES["hopper_tsinf"], with_noise=False)["obs0"], 1),
                     x0=torch.zeros(9, 3, device=DEV))
    assert tsinf._offset == offset
