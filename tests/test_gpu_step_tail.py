"""The tensor-core rollout loads a step's action words with independent loads (models with up to 8 actions) and no
longer waits at a warpgroup barrier before it does: every output below must stay bit for bit what the kernel computed
before that change.

Every output is compared with torch.equal against goldens that the kernel produced on an H100 before the change
(tests/golden/tail_*.npz), with in-kernel noise (no injected eps) and the in-kernel member draw:

* per-step ``b200pets_eval_trajectory`` outputs (next_obs, reward, done), as one window and split into windows that
  start with a one-step window (each window's first step loads the actions before the tile's first barrier, the
  others at the end of the previous step);
* expectation propagation;
* models with more actions than the registers take, which keep the word-by-word loads: humanoid_trunc (17 actions)
  and plan_in254 (243 actions), next to ant_learned_fn (8 actions, the bound);
* per-row returns of ``b200pets_eval_sequences`` on both CTA shapes: pop 500 x 20 (80 tiles: 64-row CTAs, two per SM)
  and pop 900 x 20 (160 tiles: 128-row CTAs, more tiles than CTAs, so a CTA moves on to a second tile), and the
  batched kernel with two problems (160 tiles);
* a trajectory on 128-row CTAs with more tiles than CTAs (pop 900 x 20, two one-step windows): compared through SHA-256
  digests of the outputs' bytes, which match exactly when the arrays are bit-identical (the arrays are too large to
  commit).

Regenerate (on an H100, with the library whose outputs are to be pinned):
    python tests/test_gpu_step_tail.py --write tests/golden
"""
import ctypes as C
import dataclasses
import hashlib
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from mbrl_lib_b200 import synthetic as syn  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
SEED = 0x5EED_0000_1234_ABCD
OFFSET = 29 * 1024

# name -> (case, overrides, window plans); each plan is compared with the same golden
TRAJ = {
    "tail_traj_halfcheetah": ("halfcheetah_small", dict(population=24, horizon=8), [[(0, 8)], [(0, 1), (1, 4), (4, 8)]]),
    "tail_traj_expectation": ("silu_expectation", {}, [[(0, 6)], [(0, 1), (1, 6)]]),
    "tail_traj_humanoid_trunc": ("humanoid_trunc", dict(population=12, horizon=4), [[(0, 4)], [(0, 1), (1, 4)]]),
    "tail_traj_ant": ("ant_learned_fn", dict(horizon=4), [[(0, 4)], [(0, 1), (1, 4)]]),
    "tail_traj_in254": ("plan_in254", {}, [[(0, 3)], [(0, 1), (1, 3)]]),
}
# per-row returns of the bench model (halfcheetah: 4 x 200 SiLU, 6 actions, 17 outputs) at both CTA shapes
ROWS = {"tail_rows_pop500": 500, "tail_rows_pop900": 900}
BATCH = "tail_batch_k2"  # two pop-500 problems in one launch
TRAJ_BIG = "tail_traj_pop900"  # 160 tiles, H 2 as two one-step windows: digests


def _env(name, **over):
    from test_gpu_parity import _Env

    import mbrl_lib_b200 as bp
    from mbrl_lib_b200 import functions

    spec = dataclasses.replace(syn.CASES[name], **over)
    arrays = syn.make_model_arrays(spec)
    model = bp.model_from_arrays(spec, arrays, DEV)
    rew = functions.REWARD_FNS[spec.reward_fn] if spec.reward_fn else None
    env = bp.ModelEnv(_Env(spec), model, functions.TERM_FNS[spec.term_fn], rew, generator=torch.Generator(device=DEV),
                      precision="bf16_tc", ts1="tile_shuffle")
    assert env.staged.supports_tc(spec.propagation), name
    env._few_groups = lambda *a: False  # the in-kernel member draw at every population
    env._seed = SEED
    return spec, env


def _cfg(spec):
    from mbrl_lib_b200 import _lib

    prop = spec.propagation
    return _lib.RolloutCfg(spec.population, spec.horizon, spec.particles, _lib.PREC["bf16_tc"], _lib.PROP[prop],
                           _lib.TS1_TILE_SHUFFLE, SEED, OFFSET, 0, 0)


def _inputs(spec):
    inp = syn.make_rollout_inputs(spec, with_noise=False)
    acts = torch.from_numpy(inp["actions"]).to(DEV)
    obs0 = torch.from_numpy(np.asarray(inp["obs0"], np.float32)).to(DEV)
    return acts, obs0


def trajectory(spec, env, windows):
    """b200pets_eval_trajectory over the windows: next_obs [H, B, D], reward [H, B], done [H, B] (on the device)."""
    from mbrl_lib_b200 import _lib

    lib, h = env.lib, env.staged.handle
    H, B, D = spec.horizon, spec.population * spec.particles, spec.obs_dim
    cfg = _cfg(spec)
    acts, obs0 = _inputs(spec)
    ws = torch.empty(lib.b200pets_trajectory_workspace_bytes(h, C.byref(cfg)), dtype=torch.uint8, device=DEV)
    nobs = torch.full((H, B, D), float("nan"), device=DEV)
    rew = torch.full((H, B), float("nan"), device=DEV)
    done = torch.full((H, B), 7, dtype=torch.uint8, device=DEV)
    for t0, t1 in windows:
        _lib.check(lib.b200pets_eval_trajectory(h, C.byref(cfg), t0, t1, _lib.ptr(obs0), _lib.ptr(acts), None, None,
                                                _lib.ptr(nobs[t0]), _lib.ptr(rew[t0]), _lib.ptr(done[t0]), _lib.ptr(ws),
                                                ws.numel(), _lib.stream_ptr()), "eval_trajectory")
    torch.cuda.synchronize()
    return {"next_obs": nobs, "reward": rew, "done": done}


def row_returns(spec, env):
    from mbrl_lib_b200 import _lib

    lib, h = env.lib, env.staged.handle
    cfg = _cfg(spec)
    acts, obs0 = _inputs(spec)
    ws = torch.empty(lib.b200pets_eval_workspace_bytes(h, C.byref(cfg)), dtype=torch.uint8, device=DEV)
    ret = torch.empty(spec.population, device=DEV)
    rows = torch.empty(spec.population * spec.particles, device=DEV)
    _lib.check(lib.b200pets_eval_sequences(h, C.byref(cfg), _lib.ptr(obs0), _lib.ptr(acts), None, None, _lib.ptr(ret),
                                           _lib.ptr(rows), _lib.ptr(ws), ws.numel(), _lib.stream_ptr()), "eval_sequences")
    torch.cuda.synchronize()
    return {"returns": ret, "rows": rows}


def batch_returns(spec, env, K=2):
    acts, _ = _inputs(spec)
    obs0 = np.stack([np.asarray(syn.make_rollout_inputs(spec, with_noise=False)["obs0"], np.float32) + 0.01 * k
                     for k in range(K)])
    acts = torch.stack([acts, acts.flip(0)])
    ret = env.evaluate_action_sequences_batch(acts, obs0, spec.particles, _offset=OFFSET)
    torch.cuda.synchronize()
    return {"returns": ret}


def _digest(t):
    return np.frombuffer(hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).digest(), np.uint8)


def outputs():
    """golden name -> one {array name: tensor or digest} per window plan (each must equal the golden)."""
    out = {}
    for key, (name, over, plans) in TRAJ.items():
        spec, env = _env(name, **over)
        out[key] = [trajectory(spec, env, w) for w in plans]
    for key, pop in ROWS.items():
        spec, env = _env("halfcheetah", population=pop)
        out[key] = [row_returns(spec, env)]
    spec, env = _env("halfcheetah", population=500)
    out[BATCH] = [batch_returns(spec, env)]
    spec, env = _env("halfcheetah", population=900, horizon=2)
    big = trajectory(spec, env, [(0, 1), (1, 2)])
    out[TRAJ_BIG] = [{k + "_sha256": _digest(v) for k, v in big.items()}]
    return out


def _tiles_and_shape():
    """(128-row tiles, consumer warpgroups per CTA) of the pop-500 and pop-900 launches, from the launch plan rules."""
    from test_gpu_tiles import _sm_count

    sm = _sm_count()
    return {p: (20 * -(-p // 128), 1 if 20 * -(-p // 128) < sm else 2) for p in (500, 900)}, sm


@pytest.fixture(scope="module")
def results():
    return outputs()


@pytest.mark.parametrize("key", list(TRAJ) + list(ROWS) + [BATCH, TRAJ_BIG])
def test_bit_identical_to_golden(results, golden_dir, key):
    gold = np.load(os.path.join(golden_dir, key + ".npz"))
    for i, got in enumerate(results[key]):
        for k, v in got.items():
            ref = torch.from_numpy(np.array(gold[k]))
            cur = v.cpu() if torch.is_tensor(v) else torch.from_numpy(np.array(v))
            assert cur.shape == ref.shape and cur.dtype == ref.dtype, (key, i, k, cur.shape, ref.shape)
            if not torch.equal(cur, ref):
                diff = (cur != ref) & ~(torch.isnan(cur) & torch.isnan(ref)) if cur.is_floating_point() else cur != ref
                pytest.fail(f"{key} plan {i} {k}: {int(diff.sum())} of {diff.numel()} elements differ")


def test_launch_shapes_are_covered():
    """pop 500 runs 64-row CTAs (fewer tiles than SMs), pop 900 128-row CTAs with more tiles than CTAs."""
    shapes, sm = _tiles_and_shape()
    assert shapes[500][1] == 1 and shapes[900][1] == 2 and shapes[900][0] > sm, (shapes, sm)


if __name__ == "__main__":
    if len(sys.argv) < 3 or sys.argv[1] != "--write":
        sys.exit(__doc__)
    dest = sys.argv[2]
    for key, res in outputs().items():
        first = {k: (v.cpu().numpy() if torch.is_tensor(v) else v) for k, v in res[0].items()}
        for i, other in enumerate(res[1:], 1):  # every window plan gives the same outputs
            for k, v in other.items():
                assert torch.equal(v.cpu(), torch.from_numpy(first[k])), (key, i, k)
        np.savez_compressed(os.path.join(dest, key + ".npz"), **first)
        print(key, {k: v.shape for k, v in first.items()})
