"""Launches with many more 128-row tiles than SMs, against the oracle.

The tensor-core kernel is persistent: one CTA per SM walks tiles blockIdx.x, blockIdx.x + gridDim.x, ...  Its weight
ring position carries from one tile to the next, its producer warp runs ahead into the next tile, and each tile
resets the row state (return, dead flag, observation).  The parity cases elsewhere have at most one tile per CTA;
here every launch has more than twice as many tiles as the device has SMs, in each row mapping: TS1 with injected
permutations (one launch per step), TSinf with an injected permutation (one launch over every step), expectation, and
tile shuffle with the exported member map.  The hopper model's termination ends rows part-way, so a dead flag that
leaked from one tile into the next would change returns.  The fp32 kernel runs the same inputs at its bar.
"""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

from mbrl_lib_b200 import synthetic as syn
from test_gpu_parity import DEV, _Env, assert_close_continuous, assert_close_discrete, gpu_returns
from test_gpu_shuffle import _eval_shuffle, _oracle

pytestmark = pytest.mark.gpu

TILE = 128


def _sm_count():
    from mbrl_lib_b200 import _lib

    sm = C.c_int32()
    _lib.check(_lib.load().b200pets_device_info(C.byref(sm), None, None))
    return sm.value


def _env(spec, arrays, precision, ts1):
    import mbrl_lib_b200 as bp
    from mbrl_lib_b200 import functions

    model = bp.model_from_arrays(spec, arrays, DEV)
    rew = functions.REWARD_FNS[spec.reward_fn] if spec.reward_fn else None
    env = bp.ModelEnv(_Env(spec), model, functions.TERM_FNS[spec.term_fn], rew, generator=torch.Generator(device=DEV),
                      precision=precision, ts1=ts1)
    env._few_groups = lambda *a: False
    return env


def _tc_tiles(spec, mode):
    """Tiles of one tensor-core launch (rollout_tc.cu launch_rollout_tc)."""
    N, P, M = spec.population, spec.particles, spec.num_models
    B = N * P
    if mode == "expectation":
        return -(-B // TILE)
    if mode == "tile_shuffle":
        return P * -(-N // TILE)
    return M * -(-(B // M) // TILE)


def _check(spec, got, ref, precision, discrete):
    if precision == "f32":
        if discrete:
            assert_close_discrete(got, ref, spec.particles)
        else:
            assert_close_continuous(got, ref, 2e-4)
    elif discrete:  # the bars of test_rollout_tc_discrete_rewards against the bf16-operand oracle
        d = np.abs(got - ref)
        assert np.isfinite(got).all()
        assert (d > 1e-2 * np.maximum(1.0, np.abs(ref))).mean() <= 0.01, f"{(d > 1e-2).sum()} of {d.size} differ"
        assert d.mean() <= 1e-4 * max(1.0, float(np.abs(ref).mean())), d.mean()
    else:
        assert_close_continuous(got, ref, 5e-3)


# hopper model (termination), 6 401 sequences x 6 particles: B / M = 19 203 and N are not multiples of 128
HOPPER = dict(population=6401, horizon=9, particles=6)


@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
@pytest.mark.parametrize("mode", ["ts1_perms", "tsinf_perm", "expectation", "tile_shuffle"])
def test_multi_tile_launch_matches_oracle(mode, precision):
    base = syn.CASES["hopper_tsinf"]
    prop = {"ts1_perms": "random_model", "tsinf_perm": "fixed_model", "expectation": "expectation",
            "tile_shuffle": "random_model"}[mode]
    spec = dataclasses.replace(base, propagation=prop, **HOPPER)
    arrays = syn.make_model_arrays(base)
    tiles = _tc_tiles(spec, mode)
    assert tiles > 2 * _sm_count(), tiles
    inp = syn.make_rollout_inputs(spec)
    oracle = _oracle(spec, arrays, precision == "bf16_tc")
    args = (torch.from_numpy(inp["actions"]), inp["obs0"], spec.particles)
    if mode == "tile_shuffle":
        env = _env(spec, arrays, precision, "tile_shuffle")
        offset = 17 * 1024
        got = _eval_shuffle(env, spec, inp, offset)
        assign = env.shuffle_member_assignment(spec.population, spec.horizon, spec.particles, offset)
        ref = oracle.evaluate_action_sequences(*args, None, torch.from_numpy(inp["eps"]), assign=assign).numpy()
    else:
        env = _env(spec, arrays, precision, "perms")
        got = gpu_returns(env, spec, inp)
        ref = oracle.evaluate_action_sequences(*args, torch.from_numpy(inp["perms"]), torch.from_numpy(inp["eps"])).numpy()
    _check(spec, got, ref, precision, discrete=True)


@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
def test_multi_tile_halfcheetah_matches_oracle(precision):
    """The headline model (5 members x 4 x 200 SiLU) with 2 000 sequences x 20 particles: 315 tiles of 128 rows."""
    spec = dataclasses.replace(syn.CASES["halfcheetah"], population=2000, horizon=8)
    arrays = syn.make_model_arrays(spec)
    assert _tc_tiles(spec, "ts1_perms") > 2 * _sm_count()
    inp = syn.make_rollout_inputs(spec)
    got = gpu_returns(_env(spec, arrays, precision, "perms"), spec, inp)
    ref = _oracle(spec, arrays, precision == "bf16_tc").evaluate_action_sequences(
        torch.from_numpy(inp["actions"]), inp["obs0"], spec.particles, torch.from_numpy(inp["perms"]),
        torch.from_numpy(inp["eps"])).numpy()
    _check(spec, got, ref, precision, discrete=False)


def test_bench_scale_tile_shuffle_equals_shard_launches():
    """The benched regime (pop 16 077 x H 30 x 20 particles, tile shuffle, in-kernel noise: 2 520 tiles on the SMs)
    against the same rows evaluated as shards of 499 sequences (boundaries not aligned to 128, at most 100 tiles per
    launch, one per CTA -- the regime the oracle comparisons pin): bit for bit, because every draw is keyed by global
    indices."""
    spec = syn.CASES["halfcheetah"]
    arrays = syn.make_model_arrays(spec)
    env = _env(spec, arrays, "bf16_tc", "tile_shuffle")
    N, H, P = 16077, 30, spec.particles
    sms = _sm_count()
    assert P * -(-N // TILE) > 2 * sms
    g = np.random.default_rng(16077)
    acts = torch.from_numpy(g.uniform(-1, 1, (N, H, spec.act_dim)).astype(np.float32)).to(DEV)
    obs0 = syn.make_rollout_inputs(spec, with_noise=False)["obs0"]
    offset = 19 * 1024

    def run(lo, hi):
        rr = torch.empty((hi - lo) * P, device=DEV)
        env.evaluate_action_sequences(acts[lo:hi], obs0, P, _row_returns=rr, _offset=offset, _shard=(lo, N))
        return rr

    full = run(0, N).cpu().numpy()
    bounds = list(range(0, N, 499)) + [N]
    parts = []
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        c_loc = (hi - 1) // TILE - lo // TILE + 1
        assert P * c_loc <= min(100, sms)
        parts.append(run(lo, hi))
    torch.cuda.synchronize()
    sharded = torch.cat(parts).cpu().numpy()
    assert np.isfinite(full).all()
    assert np.array_equal(sharded, full), f"{(sharded != full).sum()} of {full.size} rows differ"
