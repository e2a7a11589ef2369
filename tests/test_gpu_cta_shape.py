"""The tensor-core rollout's two CTA shapes.

A launch with fewer 128-row tiles than the device has SMs runs 64-row CTAs (one consumer warpgroup), two per SM, when
its plan fits twice in an SM's shared memory: CTA tile u is half u % 2 of 128-row tile u / 2, so a shuffle group, a
member's slot range or an expectation chunk is split over two CTAs that each walk the weights on their own.  Other
launches run 128-row CTAs, one per SM.  A row's member, keys, operands and K order are the same in both shapes, so
results do not depend on the shape.  Here: halves with no valid row at shard edges (bit for bit against the unsharded
evaluation), a launch of one 128-row tile, and the 128-row CTA with more tiles than SMs.  Small launches of models whose plan fits only once per SM
(plan_ring2, plan_k1_out256) run in the tile-shuffle and parity tests.
"""
import dataclasses

import numpy as np
import pytest
import torch

from mbrl_lib_b200 import synthetic as syn
from test_gpu_parity import DEV, assert_close_continuous, gpu_returns, make_env
from test_gpu_shuffle import _eval_shuffle, _oracle
from test_gpu_tiles import _env, _sm_count, _tc_tiles

pytestmark = pytest.mark.gpu


def test_half_tiles_at_shard_edges_equal_unsharded():
    """Shards whose edges leave one 64-row half of a 128-row shuffle group without a valid row (first half, second
    half, or the whole second half of a group with two valid rows) equal the unsharded evaluation bit for bit."""
    spec, _, env = make_env("halfcheetah", "bf16_tc", ts1="tile_shuffle")
    inp = syn.make_rollout_inputs(spec, with_noise=False)
    N, P = spec.population, spec.particles
    assert _tc_tiles(spec, "tile_shuffle") < _sm_count()  # 64-row CTAs, also for every shard
    offset = 13 * 1024

    def run(lo, hi):
        acts = torch.from_numpy(inp["actions"][lo:hi]).to(DEV)
        rr = torch.empty((hi - lo) * P, device=DEV)
        env.evaluate_action_sequences(acts, inp["obs0"], P, _row_returns=rr, _offset=offset, _shard=(lo, N))
        torch.cuda.synchronize()
        return rr.cpu().numpy()

    full = run(0, N)
    bounds = [0, 64, 130, 192, 500]  # [0, 64): group 0's second half empty; [64, 130): group 0's first, group 1's second
    parts = [run(lo, hi) for lo, hi in zip(bounds[:-1], bounds[1:])]
    sharded = np.concatenate(parts)
    assert np.isfinite(full).all()
    assert np.array_equal(sharded, full), f"{(sharded != full).sum()} of {full.size} rows differ"


def test_single_tile_launch_matches_oracle():
    """One 128-row tile (100 sequences x 1 particle, tile shuffle): two CTAs, the second with 36 valid rows."""
    spec, arrays, env = make_env("halfcheetah", "bf16_tc", ts1="tile_shuffle")
    env._few_groups = lambda *a: False
    spec = dataclasses.replace(spec, population=100, particles=1, horizon=10)
    assert _tc_tiles(spec, "tile_shuffle") == 1
    inp = syn.make_rollout_inputs(spec)
    offset = 23 * 1024
    got = _eval_shuffle(env, spec, inp, offset)
    assign = env.shuffle_member_assignment(spec.population, spec.horizon, spec.particles, offset)
    ref = _oracle(spec, arrays, True).evaluate_action_sequences(
        torch.from_numpy(inp["actions"]), inp["obs0"], spec.particles, None, torch.from_numpy(inp["eps"]),
        assign=assign).numpy()
    assert_close_continuous(got, ref, 5e-3)


def test_one_per_sm_multi_tile_launch_matches_oracle():
    """The 128-row CTA with more tiles than the device has SMs."""
    base = syn.CASES["plan_ring2"]
    spec = dataclasses.replace(base, population=8000)
    arrays = syn.make_model_arrays(base)
    env = _env(spec, arrays, "bf16_tc", "perms")
    assert _tc_tiles(spec, "ts1_perms") > _sm_count()
    inp = syn.make_rollout_inputs(spec)
    got = gpu_returns(env, spec, inp)
    ref = _oracle(spec, arrays, True).evaluate_action_sequences(
        torch.from_numpy(inp["actions"]), inp["obs0"], spec.particles, torch.from_numpy(inp["perms"]),
        torch.from_numpy(inp["eps"])).numpy()
    assert_close_continuous(got, ref, 5e-3)
