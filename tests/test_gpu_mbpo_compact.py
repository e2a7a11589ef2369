"""The MBPO device bookkeeping (b200pets_mbpo_mask, b200pets_mbpo_compact: mask, per-block count, scan, scatter) against
a numpy restatement of rollout_model_and_populate_sac_buffer's masking (mbrl/algorithms/mbpo.py:51-62) at the batch
sizes MBPO runs: B = 400 x 250 = 100 000 rows (98 blocks of 1 024 per step, the last one partial) and up to 25 steps
(2 450 blocks, so that the scan makes three passes and carries between them).  Everything is compared bit for bit."""
import numpy as np
import pytest
import torch

from mbrl_lib_b200 import synthetic as syn
from test_gpu_parity import DEV, make_env

pytestmark = pytest.mark.gpu

SENTINEL = np.float32(-31337.0)
DONE_SENTINEL = 0xAB


def _reference(done, accum0):
    """alive[i] = ~accum; accum |= done[i]   (the mask is taken before it absorbs step i's dones)."""
    accum = accum0.astype(bool).copy()
    alive = np.empty(done.shape, bool)
    for i in range(done.shape[0]):
        alive[i] = ~accum
        accum |= done[i].astype(bool)
    return alive, accum


def _run(k, B, D, A, done, accum0, g):
    from mbrl_lib_b200 import _lib

    lib = _lib.load()
    obs0 = g.standard_normal((B, D), dtype=np.float32)
    act = g.standard_normal((k, B, A), dtype=np.float32)
    nxt = g.standard_normal((k, B, D), dtype=np.float32)
    rew = g.standard_normal((k, B), dtype=np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)  # noqa: E731
    obs0_d, act_d, nxt_d, rew_d, done_d = t(obs0), t(act), t(nxt), t(rew), t(done)
    accum_d = t(accum0)
    alive_d = torch.full((k, B), 0x5A, dtype=torch.uint8, device=DEV)
    stream = _lib.stream_ptr()
    for i in range(k):
        _lib.check(lib.b200pets_mbpo_mask(B, _lib.ptr(done_d[i]), _lib.ptr(accum_d), _lib.ptr(alive_d[i]), stream), "mbpo_mask")
    o_out = torch.full((k * B, D), float(SENTINEL), device=DEV)
    a_out = torch.full((k * B, A), float(SENTINEL), device=DEV)
    n_out = torch.full((k * B, D), float(SENTINEL), device=DEV)
    r_out = torch.full((k * B,), float(SENTINEL), device=DEV)
    d_out = torch.full((k * B,), DONE_SENTINEL, dtype=torch.uint8, device=DEV)
    counts = torch.full((k + 1,), -1, dtype=torch.int64, device=DEV)
    need = lib.b200pets_mbpo_compact_workspace_bytes(k, B)
    ws = torch.full((need,), 0xFF, dtype=torch.uint8, device=DEV)  # stale workspace contents must not matter
    _lib.check(lib.b200pets_mbpo_compact(k, B, D, A, _lib.ptr(obs0_d), _lib.ptr(act_d), _lib.ptr(nxt_d), _lib.ptr(rew_d),
                                         _lib.ptr(done_d), _lib.ptr(alive_d), _lib.ptr(o_out), _lib.ptr(a_out), _lib.ptr(n_out),
                                         _lib.ptr(r_out), _lib.ptr(d_out), _lib.ptr(counts), _lib.ptr(ws), need, stream),
               "mbpo_compact")
    got = {name: x.cpu().numpy() for name, x in (("alive", alive_d), ("accum", accum_d), ("obs", o_out), ("act", a_out),
                                                 ("next", n_out), ("rew", r_out), ("done", d_out), ("counts", counts))}
    return (obs0, act, nxt, rew), got


def _bits(x):
    return np.ascontiguousarray(x).view(np.uint32 if x.dtype == np.float32 else np.uint8)


def _check(k, B, D, A, done, accum0, seed):
    g = np.random.default_rng(seed)
    (obs0, act, nxt, rew), got = _run(k, B, D, A, done, accum0, g)
    alive, accum = _reference(done, accum0)
    assert np.array_equal(got["alive"], alive.astype(np.uint8))
    assert np.array_equal(got["accum"], accum.astype(np.uint8))
    per_step = alive.sum(axis=1)
    total = int(per_step.sum())
    assert np.array_equal(got["counts"], np.append(per_step, total)), (got["counts"][:8], per_step[:8], total)
    # the rows of the reference's k add_batch calls, in (step, row) order
    obs_src = np.concatenate([obs0[None], nxt[:-1]], axis=0)
    m = alive
    want = {"obs": obs_src[m], "act": act[m], "next": nxt[m], "rew": rew[m], "done": done[m]}
    for name, w in want.items():
        assert np.array_equal(_bits(got[name][:total]), _bits(w)), f"packed {name} differs"
        past = got[name][total:]
        assert (past == (DONE_SENTINEL if name == "done" else SENTINEL)).all(), f"{name} written past the total"
    return total, per_step


SHAPES = [(1, 1, 1, 1), (3, 1023, 11, 3), (2, 1025, 17, 6), (4, 4096, 376, 17), (1, 100_000, 17, 6), (15, 100_000, 11, 3),
          (25, 100_000, 27, 8)]


@pytest.mark.parametrize("p", [0.0, 0.05, 1.0])
@pytest.mark.parametrize("k,B,D,A", SHAPES)
def test_mbpo_mask_and_compact_match_numpy(k, B, D, A, p):
    g = np.random.default_rng(k * 1000 + B + int(p * 100))
    done = (g.random((k, B)) < p).astype(np.uint8)
    total, per_step = _check(k, B, D, A, done, np.zeros(B, np.uint8), seed=B + k)
    if p == 0.0:
        assert total == k * B  # no row ever dies
    if p == 1.0:
        assert total == B and (per_step[1:] == 0).all()  # every row dies at step 0: only step 0's rows are kept
    if p == 0.05 and k > 1 and B > 1:
        assert 0 < per_step[-1] < per_step[0] == B  # some rows died, some survive


@pytest.mark.parametrize("k,B,D,A", [(3, 1023, 11, 3), (25, 100_000, 27, 8)])
def test_mbpo_compact_all_rows_dead_from_step_zero(k, B, D, A):
    g = np.random.default_rng(1)
    done = (g.random((k, B)) < 0.5).astype(np.uint8)
    total, _ = _check(k, B, D, A, done, np.ones(B, np.uint8), seed=2)
    assert total == 0


@pytest.mark.parametrize("precision", ["f32", "bf16_tc"])
def test_mbpo_device_rollout_loop_at_mbpo_scale(precision):
    """rollout_on_device with mbpo_hopper_small at B 100 000 and k 15 (hopper's longest rollout), in-kernel model noise
    with the tile shuffle, hopper termination: the packed transitions are exactly the `~accum_dones` rows of the device's
    own per-step arrays, in (step, row) order."""
    from mbrl_lib_b200 import mbpo

    spec, arrays, env = make_env("mbpo_hopper_small", precision, ts1="tile_shuffle")
    B, k = 100_000, 15
    inp = syn.make_step_inputs(spec, B)
    inp["obs"][:, 1:] *= 0.1  # most rows start inside hopper's alive region
    g = np.random.default_rng(15)
    Wd = torch.from_numpy((0.3 * g.standard_normal((spec.obs_dim, spec.act_dim))).astype(np.float32)).to(DEV)

    class _Agent:
        def act_torch(self, obs, sample):
            return torch.tanh(obs @ Wd)

    staging = {}
    obs_p, act_p, nxt_p, rew_p, done_p, counts = mbpo.rollout_on_device(env, inp["obs"], _Agent(), True, k, _staging=staging)
    st = {kk: v.cpu().numpy() for kk, v in staging.items()}
    alive, _ = _reference(st["done"], np.zeros(B, np.uint8))
    assert np.array_equal(st["alive"], alive.astype(np.uint8))
    assert 0 < alive[-1].sum() < B  # rows die along the rollout, some survive
    lo = 0
    for i in range(k):
        keep = alive[i]
        n = int(keep.sum())
        assert counts[i] == n
        src_obs = st["obs0"] if i == 0 else st["next_obs"][i - 1]
        assert np.array_equal(_bits(obs_p[lo:lo + n]), _bits(src_obs[keep]))
        assert np.array_equal(_bits(act_p[lo:lo + n]), _bits(st["act"][i][keep]))
        assert np.array_equal(_bits(nxt_p[lo:lo + n]), _bits(st["next_obs"][i][keep]))
        assert np.array_equal(_bits(rew_p[lo:lo + n]), _bits(st["reward"][i][keep]))
        assert np.array_equal(done_p[lo:lo + n], st["done"][i][keep])
        lo += n
    assert lo == len(obs_p)
