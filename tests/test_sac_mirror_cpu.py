"""CPU checks of the host side of training MBPO's SAC agent from a device-resident rollout buffer
(mbrl_lib_b200/replay.py DeviceTransitionMirror, sac.py, mbpo.py):

* ``mbpo.update_agent`` draws each update's indices as ``ReplayBuffer.sample`` draws them and leaves every generator
  (the loop's ``rng`` and both buffers') where the reference's loop (mbpo.py:258-275) leaves it;
* its ``rng.random()`` / break sequence, the buffer each update reads, and its logger calls and dumps equal a restated
  reference loop over a recording logger, for ``real_data_ratio`` 0, 0.5 and 1, a buffer shorter than the batch and a
  step that is not an update step;
* ``mbpo.scatter_positions`` puts each rollout row where the per-step ``add_batch`` calls put it, across the ring's wrap
  and when one rollout writes more rows than the capacity;
* what is refused and what falls back to the host: unmirrored buffers, a mirror on another device, dtypes the mirror
  does not store, a capacity over ``max_bytes``, and the C entry points' argument checks (before touching a device).
"""
import ctypes as C
import importlib
import types

import numpy as np
import pytest
import torch

from baseline import reference_arm as ra
from mbrl_lib_b200 import _lib, mbpo, replay, sac as bsac

mbrl, REF_SRC = ra.import_reference()
needs_ref = pytest.mark.skipif(mbrl is None, reason=f"reference not importable here: {REF_SRC}")
D, A = 3, 2


def _rb():
    return importlib.import_module("mbrl.util.replay_buffer")


def _buffer(capacity, rows, seed, rng=None):
    """A reference ReplayBuffer whose obs[:, 0] holds each row's number, so a batch names its rows."""
    buf = _rb().ReplayBuffer(capacity, (D,), (A,), rng=rng if rng is not None else np.random.default_rng(seed))
    if rows:
        g = np.random.default_rng(seed + 100)
        obs = g.standard_normal((rows, D)).astype(np.float32)
        obs[:, 0] = np.arange(rows)
        buf.add_batch(obs, g.standard_normal((rows, A)), g.standard_normal((rows, D)), g.standard_normal(rows),
                      g.random(rows) < 0.2, np.zeros(rows, bool))
    return buf


class Log:
    def __init__(self):
        self.calls = []

    def log(self, key, value, step):
        self.calls.append(("log", key, value, step))

    def dump(self, step, save=False):
        self.calls.append(("dump", step, save))


def _stats(memory, rows, updates):
    """Statistics that name the update's buffer, rows and counter, as float32 as the kernel writes them."""
    return np.array([rows.sum(), rows[0], rows[-1], len(memory), updates, updates * 0.5, -rows.mean(), 0], np.float32)


class FakeSAC:
    """mbrl_lib_b200.SAC's host interface with the launch replaced by _stats: ``update_parameters`` samples as the
    reference's does; ``update_many`` takes the rows update_agent drew."""

    log_stats = bsac.SAC.log_stats

    def __init__(self, tuning):
        self.automatic_entropy_tuning = tuning
        self.target_entropy = -float(A)
        self.many_calls = 0

    def update_parameters(self, memory, batch_size, updates, logger=None, reverse_mask=False):
        assert reverse_mask
        rows = memory.sample(batch_size).obs[:, 0].astype(np.int64)
        return self.log_stats(_stats(memory, rows, updates).tolist(), updates, logger)

    def update_many(self, batches, batch_size, first_update, reverse_mask=False):
        assert reverse_mask
        self.many_calls += 1
        return np.stack([_stats(m, m.obs[idx, 0].astype(np.int64), first_update + i) for i, (m, idx) in enumerate(batches)])


def _reference_loop(agent, replay_buffer, sac_buffer, rng, num_updates, ratio, batch_size, update_step, updates_made,
                    logger, log_frequency):
    """mbrl/algorithms/mbpo.py:258-275 as written there (not silent)."""
    for _ in range(num_updates):
        use_real_data = rng.random() < ratio
        which_buffer = replay_buffer if use_real_data else sac_buffer
        if not update_step or len(which_buffer) < batch_size:
            break
        agent.sac_agent.update_parameters(which_buffer, batch_size, updates_made, logger, reverse_mask=True)
        updates_made += 1
        if updates_made % log_frequency == 0:
            logger.dump(updates_made, save=True)
    return updates_made


def _setup(ratio_case, shared_rng):
    """(loop rng, replay_buffer, sac_buffer) for one side; the replay buffer shares the loop's generator as mbpo.train
    builds it when shared_rng."""
    rng = np.random.default_rng(11)
    real = _buffer(300, 200, seed=1, rng=rng if shared_rng else None)
    rows = {"short": 40}.get(ratio_case, 500)
    return rng, real, _buffer(1000, rows, seed=2)


def _state(*gens):
    return [g.bit_generator.state for g in gens]


@needs_ref
@pytest.mark.parametrize("shared_rng", [True, False])
@pytest.mark.parametrize("case,ratio,update_step", [("sac", 0.0, True), ("mixed", 0.5, True), ("real", 1.0, True),
                                                    ("short", 0.0, True), ("short", 0.5, True),
                                                    ("not_an_update_step", 0.5, False)])
def test_update_agent_restates_the_reference_loop(case, ratio, update_step, shared_rng):
    B, n, freq = 64, 20, 7
    out = {}
    for side in ("reference", "ours"):
        rng, real, sac_buf = _setup(case, shared_rng)
        agent = types.SimpleNamespace(sac_agent=FakeSAC(tuning=ratio != 1.0))
        log = Log()
        made = 13  # updates made before this step: the dumps fall where they would mid-run
        for _ in range(3):  # three environment steps back to back
            if side == "reference":
                made = _reference_loop(agent, real, sac_buf, rng, n, ratio, B, update_step, made, log, freq)
            else:
                made = mbpo.update_agent(agent, real, sac_buf, rng, n, ratio, B, update_step, made, logger=log,
                                         log_frequency=freq)
        out[side] = (made, log.calls, _state(rng, real._rng, sac_buf._rng), agent.sac_agent)
    ref, ours = out["reference"], out["ours"]
    assert ours[0] == ref[0]
    assert ours[1] == ref[1]
    assert ours[2] == ref[2]
    updates = ref[0] - 13
    if case == "not_an_update_step" or (case == "short" and ratio == 0.0):
        assert updates == 0 and ours[3].many_calls == 0
    else:
        assert updates > 0 and ours[3].many_calls <= 3
    if case == "mixed":  # both buffers were read: stats[3], logged as the alpha loss, is the buffer's length
        assert {c[2] for c in ours[1] if c[0] == "log" and c[1] == "train_alpha/loss"} == {200.0, 500.0}


@needs_ref
def test_indices_and_generator_equal_replay_buffer_sample():
    B = 256
    buf, twin = _buffer(1000, 700, seed=5), _buffer(1000, 700, seed=5)
    seen = []

    class Recorder(FakeSAC):
        def update_many(self, batches, batch_size, first_update, reverse_mask=False):
            seen.extend(idx for _, idx in batches)
            return super().update_many(batches, batch_size, first_update, reverse_mask)

    agent = types.SimpleNamespace(sac_agent=Recorder(True))
    mbpo.update_agent(agent, buf, buf, np.random.default_rng(0), 5, 0.0, B, True, 0)
    assert len(seen) == 5
    for idx in seen:
        want = twin.sample(B)
        np.testing.assert_array_equal(buf.obs[idx], want.obs)
        np.testing.assert_array_equal(buf.action[idx], want.act)
        np.testing.assert_array_equal(buf.terminated[idx], want.terminateds)
    assert _state(buf._rng) == _state(twin._rng)


@needs_ref
def test_pack_rows_equals_update_parameters_staging():
    """replay.pack_rows (the mirror's flush and the host half of update_many) packs as SAC.update_parameters does,
    float64 buffers included."""
    buf = _rb().ReplayBuffer(100, (D,), (A,), obs_type=np.float64, action_type=np.float64, reward_type=np.float64)
    g = np.random.default_rng(3)
    buf.add_batch(g.standard_normal((90, D)), g.standard_normal((90, A)), g.standard_normal((90, D)),
                  g.standard_normal(90), g.random(90) < 0.5, np.zeros(90, bool))
    idx = g.integers(0, 90, 37)
    b = buf._batch_from_indices(idx)
    want = np.empty((37, 2 * D + A + 2), np.float32)
    want[:, :D], want[:, D:D + A], want[:, D + A:2 * D + A] = b.obs, b.act, b.next_obs
    want[:, 2 * D + A], want[:, 2 * D + A + 1] = b.rewards, b.terminateds
    got = np.full_like(want, np.nan)
    replay.pack_rows(buf, idx, got, D, A)
    np.testing.assert_array_equal(got, want)
    assert np.array_equal(got[:, :D], torch.FloatTensor(b.obs).numpy())  # rounded as torch rounds


@needs_ref
@pytest.mark.parametrize("capacity,start,counts", [(50, 0, [10, 20, 5]), (50, 44, [3, 9, 0, 12]), (50, 49, [50]),
                                                   (50, 17, [30, 30, 30]), (50, 0, [50, 50, 7]), (7, 3, [0, 0])])
def test_scatter_positions_equal_add_batch(capacity, start, counts):
    buf = _rb().ReplayBuffer(capacity, (D,), (A,))
    if start:  # move cur_idx to start through add_batch, as a run would
        buf.add_batch(*(np.full((start, *s), -1.0) for s in ((D,), (A,), (D,), ())), np.zeros(start, bool),
                      np.zeros(start, bool))
    cur = buf.cur_idx
    total = sum(counts)
    ids = np.arange(total, dtype=np.float32)
    lo = 0
    for n in counts:
        obs = np.repeat(ids[lo:lo + n, None], D, 1)
        buf.add_batch(obs, np.zeros((n, A)), obs, ids[lo:lo + n], np.zeros(n, bool), np.zeros(n, bool))
        lo += n
    skip, first = mbpo.scatter_positions(cur, capacity, counts)
    assert skip == max(0, total - capacity)
    pos = (first + np.arange(total - skip)) % capacity
    assert len(np.unique(pos)) == len(pos)  # no two scattered rows share a position
    np.testing.assert_array_equal(buf.obs[pos, 0], ids[skip:])
    np.testing.assert_array_equal(buf.reward[pos], ids[skip:])


# ---- refusals and fall-backs ------------------------------------------------------------------------------------------

@needs_ref
@pytest.mark.parametrize("dtype", [np.float16, np.uint8, np.int32])
def test_mirror_refuses_unsupported_dtypes(dtype):
    buf = _rb().ReplayBuffer(10, (D,), (A,), obs_type=dtype)
    with pytest.raises(NotImplementedError, match="float32 or float64"):
        replay.mirror_transitions_to_device(buf, "cuda:0")
    assert replay.find_transition_mirror(buf) is None


@needs_ref
def test_mirror_refuses_trajectory_buffers_host_devices_and_oversized_capacities():
    traj = _rb().ReplayBuffer(100, (D,), (A,), max_trajectory_length=10)
    with pytest.raises(NotImplementedError, match="max_trajectory_length"):
        replay.mirror_transitions_to_device(traj, "cuda:0")
    buf = _rb().ReplayBuffer(1000, (D,), (A,))
    with pytest.raises(ValueError, match="device memory"):
        replay.mirror_transitions_to_device(buf, "cpu")
    need = 1000 * 4 * (2 * D + A + 2)
    with pytest.raises(MemoryError, match="max_bytes"):
        replay.mirror_transitions_to_device(buf, "cuda:0", max_bytes=need - 1)
    assert replay.find_transition_mirror(buf) is None
    assert "add_batch" not in buf.__dict__  # nothing was wrapped


def _agent_stub(device, obs_dim=D, act_dim=A):
    desc = types.SimpleNamespace(obs_dim=obs_dim, act_dim=act_dim)
    return types.SimpleNamespace(device=torch.device(device), _desc=desc)


@needs_ref
def test_which_buffers_are_gathered_on_the_device():
    """SAC.mirror_of: no mirror, or a mirror on another device, means the host packs the batch; a mirror on the agent's
    device with other row sizes is an error."""
    buf = _rb().ReplayBuffer(10, (D,), (A,))
    assert bsac.SAC.mirror_of(_agent_stub("cuda:0"), buf) is None  # unmirrored
    fake = types.SimpleNamespace(buffer=buf, device=torch.device("cuda", 1), obs_dim=D, act_dim=A)
    replay._TRANSITION_MIRRORS[id(buf)] = lambda: fake  # what a live weakref returns
    try:
        assert replay.find_transition_mirror(buf) is fake
        assert bsac.SAC.mirror_of(_agent_stub("cuda:0"), buf) is None  # another device: the host path
        assert bsac.SAC.mirror_of(_agent_stub("cuda:1"), buf) is fake
        with pytest.raises(ValueError, match="columns"):
            bsac.SAC.mirror_of(_agent_stub("cuda:1", obs_dim=D + 1), buf)
        other = _rb().ReplayBuffer(10, (D,), (A,))
        assert replay.find_transition_mirror(other) is None
    finally:
        del replay._TRANSITION_MIRRORS[id(buf)]


def test_write_tracker_skips_the_scan_when_nothing_was_written():
    class Buf:
        def __init__(self):
            self.obs = np.zeros((8, 2))
            self.cur_idx, self.num_stored, self.capacity = 0, 0, 8

        def add(self, *a):
            self.cur_idx, self.num_stored = self.cur_idx + 1, self.num_stored + 1

        def add_batch(self, obs, *a):
            self.cur_idx, self.num_stored = self.cur_idx + len(obs), self.num_stored + len(obs)

        def load(self, *a):
            pass

    b = Buf()
    w = replay.WriteTracker(b)
    assert w.take().size == 0
    b.add_batch(np.zeros((3, 2)))
    assert list(w.take()) == [0, 1, 2]
    assert w.take().size == 0
    b.add_batch(np.zeros((2, 2)))
    w.clear(np.array([3]))
    assert list(w.take()) == [4]
    b.add_batch(np.zeros((1, 2)))
    w.clear(np.array([5]))
    assert w.take().size == 0
    b.cur_idx = 7  # moved outside the wrappers: a resync
    assert list(w.take()) == list(range(6))
    w.close()


def _tdesc(rows=100, shift=4, obs_dim=D, act_dim=A):
    d = _lib.TransitionDesc()
    d.obs_dim, d.act_dim, d.rows, d.chunk_shift = obs_dim, act_dim, rows, shift
    return d


def test_abi_refuses_bad_arguments():
    lib = _lib.load()
    p = C.c_void_p(16)
    gather = lambda d, B=4, chunks=p, idx=p, out=p: lib.b200pets_transition_gather(  # noqa: E731
        C.byref(d) if d is not None else None, chunks, idx, B, out, None)
    assert gather(None) == -1
    assert gather(_tdesc(), chunks=None) == -1
    assert gather(_tdesc(), idx=None) == -1
    assert gather(_tdesc(), out=None) == -1
    assert gather(_tdesc(), B=0) == -1
    assert gather(_tdesc(rows=0)) == -1
    assert gather(_tdesc(obs_dim=0)) == -1
    assert gather(_tdesc(act_dim=-1)) == -1
    assert gather(_tdesc(shift=-1)) == -1
    assert gather(_tdesc(shift=_lib.REPLAY_MAX_CHUNK_SHIFT + 1)) == -1
    scatter = lambda d, first=0, count=4, arrays=(p,) * 5: lib.b200pets_transition_scatter(  # noqa: E731
        C.byref(d), p, first, count, *arrays, None)
    assert scatter(_tdesc(), count=0) == -1
    assert scatter(_tdesc(rows=10), count=11) == -1
    assert scatter(_tdesc(rows=10), first=10) == -1
    assert scatter(_tdesc(rows=10), first=-1) == -1
    for i in range(5):
        assert scatter(_tdesc(), arrays=tuple(None if j == i else p for j in range(5))) == -1
    assert lib.b200pets_sac_update_many(None, 0, 256, 0, 1, (C.c_int64 * 3)(), p, None, 0, 0, p, p, p, 1, None) == -1
    assert lib.b200pets_sac_update_many(None, 3, 256, 0, 1, (C.c_int64 * 3)(), p, None, 0, 0, p, p, p, 1, None) == -1
