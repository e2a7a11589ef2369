"""CPU checks of the replay mirror's host side (mbrl_lib_b200/replay.py, trainer.py):

* the rows :class:`replay.WriteTracker` records over random sequences of ``add`` / ``add_batch`` / ``load`` on the
  reference's own ``ReplayBuffer``, with and without ``max_trajectory_length`` (the overflow reset, the ring wrap), are
  exactly the rows whose host contents changed; a numpy stand-in for the device store, updated run by run as a flush
  copies, equals ``obs[:num_stored]``, ``action`` and ``reward`` after every flush;
* ``trainer.sequence_starts`` gives the start rows of the batches the reference's ``SequenceTransitionSampler`` /
  ``SequenceTransitionIterator`` yield and leaves their ``rng`` where iterating leaves it;
* ``b200pets_sequence_gather`` refuses bad arguments before touching a device, and the mirror refuses obs types it
  does not store.
"""
import copy
import ctypes as C
import gc
import importlib
import tempfile
import weakref

import numpy as np
import pytest

from baseline import reference_arm as ra
from mbrl_lib_b200 import _lib, replay, trainer

mbrl, REF_SRC = ra.import_reference()
needs_ref = pytest.mark.skipif(mbrl is None, reason=f"reference not importable here: {REF_SRC}")
OBS = (2, 3)


def _rb():
    return importlib.import_module("mbrl.util.replay_buffer")


def _snapshot(buf):
    return buf.obs.copy(), buf.action.copy(), buf.reward.copy()


def _changed(before, buf):
    o, a, r = before
    rows = (buf.obs != o).reshape(len(o), -1).any(1) | (buf.action != a).reshape(len(a), -1).any(1) | (buf.reward != r)
    return np.flatnonzero(rows)


class _Store:
    """The device store's stand-in: rows copied run by run, as DeviceReplayMirror._copy_run copies them."""

    def __init__(self, buf, chunk_shift):
        self.buf, self.shift = buf, chunk_shift
        self.obs = np.zeros_like(buf.obs)
        self.act = np.zeros(buf.action.shape, np.float32)
        self.rew = np.zeros(buf.reward.shape, np.float32)

    def flush(self, rows):
        for lo, hi in replay.row_runs(rows, self.shift):
            assert lo >> self.shift == (hi - 1) >> self.shift  # a run stays in one chunk
            self.obs[lo:hi] = self.buf.obs[lo:hi]
            self.act[lo:hi] = self.buf.action[lo:hi]
            self.rew[lo:hi] = self.buf.reward[lo:hi]

    def check(self):
        n = self.buf.num_stored
        np.testing.assert_array_equal(self.obs[:n], self.buf.obs[:n])
        np.testing.assert_array_equal(self.act[:n], self.buf.action[:n].astype(np.float32))
        np.testing.assert_array_equal(self.rew[:n], self.buf.reward[:n].astype(np.float32))


def _random_ops(buf, g, steps, tmp, with_load):
    """Yield after each random write (add with random terminations, add_batch of random sizes, load of a saved state)."""
    saved = False
    for _ in range(steps):
        op = g.choice(["add", "add", "add", "add_batch", "load"] if with_load else ["add", "add", "add", "add_batch"])
        if op == "add":
            buf.add(g.standard_normal(OBS).astype(np.float32), g.standard_normal(2), g.standard_normal(OBS),
                    float(g.standard_normal()), bool(g.random() < 0.1), bool(g.random() < 0.05))
        elif op == "add_batch":
            n = int(g.integers(1, buf.capacity + 1))
            if buf.cur_idx + n > buf.capacity and buf.cur_idx > buf.capacity:
                continue  # beyond the ring's end (a trajectory buffer mid-trajectory): add_batch cannot wrap from there
            buf.add_batch(g.standard_normal((n, *OBS)).astype(np.float32), g.standard_normal((n, 2)),
                          g.standard_normal((n, *OBS)), g.standard_normal(n), g.random(n) < 0.1, np.zeros(n, bool))
        else:
            if not saved or g.random() < 0.5:
                buf.save(tmp)
                saved = True
                continue
            buf.obs[:] = g.standard_normal(buf.obs.shape)  # scribble, so the load changes every row it writes
            buf.action[:] = g.standard_normal(buf.action.shape)
            buf.reward[:] = g.standard_normal(buf.reward.shape)
            yield "scribble"
            buf.load(tmp)
        yield op


@needs_ref
@pytest.mark.parametrize("max_traj", [None, 7])
@pytest.mark.parametrize("seed", range(4))
def test_tracked_rows_are_the_rows_written(max_traj, seed):
    g = np.random.default_rng(seed)
    buf = _rb().ReplayBuffer(23, OBS, (2,), obs_type=np.float32, action_type=np.float64, reward_type=np.float64,
                             rng=np.random.default_rng(0), max_trajectory_length=max_traj)
    for a in (buf.obs, buf.action, buf.reward):
        a[:] = 0  # np.empty's garbage can hold NaNs, which never compare equal
    tracker = replay.WriteTracker(buf)
    store = _Store(buf, chunk_shift=2)
    store.flush(tracker.take())
    wrapped_add = buf.add
    with tempfile.TemporaryDirectory() as tmp:
        before = _snapshot(buf)
        # (load is left to the plain buffer: it stores trajectory_indices as an array, which a later add cannot pop)
        it = _random_ops(buf, g, 300, tmp, with_load=max_traj is None)
        for op in it:
            if op == "scribble":  # a direct write no wrapper sees: resync brings the store back
                store.flush(tracker.take(resync=True))
                np.testing.assert_array_equal(store.obs[:buf.num_stored], buf.obs[:buf.num_stored])
                before = _snapshot(buf)
                continue
            want = _changed(before, buf)
            got = tracker.dirty_rows()
            np.testing.assert_array_equal(got, want, err_msg=op)
            if g.random() < 0.3:
                store.flush(tracker.take())
                store.check()
                before = _snapshot(buf)
    store.flush(tracker.take())
    store.check()
    tracker.close()
    assert "add" not in buf.__dict__ and buf.add != wrapped_add


@needs_ref
def test_a_bypassed_cur_idx_makes_the_next_take_a_resync():
    buf = _rb().ReplayBuffer(10, OBS, (2,), rng=np.random.default_rng(0))
    tracker = replay.WriteTracker(buf)
    for _ in range(4):
        buf.add(np.ones(OBS, np.float32), np.zeros(2), np.ones(OBS), 0.0, False, False)
    assert list(tracker.take()) == [0, 1, 2, 3]
    buf.obs[4] = 5.0  # writes behind the wrappers' back ...
    buf.cur_idx, buf.num_stored = 5, 5
    assert list(tracker.take()) == [0, 1, 2, 3, 4]  # ... are caught by the moved cur_idx
    buf.add(np.ones(OBS, np.float32), np.zeros(2), np.ones(OBS), 0.0, False, False)
    assert list(tracker.take()) == [5]
    buf.cur_idx = 7
    buf.add(np.ones(OBS, np.float32), np.zeros(2), np.ones(OBS), 0.0, False, False)
    assert list(tracker.take()) == list(range(buf.num_stored))  # moved before a wrapped call: still a resync


@needs_ref
def test_the_buffer_keeps_the_owner_alive_until_close():
    """``mirror_to_device(buffer, device)`` is used with its result discarded: the buffer's wrappers must keep the
    mirror (the tracker's owner) alive, and close() must let go of it."""
    class Owner:
        pass

    buf = _rb().ReplayBuffer(10, OBS, (2,), rng=np.random.default_rng(0))
    replay.WriteTracker(buf, owner=Owner())  # neither kept
    owner = weakref.ref(buf.add.func.__self__.owner)
    gc.collect()
    assert owner() is not None
    buf.add.func.__self__.close()
    gc.collect()
    assert owner() is None and "add" not in buf.__dict__


def test_row_runs_split_at_chunk_boundaries():
    rows = np.array([0, 1, 2, 3, 4, 7, 8, 9, 15, 16])
    assert replay.row_runs(rows, 2) == [(0, 4), (4, 5), (7, 8), (8, 10), (15, 16), (16, 17)]
    assert replay.row_runs(rows, 10) == [(0, 5), (7, 10), (15, 17)]
    assert replay.row_runs(np.array([], dtype=np.int64), 3) == []


def _trajectory_buffer(seed=0, trajectories=6, length=20):
    g = np.random.default_rng(seed)
    buf = _rb().ReplayBuffer(500, OBS, (2,), rng=np.random.default_rng(seed), max_trajectory_length=length)
    for _ in range(trajectories):
        n = int(g.integers(length // 2, length + 1))
        for t in range(n):
            buf.add(g.standard_normal(OBS).astype(np.float32), g.standard_normal(2).astype(np.float32),
                    g.standard_normal(OBS).astype(np.float32), float(g.standard_normal()), False, t == n - 1)
    return buf


@needs_ref
@pytest.mark.parametrize("kind,kwargs", [
    ("sampler", dict(use_simple_sampler=True, max_batches_per_loop_train=5)),
    ("iterator", dict(shuffle_each_epoch=True)),  # every valid start once, the last batch short
    ("iterator", dict(shuffle_each_epoch=True, max_batches_per_loop_train=3)),
    ("iterator", dict(shuffle_each_epoch=False)),
])
def test_sequence_starts_reproduce_the_reference_batches(kind, kwargs):
    common = importlib.import_module("mbrl.util.common")
    buf = _trajectory_buffer()
    ds, _ = common.get_sequence_buffer_iterator(buf, 7, 0, 6, **kwargs)
    assert trainer._sequence_kind(ds) == kind
    twin = copy.deepcopy(ds)  # its own copy of the rng
    for epoch in range(2):
        ref = [np.asarray(b.obs) for b in twin]
        got = list(trainer.sequence_starts(ds, kind))
        assert len(got) == len(ref) > 0
        for starts, obs in zip(got, ref):
            assert starts.dtype == np.int64 and obs.shape[0] == len(starts)
            want = buf.obs[starts[:, None] + np.arange(6)[None]]
            np.testing.assert_array_equal(want, obs)
        assert ds._rng.bit_generator.state == twin._rng.bit_generator.state, epoch
        if kind == "iterator" and "max_batches_per_loop_train" not in kwargs:
            n = len(ds._valid_starts)
            assert n % 7 and sum(len(s) for s in got) == n and len(got[-1]) == n % 7  # a short last batch


@needs_ref
def test_other_iterators_are_not_sequence_iterators():
    rb = _rb()
    buf = _trajectory_buffer()
    it = rb.TransitionIterator(buf.get_all(), 4)
    assert trainer._sequence_kind(it) is None
    common = importlib.import_module("mbrl.util.common")
    ds, _ = common.get_sequence_buffer_iterator(buf, 4, 0, 5, use_simple_sampler=True, max_batches_per_loop_train=2)

    class Sub(type(ds)):
        def __getitem__(self, item):
            return super().__getitem__(item)

    sub = copy.copy(ds)
    sub.__class__ = Sub
    assert trainer._sequence_kind(ds) == "sampler" and trainer._sequence_kind(sub) is None


def _desc(**kw):
    d = _lib.ReplayDesc()
    d.frame_elems, d.rows, d.action_size, d.dtype, d.chunk_shift = 12288, 100, 6, _lib.DTYPE["uint8"], 10
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def test_abi_refuses_bad_arguments():
    lib = _lib.load()
    dummy = C.c_void_p(8)

    def call(d=None, B=5, T=8, chunks=dummy, out=dummy):
        return lib.b200pets_sequence_gather(C.byref(d or _desc()), chunks, dummy, dummy, dummy, B, T, out, dummy, dummy,
                                            None)

    assert call(B=0) == -1 and call(T=1) == -1
    assert call(chunks=None) == -1 and call(out=None) == -1
    assert lib.b200pets_sequence_gather(None, dummy, dummy, dummy, dummy, 5, 8, dummy, dummy, dummy, None) == -1
    assert call(_desc(dtype=_lib.DTYPE["float64"])) == -1 and call(_desc(dtype=7)) == -1
    assert call(_desc(chunk_shift=-1)) == -1 and call(_desc(chunk_shift=_lib.REPLAY_MAX_CHUNK_SHIFT + 1)) == -1
    assert call(_desc(frame_elems=0)) == -1 and call(_desc(action_size=0)) == -1
    assert call(_desc(rows=7)) == -1  # fewer rows than one sequence
    assert "sequence_gather" in lib.b200pets_last_error().decode()


@needs_ref
@pytest.mark.parametrize("dtype", [np.float64, np.float16, np.int32])
def test_mirror_refuses_unsupported_obs_types(dtype):
    buf = _rb().ReplayBuffer(10, OBS, (2,), obs_type=dtype)
    with pytest.raises(NotImplementedError, match="uint8 or float32"):
        replay.mirror_to_device(buf, "cuda:0")
    assert "add" not in buf.__dict__  # nothing wrapped


def test_mirror_refuses_a_host_device():
    class Buf:
        obs = np.zeros((4, 3), np.float32)
        action = np.zeros((4, 1), np.float32)
        reward = np.zeros(4, np.float32)
        cur_idx = num_stored = 0
        capacity = 4

    with pytest.raises(ValueError, match="device memory"):
        replay.mirror_to_device(Buf(), "cpu")
