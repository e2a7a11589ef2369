"""Transition batches and the two dataset iterators ``ModelTrainer.train`` consumes, with the semantics of mbrl-lib's
``mbrl.types.TransitionBatch`` and ``mbrl.util.replay_buffer.{TransitionIterator, BootstrapIterator}``
(replay_buffer.py:33-180): what users without mbrl-lib hand to :class:`mbrl_lib_b200.ModelTrainer`, and what its tests
drive it with.  ``ModelTrainer`` recognises these classes and mbrl-lib's own by their attributes, not their type.

And :func:`mirror_to_device`: a copy of an mbrl-lib ``ReplayBuffer``'s observations, actions and rewards in device
memory, kept current by wrapping the buffer's writers, from which ``ModelTrainer`` gathers PlaNet's sequence batches
on the device (:class:`DeviceReplayMirror`).

* ``TransitionIterator``: batches of ``batch_size`` consecutive entries of ``_order`` (the last one shorter), with
  ``_order`` re-drawn as a permutation from ``_rng`` at every ``iter()`` when ``shuffle_each_epoch``.
* ``BootstrapIterator``: one index row per member (``member_indices [E, n]``, permutations or draws with replacement,
  made once at construction); in bootstrap mode a batch stacks, per member, the entries ``member_indices[m][indices]``
  along a leading member axis.  ``toggle_bootstrap()`` switches to plain batches (evaluation).
"""
from __future__ import annotations

import ctypes as C
import functools
import weakref
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import numpy as np
import torch

from . import _lib


@dataclass
class TransitionBatch:
    obs: np.ndarray
    act: np.ndarray
    next_obs: np.ndarray
    rewards: np.ndarray
    terminateds: np.ndarray
    truncateds: np.ndarray

    def __len__(self):
        return self.obs.shape[0]

    def astuple(self):
        return self.obs, self.act, self.next_obs, self.rewards, self.terminateds, self.truncateds

    def __getitem__(self, item):
        return TransitionBatch(*(x[item] for x in self.astuple()))


def _stack_members(batches) -> TransitionBatch:
    return TransitionBatch(*(np.stack(cols) for cols in zip(*(b.astuple() for b in batches))))


class TransitionIterator:
    def __init__(self, transitions: TransitionBatch, batch_size: int, shuffle_each_epoch: bool = False,
                 rng: Optional[np.random.Generator] = None):
        self.transitions = transitions
        self.num_stored = len(transitions)
        self._order = np.arange(self.num_stored)
        self.batch_size = batch_size
        self._current_batch = 0
        self._shuffle_each_epoch = shuffle_each_epoch
        self._rng = rng if rng is not None else np.random.default_rng()

    def _get_indices_next_batch(self):
        start = self._current_batch * self.batch_size
        if start >= self.num_stored:
            raise StopIteration
        self._current_batch += 1
        return self._order[start:min(start + self.batch_size, self.num_stored)]

    def __iter__(self):
        self._current_batch = 0
        if self._shuffle_each_epoch:
            self._order = self._rng.permutation(self.num_stored)
        return self

    def __next__(self):
        return self[self._get_indices_next_batch()]

    def ensemble_size(self):
        return 0

    def __len__(self):
        return (self.num_stored - 1) // self.batch_size + 1

    def __getitem__(self, item):
        return self.transitions[item]


class BootstrapIterator(TransitionIterator):
    def __init__(self, transitions: TransitionBatch, batch_size: int, ensemble_size: int, shuffle_each_epoch: bool = False,
                 permute_indices: bool = True, rng: Optional[np.random.Generator] = None):
        super().__init__(transitions, batch_size, shuffle_each_epoch=shuffle_each_epoch, rng=rng)
        self._ensemble_size = ensemble_size
        self._permute_indices = permute_indices
        self._bootstrap_iter = ensemble_size > 1
        if permute_indices:
            self.member_indices = np.stack([self._rng.permutation(self.num_stored) for _ in range(ensemble_size)]) \
                if ensemble_size > 0 else np.empty((0, self.num_stored), dtype=int)
        else:
            self.member_indices = self._rng.choice(self.num_stored, size=(ensemble_size, self.num_stored), replace=True)

    def __next__(self):
        if not self._bootstrap_iter:
            return super().__next__()
        indices = self._get_indices_next_batch()
        return _stack_members([self[member[indices]] for member in self.member_indices])

    def toggle_bootstrap(self):
        if self.ensemble_size > 1:
            self._bootstrap_iter = not self._bootstrap_iter

    @property
    def ensemble_size(self):
        return self._ensemble_size


# ---- the device-resident mirror ---------------------------------------------------------------------------------------

_CHUNK_BYTES = 64 << 20  # frames per chunk: the largest power of two of rows within this (1024 rows at 3x64x64 fp32)
_STAGING_SLOT_BYTES = 16 << 20  # each of the two pinned staging slots a flush copies frames through
_STORAGE = {np.dtype(np.uint8): (torch.uint8, "uint8"), np.dtype(np.float32): (torch.float32, "float32")}
_HOOKED = ("add", "add_batch", "load")
_MISSING = object()
_MIRRORS: Dict[int, "weakref.ref[DeviceReplayMirror]"] = {}  # data address of a mirrored buffer's obs -> its mirror


def _address(a: np.ndarray) -> int:
    return int(a.__array_interface__["data"][0])


def _cuda_device(device) -> torch.device:
    dev = torch.device(device)
    if dev.type != "cuda":
        raise ValueError(f"the replay mirror lives in device memory; got device {dev}")
    return dev if dev.index is not None else torch.device("cuda", torch.cuda.current_device())


class WriteTracker:
    """The rows of a replay buffer written since the last :meth:`take`, recorded by wrapping the buffer's ``add``,
    ``add_batch`` and ``load``: ``add`` writes the row at ``cur_idx`` before the call (also when a buffer that stores
    trajectories resets ``cur_idx`` to 0 on overflow), ``add_batch`` the rows from ``cur_idx`` on, wrapping at
    ``capacity`` (replay_buffer.py:553-599), ``load`` rows ``[0, num_stored)``.  Rows ``[0, num_stored)`` count as
    written at construction.  The wrappers hold the tracker, and the tracker holds ``owner``: the buffer keeps both
    alive until :meth:`close`."""

    def __init__(self, buffer, owner=None):
        self.buffer = buffer
        self.owner = owner
        self.rows = len(buffer.obs)  # capacity, plus max_trajectory_length for a buffer that stores trajectories
        self._dirty = np.zeros(self.rows, dtype=bool)
        self._dirty[:int(buffer.num_stored)] = True
        self._pending = buffer.num_stored > 0  # whether _dirty may have a set bit (take() skips the scan when not)
        self._seen = self._state()
        self._stale = False
        self._hooks = {}
        for name in _HOOKED:
            self._hooks[name] = buffer.__dict__.get(name, _MISSING)
            orig = getattr(buffer, name)
            setattr(buffer, name, functools.wraps(orig)(functools.partial(getattr(self, f"_on_{name}"), orig)))

    def _state(self) -> Tuple[int, int]:
        return int(self.buffer.cur_idx), int(self.buffer.num_stored)

    def _before(self):
        if self._state() != self._seen:  # cur_idx / num_stored moved outside the wrappers: writes they did not see
            self._stale = True

    def _on_add(self, orig, *args, **kwargs):
        self._before()
        cur = int(self.buffer.cur_idx)
        if 0 <= cur < self.rows:
            self._dirty[cur] = True
            self._pending = True
        out = orig(*args, **kwargs)
        self._seen = self._state()
        return out

    def _on_add_batch(self, orig, *args, **kwargs):
        self._before()
        n = len(args[0] if args else kwargs["obs"])
        cur, cap = int(self.buffer.cur_idx), int(self.buffer.capacity)
        first = 0  # the slices replay_buffer.py:588-597 copies into, sliced as numpy slices them there
        if cur + n > cap:
            self._dirty[cur:cur + (cap - cur)] = True
            first, cur = cap - cur, 0
        self._dirty[cur:cur + (n - first)] = True
        self._pending = True
        out = orig(*args, **kwargs)
        self._seen = self._state()
        return out

    def _on_load(self, orig, *args, **kwargs):
        out = orig(*args, **kwargs)
        self._dirty[:int(self.buffer.num_stored)] = True
        self._pending = True
        self._seen = self._state()
        return out

    def dirty_rows(self) -> np.ndarray:
        """Rows written since the last :meth:`take`, as the wrappers recorded them."""
        return np.flatnonzero(self._dirty)

    def take(self, resync: bool = False) -> np.ndarray:
        """The rows to copy, now counted as copied: those written since the last call, or all of ``[0, num_stored)``
        with ``resync`` or when ``cur_idx`` / ``num_stored`` changed outside the wrappers since they last ran."""
        if resync or self._stale or self._state() != self._seen:
            self._dirty[:] = False
            self._dirty[:int(self.buffer.num_stored)] = True
            self._seen = self._state()
            self._stale = False
            self._pending = True
        if not self._pending:
            return np.empty(0, dtype=np.int64)
        rows = np.flatnonzero(self._dirty)
        self._dirty[rows] = False
        self._pending = False
        return rows

    def clear(self, rows: np.ndarray):
        """Count ``rows`` as copied (rows the caller wrote to the device copy itself)."""
        self._dirty[rows] = False
        self._pending = bool(self._dirty.any())

    def mark_stale(self):
        """Make the next :meth:`take` a resync (a copy that failed part-way)."""
        self._stale = True

    def close(self):
        """Restore the buffer's methods and let go of ``owner``."""
        for name, prev in self._hooks.items():
            if prev is _MISSING:
                self.buffer.__dict__.pop(name, None)
            else:
                setattr(self.buffer, name, prev)
        self._hooks = {}
        self.owner = None


def row_runs(rows: np.ndarray, chunk_shift: int):
    """Sorted rows as ``(lo, hi)`` runs of consecutive rows, none crossing a multiple of ``2 ** chunk_shift``."""
    if rows.size == 0:
        return []
    cut = np.flatnonzero((np.diff(rows) != 1) | (np.diff(rows >> chunk_shift) != 0)) + 1
    return [(int(r[0]), int(r[-1]) + 1) for r in np.split(rows, cut)]


class _ChunkedMirror:
    """The device store both mirrors keep: ``rows`` rows of a buffer, each ``row_elems`` elements of ``storage``.

    Rows live in chunks of ``2 ** chunk_shift`` rows, each allocated through torch's allocator the first time a row in
    it is written, plus a device table of chunk pointers, so the device memory follows the rows written rather than the
    capacity.

    A :class:`WriteTracker` records the rows the buffer's ``add``, ``add_batch`` and ``load`` write; :meth:`flush` copies
    them through two pinned staging slots, each filled by the subclass's :meth:`_fill`.  Writes no wrapper sees
    (assignments to the buffer's arrays) need :meth:`resync`; a ``cur_idx`` or ``num_stored`` that changed outside the
    wrappers makes :meth:`flush` resync by itself, and so does a copy that failed part-way."""

    _registry: Dict[int, "weakref.ref[_ChunkedMirror]"]  # a subclass's _key(buffer) -> its mirror, one per subclass

    def __init__(self, buffer, device: torch.device, rows: int, row_elems: int, storage: torch.dtype,
                 _rows_per_chunk: Optional[int] = None):
        self.buffer, self.device = buffer, device
        self.rows, self._row_elems, self.storage = rows, row_elems, storage
        row_bytes = row_elems * storage.itemsize
        rows_per_chunk = _rows_per_chunk or max(1, _CHUNK_BYTES // row_bytes)
        # a power of two, and no more rows than the whole store needs
        self.chunk_shift = min(int(rows_per_chunk).bit_length() - 1, max(0, (self.rows - 1).bit_length()))
        self._chunks = [None] * ((self.rows + (1 << self.chunk_shift) - 1) >> self.chunk_shift)
        self._slot_rows = max(1, min(self.rows, _STAGING_SLOT_BYTES // row_bytes))
        with torch.cuda.device(device):
            self._chunk_table = torch.zeros(len(self._chunks), dtype=torch.int64, device=device)
        self.rows_held = 0  # rows [0, rows_held) are current on the device (the buffer's num_stored at the last flush)
        self._staging = None
        self._events = None
        self._slot = 0
        self._rows_copied = 0  # rows copied by the last flush (tests)
        self._writes = WriteTracker(buffer, owner=self)  # the buffer's wrappers keep this mirror alive

    @classmethod
    def _registered(cls, buffer):
        """The live mirror of this kind whose buffer is ``buffer``, or None."""
        found = cls._registry.get(cls._key(buffer))
        m = found() if found is not None else None
        return m if m is not None and m.buffer is buffer else None

    @classmethod
    def _get_or_make(cls, buffer, device, **kwargs):
        """``buffer``'s mirror of this kind on ``device``: the one already made, or a new one, registered."""
        m = cls._registered(buffer)
        if m is not None:
            if m.device == _cuda_device(device):
                return m
            raise ValueError(f"this buffer is already mirrored on {m.device}; close() that mirror first")
        m = cls(buffer, device, **kwargs)
        cls._registry[cls._key(buffer)] = weakref.ref(m)
        return m

    # ---- copies ----------------------------------------------------------------------------------------------------
    def flush(self) -> int:
        """Copy the rows written since the last flush to the device, as contiguous runs per chunk through a pinned
        staging buffer, on the current stream; resync instead when ``cur_idx`` / ``num_stored`` changed outside the
        wrappers.  Returns the number of rows copied."""
        return self._copy(self._writes.take())

    def resync(self) -> int:
        """Re-copy rows ``[0, num_stored)``: for code that writes the buffer's arrays directly, which no wrapper sees."""
        return self._copy(self._writes.take(resync=True))

    def _copy(self, rows: np.ndarray) -> int:
        try:
            with torch.cuda.device(self.device):
                for lo, hi in row_runs(rows, self.chunk_shift):
                    self._copy_run(lo, hi)
        except BaseException:
            self._writes.mark_stale()
            raise
        self.rows_held = min(int(self.buffer.num_stored), self.rows)
        self._rows_copied = int(rows.size)
        return self._rows_copied

    def _chunk(self, c: int) -> torch.Tensor:
        t = self._chunks[c]
        if t is None:
            n = min(1 << self.chunk_shift, self.rows - (c << self.chunk_shift))
            t = torch.empty(n, self._row_elems, dtype=self.storage, device=self.device)
            self._chunks[c] = t
            self._chunk_table[c] = t.data_ptr()
        return t

    def _copy_run(self, lo: int, hi: int):
        """Rows [lo, hi) of one chunk, through two pinned staging slots."""
        if self._staging is None:
            self._staging = [torch.empty(self._slot_rows, self._row_elems, dtype=self.storage, pin_memory=True)
                             for _ in range(2)]
            self._events = [torch.cuda.Event() for _ in range(2)]
        c = lo >> self.chunk_shift
        chunk, base = self._chunk(c), c << self.chunk_shift
        for s in range(lo, hi, self._slot_rows):
            e = min(hi, s + self._slot_rows)
            k = self._slot
            self._slot ^= 1
            self._events[k].synchronize()  # the slot's previous copy has left it
            stage = self._staging[k][:e - s]
            self._fill(stage.numpy(), s, e)
            chunk[s - base:e - base].copy_(stage, non_blocking=True)
            self._events[k].record()
        self._run_copied(lo, hi)

    def _fill(self, stage: np.ndarray, s: int, e: int):
        """Put the buffer's rows [s, e) into ``stage`` [e - s, row_elems] as the device store holds them."""
        raise NotImplementedError

    def _run_copied(self, lo: int, hi: int):
        """What else a subclass copies with rows [lo, hi), once their staging copies are queued."""

    def device_rows(self, lo: int, hi: int) -> torch.Tensor:
        """Rows [lo, hi) of the device store (tests; one chunk per call)."""
        c = lo >> self.chunk_shift
        base = c << self.chunk_shift
        if (hi - 1) >> self.chunk_shift != c:
            raise ValueError("rows of one chunk only")
        return self._chunk(c)[lo - base:hi - base]

    def close(self):
        """Restore the buffer's methods and free the device and pinned memory."""
        self._writes.close()
        if self._events is not None:
            for ev in self._events:
                ev.synchronize()
        key = self._key(self.buffer)
        if key in self._registry and self._registry[key]() is self:
            del self._registry[key]
        self._chunks, self._staging, self._events = [], None, None
        self._chunk_table = None
        self.rows_held = 0


class DeviceReplayMirror(_ChunkedMirror):
    """A copy in device memory of what PlaNet's sequence loss reads from an mbrl-lib ``ReplayBuffer``
    (mbrl/models/planet.py:274-287): ``obs`` in the buffer's own element type (uint8 or float32), and ``action`` and
    ``reward`` as float32, converted as ``.float()`` converts them.  ``next_obs``, ``terminated`` and ``truncated`` are
    not mirrored.  Made by :func:`mirror_to_device`.

    Frames live in the chunked store (:class:`_ChunkedMirror`): PlaNet's buffer has room for a million frames, far more
    than a run writes.  Actions and rewards are allocated for every row."""

    _registry = _MIRRORS

    def __init__(self, buffer, device, _rows_per_chunk: Optional[int] = None):
        obs = buffer.obs
        if obs.dtype not in _STORAGE:
            raise NotImplementedError(f"the replay mirror stores uint8 or float32 observations, not {obs.dtype}")
        if not obs.flags.c_contiguous:
            raise ValueError("the replay mirror copies rows of a C-contiguous obs array")
        dev = _cuda_device(device)
        rows = len(obs)
        self.frame_shape = tuple(int(n) for n in obs.shape[1:])
        self.frame_elems = int(np.prod(self.frame_shape, dtype=np.int64))
        self.action_size = int(np.prod(buffer.action.shape[1:], dtype=np.int64))
        storage, self._dtype_name = _STORAGE[obs.dtype]
        with torch.cuda.device(dev):  # before the store's tracker wraps the buffer's writers
            self.act = torch.zeros(rows, self.action_size, device=dev)
            self.rew = torch.zeros(rows, device=dev)
        super().__init__(buffer, dev, rows, self.frame_elems, storage, _rows_per_chunk)

    @staticmethod
    def _key(buffer) -> int:
        return _address(buffer.obs)  # find_mirror starts from get_all()'s views, which share the obs data

    def _fill(self, stage: np.ndarray, s: int, e: int):
        np.copyto(stage, self.buffer.obs.reshape(self.rows, self.frame_elems)[s:e])

    def _run_copied(self, lo: int, hi: int):
        b = self.buffer
        act = torch.from_numpy(np.ascontiguousarray(b.action[lo:hi]).reshape(hi - lo, self.action_size)).float()
        rew = torch.from_numpy(np.ascontiguousarray(b.reward[lo:hi])).float()
        self.act[lo:hi].copy_(act)
        self.rew[lo:hi].copy_(rew)

    def device_obs(self, lo: int, hi: int) -> torch.Tensor:
        """Rows [lo, hi) of the device store's frames (tests; one chunk per call)."""
        return self.device_rows(lo, hi).view(hi - lo, *self.frame_shape)

    # ---- the gather ------------------------------------------------------------------------------------------------
    def desc(self) -> _lib.ReplayDesc:
        d = _lib.ReplayDesc()
        d.frame_elems, d.rows, d.action_size = self.frame_elems, self.rows_held, self.action_size
        d.dtype, d.chunk_shift = _lib.DTYPE[self._dtype_name], self.chunk_shift
        return d

    def gather(self, starts: torch.Tensor, T: int, obs_out: torch.Tensor, act_out: torch.Tensor,
               rew_out: torch.Tensor):
        """``b200pets_sequence_gather``: the B sequences of T rows that start at ``starts`` (int64 [B] on the device,
        checked by the caller) into ``obs_out`` [B, T-1, *obs_shape], ``act_out`` [B, T-1, A], ``rew_out`` [B, T-1]."""
        B = int(starts.shape[0])
        for t, shape in ((obs_out, (B, T - 1, *self.frame_shape)), (act_out, (B, T - 1, self.action_size)),
                         (rew_out, (B, T - 1))):
            if tuple(t.shape) != shape or t.dtype != torch.float32 or not t.is_contiguous() or t.device != self.device:
                raise ValueError(f"gather output {tuple(t.shape)} {t.dtype} on {t.device}: expected contiguous float32 "
                                 f"{shape} on {self.device}")
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().b200pets_sequence_gather(
                C.byref(self.desc()), _lib.ptr(self._chunk_table), _lib.ptr(self.act), _lib.ptr(self.rew),
                _lib.ptr(starts), B, int(T), _lib.ptr(obs_out), _lib.ptr(act_out), _lib.ptr(rew_out),
                _lib.stream_ptr()), "sequence_gather")

    def close(self):
        super().close()
        self.act = self.rew = None


def mirror_to_device(buffer, device, *, _rows_per_chunk: Optional[int] = None) -> DeviceReplayMirror:
    """Mirror an mbrl-lib ``ReplayBuffer`` (or any object with its ``obs``, ``action``, ``reward``, ``cur_idx``,
    ``num_stored``, ``capacity``, ``add``, ``add_batch`` and ``load``) in ``device`` memory; see
    :class:`DeviceReplayMirror`.  From then on ``mbrl_lib_b200.ModelTrainer`` trains a PlaNet model from the mirror when
    it is handed a sequence sampler or iterator over ``buffer.get_all()``.  The buffer keeps the mirror alive until
    :meth:`DeviceReplayMirror.close`.  Mirroring a buffer again on the same device returns its mirror."""
    return DeviceReplayMirror._get_or_make(buffer, device, _rows_per_chunk=_rows_per_chunk)


def find_mirror(transitions) -> Optional[DeviceReplayMirror]:
    """The mirror whose buffer ``transitions`` views from row 0 (``obs``, ``act`` and ``rewards`` all), as
    ``ReplayBuffer.get_all()`` returns them (replay_buffer.py:685-703); None otherwise (``get_all(shuffle=True)``
    returns copies)."""
    obs = getattr(transitions, "obs", None)
    if not isinstance(obs, np.ndarray) or obs.ndim < 1:
        return None
    found = _MIRRORS.get(_address(obs))
    m = found() if found is not None else None
    if m is None:
        return None
    b = m.buffer

    def views(part, whole):
        return isinstance(part, np.ndarray) and isinstance(whole, np.ndarray) and part.dtype == whole.dtype and \
            part.shape[1:] == whole.shape[1:] and part.strides == whole.strides and len(part) <= len(whole) and \
            _address(part) == _address(whole)

    if views(obs, b.obs) and views(getattr(transitions, "act", None), b.action) and \
            views(getattr(transitions, "rewards", None), b.reward):
        return m
    return None


class SequenceGather:
    """Gathers batches of one mirror into output buffers reused from batch to batch (one ``ModelTrainer.train`` /
    ``evaluate`` call): the batch's start rows go to the device through a pinned buffer, then one
    ``b200pets_sequence_gather``."""

    def __init__(self, mirror: DeviceReplayMirror):
        self.mirror = mirror
        self._cap, self._T = 0, 0
        self._copied = None

    def __call__(self, starts: np.ndarray, T: int, limit: int):
        """A ``latent_train.SequenceBatch`` of the sequences of T rows at ``starts``; IndexError when one leaves
        rows ``[0, limit)`` (``limit`` is at most the rows the mirror holds)."""
        from .latent_train import SequenceBatch

        m = self.mirror
        B = len(starts)
        limit = min(int(limit), m.rows_held)
        if B == 0 or int(starts.min()) < 0 or int(starts.max()) + T > limit:
            raise IndexError(f"sequences of {T} rows at starts in [{starts.min() if B else None}, "
                             f"{starts.max() if B else None}] leave the {limit} rows stored")
        if B > self._cap or T != self._T:
            self._cap, self._T = max(B, self._cap), T
            dev = m.device
            self._starts_host = torch.empty(self._cap, dtype=torch.int64, pin_memory=True)
            self._starts = torch.empty(self._cap, dtype=torch.int64, device=dev)
            self._obs = torch.empty(self._cap, T - 1, *m.frame_shape, device=dev)
            self._act = torch.empty(self._cap, T - 1, m.action_size, device=dev)
            self._rew = torch.empty(self._cap, T - 1, device=dev)
            self._copied = None
        with torch.cuda.device(m.device):
            if self._copied is not None:
                self._copied.synchronize()  # the previous batch's starts have left the pinned buffer
            self._starts_host[:B].numpy()[:] = starts
            self._starts[:B].copy_(self._starts_host[:B], non_blocking=True)
            self._copied = torch.cuda.Event()
            self._copied.record()
            out = SequenceBatch(self._obs[:B], self._act[:B], self._rew[:B])
            m.gather(self._starts[:B], T, *out)
        return out


# ---- MBPO's SAC transitions in device memory --------------------------------------------------------------------------

_TRANSITION_DTYPES = (np.dtype(np.float32), np.dtype(np.float64))
_TRANSITION_MIRRORS: Dict[int, "weakref.ref[DeviceTransitionMirror]"] = {}  # id of a mirrored buffer -> its mirror


class DeviceTransitionMirror(_ChunkedMirror):
    """A copy in device memory of what ``SAC.update_parameters`` reads from an mbrl-lib ``ReplayBuffer``
    (pytorch_sac_pranz24/sac.py:76-97): ``obs``, ``action``, ``next_obs``, ``reward`` and ``terminated``, one packed
    float32 row per transition in the layout ``b200pets_sac_update`` reads, ``[obs | action | next_obs | reward |
    terminated]`` (W = 2 D + A + 2 floats).  float64 buffers are converted as ``torch.FloatTensor`` converts them
    (round to nearest).  Made by :func:`mirror_transitions_to_device`.

    Rows live in the chunked store (:class:`_ChunkedMirror`); ``mbpo.rollout_model_and_populate_sac_buffer`` writes its
    rows device-to-device (:meth:`scatter`)."""

    _registry = _TRANSITION_MIRRORS

    def __init__(self, buffer, device, max_bytes: Optional[int] = None, _rows_per_chunk: Optional[int] = None):
        for name in ("obs", "action", "next_obs", "reward"):
            a = getattr(buffer, name)
            if a.dtype not in _TRANSITION_DTYPES:
                raise NotImplementedError(f"the transition mirror stores float32 or float64 arrays, not {name} {a.dtype}")
        if getattr(buffer, "trajectory_indices", None) is not None:
            raise NotImplementedError("the transition mirror covers buffers without max_trajectory_length")
        dev = _cuda_device(device)
        self.obs_dim = int(np.prod(buffer.obs.shape[1:], dtype=np.int64))
        self.act_dim = int(np.prod(buffer.action.shape[1:], dtype=np.int64))
        self.width = 2 * self.obs_dim + self.act_dim + 2
        rows = int(buffer.capacity)
        row_bytes = 4 * self.width
        if max_bytes is not None and rows * row_bytes > max_bytes:
            raise MemoryError(f"mirroring {rows} rows of {row_bytes} bytes takes up to {rows * row_bytes} "
                              f"bytes of device memory, more than max_bytes = {max_bytes}")
        self.max_bytes = max_bytes
        super().__init__(buffer, dev, rows, self.width, torch.float32, _rows_per_chunk)

    @staticmethod
    def _key(buffer) -> int:
        return id(buffer)

    def _fill(self, stage: np.ndarray, s: int, e: int):
        pack_rows(self.buffer, slice(s, e), stage, self.obs_dim, self.act_dim)

    def allocated_bytes(self) -> int:
        """Device memory the allocated chunks take."""
        return sum(4 * self.width * int(t.shape[0]) for t in self._chunks if t is not None)

    def desc(self, rows: int) -> _lib.TransitionDesc:
        d = _lib.TransitionDesc()
        d.obs_dim, d.act_dim, d.rows, d.chunk_shift = self.obs_dim, self.act_dim, int(rows), self.chunk_shift
        return d

    # ---- device-side reads and writes ------------------------------------------------------------------------------
    def gather(self, indices: torch.Tensor, out: torch.Tensor):
        """``b200pets_transition_gather``: rows ``indices`` (int64 [B] on the device, each below the rows held) into
        ``out`` [B, W] float32, on the current stream.  Call :meth:`flush` first."""
        B = int(indices.shape[0])
        if tuple(out.shape) != (B, self.width) or out.dtype != torch.float32 or not out.is_contiguous() or \
                out.device != self.device:
            raise ValueError(f"gather output {tuple(out.shape)} {out.dtype} on {out.device}: expected contiguous float32 "
                             f"{(B, self.width)} on {self.device}")
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().b200pets_transition_gather(C.byref(self.desc(self.rows_held)),
                                                               _lib.ptr(self._chunk_table), _lib.ptr(indices), B,
                                                               _lib.ptr(out), _lib.stream_ptr()), "transition_gather")

    def scatter(self, first: int, obs, act, next_obs, reward, terminated):
        """``b200pets_transition_scatter``: the packed device rows (float32 [n, D], [n, A], [n, D], [n], uint8 [n]) to
        positions ``(first + j) mod capacity``, on the current stream, allocating the chunks they fall in.  n must not
        exceed the capacity.  The caller clears the positions' dirty bits once the host buffer holds the same rows."""
        n = int(reward.shape[0])
        pos = (first + np.arange(n, dtype=np.int64)) % self.rows
        for c in np.unique(pos >> self.chunk_shift):
            self._chunk(int(c))
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().b200pets_transition_scatter(
                C.byref(self.desc(self.rows)), _lib.ptr(self._chunk_table), int(first), n, _lib.ptr(obs), _lib.ptr(act),
                _lib.ptr(next_obs), _lib.ptr(reward), _lib.ptr(terminated), _lib.stream_ptr()), "transition_scatter")
        return pos


def pack_rows(buffer, rows, out: np.ndarray, D: int, A: int):
    """``buffer``'s rows ``rows`` as SAC staging rows ``[obs | action | next_obs | reward | terminated]`` in ``out``
    [n, 2D + A + 2] float32: numpy's float32 conversion, which rounds to nearest as ``torch.FloatTensor`` does."""
    n = out.shape[0]
    out[:, :D] = buffer.obs[rows].reshape(n, D)
    out[:, D:D + A] = buffer.action[rows].reshape(n, A)
    out[:, D + A:2 * D + A] = buffer.next_obs[rows].reshape(n, D)
    out[:, 2 * D + A] = buffer.reward[rows]
    out[:, 2 * D + A + 1] = buffer.terminated[rows]


def mirror_transitions_to_device(buffer, device, max_bytes: Optional[int] = None, *,
                                 _rows_per_chunk: Optional[int] = None) -> DeviceTransitionMirror:
    """Mirror what ``SAC.update_parameters`` reads from an mbrl-lib ``ReplayBuffer`` (float32 or float64 arrays, no
    ``max_trajectory_length``) in ``device`` memory; see :class:`DeviceTransitionMirror`.  From then on
    ``mbrl_lib_b200.SAC.update_parameters`` and ``mbpo.update_agent`` gather their batches from the mirror on the
    device, and ``mbpo.rollout_model_and_populate_sac_buffer`` writes its rollouts into it.  ``max_bytes``: refuse
    (``MemoryError``, before allocating anything) a buffer whose full capacity would take more device memory.  The
    buffer keeps the mirror alive until :meth:`DeviceTransitionMirror.close`.  Mirroring a buffer again on the same
    device returns its mirror."""
    return DeviceTransitionMirror._get_or_make(buffer, device, max_bytes=max_bytes, _rows_per_chunk=_rows_per_chunk)


def find_transition_mirror(buffer) -> Optional[DeviceTransitionMirror]:
    """The transition mirror of ``buffer``, or None."""
    return DeviceTransitionMirror._registered(buffer)
