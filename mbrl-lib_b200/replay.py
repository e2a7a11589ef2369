"""Transition batches and the two dataset iterators ``ModelTrainer.train`` consumes, with the semantics of mbrl-lib's
``mbrl.types.TransitionBatch`` and ``mbrl.util.replay_buffer.{TransitionIterator, BootstrapIterator}``
(replay_buffer.py:33-180): what users without mbrl-lib hand to :class:`mbrl_lib_b200.ModelTrainer`, and what its tests
drive it with.  ``ModelTrainer`` recognises these classes and mbrl-lib's own by their attributes, not their type.

* ``TransitionIterator``: batches of ``batch_size`` consecutive entries of ``_order`` (the last one shorter), with
  ``_order`` re-drawn as a permutation from ``_rng`` at every ``iter()`` when ``shuffle_each_epoch``.
* ``BootstrapIterator``: one index row per member (``member_indices [E, n]``, permutations or draws with replacement,
  made once at construction); in bootstrap mode a batch stacks, per member, the entries ``member_indices[m][indices]``
  along a leading member axis.  ``toggle_bootstrap()`` switches to plain batches (evaluation).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import numpy as np


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
