"""MBPO model rollouts kept on the device: ``rollout_model_and_populate_sac_buffer`` with the reference's signature
(mbrl/algorithms/mbpo.py:31-63).

The reference moves every step's ``(next_obs, rewards, dones)`` to the host, masks them with numpy and calls
``sac_buffer.add_batch`` per step.  Here the observation batch, the predictions of all ``rollout_horizon`` steps and the
``accum_dones`` mask stay in HBM; one ordered compaction (``b200pets_mbpo_compact``) packs the alive transitions of all
steps, ONE device->host copy brings them back, and ``add_batch`` is then called once per step on host slices -- the
replay buffer ends up with exactly the rows, in exactly the order, the reference would have stored.

The policy: ``agent.act(obs, sample=..., batched=True)`` is numpy-in / numpy-out in the reference
(mbrl/planning/sac_wrapper.py:27-46).  To keep the loop on the device the actor is taken as an opaque torch callable:
``agent.act_torch(obs_tensor, sample)`` when the agent offers it, else ``agent.sac_agent.policy.sample`` (the
pytorch_sac policy the reference's SACAgent wraps), else the numpy ``agent.act`` with a per-step round trip of the
observations / actions only.

When ``sac_buffer`` has a transition mirror on the model's device (``replay.mirror_transitions_to_device``), the
compacted rows are also scattered device-to-device into the mirror, at the ring positions the ``add_batch`` calls write,
so the SAC updates gather them without a host-to-device copy.  ``update_agent`` runs one environment step's SAC updates
(mbpo.py:258-275) as one ``b200pets_sac_update_many`` call, and ``maybe_replace_sac_buffer`` (mbpo.py:88-113) carries the
mirror over to the replacement buffer.
"""
from __future__ import annotations

from typing import Sequence, Tuple

import numpy as np
import torch

from . import _lib, replay


def _policy(agent, device):
    if hasattr(agent, "act_torch"):
        return lambda obs, sample: agent.act_torch(obs, sample)
    sac = getattr(agent, "sac_agent", None)
    if sac is not None and hasattr(sac, "policy") and hasattr(sac.policy, "sample"):
        def f(obs, sample):  # pytorch_sac select_action: (action, log_prob, mean) = policy.sample(state)
            with torch.no_grad():
                action, _, mean = sac.policy.sample(obs.to(getattr(sac, "device", device)))
            return (action if sample else mean).to(device)
        return f

    def g(obs, sample):  # opaque numpy agent: only the observations / actions cross PCIe
        a = agent.act(obs.cpu().numpy(), sample=sample, batched=True)
        return torch.from_numpy(np.asarray(a, dtype=np.float32)).to(device)
    return g


def rollout_on_device(model_env, initial_obs: np.ndarray, agent, sac_samples_action: bool, rollout_horizon: int, *,
                      _noise=None, _staging=None):
    """The device part of the rollout: returns host arrays ``(obs, act, next_obs, reward, done, counts)`` holding the
    alive transitions of all steps packed in (step, row) order; ``counts[i]`` rows belong to step i.
    (``_noise``: per-step ``(perm, eps)`` device tensors injected into ModelEnv.step; ``_staging``: a dict that receives
    the un-compacted device buffers -- both for parity tests.)"""
    rows, counts = _rollout_compacted(model_env, initial_obs, agent, sac_samples_action, rollout_horizon, _noise,
                                      _staging)
    return (*[t.cpu().numpy() for t in rows], counts)


def _rollout_compacted(model_env, initial_obs, agent, sac_samples_action, rollout_horizon, _noise=None, _staging=None):
    """``rollout_on_device``'s packed rows as device tensors ``(obs, act, next_obs, reward, done)``, and the host
    array of per-step counts."""
    lib = _lib.load()
    dev = model_env.device
    k = int(rollout_horizon)
    state = model_env.reset(np.asarray(initial_obs), return_as_np=False)
    obs0 = state["obs"]
    B, D = obs0.shape
    A = int(model_env.action_space.shape[0])
    policy = _policy(agent, dev)
    act = torch.empty(k, B, A, device=dev)
    nxt = torch.empty(k, B, D, device=dev)
    rew = torch.empty(k, B, device=dev)
    done = torch.empty(k, B, dtype=torch.uint8, device=dev)
    alive = torch.empty(k, B, dtype=torch.uint8, device=dev)
    accum = torch.zeros(B, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        for i in range(k):
            a = policy(state["obs"], sac_samples_action)
            act[i].copy_(a.reshape(B, A))
            pn, en = _noise[i] if _noise is not None else (None, None)
            model_env.step(act[i], state, sample=True, _out=(nxt[i], rew[i], done[i]), _perm=pn, _eps=en)
            _lib.check(lib.b200pets_mbpo_mask(B, _lib.ptr(done[i]), _lib.ptr(accum), _lib.ptr(alive[i]), _lib.stream_ptr()),
                       "mbpo_mask")
            state = dict(state)
            state["obs"] = nxt[i]
        o_out = torch.empty(k * B, D, device=dev)
        a_out = torch.empty(k * B, A, device=dev)
        n_out = torch.empty(k * B, D, device=dev)
        r_out = torch.empty(k * B, device=dev)
        d_out = torch.empty(k * B, dtype=torch.uint8, device=dev)
        counts = torch.empty(k + 1, dtype=torch.int64, device=dev)
        need = lib.b200pets_mbpo_compact_workspace_bytes(k, B)
        ws = torch.empty(need, dtype=torch.uint8, device=dev)
        _lib.check(lib.b200pets_mbpo_compact(k, B, D, A, _lib.ptr(obs0), _lib.ptr(act), _lib.ptr(nxt), _lib.ptr(rew),
                                             _lib.ptr(done), _lib.ptr(alive), _lib.ptr(o_out), _lib.ptr(a_out), _lib.ptr(n_out),
                                             _lib.ptr(r_out), _lib.ptr(d_out), _lib.ptr(counts), _lib.ptr(ws), need,
                                             _lib.stream_ptr()), "mbpo_compact")
    if _staging is not None:
        _staging.update(obs0=obs0, act=act, next_obs=nxt, reward=rew, done=done, alive=alive)
    counts_h = counts.cpu().numpy()  # synchronises: the number of rows to bring back
    total = int(counts_h[k])
    return [t[:total] for t in (o_out, a_out, n_out, r_out, d_out)], counts_h[:k]


def scatter_positions(cur_idx: int, capacity: int, counts) -> Tuple[int, int]:
    """Where consecutive ``add_batch`` calls of ``counts`` rows each, from ``cur_idx``, leave the packed rows: row J
    of the concatenation at ``(cur_idx + J) mod capacity`` (replay_buffer.py:588-597 for each call of at most
    ``capacity`` rows).  Returns ``(skip, first)``: the first ``skip`` rows are overwritten by later ones, and the rest
    go to ``(first + j) mod capacity``."""
    total = int(np.sum(counts))
    skip = max(0, total - capacity)
    return skip, (cur_idx + skip) % capacity


def rollout_model_and_populate_sac_buffer(model_env, replay_buffer, agent, sac_buffer, sac_samples_action: bool,
                                          rollout_horizon: int, batch_size: int):
    """Drop-in for mbrl/algorithms/mbpo.py:31-63."""
    batch = replay_buffer.sample(batch_size)
    initial_obs, *_ = batch.astuple()
    rows, counts = _rollout_compacted(model_env, initial_obs, agent, sac_samples_action, rollout_horizon)
    m = replay.find_transition_mirror(sac_buffer)  # any object with add_batch is accepted; only a mirrored one is read
    positions = None
    if m is not None and m.device == rows[0].device and int(np.sum(counts)) > 0 and int(np.max(counts)) <= m.rows:
        skip, first = scatter_positions(int(sac_buffer.cur_idx), m.rows, counts)
        with torch.cuda.device(m.device):
            positions = m.scatter(first, *(t[skip:] for t in rows))
    obs, act, nxt, rew, done = (t.cpu().numpy() for t in rows)
    lo = 0
    for n in counts:  # one add_batch per step, as the reference issues them (replay_buffer.py:553-599 wraps per call)
        hi = lo + int(n)
        sac_buffer.add_batch(obs[lo:hi], act[lo:hi], nxt[lo:hi], rew[lo:hi], done[lo:hi].astype(bool),
                             np.zeros(hi - lo, dtype=bool))
        lo = hi
    if positions is not None:  # the device already holds these rows: the next flush need not copy them
        m._writes.clear(positions)


def update_agent(agent, replay_buffer, sac_buffer, rng, num_updates, real_data_ratio, batch_size, update_step,
                 updates_made, logger=None, log_frequency=None):
    """One environment step's SAC updates, mbrl/algorithms/mbpo.py:258-275, with ``agent.sac_agent`` an
    ``mbrl_lib_b200.SAC``: the same ``rng.random()`` per iteration before the break test, the same choice of buffer and
    break rule (``update_step`` is ``(env_steps + 1) % sac_updates_every_steps == 0``), and each update's indices drawn
    from the chosen buffer's generator in order, as its ``sample`` draws them.  The updates then run as one
    ``SAC.update_many`` (one index copy, one launch call, one statistics copy), and the seven log calls per update and
    ``logger.dump(updates_made, save=True)`` every ``log_frequency`` updates are replayed in the reference's order
    (no dump when ``log_frequency`` is None, as with ``silent``).  Returns the new ``updates_made``."""
    sac = getattr(agent, "sac_agent", agent)
    batches = []
    for _ in range(num_updates):
        use_real_data = rng.random() < real_data_ratio
        which_buffer = replay_buffer if use_real_data else sac_buffer
        if not update_step or len(which_buffer) < batch_size:
            break
        batches.append((which_buffer, which_buffer._rng.choice(which_buffer.num_stored, size=batch_size)))
    if not batches:
        return updates_made
    stats = sac.update_many(batches, batch_size, updates_made, reverse_mask=True)
    for row in stats:
        sac.log_stats(row.tolist(), updates_made, logger)
        updates_made += 1
        if logger is not None and log_frequency is not None and updates_made % log_frequency == 0:
            logger.dump(updates_made, save=True)
    return updates_made


def maybe_replace_sac_buffer(sac_buffer, obs_shape: Sequence[int], act_shape: Sequence[int], new_capacity: int,
                             seed: int):
    """mbrl/algorithms/mbpo.py:88-113.  When ``sac_buffer`` has a transition mirror, the replacement is mirrored on the
    same device with the same ``max_bytes`` (its rows are copied by the next flush) and the old mirror is closed."""
    if sac_buffer is not None and new_capacity == sac_buffer.capacity:
        return sac_buffer
    if sac_buffer is None:
        from mbrl.util import ReplayBuffer

        return ReplayBuffer(new_capacity, obs_shape, act_shape, rng=np.random.default_rng(seed=seed))
    new_buffer = type(sac_buffer)(new_capacity, obs_shape, act_shape, rng=sac_buffer.rng)
    new_buffer.add_batch(*sac_buffer.get_all().astuple())
    old = replay.find_transition_mirror(sac_buffer)
    if old is not None:
        replay.mirror_transitions_to_device(new_buffer, old.device, old.max_bytes)
        old.close()
    return new_buffer
