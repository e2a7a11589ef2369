"""Population-sharded CEM across GPUs (SURVEY.md section 8e): one process per GPU, weights / normaliser /
observation / (mu, sigma) replicated, every rank evaluates its own contiguous slice of the GLOBAL population, and
the only exchange per CEM iteration is ONE all-gather of each rank's local top-k records ``[value, sequence]``
(NCCL over NVLink / NVSwitch; <= 290 KB at config 2 on 8 GPUs, latency bound).  Every rank then refits from
the identical gathered records, so (mu, sigma, best) stay bit-identical on all ranks without a broadcast.

Results do not depend on the number of GPUs: the population noise is keyed by global sequence index
(``b200pets_cem_sample_shard``), the model noise by global row id and the TS1 member draw by global shuffle group
(``b200pets_rollout_cfg.first_sequence / global_population``), records arrive in global index order (contiguous
shards, rank-major gather) and the refit sums the elites in that order.  ``tests/test_gpu_parity.py`` checks that
two shards evaluated one after the other on one GPU reproduce the unsharded plan bit for bit, and
``tests/test_gpu_multi.py`` does the same across two processes with NCCL.

The reference has no multi-GPU path (SURVEY.md section 5); semantics are those of ``CEMOptimizer.optimize``
(mbrl/planning/trajectory_opt.py:142-188) over the union population.
"""
from __future__ import annotations

import ctypes as C
from typing import Callable, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.distributed as dist

from . import _lib


def shard_bounds(total: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous slice [lo, hi) of ``total`` units owned by ``rank`` (remainder spread over the first ranks)."""
    base, rem = divmod(total, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def records_per_rank(elite_num: int, local_population: int) -> int:
    """A rank can hold at most all global elites, and never more records than it has sequences."""
    return min(elite_num, local_population)


def gather_records(local_records: torch.Tensor, group=None) -> torch.Tensor:
    """The one collective of an iteration: all ranks' [k, 1 + dims] records, concatenated in rank order."""
    world = dist.get_world_size(group)
    out = torch.empty((world,) + tuple(local_records.shape), dtype=local_records.dtype, device=local_records.device)
    if dist.get_backend(group) == "nccl":
        dist.all_gather_into_tensor(out.view(-1), local_records.contiguous().view(-1), group=group)  # one NCCL kernel
    else:  # gloo (CPU tests)
        dist.all_gather([out[r] for r in range(world)], local_records.contiguous(), group=group)
    return out.view(world * local_records.shape[0], local_records.shape[1])


class ShardedCEMOptimizer:
    """CEM whose population of ``population_size`` (global) is split over the ranks of ``group``.

    ``population_size`` / ``elite_ratio`` keep their reference meaning for the *global* population.
    ``rank`` / ``world`` / ``gather`` default to the process group's; tests pass them explicitly to run several
    shards in one process (``gather`` maps this rank's ``[k, 1 + dims]`` records to the ``[world * k, 1 + dims]``
    union in rank order)."""

    def __init__(self, num_iterations: int, elite_ratio: float, population_size: int,
                 lower_bound: Sequence[Sequence[float]], upper_bound: Sequence[Sequence[float]], alpha: float, device,
                 return_mean_elites: bool = False, group=None, *, rank: Optional[int] = None, world: Optional[int] = None,
                 gather: Optional[Callable[[torch.Tensor], torch.Tensor]] = None):
        self.num_iterations = num_iterations
        self.population_size = population_size
        self.elite_num = int(np.ceil(population_size * elite_ratio).astype(np.int32))
        self.alpha = alpha
        self.return_mean_elites = return_mean_elites
        self.device = torch.device(device)
        self.group = group
        self.rank = dist.get_rank(group) if rank is None else rank
        self.world = dist.get_world_size(group) if world is None else world
        self._gather = gather if gather is not None else (lambda rec: gather_records(rec, self.group))
        lo, hi = shard_bounds(population_size, self.rank, self.world)
        self.local_population = hi - lo
        self.local_offset = lo
        self.k_local = records_per_rank(self.elite_num, self.local_population)
        counts = [records_per_rank(self.elite_num, shard_bounds(population_size, r, self.world)[1]
                                   - shard_bounds(population_size, r, self.world)[0]) for r in range(self.world)]
        if len(set(counts)) != 1:
            raise ValueError("population must split so that every rank contributes the same number of records")
        if self.k_local * self.world < self.elite_num:
            raise ValueError("not enough sequences per rank to cover the global elite set")
        self.lower_bound = torch.tensor(lower_bound, device=self.device, dtype=torch.float32).contiguous()
        self.upper_bound = torch.tensor(upper_bound, device=self.device, dtype=torch.float32).contiguous()
        self.lib = _lib.load()
        self._seed = int(torch.initial_seed()) & 0xFFFFFFFFFFFFFFFF
        self._offset = 0
        self._buf = None
        self.record_values = False
        self.last_values = None
        self.comm_events = None  # set to [] to record (start, end) CUDA events around every collective
        # Exchange over NVLink peer memory fused into the select / refit kernels (b200pets_cem_values_push / _elites_refit:
        # all values first, then only the rows of the global elites) instead of a host-issued NCCL all-gather of every
        # rank's local top-k: set up lazily (needs dims), only for a real NCCL group on ONE node with equal shards.
        # B200PETS_PEER_EXCHANGE=0 keeps the NCCL collective.
        import os
        self.peer_exchange = os.environ.get("B200PETS_PEER_EXCHANGE", "1") != "0" and gather is None
        self._peer = None  # {"own": ptr, "ptrs": (c_void_p * world), "key": (k, dims), "tag": tensor}
        self._epoch = 0

    # ---- peer-memory gather buffers ---------------------------------------------------------------------------
    def _setup_peers(self, dims: int):
        import socket

        if not self.peer_exchange or self.world < 2 or self.world > 16 or not dist.is_initialized():
            return None
        if dist.get_backend(self.group) != "nccl":
            return None
        key = (self.local_population, dims)
        if self._peer is not None and self._peer["key"] == key:
            return self._peer
        if self._peer is not None:
            self._close_peers()
        if self.population_size % self.world != 0 or self.local_population > 40960 or self.elite_num < 2:
            self.peer_exchange = False  # unequal shards / very large shards: keep the collective
            return None
        # Every decision below is taken from information ALL ranks hold (gathered tuples), so that either every rank uses the
        # peer path or none does: a rank that cannot allocate / map a buffer makes everybody fall back to the NCCL collective.
        nbytes = self.lib.b200pets_peer_buffer_bytes(self.world, self.local_population, dims, self.elite_num)
        own, handle, ok = C.c_void_p(), C.create_string_buffer(64), True
        try:
            with torch.cuda.device(self.device):
                _lib.check(self.lib.b200pets_peer_alloc(nbytes, C.byref(own), handle), "peer_alloc")
        except Exception:
            ok, own = False, C.c_void_p()
        infos = [None] * self.world
        dist.all_gather_object(infos, (socket.gethostname(), bytes(handle.raw), ok), group=self.group)
        opened = []
        if all(i[2] for i in infos) and len({i[0] for i in infos}) == 1:  # (another node: IPC handles do not travel)
            ptrs = (C.c_void_p * self.world)()
            try:
                with torch.cuda.device(self.device):
                    for r, (_, hb, _) in enumerate(infos):
                        if r == self.rank:
                            ptrs[r] = own.value
                        else:
                            q = C.c_void_p()
                            _lib.check(self.lib.b200pets_peer_open(hb, C.byref(q)), "peer_open")
                            opened.append(q)
                            ptrs[r] = q.value
            except Exception:
                ok = False
        else:
            ok = False
        oks = [None] * self.world
        dist.all_gather_object(oks, ok, group=self.group)
        if not all(oks):
            with torch.cuda.device(self.device):
                for q in opened:
                    self.lib.b200pets_peer_close(q, 0)
                if own.value:
                    self.lib.b200pets_peer_close(own, 1)
            self.peer_exchange = False
            return None
        dist.barrier(group=self.group)
        self._peer = {"own": own, "ptrs": ptrs, "key": key,
                      "tag": torch.zeros(1, dtype=torch.int32, device=self.device)}
        return self._peer

    def _close_peers(self):
        if getattr(self, "_peer", None) is None:  # (also a constructor that refused its arguments: __del__ still runs)
            return
        try:
            with torch.cuda.device(self.device):
                torch.cuda.synchronize()
                for r in range(self.world):
                    if r != self.rank and self._peer["ptrs"][r]:
                        self.lib.b200pets_peer_close(C.c_void_p(self._peer["ptrs"][r]), 0)
                self.lib.b200pets_peer_close(self._peer["own"], 1)
        except Exception:
            pass
        self._peer = None

    def __del__(self):
        self._close_peers()

    def _buffers(self, shape):
        dims = int(np.prod(shape))
        key = (tuple(shape), self.local_population)
        if self._buf is None or self._buf["key"] != key:
            dev, n_loc, k = self.device, self.local_population, self.k_local
            nbytes = max(self.lib.b200pets_cem_update_workspace_bytes(n_loc, dims, k),
                         self.lib.b200pets_cem_update_workspace_bytes(k * self.world, dims, self.elite_num))
            self._buf = {
                "key": key,
                "mu": torch.empty(dims, device=dev), "disp": torch.empty(dims, device=dev),
                "best_val": torch.empty(1, device=dev), "best_sol": torch.empty(dims, device=dev),
                "pop": torch.empty((n_loc,) + tuple(shape), device=dev),
                "records": torch.empty(k, 1 + dims, device=dev),
                "values": torch.empty(n_loc, dtype=torch.float32, device=dev),
                "ws": torch.empty(nbytes, dtype=torch.uint8, device=dev),
            }
        return self._buf

    def optimize(self, obj_fun: Callable[[torch.Tensor], torch.Tensor], x0: torch.Tensor,
                 callback: Optional[Callable] = None) -> torch.Tensor:
        dev = self.device
        x0 = x0.to(dev, torch.float32).contiguous()
        shape = tuple(x0.shape)
        dims = int(np.prod(shape))
        n_loc, k = self.local_population, self.k_local
        b = self._buffers(shape)
        mu, disp, best_val, best_sol, pop, records, ws = (b["mu"], b["disp"], b["best_val"], b["best_sol"], b["pop"],
                                                          b["records"], b["ws"])
        mu.copy_(x0.reshape(-1))
        disp.copy_((((self.upper_bound - self.lower_bound) ** 2) / 16).reshape(-1))
        best_val.fill_(float("-inf"))
        nbytes = ws.numel()
        self._offset += 1
        from .planning import _FusedObjective

        fused = obj_fun if isinstance(obj_fun, _FusedObjective) and obj_fun.model_env.ts1 == "tile_shuffle" else None
        values = b["values"]
        if self.record_values:
            self.last_values = torch.empty(self.num_iterations, n_loc, device=dev)
        if fused is not None:
            env = fused.model_env
            env._fresh()
            prop = env._propagation()
            H = shape[0]
            # the same (seed, offset) on every rank: draws are keyed by GLOBAL sequence / row / group indices
            call = env._next_offset()
            rcfg = _lib.RolloutCfg(n_loc, H, fused.num_particles, _lib.PREC[env.precision_for(prop)], _lib.PROP[prop],
                                   _lib.TS1_TILE_SHUFFLE, env._seed, 0, self.local_offset, self.population_size)
            obs0 = env._obs_to_device(fused.obs)
            eval_ws = env._workspace(self.lib.b200pets_eval_workspace_bytes(env.staged.handle, C.byref(rcfg)))
            seed = env._seed
        else:
            call = self._offset
            seed = self._seed
        peer = self._setup_peers(dims)
        with torch.cuda.device(dev):
            stream = _lib.stream_ptr()
            for i in range(self.num_iterations):
                off = call * 1024 + i
                if peer is None or i == 0:  # (peer path: later populations are drawn by the refit kernel)
                    _lib.check(self.lib.b200pets_cem_sample_shard(
                        n_loc, self.local_offset, dims, _lib.ptr(mu), _lib.ptr(disp), _lib.ptr(self.lower_bound),
                        _lib.ptr(self.upper_bound), None, seed, off, 0, _lib.ptr(pop), stream), "cem_sample_shard")
                if fused is not None:  # ModelEnv objective: one C call, no per-iteration host staging
                    rcfg.offset = off
                    _lib.check(self.lib.b200pets_eval_sequences(env.staged.handle, C.byref(rcfg), _lib.ptr(obs0), _lib.ptr(pop), None,
                                                                None, _lib.ptr(values), None, _lib.ptr(eval_ws), eval_ws.numel(),
                                                                stream), "eval_sequences")
                else:
                    values = obj_fun(pop).to(dev, torch.float32).contiguous()
                if callback is not None:
                    callback(pop, values, i)
                if self.record_values:
                    self.last_values[i].copy_(values)
                if peer is not None:
                    # values -> every rank over NVLink + flag; the refit kernel waits for them, selects the GLOBAL elites, ships
                    # the rows this rank owns, waits for everybody's, refits and draws the next shard: two launches after the
                    # rollout and no host-issued collective on the iteration's critical path
                    self._epoch += 1
                    if self.comm_events is not None:
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                    _lib.check(self.lib.b200pets_cem_values_push(n_loc, dims, self.elite_num, _lib.ptr(values), self.rank, self.world,
                                                                 self._epoch, peer["ptrs"], stream), "cem_values_push")
                    more = 1 if i + 1 < self.num_iterations else 0
                    _lib.check(self.lib.b200pets_cem_elites_refit(
                        n_loc, self.local_offset, dims, self.elite_num, float(self.alpha), 0, self.rank, self.world, self._epoch,
                        peer["ptrs"], _lib.ptr(pop), _lib.ptr(mu), _lib.ptr(disp), _lib.ptr(best_val), _lib.ptr(best_sol), more,
                        _lib.ptr(self.lower_bound), _lib.ptr(self.upper_bound), seed, call * 1024 + i + 1, 0, _lib.ptr(peer["tag"]),
                        _lib.ptr(pop), stream), "cem_elites_refit")
                    if self.comm_events is not None:  # (exchange + select + refit + next population: the waits are in here)
                        e1.record()
                        self.comm_events.append((e0, e1))
                    continue
                _lib.check(self.lib.b200pets_cem_local_topk(n_loc, dims, k, _lib.ptr(pop), _lib.ptr(values), _lib.ptr(records),
                                                            _lib.ptr(ws), nbytes, stream), "cem_local_topk")
                if self.comm_events is not None:
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                allrec = self._gather(records)  # <- the single collective of this iteration
                if self.comm_events is not None:
                    e1.record()
                    self.comm_events.append((e0, e1))
                _lib.check(self.lib.b200pets_cem_update_from_records(
                    allrec.shape[0], dims, self.elite_num, float(self.alpha), 1, 0, _lib.ptr(allrec), _lib.ptr(mu),
                    _lib.ptr(disp), _lib.ptr(best_val), _lib.ptr(best_sol), None, _lib.ptr(ws), nbytes, stream),
                    "cem_update_from_records")
        out = mu if self.return_mean_elites else best_sol
        return out.view(shape).clone()
