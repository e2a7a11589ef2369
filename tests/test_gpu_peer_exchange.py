"""The peer-memory exchange kernels of the sharded CEM (csrc/cem.cu: cem_values_push_kernel, cem_elites_refit_sample_kernel)
on ONE GPU, so that the single-GPU suite covers them (tests/test_gpu_multi.py needs two):

* world = 1: values push + global select + elite push + refit + next population must equal, bit for bit,
  b200pets_cem_update (the single-GPU refit) followed by b200pets_cem_sample_shard on the refitted distribution;
* world = 2 emulated in one process: two "ranks" with their own buffers, kernels on two streams (they wait for each other's
  flags, so they must be co-resident: two single-CTA selects + sampling CTAs fit an H100 many times over); both must end
  with the refit of the UNION population and draw their own shard of the next one.
NaNs, ties at the selection threshold and a -inf are in the values on purpose.
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from mbrl_lib_b200 import _lib  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _problem(n, dims, seed=0):
    g = torch.Generator().manual_seed(seed)
    pop = torch.rand(n, dims, generator=g) * 2 - 1
    values = torch.randn(n, generator=g)
    values[7] = float("nan")
    values[n // 2] = float("nan")
    values[11] = values[3]          # ties ...
    values[n - 5:] = values[n - 6]  # ... a run of equal values that straddles the elite threshold when it is an elite
    values[19] = float("-inf")
    mu = torch.rand(dims, generator=g) * 0.2 - 0.1
    disp = torch.rand(dims, generator=g) * 0.2 + 0.05
    lb, ub = -torch.ones(dims), torch.ones(dims)
    return pop, values, mu, disp, lb, ub


def _single_gpu_reference(lib, pop, values, mu, disp, lb, ub, k, alpha, seed, offset, first, n_next):
    """b200pets_cem_update on the whole population, then the next population shard [first, first + n_next)."""
    n, dims = pop.shape
    pop_d, val_d, mu_d, disp_d = pop.to(DEV), values.to(DEV).clone(), mu.to(DEV).clone(), disp.to(DEV).clone()
    best_v = torch.full((1,), float("-inf"), device=DEV)
    best_s = torch.zeros(dims, device=DEV)
    ws = torch.empty(lib.b200pets_cem_update_workspace_bytes(n, dims, k), dtype=torch.uint8, device=DEV)
    _lib.check(lib.b200pets_cem_update(n, dims, k, alpha, 1, 0, _lib.ptr(pop_d), _lib.ptr(val_d), _lib.ptr(mu_d), _lib.ptr(disp_d),
                                       _lib.ptr(best_v), _lib.ptr(best_s), None, None, _lib.ptr(ws), ws.numel(), _lib.stream_ptr()))
    nxt = torch.empty(n_next, dims, device=DEV)
    lb_d, ub_d = lb.to(DEV), ub.to(DEV)  # (kept alive until the synchronize: the launch only takes their addresses)
    _lib.check(lib.b200pets_cem_sample_shard(n_next, first, dims, _lib.ptr(mu_d), _lib.ptr(disp_d), _lib.ptr(lb_d),
                                             _lib.ptr(ub_d), None, seed, offset, 0, _lib.ptr(nxt), _lib.stream_ptr()))
    torch.cuda.synchronize()
    return mu_d.cpu(), disp_d.cpu(), best_v.cpu(), best_s.cpu(), nxt.cpu(), val_d.cpu()


def _alloc(lib, world, n_loc, dims, k):
    nbytes = lib.b200pets_peer_buffer_bytes(world, n_loc, dims, k)
    assert nbytes > 0
    ptr, handle = C.c_void_p(), C.create_string_buffer(64)
    _lib.check(lib.b200pets_peer_alloc(nbytes, C.byref(ptr), handle))
    return ptr


@pytest.mark.parametrize("n,dims,k", [(500, 180, 50), (96, 12, 7), (3000, 30, 300)])
def test_peer_exchange_world1_equals_single_gpu_refit(n, dims, k):
    lib = _lib.load()
    pop, values, mu, disp, lb, ub = _problem(n, dims)
    alpha, seed, offset = 0.1, 1234, 77
    want = _single_gpu_reference(lib, pop, values, mu, disp, lb, ub, k, alpha, seed, offset, 0, n)
    buf = _alloc(lib, 1, n, dims, k)
    try:
        ptrs = (C.c_void_p * 1)(buf.value)
        pop_d, val_d, mu_d, disp_d = pop.to(DEV), values.to(DEV).clone(), mu.to(DEV).clone(), disp.to(DEV).clone()
        lb_d, ub_d = lb.to(DEV), ub.to(DEV)
        best_v = torch.full((1,), float("-inf"), device=DEV)
        best_s = torch.zeros(dims, device=DEV)
        tag = torch.zeros(1, dtype=torch.int32, device=DEV)
        nxt = torch.empty(n, dims, device=DEV)
        for epoch in (1, 2):  # twice: both parities of the tables, and the second refit starts from the first one's result
            _lib.check(lib.b200pets_cem_values_push(n, dims, k, _lib.ptr(val_d), 0, 1, epoch, ptrs, _lib.stream_ptr()))
            _lib.check(lib.b200pets_cem_elites_refit(n, 0, dims, k, alpha, 0, 0, 1, epoch, ptrs, _lib.ptr(pop_d), _lib.ptr(mu_d),
                                                     _lib.ptr(disp_d), _lib.ptr(best_v), _lib.ptr(best_s), 1, _lib.ptr(lb_d),
                                                     _lib.ptr(ub_d), seed, offset, 0, _lib.ptr(tag), _lib.ptr(nxt), _lib.stream_ptr()))
            torch.cuda.synchronize()
            if epoch == 1:
                got = (mu_d.cpu(), disp_d.cpu(), best_v.cpu(), best_s.cpu(), nxt.cpu(), val_d.cpu())
                exact = n <= 2048  # above, the single-GPU refit sums the elites in 32 interleaved partial sums (another rounding)
                for name, g, w in zip(("mu", "disp", "best_value", "best_solution", "next population", "values (NaN rule)"), got, want):
                    if exact or name in ("best_value", "best_solution", "values (NaN rule)"):
                        assert torch.equal(g, w, ) or (torch.isnan(g) == torch.isnan(w)).all() and torch.equal(torch.nan_to_num(g), torch.nan_to_num(w)), \
                            f"{name} differs from the single-GPU refit: max |diff| {(g - w).abs().max()}"
                    else:
                        assert torch.allclose(g, w, rtol=1e-5, atol=1e-6), f"{name}: max |diff| {(g - w).abs().max()}"
        # second refit over the same population from the first one's (mu, disp): the single-GPU path again
        want2 = _single_gpu_reference(lib, pop, values, got[0], got[1], lb, ub, k, alpha, seed, offset, 0, n)
        if n <= 2048:
            assert torch.equal(mu_d.cpu(), want2[0]) and torch.equal(disp_d.cpu(), want2[1])
        else:
            assert torch.allclose(mu_d.cpu(), want2[0], rtol=1e-5, atol=1e-6)
    finally:
        lib.b200pets_peer_close(buf, 1)


def test_peer_exchange_two_ranks_on_two_streams_equal_the_union_refit():
    lib = _lib.load()
    n, dims, k, world = 500, 180, 50, 2
    n_loc = n // world
    pop, values, mu, disp, lb, ub = _problem(n, dims, seed=5)
    alpha, seed, offset = 0.1, 99, 2049
    bufs = [_alloc(lib, world, n_loc, dims, k) for _ in range(world)]
    try:
        ptrs = (C.c_void_p * world)(*[b.value for b in bufs])  # same device: every "rank" sees every buffer directly
        streams = [torch.cuda.Stream(device=DEV) for _ in range(world)]
        state = []
        for r in range(world):
            sl = slice(r * n_loc, (r + 1) * n_loc)
            state.append(dict(pop=pop[sl].contiguous().to(DEV), val=values[sl].contiguous().to(DEV), mu=mu.to(DEV).clone(),
                              disp=disp.to(DEV).clone(), best_v=torch.full((1,), float("-inf"), device=DEV),
                              best_s=torch.zeros(dims, device=DEV), tag=torch.zeros(1, dtype=torch.int32, device=DEV),
                              nxt=torch.empty(n_loc, dims, device=DEV)))
        lb_d, ub_d = lb.to(DEV), ub.to(DEV)
        torch.cuda.synchronize()
        for r in range(world):  # enqueue both ranks; the kernels of one wait for the other's flags
            st = state[r]
            with torch.cuda.stream(streams[r]):
                sp = C.c_void_p(streams[r].cuda_stream)
                _lib.check(lib.b200pets_cem_values_push(n_loc, dims, k, _lib.ptr(st["val"]), r, world, 1, ptrs, sp))
                _lib.check(lib.b200pets_cem_elites_refit(n_loc, r * n_loc, dims, k, alpha, 0, r, world, 1, ptrs, _lib.ptr(st["pop"]),
                                                         _lib.ptr(st["mu"]), _lib.ptr(st["disp"]), _lib.ptr(st["best_v"]),
                                                         _lib.ptr(st["best_s"]), 1, _lib.ptr(lb_d), _lib.ptr(ub_d), seed, offset, 0,
                                                         _lib.ptr(st["tag"]), _lib.ptr(st["nxt"]), sp))
        torch.cuda.synchronize()
        for r in range(world):
            want = _single_gpu_reference(lib, pop, values, mu, disp, lb, ub, k, alpha, seed, offset, r * n_loc, n_loc)
            st = state[r]
            assert torch.equal(st["mu"].cpu(), want[0]) and torch.equal(st["disp"].cpu(), want[1]), f"rank {r}: refit differs"
            assert torch.equal(st["best_v"].cpu(), want[2]) and torch.equal(st["best_s"].cpu(), want[3]), f"rank {r}: best differs"
            assert torch.equal(st["nxt"].cpu(), want[4]), f"rank {r}: next population shard differs"
    finally:
        for b in bufs:
            lib.b200pets_peer_close(b, 1)
