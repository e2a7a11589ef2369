"""CPU-only checks of the CEM plan entry points: the single and the batched plan of the ensemble refuse a bad elite count
or a population the members do not divide before their first launch, and every single workspace query is its batched
query at one problem."""
import ctypes as C

import pytest
import torch

from mbrl_lib_b200 import _lib

# A plan that refused too late would launch on the dummy pointers below, so these run only where there is no device.
pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="checks that no call reaches a device")


def _handle(desc):
    """A host block standing in for an opaque model handle: the descriptor, which is the handle's first member, then
    zeros.  The checks read nothing else."""
    block = C.create_string_buffer(4096)
    C.memmove(block, C.byref(desc), C.sizeof(desc))
    return block, C.cast(block, C.c_void_p)


def _ensemble():
    d = _lib.ModelDesc()
    d.ensemble_size, d.num_members, d.obs_dim, d.act_dim = 7, 5, 17, 6
    d.in_size, d.out_size, d.hid_size, d.num_hidden = 23, 18, 200, 4
    d.learned_rewards, d.reward_fn, d.term_fn = 1, _lib.REWARD["learned"], _lib.TERM["no_termination"]
    return _handle(d)


def _cfg(population=50, particles=1):
    return _lib.RolloutCfg(population, 4, particles, _lib.PREC["f32"], _lib.PROP["random_model"], _lib.TS1_TILE_SHUFFLE,
                           1, 2, 0, 0)


def test_ensemble_plans_refuse_before_launching():
    lib = _lib.load()
    block, h = _ensemble()
    dummy = C.c_void_p(16)

    def single(rcfg, ccfg):
        return lib.b200pets_cem_plan(h, C.byref(rcfg), C.byref(ccfg), dummy, dummy, dummy, dummy, None, None, None, dummy,
                                     None, dummy, 1 << 30, None)

    def batch(rcfg, ccfg):
        return lib.b200pets_cem_plan_batch(h, C.byref(rcfg), C.byref(ccfg), 2, dummy, dummy, dummy, dummy, None, None, None,
                                           dummy, None, dummy, 1 << 30, None)

    for plan in (single, batch):
        for elites in (0, 51):
            assert plan(_cfg(), _lib.CemCfg(3, elites, 0.1, 0, 0)) == -1
            assert "elites" in lib.b200pets_last_error().decode()
        assert plan(_cfg(population=51), _lib.CemCfg(3, 5, 0.1, 0, 0)) == -1
        assert "multiple of the number of models" in lib.b200pets_last_error().decode()


def test_single_workspace_queries_are_the_batch_of_one():
    lib = _lib.load()
    block, h = _ensemble()
    ld = _lib.LatentDesc()
    ld.action_size, ld.latent_size, ld.belief_size, ld.hidden_size, ld.min_std = 6, 30, 200, 200, 0.1
    lblock, lh = _handle(ld)
    ccfg = _lib.CemCfg(5, 50, 0.1, 0, 0)
    for population, particles in ((50, 1), (500, 20), (1000, 1)):
        r = C.byref(_cfg(population, particles))
        pairs = [
            (lib.b200pets_eval_workspace_bytes(h, r), lib.b200pets_eval_batch_workspace_bytes(h, r, 1)),
            (lib.b200pets_cem_plan_workspace_bytes(h, r, C.byref(ccfg)),
             lib.b200pets_cem_plan_batch_workspace_bytes(h, r, C.byref(ccfg), 1)),
            (lib.b200pets_latent_eval_workspace_bytes(lh, r), lib.b200pets_latent_eval_batch_workspace_bytes(lh, r, 1)),
            (lib.b200pets_latent_cem_plan_workspace_bytes(lh, r, C.byref(ccfg)),
             lib.b200pets_latent_cem_plan_batch_workspace_bytes(lh, r, C.byref(ccfg), 1)),
        ]
        for one, batch_of_one in pairs:
            assert one == batch_of_one > 0
