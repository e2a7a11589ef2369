"""CPU-only checks of the fused iCEM plan's host side: the torch generator draws it makes before its one C call follow the
per-iteration loop's schedule (which iterations draw a kept-elite permutation and an evaluation's permutations, of which
sizes, in which order), and ``b200pets_icem_plan`` refuses bad arguments before its first launch."""
import ctypes as C

import pytest
import torch

import mbrl_lib_b200 as bp
from mbrl_lib_b200 import _lib


class _StubEnv:
    """Records the ``_eval_perms`` calls the draws make and returns no permutations."""

    def __init__(self, log):
        self.log = log

    def _eval_perms(self, prop, population, horizon, particles):
        self.log.append(("eval", prop, population, horizon, particles))
        return None


def _draws(opt, monkeypatch, horizon=10, particles=20):
    log = []
    real = torch.randperm

    def randperm(n, *args, **kwargs):
        log.append(("keep", n))
        return real(n, *args, **kwargs)

    monkeypatch.setattr(torch, "randperm", randperm)
    rows, keep_index, perms = opt._fused_draws(_StubEnv(log), "random_model", horizon, particles)
    monkeypatch.setattr(torch, "randperm", real)
    return log, rows, keep_index, perms


def _cartpole(iters=5):
    """pets_icem_cartpole's optimiser: population 200 decaying by 1.3, 20 elites, keep 0.3 rounded up to module 7."""
    return bp.ICEMOptimizer(iters, 0.1, 200, 1.3, 2.0, [[-1.0]] * 10, [[1.0]] * 10, 0.3, 0.1, "cpu", population_size_module=7)


def test_first_call_draws_like_the_loop(monkeypatch):
    opt = _cartpole()
    assert opt.population_sizes() == [203, 154, 119, 98, 77] and opt.elite_num == 20 and opt.keep_elite_size == 7
    log, rows, keep_index, perms = _draws(opt, monkeypatch)
    # no elites yet at iteration 0; kept elites at 1-3; the mean as the one extra row of the last iteration
    assert log == [("eval", "random_model", 203, 10, 20),
                   ("keep", 20), ("eval", "random_model", 161, 10, 20),
                   ("keep", 20), ("eval", "random_model", 126, 10, 20),
                   ("keep", 20), ("eval", "random_model", 105, 10, 20),
                   ("eval", "random_model", 78, 10, 20)]
    assert rows == [203, 161, 126, 105, 78] and perms == [None] * 5
    assert keep_index.shape == (5, 7) and keep_index.dtype == torch.int64


def test_carried_elites_draw_at_iteration_zero(monkeypatch):
    opt = _cartpole()
    opt.elite = torch.zeros(20, 10, 1)
    log, rows, keep_index, _ = _draws(opt, monkeypatch)
    assert [e[0] for e in log] == ["keep", "eval"] * 4 + ["eval"]
    assert rows == [210, 161, 126, 105, 78]
    # the permutation of iteration i is the one drawn right before its evaluation
    torch.manual_seed(3)
    opt.elite = torch.zeros(20, 10, 1)
    _, _, first, _ = _draws(opt, monkeypatch)
    torch.manual_seed(3)
    want = [torch.randperm(20)[:7] for _ in range(4)]
    assert all(torch.equal(first[i], want[i]) for i in range(4))


@pytest.mark.parametrize("iters,carried,expect", [
    (1, False, ([("eval", 203)], [203])),  # one iteration: never a mean row, no elites yet
    (1, True, ([("keep", 20), ("eval", 210)], [210])),  # one iteration with carried elites: kept, shifted
    (2, False, ([("eval", 203), ("eval", 155)], [203, 155])),
    (2, True, ([("keep", 20), ("eval", 210), ("eval", 155)], [210, 155])),
])
def test_short_plans(monkeypatch, iters, carried, expect):
    opt = _cartpole(iters)
    if carried:
        opt.elite = torch.zeros(20, 10, 1)
    log, rows, keep_index, _ = _draws(opt, monkeypatch)
    assert [e if e[0] == "keep" else (e[0], e[2]) for e in log] == expect[0] and rows == expect[1]
    assert (keep_index is None) == (not carried and iters <= 2)


def test_keep_rounded_above_elite_num_and_no_keep(monkeypatch):
    lb, ub = [[-1.0]] * 8, [[1.0]] * 8
    opt = bp.ICEMOptimizer(3, 0.1, 30, 1.3, 2.0, lb, ub, 0.5, 0.1, "cpu", population_size_module=7)
    assert opt.population_sizes() == [35, 28, 21] and opt.elite_num == 3 and opt.keep_elite_size == 7
    log, rows, keep_index, _ = _draws(opt, monkeypatch, horizon=8, particles=5)
    assert rows == [35, 31, 22] and keep_index.shape == (3, 3)  # only the 3 elites that exist are kept
    assert [e[0] for e in log] == ["eval", "keep", "eval", "eval"]
    opt = bp.ICEMOptimizer(3, 0.1, 100, 1.3, 2.0, lb, ub, 0.0, 0.1, "cpu")
    log, rows, keep_index, _ = _draws(opt, monkeypatch, horizon=8, particles=5)
    assert keep_index is None and rows == [100, 77, 61]
    assert [e[0] for e in log] == ["eval", "keep", "eval", "eval"]  # the loop draws the permutation of no rows too


# A plan that refused too late would launch on the dummy pointers below, so this runs only where there is no device.
@pytest.mark.skipif(torch.cuda.is_available(), reason="checks that no call reaches a device")
def test_plan_refuses_before_launching():
    lib = _lib.load()
    d = _lib.ModelDesc()
    d.ensemble_size, d.num_members, d.obs_dim, d.act_dim = 7, 5, 17, 6
    d.in_size, d.out_size, d.hid_size, d.num_hidden = 23, 18, 200, 4
    d.learned_rewards, d.reward_fn, d.term_fn = 1, _lib.REWARD["learned"], _lib.TERM["no_termination"]
    block = C.create_string_buffer(4096)  # the descriptor is the handle's first member; the checks read nothing else
    C.memmove(block, C.byref(d), C.sizeof(d))
    h = C.cast(block, C.c_void_p)
    dummy = C.c_void_p(16)
    sizes = (C.c_int32 * 3)(100, 77, 60)

    def plan(horizon=8, particles=5, elite_num=10, keep=3, iters=3, s=sizes, first_sequence=0, external=False):
        r = _lib.RolloutCfg(0, horizon, particles, _lib.PREC["f32"], _lib.PROP["random_model"], _lib.TS1_TILE_SHUFFLE, 1, 2,
                            first_sequence, 0)
        c = _lib.IcemCfg(iters, elite_num, keep, 0.1, 2.0, 1, 7, 1)
        d.reward_fn = _lib.REWARD["external"] if external else _lib.REWARD["learned"]
        C.memmove(block, C.byref(d), C.sizeof(d))
        return lib.b200pets_icem_plan(h, C.byref(r), C.byref(c), s, dummy, dummy, dummy, dummy, None, None, None, dummy, dummy,
                                      None, dummy, 1 << 40, None)

    def refused(rc, text, code=-1):
        assert rc == code and text in lib.b200pets_last_error().decode(), (rc, lib.b200pets_last_error().decode())

    refused(plan(iters=0), "num_iterations")
    refused(plan(horizon=1), "horizon of at least 2")
    refused(plan(keep=11), "kept elites")
    refused(plan(elite_num=62), "62 elites of a smallest population of 61")  # rows 100, 80, 61
    refused(plan(particles=1), "multiple of the number of models")
    refused(plan(first_sequence=5), "sharded", -2)
    refused(plan(external=True), "external reward/termination", -2)
    refused(plan(s=None), "null argument")
    r = _lib.RolloutCfg(0, 8, 5, 0, 0, 1, 1, 2, 0, 0)
    assert lib.b200pets_icem_plan_workspace_bytes(h, C.byref(r), C.byref(_lib.IcemCfg(0, 10, 3, 0.1, 2.0, 1, 7, 1)), sizes) == 0
    assert lib.b200pets_icem_plan_workspace_bytes(h, C.byref(r), C.byref(_lib.IcemCfg(3, 10, 3, 0.1, 2.0, 1, 7, 1)), sizes) > 0
