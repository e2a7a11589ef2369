"""Training MBPO's SAC agent from a device-resident copy of its rollout buffer (replay.DeviceTransitionMirror,
``b200pets_transition_gather`` / ``_scatter``, ``b200pets_sac_update_many``, ``mbpo.update_agent``), compared with
``torch.equal`` throughout:

* the gather kernel, row for row against numpy's packing, at B = 1, 255, 256 and 257, with rows on both sides of chunk
  boundaries, float32 and float64 buffers, and nothing written past its output;
* ``rollout_model_and_populate_sac_buffer`` into a mirrored buffer: the device rows equal the host rows after every
  rollout, across the ring's wrap, a rollout larger than the capacity and ``maybe_replace_sac_buffer``, and the next
  ``flush()`` copies no row;
* at the five shipped MBPO shapes, entropy tuning on and off and target intervals 1 and 4: 50 mirrored
  ``update_parameters`` against 50 unmirrored ones, and ``update_agent`` (mirrored, and unmirrored through its host
  packing) against the same 50 sequential ``update_parameters``: parameters, targets, Adam moments and steps,
  ``log_alpha``, every logged value and the generators' states are equal;
* ``update_agent`` mixing an unmirrored real buffer and the mirrored rollout buffer (``real_data_ratio`` 0.5) against
  the reference loop;
* the draws injected through ``update_many`` still give the float64 oracle's update (oracle/sac_f64.py).
"""
import os
import sys
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import test_gpu_sac as base  # noqa: E402  its agent, oracle and comparison helpers
from baseline import reference_arm as ra  # noqa: E402
from mbrl_lib_b200 import mbpo, replay  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
mbrl, REF_SRC = ra.import_reference()
needs_ref = pytest.mark.skipif(mbrl is None, reason=f"reference not importable here: {REF_SRC}")
SHAPES = [  # the shipped MBPO configs' obs / act / hidden
    ("cartpole", 4, 1, 256), ("hopper", 11, 3, 512), ("halfcheetah", 17, 6, 512), ("ant", 27, 8, 1024),
    ("humanoid", 45, 17, 1024)]


def _rb():
    from mbrl.util.replay_buffer import ReplayBuffer

    return ReplayBuffer


def _filled(capacity, rows, D, A, seed, dtype=np.float32, rng_seed=0):
    buf = _rb()(capacity, (D,), (A,), obs_type=dtype, action_type=dtype, reward_type=dtype,
                rng=np.random.default_rng(rng_seed))
    g = np.random.default_rng(seed)
    buf.add_batch(g.standard_normal((rows, D)), g.uniform(-1, 1, (rows, A)), g.standard_normal((rows, D)),
                  g.standard_normal(rows), g.random(rows) < 0.1, np.zeros(rows, bool))
    return buf


def _host_rows(buf, rows, D, A):
    out = np.empty((len(rows), 2 * D + A + 2), np.float32)
    replay.pack_rows(buf, rows, out, D, A)
    return torch.from_numpy(out)


def _device_store(m, n):
    """Rows [0, n) of the mirror, chunk by chunk, on the host."""
    step = 1 << m.chunk_shift
    return torch.cat([m.device_rows(lo, min(n, lo + step)).cpu() for lo in range(0, n, step)])


# ---- the gather -------------------------------------------------------------------------------------------------------

@needs_ref
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("B", [1, 255, 256, 257])
def test_gather_matches_numpy_row_for_row(B, dtype):
    D, A = 11, 3
    buf = _filled(1000, 900, D, A, seed=B, dtype=dtype)
    m = replay.mirror_transitions_to_device(buf, DEV, _rows_per_chunk=64)
    try:
        assert m.flush() == 900
        g = np.random.default_rng(B)
        edges = np.array([0, 63, 64, 127, 128, 511, 512, 895, 899])  # both sides of chunk boundaries
        idx = np.concatenate([edges, g.integers(0, 900, max(0, B - len(edges)))])[:B]
        out = torch.full((B + 8, m.width), float("nan"), device=DEV)
        m.gather(torch.from_numpy(idx).to(DEV), out[:B])
        got = out.cpu()
        assert torch.equal(got[:B], _host_rows(buf, idx, D, A))
        assert torch.isnan(got[B:]).all()  # nothing past the output
    finally:
        m.close()


# ---- the rollout's scatter --------------------------------------------------------------------------------------------

def _model_env(term):
    import mbrl_lib_b200 as bp
    from mbrl_lib_b200 import functions, synthetic as syn

    spec = syn.CASES["halfcheetah_small"]
    model = bp.model_from_arrays(spec, syn.make_model_arrays(spec), DEV)

    class Env:
        observation_space = base.Box(spec.obs_dim, -np.inf, np.inf)
        action_space = base.Box(spec.act_dim)

    env = bp.ModelEnv(Env(), model, getattr(functions, term), functions.reward_halfcheetah,
                      generator=torch.Generator(device=DEV).manual_seed(0))
    return env, spec.obs_dim, spec.act_dim


@needs_ref
@pytest.mark.parametrize("capacity,term", [(700, "term_hopper"), (250, "no_termination")])
def test_rollouts_land_in_the_mirror(capacity, term):
    """Rollouts of up to 300 rows: with terminations (the done column) over 8 rollouts the ring wraps; without, every
    rollout writes more rows than a capacity of 250 holds."""
    env, D, A = _model_env(term)
    agent = types.SimpleNamespace(sac_agent=base._agent(D, A, 256, seed=3))
    real = _filled(2000, 1000, D, A, seed=4, rng_seed=5)
    sac_buf = mbpo.maybe_replace_sac_buffer(None, (D,), (A,), capacity, seed=6)
    m = replay.mirror_transitions_to_device(sac_buf, DEV, _rows_per_chunk=128)
    copied = []

    def check(buf, mirror):
        n = buf.num_stored
        assert torch.equal(_device_store(mirror, n), _host_rows(buf, np.arange(n), D, A))
        copied.append(mirror.flush())

    for _ in range(8):  # 100 rows x 3 steps per rollout, less what terminates (step 0 keeps all 100)
        mbpo.rollout_model_and_populate_sac_buffer(env, real, agent, sac_buf, True, 3, 100)
        check(sac_buf, m)
    assert sac_buf.num_stored == capacity  # it wrapped
    assert sac_buf.terminated.any() == (term != "no_termination")
    new = mbpo.maybe_replace_sac_buffer(sac_buf, (D,), (A,), capacity + 300, seed=6)
    assert replay.find_transition_mirror(sac_buf) is None
    m2 = replay.find_transition_mirror(new)
    assert m2 is not None and m2.device == m.device
    assert m2.flush() == new.num_stored  # the replacement's rows go up once
    check(new, m2)
    mbpo.rollout_model_and_populate_sac_buffer(env, real, agent, new, True, 3, 100)
    check(new, m2)
    assert copied == [0] * len(copied)
    m2.close()


# ---- the updates ------------------------------------------------------------------------------------------------------

class Log:
    def __init__(self):
        self.calls = []

    def log(self, key, value, step):
        self.calls.append((key, value, step))

    def dump(self, step, save=False):
        self.calls.append(("dump", step, save))


def _contract(agent):
    """Every tensor the update changes: parameters, targets, Adam moments and steps, log_alpha."""
    out = [p.detach().clone() for p in list(agent.critic.parameters()) + list(agent.critic_target.parameters())
           + list(agent.policy.parameters())]
    for opt, ps in agent._optimizers():
        for p in ps:
            st = opt.state[p]
            out += [st["step"].clone(), st["exp_avg"].clone(), st["exp_avg_sq"].clone()]
    if agent.automatic_entropy_tuning:
        out.append(agent.log_alpha.detach().clone())
    return out


def _assert_same(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), f"tensor {i} differs"


def _reference_loop(agent, replay_buffer, sac_buffer, rng, n, ratio, B, updates_made, logger, freq):
    for _ in range(n):  # mbrl/algorithms/mbpo.py:258-275
        use_real_data = rng.random() < ratio
        which = replay_buffer if use_real_data else sac_buffer
        if len(which) < B:
            break
        agent.sac_agent.update_parameters(which, B, updates_made, logger, reverse_mask=True)
        updates_made += 1
        if updates_made % freq == 0:
            logger.dump(updates_made, save=True)
    return updates_made


@needs_ref
@pytest.mark.parametrize("tuning,interval", [(False, 1), (True, 1), (False, 4), (True, 4)])
@pytest.mark.parametrize("name,D,A,H", SHAPES)
def test_mirrored_and_many_updates_equal_sequential_updates(name, D, A, H, tuning, interval):
    B, n_updates, per_step = 256, 50, 25
    runs = {}
    for kind in ("host", "mirror", "many_mirror", "many_host"):
        agent = types.SimpleNamespace(sac_agent=base._agent(D, A, H, seed=D + H, tuning=tuning, interval=interval))
        rng = np.random.default_rng(1)
        buf = _filled(5000, 4000, D, A, seed=2, rng_seed=3)
        if kind in ("mirror", "many_mirror"):
            replay.mirror_transitions_to_device(buf, DEV, _rows_per_chunk=1024)
        log = Log()
        made = 0
        while made < n_updates:
            if kind.startswith("many"):
                made = mbpo.update_agent(agent, None, buf, rng, per_step, 0.0, B, True, made, logger=log,
                                         log_frequency=10)
            else:
                made = _reference_loop(agent, None, buf, rng, per_step, 0.0, B, made, log, 10)
        assert made == n_updates
        runs[kind] = (_contract(agent.sac_agent), log.calls, rng.bit_generator.state, buf._rng.bit_generator.state,
                      agent.sac_agent._updates_done)
        m = replay.find_transition_mirror(buf)
        if m is not None:
            m.close()
    want = runs["host"]
    assert len(want[1]) == n_updates * 7 + n_updates // 10
    for kind in ("mirror", "many_mirror", "many_host"):
        got = runs[kind]
        _assert_same(got[0], want[0])
        assert got[1] == want[1], kind
        assert got[2:] == want[2:], kind


@needs_ref
def test_update_agent_mixes_a_host_and_a_mirrored_buffer():
    D, A, H, B = 17, 6, 512, 256
    runs = {}
    for kind in ("reference", "ours"):
        agent = types.SimpleNamespace(sac_agent=base._agent(D, A, H, seed=7, tuning=True, interval=4))
        rng = np.random.default_rng(8)
        real = _filled(3000, 2000, D, A, seed=9, dtype=np.float64)
        real._rng = rng  # mbpo.train builds the real buffer on the loop's generator
        sac_buf = _filled(5000, 4000, D, A, seed=10, rng_seed=11)
        replay.mirror_transitions_to_device(sac_buf, DEV)
        log = Log()
        made = 0
        for _ in range(3):
            if kind == "reference":
                made = _reference_loop(agent, real, sac_buf, rng, 20, 0.5, B, made, log, 7)
            else:
                made = mbpo.update_agent(agent, real, sac_buf, rng, 20, 0.5, B, True, made, logger=log, log_frequency=7)
        runs[kind] = (_contract(agent.sac_agent), log.calls, made, rng.bit_generator.state,
                      sac_buf._rng.bit_generator.state)
        replay.find_transition_mirror(sac_buf).close()
    _assert_same(runs["ours"][0], runs["reference"][0])
    assert runs["ours"][1:] == runs["reference"][1:]
    assert runs["ours"][2] == 60


@needs_ref
@pytest.mark.parametrize("D,A,H,B,tuning,reverse", [(17, 6, 512, 256, True, False), (27, 8, 1024, 256, False, True)])
def test_injected_draws_through_update_many_match_float64(D, A, H, B, tuning, reverse):
    """test_gpu_sac.py's one-update cases (same agent, Adam state, batch and draws), the batch gathered from a mirror."""
    agent = base._agent(D, A, H, seed=D * 100 + H + B, tuning=tuning,
                        box=base.Box(A, -np.linspace(1, 2, A), np.linspace(1, 3, A)))
    base._prefill(agent, seed=B)
    batch = base._batch(B, D, A, seed=B + D)
    buf = _rb()(2 * B, (D,), (A,), obs_type=np.float64, action_type=np.float64, reward_type=np.float64)
    buf.add_batch(*batch.astuple())
    m = replay.mirror_transitions_to_device(buf, DEV)
    try:
        eps = torch.randn(2, B, A, generator=torch.Generator().manual_seed(5)).to(DEV)
        before = base._snapshot(agent)
        want = base._oracle(agent, before, batch, eps, 0, reverse)
        stats = agent.update_many([(buf, np.arange(B))], B, 0, reverse_mask=reverse, _eps=eps[None])
        base._compare(f"update_many,{D},{tuning}", before, base._snapshot(agent), want, fresh=False)
        for got, w in zip(stats[0][:5].tolist(), want["stats"][:5]):
            assert abs(got - w) <= 1e-5 * max(1.0, abs(w))
    finally:
        m.close()
