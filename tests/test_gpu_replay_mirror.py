"""PlaNet's sequence batches from a device-resident mirror of the reference's own ``ReplayBuffer``
(mbrl_lib_b200/replay.py, csrc/replay.cu, the sequence path of trainer.py).

* Content: after mixed ``add`` / ``add_batch`` / ``load`` writes, with chunks of a few rows so that writes cross chunk
  boundaries, the device store is ``torch.equal`` to the host arrays, for uint8 and float32 frames.
* Gather: for uint8 and float32 frames at 3x64x64 (16-byte path), 3x15x15 (scalar path) and 4x8x20 (16-byte path, the
  uint8 kernel's last warp span partly past the frame), (B, T) in {(1, 2), (5, 8), (50, 50)}, sequences straddling chunks, the sampler's batches and the iterator's short last batch: the three outputs
  are ``torch.equal`` to ``latent_train._process_batch`` of the reference's own host batch, shifted as the loss shifts
  it; guard words after each output stay untouched.
* Drop-in, bit for bit: the sequence ``mbrl/algorithms/planet.py`` runs (5 trajectories of ``add``, a sequence sampler,
  ``train(num_epochs=1, batch_callback, evaluate=False)``, one more episode, train again), once mirrored and once not,
  from identical state: the callback's losses and meta, every parameter and Adam moment, and the buffer's rng are equal;
  the second flush copied only the new episode's rows.  Also with ``mirror_to_device``'s result discarded, as the
  one-line opt-in in planet.py discards it.  ``evaluate()`` over a ``SequenceTransitionIterator`` too.
* Fallbacks: an unmirrored buffer, a ``get_all(shuffle=True)`` copy and a mirror on another device take the host path;
  a bypassed ``cur_idx`` makes the flush resync; each gives the host path's results.
"""
import copy
import gc
import importlib
import tempfile
import types

import numpy as np
import pytest
import torch

import mbrl_lib_b200 as bp
from baseline import reference_arm as ra
from mbrl_lib_b200 import latent_train, models, replay, trainer as tr

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
mbrl, REF_SRC = ra.import_reference()
if mbrl is None:  # the reference travels with the build (oracle/_ref); these tests run it, so its absence is a failure
    raise RuntimeError(f"the reference is not importable: {REF_SRC}")
rb = importlib.import_module("mbrl.util.replay_buffer")
common = importlib.import_module("mbrl.util.common")

ENC = ((3, 8, 4, 2), (8, 16, 4, 2))  # 3 x 16 x 16 frames -> 16 x 2 x 2
DEC = ((32, 1, 1), ((32, 16, 5, 2), (16, 8, 5, 2), (8, 3, 4, 1)))
A, L, H, EP = 3, 8, 48, 30  # action, latent, belief = hidden sizes; episode length


def _frames(g, n, shape, dtype):
    """dmc2gym-style pixels: 5-bit values plus uniform noise below the quantum (float32), or plain bytes (uint8)."""
    if dtype == np.uint8:
        return g.integers(0, 256, (n, *shape), dtype=np.uint8)
    return (g.integers(0, 32, (n, *shape)) * 8 + g.uniform(0, 8, (n, *shape))).astype(np.float32)


def _stub(dev=DEV):
    return types.SimpleNamespace(parameters=lambda: iter([torch.empty(0, device=dev)]))


# ---- content -----------------------------------------------------------------------------------------------------------
def _check_content(buf, m):
    n = buf.num_stored
    assert m.rows_held == n
    for lo in range(0, n, 1 << m.chunk_shift):
        hi = min(n, lo + (1 << m.chunk_shift))
        assert torch.equal(m.device_obs(lo, hi).cpu(), torch.from_numpy(buf.obs[lo:hi])), (lo, hi)
    assert torch.equal(m.act[:n].cpu(), torch.from_numpy(buf.action[:n]).float().reshape(n, -1))
    assert torch.equal(m.rew[:n].cpu(), torch.from_numpy(buf.reward[:n]).float())


@pytest.mark.parametrize("dtype", [np.uint8, np.float32])
def test_device_store_equals_the_host_arrays(dtype):
    g = np.random.default_rng(1)
    shape = (3, 5, 7)
    buf = rb.ReplayBuffer(61, shape, (2,), obs_type=dtype, action_type=np.float64, reward_type=np.float64,
                          rng=np.random.default_rng(0))
    buf.add_batch(_frames(g, 9, shape, dtype), g.standard_normal((9, 2)), _frames(g, 9, shape, dtype),
                  g.standard_normal(9), np.zeros(9, bool), np.zeros(9, bool))
    m = replay.mirror_to_device(buf, DEV, _rows_per_chunk=8)
    try:
        assert m.chunk_shift == 3 and replay.mirror_to_device(buf, DEV) is m
        assert m.flush() == 9
        _check_content(buf, m)
        with tempfile.TemporaryDirectory() as tmp:
            for step in range(40):
                if step % 3 == 0:
                    n = int(g.integers(1, 30))
                    buf.add_batch(_frames(g, n, shape, dtype), g.standard_normal((n, 2)), _frames(g, n, shape, dtype),
                                  g.standard_normal(n), np.zeros(n, bool), np.zeros(n, bool))
                else:
                    buf.add(_frames(g, 1, shape, dtype)[0], g.standard_normal(2), _frames(g, 1, shape, dtype)[0],
                            float(g.standard_normal()), False, False)
                if step == 20:
                    buf.save(tmp)
                if step % 7 == 6:
                    m.flush()
                    _check_content(buf, m)
            buf.obs[:] = _frames(g, len(buf.obs), shape, dtype)  # overwritten, then restored by load
            buf.load(tmp)
            m.flush()
            _check_content(buf, m)
            buf.obs[3] = _frames(g, 1, shape, dtype)[0]  # a direct write: resync() picks it up
            assert m.resync() == buf.num_stored
            _check_content(buf, m)
        assert sum(c is not None for c in m._chunks) == len(m._chunks)  # all rows written by now
    finally:
        m.close()
    assert "add" not in buf.__dict__ and replay.find_mirror(buf.get_all()) is None


def test_chunks_are_allocated_when_first_written():
    shape = (3, 64, 64)
    buf = rb.ReplayBuffer(20000, shape, (A,), obs_type=np.float32, rng=np.random.default_rng(0))
    m = replay.mirror_to_device(buf, DEV)
    try:
        assert (1 << m.chunk_shift) == 1024  # 48 MiB of 3x64x64 float32 frames
        g = np.random.default_rng(0)
        for _ in range(1030):
            buf.add(_frames(g, 1, shape, np.float32)[0], np.zeros(A), _frames(g, 1, shape, np.float32)[0], 0.0, False,
                    False)
        m.flush()
        assert [c is not None for c in m._chunks[:3]] == [True, True, False] and len(m._chunks) == 20
        _check_content(buf, m)
    finally:
        m.close()


# ---- gather ------------------------------------------------------------------------------------------------------------
def _sequence_buffer(shape, dtype, trajectories, length, seed=0):
    g = np.random.default_rng(seed)
    buf = rb.ReplayBuffer(trajectories * length, shape, (A,), obs_type=dtype, rng=np.random.default_rng(seed),
                          max_trajectory_length=length)
    for _ in range(trajectories):
        for t in range(length):
            buf.add(_frames(g, 1, shape, dtype)[0], g.uniform(-1, 1, A).astype(np.float32),
                    _frames(g, 1, shape, dtype)[0], float(g.standard_normal()), False, t == length - 1)
    return buf


def _guarded(shape, guard=64):
    n = int(np.prod(shape))
    t = torch.full((n + guard,), float("nan"), device=DEV)
    t[n:] = 12345.0
    return t, t[:n].view(shape)


@pytest.mark.parametrize("dtype", [np.uint8, np.float32])
@pytest.mark.parametrize("frame", [(3, 64, 64), (3, 15, 15), (4, 8, 20)])
@pytest.mark.parametrize("B,T", [(1, 2), (5, 8), (50, 50)])
def test_gather_equals_the_reference_batch(dtype, frame, B, T):
    buf = _sequence_buffer(frame, dtype, trajectories=4, length=max(T + 10, 2 * B))
    m = replay.mirror_to_device(buf, DEV, _rows_per_chunk=16)  # sequences straddle chunks
    try:
        m.flush()
        for kind, kw in (("sampler", dict(use_simple_sampler=True, max_batches_per_loop_train=2)),
                         ("iterator", dict(shuffle_each_epoch=True))):
            ds, _ = common.get_sequence_buffer_iterator(buf, B, 0, T, **kw)
            twin = copy.deepcopy(ds)
            host = list(twin)
            starts = list(tr.sequence_starts(ds, kind))
            assert len(starts) == len(host)
            if kind == "iterator" and len(ds._valid_starts) % B:
                assert len(starts[-1]) < B  # the iterator's short last batch
            for st, hb in zip(starts, host):
                b = len(st)
                obs, act, rew = latent_train._process_batch(_stub(), hb)
                outs = [_guarded((b, T - 1, *frame)), _guarded((b, T - 1, A)), _guarded((b, T - 1))]
                m.gather(torch.from_numpy(st).to(DEV), T, *(o[1] for o in outs))
                for (full, got), want in zip(outs, (obs[:, 1:], act[:, :-1], rew[:, :-1])):
                    assert torch.equal(got, want.contiguous())
                    assert bool((full[got.numel():] == 12345.0).all())
    finally:
        m.close()


def test_gather_refuses_sequences_outside_the_store():
    buf = _sequence_buffer((3, 15, 15), np.uint8, trajectories=2, length=20)
    m = replay.mirror_to_device(buf, DEV)
    try:
        m.flush()
        g = replay.SequenceGather(m)
        g(np.array([0, 30], dtype=np.int64), 10, buf.num_stored)
        with pytest.raises(IndexError):
            g(np.array([0, 31], dtype=np.int64), 10, buf.num_stored)
        with pytest.raises(IndexError):
            g(np.array([-1], dtype=np.int64), 10, buf.num_stored)
    finally:
        m.close()


# ---- the trainer -------------------------------------------------------------------------------------------------------
@pytest.fixture
def deterministic():
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32, torch.backends.cudnn.deterministic,
           torch.backends.cudnn.benchmark)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    yield
    (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32, torch.backends.cudnn.deterministic,
     torch.backends.cudnn.benchmark) = old


@pytest.fixture
def gathers(monkeypatch):
    calls = []
    orig = replay.DeviceReplayMirror.gather
    monkeypatch.setattr(replay.DeviceReplayMirror, "gather", lambda self, *a: (calls.append(1), orig(self, *a))[1])
    return calls


def _setup(dtype=np.float32):
    torch.manual_seed(0)
    rng = torch.Generator(device=DEV)
    rng.manual_seed(9)
    model = models.PlaNetModel(A, L, H, H, device=DEV, obs_shape=(3, 16, 16), obs_encoding_size=32, encoder_config=ENC,
                               decoder_config=DEC, rng=rng)
    trainer = bp.ModelTrainer(model, optim_lr=1e-3, optim_eps=1e-4)
    buf = rb.ReplayBuffer(1000, (3, 16, 16), (A,), obs_type=dtype, rng=np.random.default_rng(3),
                          max_trajectory_length=EP)
    return model, trainer, buf


def _episode(buf, g, dtype=np.float32):
    for t in range(EP):
        buf.add(_frames(g, 1, (3, 16, 16), dtype)[0], g.uniform(-1, 1, A).astype(np.float32),
                _frames(g, 1, (3, 16, 16), dtype)[0], float(g.standard_normal()), False, t == EP - 1)


def _state(model, trainer, buf, record):
    return {"record": record, "params": [p.detach().clone() for p in model.parameters()],
            "moments": [(s["exp_avg"].clone(), s["exp_avg_sq"].clone(), float(s["step"]))
                        for s in trainer.optimizer.state.values()],
            "rng": copy.deepcopy(buf.rng.bit_generator.state)}


def _assert_same(a, b):
    assert len(a["record"]) == len(b["record"]) > 0
    for (ea, la, ma, wa), (eb, lb, mb, wb) in zip(a["record"], b["record"]):
        assert (ea, la, wa) == (eb, lb, wb)
        assert ma.keys() == mb.keys()
        for k in ma:
            if isinstance(ma[k], torch.Tensor):
                assert torch.equal(ma[k], mb[k]), k
            else:
                assert ma[k] == mb[k], k
    assert all(torch.equal(x, y) for x, y in zip(a["params"], b["params"]))
    assert len(a["moments"]) == len(b["moments"])
    for (m1, v1, s1), (m2, v2, s2) in zip(a["moments"], b["moments"]):
        assert torch.equal(m1, m2) and torch.equal(v1, v2) and s1 == s2
    assert a["rng"] == b["rng"]


def _planet_loop(mirror_fn=None, dtype=np.float32, between=None, dataset_fn=None):
    """What mbrl/algorithms/planet.py does with the model and the buffer, on a small model: 5 random trajectories,
    train on a sequence sampler with a batch_callback, one more episode, train again."""
    model, trainer, buf = _setup(dtype)
    mirror = mirror_fn(buf) if mirror_fn else None
    g = np.random.default_rng(7)
    record = []
    cb = lambda epoch, loss, meta, mode: record.append((epoch, loss, meta, mode))  # noqa: E731
    make = dataset_fn or (lambda b: common.get_sequence_buffer_iterator(b, 6, 0, 10, max_batches_per_loop_train=4,
                                                                        use_simple_sampler=True)[0])
    copied = []
    for _ in range(5):
        _episode(buf, g, dtype)
    trainer.train(make(buf), num_epochs=1, batch_callback=cb, evaluate=False)
    copied.append(mirror._rows_copied if mirror else None)
    _episode(buf, g, dtype)
    if between:
        between(buf, g)
    trainer.train(make(buf), num_epochs=1, batch_callback=cb, evaluate=False)
    copied.append(mirror._rows_copied if mirror else None)
    out = _state(model, trainer, buf, record)
    if mirror is not None:
        mirror.close()
    return out, copied, (model, trainer, buf)


@pytest.mark.parametrize("dtype", [np.float32, np.uint8])
def test_planet_loop_bit_for_bit(deterministic, gathers, dtype):
    host, _, _ = _planet_loop(dtype=dtype)
    assert not gathers
    dev, copied, _ = _planet_loop(lambda b: replay.mirror_to_device(b, DEV), dtype=dtype)
    assert len(gathers) == 8  # every batch of both train() calls was gathered
    assert copied == [5 * EP, EP]  # the second flush copied only the new episode
    _assert_same(host, dev)


def test_the_one_line_opt_in(deterministic, gathers):
    """``mirror_to_device(replay_buffer, device)`` with its result discarded, as planet.py would call it: the buffer
    keeps the mirror alive, and every batch is gathered from it."""
    def opt_in(b):
        replay.mirror_to_device(b, DEV)
        gc.collect()
        return None

    host, _, _ = _planet_loop()
    got, _, (_, _, buf) = _planet_loop(opt_in)
    assert len(gathers) == 8
    _assert_same(host, got)
    m = replay.find_mirror(buf.get_all())
    assert m is not None and m._rows_copied == EP  # the second train()'s flush: the new episode
    m.close()
    assert replay.find_mirror(buf.get_all()) is None and "add" not in buf.__dict__


def test_evaluate_over_a_sequence_iterator(deterministic, gathers):
    def make(b):
        return common.get_sequence_buffer_iterator(b, 7, 0, 9, shuffle_each_epoch=True)[0]

    results = []
    for mirrored in (False, True):
        model, trainer, buf = _setup()
        m = replay.mirror_to_device(buf, DEV) if mirrored else None
        g = np.random.default_rng(7)
        for _ in range(3):
            _episode(buf, g)
        ds = make(buf)
        seen = []
        score = trainer.evaluate(ds, batch_callback=lambda *a: seen.append(a))
        results.append((score, seen, copy.deepcopy(buf.rng.bit_generator.state)))
        if m:
            m.close()
    assert len(gathers) == len(results[1][1]) == len(results[0][1]) > 1
    assert torch.equal(results[0][0], results[1][0]) and results[0][2] == results[1][2]
    for a, b in zip(results[0][1], results[1][1]):
        assert torch.equal(a[0], b[0]) and torch.equal(a[1]["reconstruction"], b[1]["reconstruction"])


def test_fallbacks_give_the_host_results(deterministic, gathers):
    host, _, _ = _planet_loop()
    assert not gathers

    # an unmirrored buffer next to a mirrored one: the host path
    other = rb.ReplayBuffer(10, (3, 16, 16), (A,), rng=np.random.default_rng(0))
    om = replay.mirror_to_device(other, DEV)
    got, _, _ = _planet_loop()
    om.close()
    assert not gathers
    _assert_same(host, got)

    # a sampler over get_all(shuffle=True), a shuffled copy: no mirror matches, the host path (on both sides)
    def shuffled(b):
        ds, _ = common.get_sequence_buffer_iterator(b, 6, 0, 10, max_batches_per_loop_train=4, use_simple_sampler=True)
        ds.transitions = b.get_all(shuffle=True)
        return ds

    want, _, _ = _planet_loop(dataset_fn=shuffled)
    got, _, _ = _planet_loop(lambda b: replay.mirror_to_device(b, DEV), dataset_fn=shuffled)
    assert not gathers
    _assert_same(want, got)

    # a mirror on another device than the model's: the host path
    def elsewhere(b):
        m = replay.mirror_to_device(b, DEV)
        m.device = torch.device("cuda", 1)  # (one device here: only the comparison the trainer makes is exercised)
        return m

    got, _, _ = _planet_loop(elsewhere)
    assert not gathers
    _assert_same(host, got)


def test_a_bypassed_cur_idx_resyncs(deterministic, gathers):
    def bypass(buf, g):  # a trajectory written into the arrays directly, cur_idx and num_stored moved by hand
        n0 = buf.cur_idx
        buf.obs[n0:n0 + EP] = _frames(g, EP, (3, 16, 16), np.float32)
        buf.action[n0:n0 + EP] = g.uniform(-1, 1, (EP, A))
        buf.reward[n0:n0 + EP] = g.standard_normal(EP)
        buf.trajectory_indices.append((n0, n0 + EP))
        buf.cur_idx = buf.num_stored = n0 + EP
        buf._start_last_trajectory = buf.cur_idx

    host, _, _ = _planet_loop(between=bypass)
    assert not gathers
    dev, copied, (_, _, buf) = _planet_loop(lambda b: replay.mirror_to_device(b, DEV), between=bypass)
    assert len(gathers) == 8 and copied == [5 * EP, 7 * EP]  # the second flush re-copied every row
    _assert_same(host, dev)
