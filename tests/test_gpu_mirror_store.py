"""The chunked device store both replay mirrors share (mbrl_lib_b200/replay.py ``_ChunkedMirror``): a flush whose
staging fill fails part-way leaves the next flush to copy every stored row, after which the device rows equal the
buffer's, for PlaNet's frame mirror and MBPO's SAC transition mirror alike."""
import importlib

import numpy as np
import pytest
import torch

from baseline import reference_arm as ra
from mbrl_lib_b200 import replay

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
mbrl, REF_SRC = ra.import_reference()
needs_ref = pytest.mark.skipif(mbrl is None, reason=f"reference not importable here: {REF_SRC}")
OBS, A = (3, 4, 5), 2


def _write(buf, g, n):
    buf.add_batch(g.standard_normal((n, *OBS)).astype(np.float32), g.standard_normal((n, A)),
                  g.standard_normal((n, *OBS)), g.standard_normal(n), g.random(n) < 0.2, np.zeros(n, bool))


def _check(kind, buf, m):
    n = buf.num_stored
    assert m.rows_held == n
    for lo in range(0, n, 1 << m.chunk_shift):
        hi = min(n, lo + (1 << m.chunk_shift))
        if kind == "planet":
            assert torch.equal(m.device_obs(lo, hi).cpu(), torch.from_numpy(buf.obs[lo:hi])), (lo, hi)
        else:
            want = np.empty((hi - lo, m.width), np.float32)
            replay.pack_rows(buf, slice(lo, hi), want, m.obs_dim, m.act_dim)
            assert torch.equal(m.device_rows(lo, hi).cpu(), torch.from_numpy(want)), (lo, hi)
    if kind == "planet":
        assert torch.equal(m.act[:n].cpu(), torch.from_numpy(buf.action[:n]).float())
        assert torch.equal(m.rew[:n].cpu(), torch.from_numpy(buf.reward[:n]).float())


@needs_ref
@pytest.mark.parametrize("kind", ["planet", "sac"])
def test_a_copy_that_fails_part_way_makes_the_next_flush_a_resync(kind):
    rb = importlib.import_module("mbrl.util.replay_buffer")
    g = np.random.default_rng(0)
    buf = rb.ReplayBuffer(100, OBS, (A,), rng=np.random.default_rng(0))
    mirror = replay.mirror_to_device if kind == "planet" else replay.mirror_transitions_to_device
    m = mirror(buf, DEV, _rows_per_chunk=8)
    try:
        _write(buf, g, 40)  # five chunks of 8 rows, each one run and one staging fill
        starts = []
        fill = m._fill

        def fails_second(stage, s, e):
            starts.append(s)
            if len(starts) == 2:
                raise RuntimeError("staging fill failed")
            fill(stage, s, e)

        m._fill = fails_second
        with pytest.raises(RuntimeError, match="staging fill failed"):
            m.flush()
        assert starts == [0, 8]  # the first chunk was copied, the second was not
        del m._fill
        _write(buf, g, 1)
        assert m.flush() == buf.num_stored == 41 and m._rows_copied == 41
        _check(kind, buf, m)
    finally:
        m.close()
