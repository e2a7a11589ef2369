"""CPU checks of planning PlaNet's latent model for K observations at once:

* ``PosteriorBatch.update`` (what ``LatentModelEnv.update_posterior_batch`` runs) row by row against the reference's
  own ``PlaNetModel.update_posterior`` (oracle/_ref, skipped without it) and a float64 restatement, over two steps, with
  a reset entry restarting from the state ``reset_posterior()`` leaves;
* the batch's refusals;
* the C entry points' refusals, returned before anything touches a device;
* the single-problem rollout kernel's SASS is that of the kernel before the batched instantiation existed, and neither
  instantiation has a stack frame.
"""
import ctypes as C
import importlib.util
import json
import os
import re
import shutil
import subprocess

import hashlib
import numpy as np
import pytest
import torch

from baseline import reference_arm as ra
from mbrl_lib_b200 import _lib, models
from mbrl_lib_b200.latent import PosteriorBatch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
mbrl, REF_SRC = ra.import_reference()
needs_ref = pytest.mark.skipif(mbrl is None, reason=f"reference not importable here: {REF_SRC}")
ENC = ((3, 8, 4, 2), (8, 16, 4, 2))
DEC = ((32, 1, 1), ((32, 16, 5, 2), (16, 8, 5, 2), (8, 3, 4, 1)))
KW = dict(obs_shape=(3, 16, 16), obs_encoding_size=32, encoder_config=ENC, decoder_config=DEC)
A, L, HB, HF = 2, 4, 16, 16


def _local_model():
    return models.PlaNetModel(A, L, HB, HF, device="cpu", seed=3, scale=0.2, **KW)


def _frames(K, seed):
    return np.random.default_rng(seed).integers(0, 256, (K, 3, 16, 16), dtype=np.uint8)


@torch.no_grad()
def _f64_update(model, obs, latent, belief, action, eps):
    """PlaNetModel.update_posterior (planet.py:592-641) for one row in float64."""
    def lin(m, x):
        return x @ m.weight.double().T + m.bias.double()

    rnn = model.belief_model.rnn
    e = torch.relu(lin(model.belief_model.embedding_layer[0], torch.cat([latent, action]).double()))
    h = belief.double()
    gi, gh = e @ rnn.weight_ih.double().T + rnn.bias_ih.double(), h @ rnn.weight_hh.double().T + rnn.bias_hh.double()
    r, z = torch.sigmoid(gi[:HB] + gh[:HB]), torch.sigmoid(gi[HB:2 * HB] + gh[HB:2 * HB])
    n = torch.tanh(gi[2 * HB:] + r * gh[2 * HB:])
    h1 = (1 - z) * n + z * h
    x = torch.as_tensor(obs).double()[None] / 256.0 - 0.5
    for conv in model.encoder.convs:
        x = torch.relu(torch.nn.functional.conv2d(x, conv[0].weight.double(), conv[0].bias.double(),
                                                  stride=conv[0].stride))
    enc = x.reshape(-1)
    if not isinstance(model.encoder.fc, torch.nn.Identity):
        enc = lin(model.encoder.fc, enc)
    q = model.posterior_transition_model
    p = lin(q[2], torch.relu(lin(q[0], torch.cat([h1, enc]))))
    std = torch.nn.functional.softplus(p[L:]) + q[3].min_std
    return p[:L] + std * eps.double(), h1


def _run_batch(model, frames, actions, eps, reset_after_first):
    pb = PosteriorBatch(model, L, HB, A, "cpu")
    out = [pb.update(frames[0], None, _eps=eps[0])]
    out = [{k: v.clone() for k, v in out[0].items()}]
    pb.reset(reset_after_first)
    out.append(pb.update(frames[1], actions, _eps=eps[1]))
    return out


def test_rows_match_float64_and_reset_entries_restart():
    torch.manual_seed(0)
    K = 5
    model = _local_model()
    frames = [_frames(K, 1), _frames(K, 2)]
    actions = torch.rand(K, A) * 2 - 1
    eps = torch.randn(2, K, L)
    got = _run_batch(model, frames, actions, eps, [1, 3])
    for k in range(K):
        s1, h1 = _f64_update(model, frames[0][k], torch.zeros(L), torch.zeros(HB), torch.zeros(A), eps[0, k])
        np.testing.assert_allclose(got[0]["latent"][k].double(), s1, rtol=0, atol=2e-6)
        np.testing.assert_allclose(got[0]["belief"][k].double(), h1, rtol=0, atol=2e-6)
        start = (torch.zeros(L), torch.zeros(HB), torch.zeros(A)) if k in (1, 3) else \
            (got[0]["latent"][k], got[0]["belief"][k], actions[k])
        s2, h2 = _f64_update(model, frames[1][k], *start, eps[1, k])
        np.testing.assert_allclose(got[1]["latent"][k].double(), s2, rtol=0, atol=2e-6)
        np.testing.assert_allclose(got[1]["belief"][k].double(), h2, rtol=0, atol=2e-6)


@needs_ref
def test_rows_equal_the_reference_update_posterior():
    torch.manual_seed(0)
    model = mbrl.models.PlaNetModel(latent_state_size=L, action_size=A, belief_size=HB, hidden_size_fcs=HF, device="cpu",
                                    **KW)
    K = 4
    frames = [_frames(K, 5), _frames(K, 6)]
    actions = torch.rand(K, A) * 2 - 1
    eps = torch.randn(2, K, L)
    got = _run_batch(model, frames, actions, eps, [2])
    orig = torch.randn
    for k in range(K):
        queue = [eps[0, k][None].clone(), eps[1, k][None].clone()]
        torch.randn = lambda *a, **kw: queue.pop(0)
        try:
            model.reset_posterior()
            want0 = {n: v.clone() for n, v in model.update_posterior(frames[0][k]).items()}
            if k == 2:  # a reset entry: reset_posterior() then update_posterior(obs, action=None)
                model.reset_posterior()
                want1 = model.update_posterior(frames[1][k])
            else:
                want1 = model.update_posterior(frames[1][k], actions[k].numpy())
        finally:
            torch.randn = orig
        for step, want in ((0, want0), (1, want1)):
            for n in ("latent", "belief"):
                torch.testing.assert_close(got[step][n][k], want[n][0], rtol=0, atol=1e-6)


def test_batch_refusals():
    model = _local_model()
    pb = PosteriorBatch(model, L, HB, A, "cpu")
    with pytest.raises(NotImplementedError, match="one posterior"):
        pb.get()
    pb.update(_frames(3, 0))
    assert pb.get(3)[0].shape == (3, L)
    with pytest.raises(ValueError, match="batch of 3"):
        pb.get(2)
    with pytest.raises(ValueError, match="3 posteriors"):
        pb.update(_frames(2, 0), torch.zeros(2, A))
    with pytest.raises(ValueError, match="action is None"):
        pb.update(_frames(3, 0))
    pb.reset([0])
    with pytest.raises(RuntimeError, match=r"\[0\] were reset"):
        pb.get(3)
    pb.reset()
    pb.update(_frames(2, 0), torch.zeros(2, A))  # a new batch: K from the observations, every entry from zeros
    assert pb.get(2)[0].shape == (2, L)
    with pytest.raises(ValueError, match="must be"):
        pb.set(torch.zeros(2, L + 1), torch.zeros(2, HB))
    with pytest.raises(NotImplementedError, match="encoder"):
        PosteriorBatch(models.PlaNetModel(A, L, HB, HF), L, HB, A, "cpu").update(_frames(2, 0))


# ---- the C entry points refuse bad arguments before anything touches a device -------------------------------------------
def test_abi_refusals_need_no_device():
    lib = _lib.load()
    # A host block standing in for the opaque handle.  These checks read nothing of it but its descriptor, which is the
    # handle's first member; a wrong field read anywhere else would touch no device either, only host memory.
    desc = _lib.LatentDesc()
    desc.action_size, desc.latent_size, desc.belief_size, desc.hidden_size, desc.min_std = 6, 30, 200, 200, 0.1
    handle = C.create_string_buffer(4096)
    C.memmove(handle, C.byref(desc), C.sizeof(desc))
    h = C.cast(handle, C.c_void_p)
    dummy = C.c_void_p(16)

    def cfg(**kw):
        c = _lib.RolloutCfg(50, 4, 1, _lib.PREC["f32"], _lib.PROP["expectation"], _lib.TS1_PERMS, 1, 2, 0, 0)
        for k, v in kw.items():
            setattr(c, k, v)
        return c

    ccfg = _lib.CemCfg(3, 5, 0.1, 1, 1)

    def ev(c, K=2, ws=1 << 30, latent0=dummy, returns=dummy):
        return lib.b200pets_latent_eval_sequences_batch(h, C.byref(c), K, latent0, dummy, dummy, None, returns, None, dummy,
                                                        ws, None)

    def plan(c, K=2, ws=1 << 30, x0=dummy, cc=ccfg):
        return lib.b200pets_latent_cem_plan_batch(h, C.byref(c), C.byref(cc), K, dummy, dummy, x0, dummy, dummy, None, None,
                                                  dummy, None, dummy, ws, None)

    # the single entry points: the same refusals, less the problem count
    def ev1(c, K=None, ws=1 << 30, latent0=dummy, returns=dummy):
        return lib.b200pets_latent_eval_sequences(h, C.byref(c), latent0, dummy, dummy, None, returns, None, dummy, ws, None)

    def plan1(c, K=None, ws=1 << 30, x0=dummy, cc=ccfg):
        return lib.b200pets_latent_cem_plan(h, C.byref(c), C.byref(cc), dummy, dummy, x0, dummy, dummy, None, None, dummy,
                                            None, dummy, ws, None)

    for call in (ev, plan, ev1, plan1):
        if call in (ev, plan):
            assert call(cfg(), K=0) == -1 and "num_problems" in lib.b200pets_last_error().decode()
        assert call(cfg(first_sequence=10)) == -2 and "sharded" in lib.b200pets_last_error().decode()
        assert call(cfg(global_population=100)) == -2
        assert call(cfg(precision=_lib.PREC["bf16_tc"])) == -2 and "fp32" in lib.b200pets_last_error().decode()
        assert call(cfg(population=0)) == -1
        assert call(cfg(), ws=0) == -1 and "workspace too small" in lib.b200pets_last_error().decode()
    for call in (ev, ev1):
        assert call(cfg(), latent0=None) == -1 and "null" in lib.b200pets_last_error().decode()
        assert call(cfg(), returns=None) == -1
    for call in (plan, plan1):
        assert call(cfg(), x0=None) == -1 and "null" in lib.b200pets_last_error().decode()
        assert call(cfg(), cc=_lib.CemCfg(3, 51, 0.1, 1, 1)) == -1 and "elites" in lib.b200pets_last_error().decode()
        assert call(cfg(), cc=_lib.CemCfg(3, 0, 0.1, 1, 1)) == -1 and "elites" in lib.b200pets_last_error().decode()
    assert lib.b200pets_latent_eval_sequences_batch(None, C.byref(cfg()), 2, dummy, dummy, dummy, None, dummy, None, dummy,
                                                    1 << 30, None) == -1
    need1 = lib.b200pets_latent_eval_batch_workspace_bytes(h, C.byref(cfg()), 1)
    assert lib.b200pets_latent_eval_batch_workspace_bytes(h, C.byref(cfg()), 4) >= 4 * 50 * 4 > need1 > 0
    assert lib.b200pets_latent_eval_batch_workspace_bytes(h, C.byref(cfg()), 0) == 0
    assert lib.b200pets_latent_cem_plan_batch_workspace_bytes(h, C.byref(cfg()), C.byref(ccfg), 3) > \
        lib.b200pets_latent_cem_plan_batch_workspace_bytes(h, C.byref(cfg()), C.byref(ccfg), 1) > 0


# ---- SASS -------------------------------------------------------------------------------------------------------------
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CUOBJDUMP = shutil.which("cuobjdump") or os.path.join(os.path.dirname(NVCC), "cuobjdump")


@pytest.fixture(scope="module")
def library():
    if not (os.path.exists(NVCC) and os.path.exists(CUOBJDUMP)):
        pytest.skip("needs nvcc and cuobjdump")
    spec = importlib.util.spec_from_file_location("b200pets_build_latent_batch", os.path.join(ROOT, "mbrl-lib_b200", "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.build()


def _sass(lib, name):
    """{rows per CTA: instruction text} of the kernels `name`<R>, addresses and comments dropped."""
    out = subprocess.run([CUOBJDUMP, "-sass", lib], capture_output=True, text=True, check=True).stdout
    res, r = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            mm = re.search(name + r"ILi(\d+)E", m.group(1))
            r = mm.group(1) if mm else None
            if r:
                res[r] = []
            continue
        if r:
            m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s*(.*?)\s*;", line)
            if m:
                res[r].append(m.group(1))
    return res


def test_single_rollout_sass_is_unchanged(library):
    """tests/golden/latent_rollout_sass.json holds the digests of latent_rollout_kernel<R> as built before the batched
    instantiation was added; SASS is the compiler's, so the check runs under the nvcc release that recorded them."""
    with open(os.path.join(ROOT, "tests", "golden", "latent_rollout_sass.json")) as f:
        golden = json.load(f)
    version = subprocess.run([NVCC, "--version"], capture_output=True, text=True, check=True).stdout
    if golden["nvcc"] not in version:
        pytest.skip(f"digests recorded with nvcc {golden['nvcc']}")
    got = {r: hashlib.sha256("\n".join(ins).encode()).hexdigest() for r, ins in _sass(library, "latent_rollout_kernel").items()}
    assert got == golden["sha256"]


def test_batched_rollout_has_no_stack_frame(library):
    out = subprocess.run([CUOBJDUMP, "-res-usage", library], capture_output=True, text=True, check=True).stdout
    res, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+) .*LOCAL:(\d+)", line)
        if m and name:
            res[name] = tuple(int(g) for g in m.groups())
            name = None
    for kernel in ("latent_rollout_kernel", "latent_rollout_batch_kernel"):
        found = {n: r for n, r in res.items() if kernel + "ILi" in n}
        assert sorted(int(re.search(r"ILi(\d+)E", n).group(1)) for n in found) == [1, 2, 4, 8, 16, 32], sorted(found)
        for n, (regs, stack, local) in found.items():
            assert stack == 0 and local == 0, f"{n}: {stack} B stack, {local} B local"
            assert regs <= 255, n
