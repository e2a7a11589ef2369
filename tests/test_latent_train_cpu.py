"""CPU checks of PlaNet's training path: the float64 oracle against the reference's own PlaNetModel.update recorded in
tests/golden/planet_train.npz (oracle/gen_golden_planet_train.py) and, where oracle/_ref exists, against the live
reference (with the draws injected into the reference's sampler), the container's training layout against a reference model's state_dict,
the sequence kernels' resource use and the C ABI's refusals of bad arguments."""
import copy
import ctypes as C
import importlib.util
import os
import re
import shutil
import subprocess
import types

import numpy as np
import pytest
import torch

from baseline import reference_arm as ra
from mbrl_lib_b200 import _lib, latent_train, models
from oracle import planet_train_f64 as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
mbrl, REF_SRC = ra.import_reference()
needs_ref = pytest.mark.skipif(mbrl is None, reason=f"reference not importable here: {REF_SRC}")
ENC = ((3, 8, 4, 2), (8, 16, 4, 2))
DEC = ((32, 1, 1), ((32, 16, 5, 2), (16, 8, 5, 2), (8, 3, 4, 1)))
KW = dict(obs_shape=(3, 16, 16), obs_encoding_size=32, encoder_config=ENC, decoder_config=DEC)


def _ref_model():
    torch.manual_seed(0)
    return mbrl.models.PlaNetModel(latent_state_size=4, action_size=2, belief_size=16, hidden_size_fcs=16, device="cpu",
                                   **KW)


def _inject(model, draws):
    """Make the reference's _sample_state_from_params read ``draws`` (posterior, prior, posterior, ... per step)."""
    it = iter(draws)
    orig = model._sample_state_from_params

    def sample(params, generator, deterministic=False):
        if deterministic:
            return orig(params, generator, deterministic)
        L = model.latent_state_size
        return params[:, :L] + params[:, L:] * next(it).to(params.dtype)

    model._sample_state_from_params = sample


def test_oracle_reproduces_the_recorded_reference_update(golden_dir):
    g = np.load(os.path.join(golden_dir, "planet_train.npz"))
    model = models.PlaNetModel(2, 4, 16, 16, min_std=0.1, free_nats=0.1, **KW)
    with torch.no_grad():
        for n, p in model.named_parameters():
            p.copy_(torch.from_numpy(g[f"param/{n}"]))
    m64 = po.as_f64(model)
    opt64 = torch.optim.Adam(m64.parameters(), lr=1e-3, eps=1e-4)
    obs = torch.from_numpy(g["obs"].astype(np.float64)) / 256.0 - 0.5
    got = po.update(m64, obs, torch.from_numpy(g["act"]).double(), torch.from_numpy(g["rewards"]).double(),
                    torch.from_numpy(g["eps_q"]), torch.from_numpy(g["eps_p"]), opt64)
    for what, a in zip(("loss", "observations_loss", "reward_loss", "kl_loss", "grad_norm"), got):
        b = float(g[what])
        assert abs(a - b) <= 2e-5 * max(1.0, abs(b)), (what, a, b)
    for n, p in m64.named_parameters():
        want = torch.from_numpy(g[f"grad/{n}"]).double()
        assert float((p.grad - want).norm() / want.norm()) <= 1e-4, n
        assert float((p.detach() - torch.from_numpy(g[f"after/{n}"]).double()).abs().max()) <= 1e-6, n


@needs_ref
def test_oracle_reproduces_the_reference_loss_and_update():
    ref = _ref_model()
    B, S = 3, 6
    g = np.random.default_rng(1)
    batch = types.SimpleNamespace(obs=g.integers(0, 256, (B, S, 3, 16, 16)).astype(np.float32),
                                  act=g.uniform(-1, 1, (B, S, 2)).astype(np.float32),
                                  rewards=g.standard_normal((B, S)).astype(np.float32),
                                  next_obs=None, terminateds=None, truncateds=None)
    eq, ep = (torch.from_numpy(g.standard_normal((S - 1, B, 4))) for _ in range(2))
    m64 = po.as_f64(ref)
    _inject(ref, [e.float() for pair in zip(eq, ep) for e in pair])
    opt = torch.optim.Adam(ref.parameters(), lr=1e-3, eps=1e-4)
    opt64 = torch.optim.Adam(m64.parameters(), lr=1e-3, eps=1e-4)
    loss, meta = ref.update(batch, opt)
    obs = torch.from_numpy(batch.obs).double() / 256.0 - 0.5
    got = po.update(m64, obs, torch.from_numpy(batch.act).double(), torch.from_numpy(batch.rewards).double(), eq, ep, opt64)
    want = (loss, meta["observations_loss"], meta["reward_loss"], meta["kl_loss"], meta["grad_norm"])
    for a, b in zip(got, want):
        assert abs(a - b) <= 2e-5 * max(1.0, abs(b)), (got, want)
    for (n, p), p64 in zip(ref.named_parameters(), m64.parameters()):
        assert float((p.double() - p64).abs().max()) <= 1e-6, n


@needs_ref
def test_container_layout_matches_the_reference_state_dict():
    ref = _ref_model()
    mine = models.PlaNetModel(2, 4, 16, 16, **KW)
    want = {k: tuple(v.shape) for k, v in ref.state_dict().items()}
    assert {k: tuple(v.shape) for k, v in mine.state_dict().items()} == want
    mine.load_state_dict(ref.state_dict())
    assert [n for n, _ in mine.named_parameters()] == [n for n, _ in ref.named_parameters()]
    assert latent_train.is_trainable_latent_model(ref) and latent_train.is_trainable_latent_model(mine)
    d0, d1 = latent_train.train_desc(ref), latent_train.train_desc(mine)
    assert [getattr(d0, f) for f, _ in d0._fields_] == [getattr(d1, f) for f, _ in d1._fields_]
    assert (d0.action_size, d0.latent_size, d0.belief_size, d0.hidden_size, d0.encoding_size) == (2, 4, 16, 16, 32)


def test_container_without_observation_arguments_is_the_planning_container():
    m = models.PlaNetModel(6, 30, 200, 200)
    assert not hasattr(m, "encoder") and not hasattr(m, "decoder") and not hasattr(m, "posterior_transition_model")
    assert not latent_train.is_trainable_latent_model(m)
    assert sum(p.numel() for p in m.parameters()) == 387_461


def test_draw_key_follows_the_model_rng():
    m = models.PlaNetModel(2, 4, 16, 16, **KW)
    m.rng = torch.Generator()
    m.rng.manual_seed(5)
    assert latent_train.draw_key(m) == (5, 0) and latent_train.draw_key(m) == (5, 1)


def test_sequence_kernels_have_no_stack_frame():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cuobjdump = shutil.which("cuobjdump") or os.path.join(os.path.dirname(nvcc), "cuobjdump")
    if not (os.path.exists(nvcc) and os.path.exists(cuobjdump)):
        pytest.skip("needs nvcc and cuobjdump")
    spec = importlib.util.spec_from_file_location("b200pets_build_lt", os.path.join(ROOT, "mbrl-lib_b200", "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    out = subprocess.run([cuobjdump, "-res-usage", mod.build()], capture_output=True, text=True, check=True).stdout
    res, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+)", line)
        if m and name:
            res[name] = (int(m.group(1)), int(m.group(2)))
            name = None
    for kind in ("rssm_seq_forward_kernel", "rssm_seq_backward_kernel"):
        got = {n: r for n, r in res.items() if kind in n}
        assert sorted(int(re.search(r"ILi(\d+)E", n).group(1)) for n in got) == [1, 2, 4, 8, 16, 32], sorted(got)
        for n, (regs, stack) in got.items():
            assert stack == 0, f"{n}: {stack} B stack frame"
            assert regs <= 255, n


def test_abi_refuses_bad_arguments():
    lib = _lib.load()
    d = _lib.LatentTrainDesc(6, 30, 200, 200, 1024, 0.1)
    params = (C.c_void_p * _lib.LATENT_TRAIN_NUM_PARAMS)(*([8] * _lib.LATENT_TRAIN_NUM_PARAMS))
    dummy = C.c_void_p(8)
    fwd = lambda B, T, p=params, eq=None, tape=None: lib.b200pets_latent_seq_forward(  # noqa: E731
        C.byref(d), p, B, T, dummy, dummy, eq, None, 0, 0, dummy, dummy, dummy, dummy, dummy, tape, dummy, 1 << 30, None)
    assert fwd(0, 5) == -1 and fwd(5, 0) == -1
    assert fwd(5, 5, p=(C.c_void_p * _lib.LATENT_TRAIN_NUM_PARAMS)()) == -1
    assert fwd(5, 5, eq=dummy) == -1  # eps_q without eps_p
    assert fwd(5, 5, tape=C.byref(_lib.LatentTape())) == -1  # a tape with NULL fields
    bwd = lib.b200pets_latent_seq_backward(C.byref(d), params, 5, 5, dummy, None, None, None, None, None, None, dummy, None)
    assert bwd == -1  # the backward pass needs the tape
    assert lib.b200pets_latent_train_workspace_bytes(C.byref(d), 0, 5) == 0
    bad = copy.copy(d)
    bad.encoding_size = 0
    assert lib.b200pets_latent_train_supported(C.byref(bad)) == -1
