"""CPU checks of the SAC path: the float64 oracle against the reference's own updates (tests/golden/sac_*.npz, written by
oracle/gen_golden_sac.py), state_dict compatibility of the drop-in's networks, the kernel's resources, and the refusals
that need no device."""
import ctypes as C
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from baseline import reference_arm as ra  # noqa: E402
from mbrl_lib_b200 import _lib, sac as bsac  # noqa: E402
from oracle import sac_f64  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
mbrl, REF_SRC = ra.import_reference()
needs_ref = pytest.mark.skipif(mbrl is None, reason=f"reference not importable here: {REF_SRC}")


class Box:
    def __init__(self, A):
        self.low, self.high, self.shape = -np.ones(A, np.float32), np.ones(A, np.float32), (A,)


@pytest.mark.parametrize("name", ["sac_tuning", "sac_interval2"])
def test_oracle_reproduces_the_references_updates(name):
    """Three consecutive updates of the oracle, each from its own previous result, against the reference's fp32 CPU
    updates on the same batches and draws: within 5e-3 of each tensor's change in the update, or since the start when
    that is larger (the target between soft updates; measured 1.1e-3: from a fresh Adam
    state an element whose gradient is near zero moves by up to lr in either direction, so fp32 rounding of the
    reference's gradient shows at that scale; most elements agree to 1e-6 of the change)."""
    z = np.load(os.path.join(GOLDEN, f"{name}.npz"))
    D, A, H, B, tuning, interval, reverse = (int(x) for x in z["cfg"])
    gamma, tau, alpha, lr = (float(x) for x in z["hyper"])
    t = lambda a: torch.from_numpy(np.asarray(a)).double()  # noqa: E731
    nets = {p: {k: t(z[f"init/{p}/{k}"]) for k in (sac_f64.POLICY_KEYS if p == "policy" else sac_f64.CRITIC_KEYS)}
            for p in ("critic", "target", "policy")}
    zero = lambda keys, P: {k: (0, torch.zeros_like(P[k]), torch.zeros_like(P[k])) for k in keys}  # noqa: E731
    cst, pst = zero(sac_f64.CRITIC_KEYS, nets["critic"]), zero(sac_f64.POLICY_KEYS, nets["policy"])
    la, ast = torch.zeros(1, dtype=torch.float64), (0, torch.zeros(1, dtype=torch.float64), torch.zeros(1, dtype=torch.float64))
    te = -float(A)
    for u in range(3):
        batch = [z[f"u{u}/batch/{k}"].astype(np.float64) for k in ("obs", "act", "next_obs", "rewards", "terminateds")]
        cfg = dict(gamma=gamma, tau=tau, lr=lr, alpha=alpha, tuning=bool(tuning), target_entropy=te,
                   target_update_interval=interval, updates=u, reverse_mask=bool(reverse), scale=t(z["scale"]),
                   bias=t(z["bias"]))
        prev = {p: dict(v) for p, v in nets.items()}
        out = sac_f64.sac_update(nets["critic"], nets["target"], nets["policy"], cst, pst, batch, t(z[f"u{u}/eps"]), cfg,
                                 la, ast)
        for p in ("critic", "target", "policy"):
            for k, v in out[p].items():
                ref = t(z[f"u{u}/{p}/{k}"])
                change = torch.maximum((ref - prev[p][k]).abs().max(), (ref - t(z[f"init/{p}/{k}"])).abs().max())
                assert float((v - ref).abs().max() / change) <= 5e-3, (u, p, k)
        for k, (_, m, v) in out["critic_state"].items():
            assert float((m - t(z[f"u{u}/critic_m/{k}"])).abs().max()) <= 1e-4 * float(m.abs().max()) + 1e-9  # measured 1.2e-5
        stats = z[f"u{u}/stats"]
        # the policy loss is a difference of two terms (measured 1.9e-4 relative)
        assert np.allclose(out["stats"][:5], stats, rtol=1e-3, atol=1e-6), (out["stats"][:5], stats)
        if tuning:
            assert abs(float(out["log_alpha"]) - float(z[f"u{u}/log_alpha"][0])) <= 1e-6
            la, ast, alpha = out["log_alpha"], out["alpha_state"], out["alpha"]
        nets = {p: out[p] for p in ("critic", "target", "policy")}
        cst, pst = out["critic_state"], out["policy_state"]


@needs_ref
def test_state_dict_keys_match_the_reference():
    from mbrl.third_party.pytorch_sac_pranz24.model import GaussianPolicy, QNetwork

    for ours, theirs in ((bsac.QNetwork(5, 2, 8), QNetwork(5, 2, 8)),
                         (bsac.GaussianPolicy(5, 2, 8, Box(2)), GaussianPolicy(5, 2, 8, Box(2)))):
        assert [(k, v.shape) for k, v in ours.state_dict().items()] == [(k, v.shape) for k, v in theirs.state_dict().items()]
        ours.load_state_dict(theirs.state_dict())
        theirs.load_state_dict(ours.state_dict())
    # the parameter orders the C ABI documents
    assert [k for k, _ in bsac.QNetwork(5, 2, 8).named_parameters()] == sac_f64.CRITIC_KEYS
    assert [k for k, _ in bsac.GaussianPolicy(5, 2, 8).named_parameters()] == sac_f64.POLICY_KEYS


def test_sac_kernel_has_no_stack_frame():
    lib = os.path.join(ROOT, "mbrl-lib_b200", "libb200pets.so")
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-res-usage", lib], capture_output=True, text=True).stdout
    lines = out.splitlines()
    idx = [i for i, s in enumerate(lines) if "sac_update_kernel" in s]
    assert idx, "sac_update_kernel not found in the library"
    for i in idx:
        res = lines[i + 1]
        assert "STACK:0" in res, res


def _desc(**kw):
    args = types.SimpleNamespace(gamma=0.99, tau=0.005, alpha=0.2, policy="Gaussian", target_update_interval=1,
                                 automatic_entropy_tuning=False, target_entropy=None, hidden_size=32, device="cuda", lr=3e-4)
    A = kw.pop("A", 3)
    d = bsac.sac_desc(kw.pop("D", 5), Box(A) if A > 0 else types.SimpleNamespace(shape=(A,), low=[], high=[]), args, -3.0)
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def _ptrs(n, null_at=None):
    return (C.c_void_p * n)(*[None if i == null_at else 0x1000 + 256 * i for i in range(n)])


def test_sac_abi_refusals():
    lib = _lib.load()
    assert lib.b200pets_sac_supported(C.byref(_desc())) == 0
    assert lib.b200pets_sac_supported(C.byref(_desc(A=32))) == 0
    assert lib.b200pets_sac_supported(C.byref(_desc(A=33))) == -2 and b"one tile" in lib.b200pets_last_error()
    assert lib.b200pets_sac_supported(C.byref(_desc(hidden=0))) == -1
    assert lib.b200pets_sac_supported(C.byref(_desc(obs_dim=0))) == -1
    assert lib.b200pets_sac_supported(C.byref(_desc(target_update_interval=0))) == -1
    assert lib.b200pets_sac_supported(None) == -1
    n = _lib.SAC_NUM_PARAMS
    p = C.c_void_p(0x1000)

    def create(d=None, P=None, T=None, M=None, V=None, la=(p, p, p)):
        h = C.c_void_p()
        rc = lib.b200pets_sac_create(C.byref(d or _desc()), P or _ptrs(n), T or _ptrs(12), M or _ptrs(n), V or _ptrs(n),
                                     *la, C.byref(h))
        if rc == 0:
            lib.b200pets_sac_destroy(h)
        return rc

    assert create() == 0
    assert create(P=_ptrs(n, null_at=19)) == -1
    assert create(T=_ptrs(12, null_at=11)) == -1
    assert create(M=_ptrs(n, null_at=0)) == -1
    assert create(la=(None, None, None)) == 0  # no entropy tuning: log_alpha is not read
    assert create(d=_desc(automatic_entropy_tuning=1), la=(p, None, p)) == -1
    assert create(d=_desc(A=40)) == -2

    h = C.c_void_p()
    assert lib.b200pets_sac_create(C.byref(_desc()), _ptrs(n), _ptrs(12), _ptrs(n), _ptrs(n), None, None, None,
                                   C.byref(h)) == 0
    try:
        need = lib.b200pets_sac_workspace_bytes(h, 256)
        assert need > 0 and lib.b200pets_sac_workspace_bytes(h, 257) > need and lib.b200pets_sac_workspace_bytes(h, 0) == 0
        steps = (C.c_int64 * 3)(0, 0, 0)

        def update(batch=256, updates=0, st=steps, trans=p, alpha=p, stats=p, ws=p, nbytes=need):
            return lib.b200pets_sac_update(h, batch, updates, 1, st, trans, None, 1, 0, alpha, stats, ws, nbytes, None)

        assert update(trans=None) == -1 and update(alpha=None) == -1 and update(stats=None) == -1 and update(ws=None) == -1
        assert update(st=None) == -1
        assert update(batch=0) == -1 and update(updates=-1) == -1
        assert update(nbytes=need - 1) == -1 and b"workspace" in lib.b200pets_last_error()
        assert update(st=(C.c_int64 * 3)(0, -1, 0)) == -1
    finally:
        lib.b200pets_sac_destroy(h)


def test_drop_in_refusals_at_construction():
    args = types.SimpleNamespace(gamma=0.99, tau=0.005, alpha=0.2, policy="Deterministic", target_update_interval=1,
                                 automatic_entropy_tuning=False, target_entropy=None, hidden_size=32, device="cuda", lr=3e-4)
    with pytest.raises(NotImplementedError, match="Gaussian"):
        bsac.SAC(5, Box(2), args)
    args.policy, args.device = "Gaussian", "cpu"
    with pytest.raises(NotImplementedError, match="CUDA"):
        bsac.SAC(5, Box(2), args)
    args.device = "cuda:0"
    with pytest.raises(NotImplementedError, match="act_dim 33"):  # refused before any tensor is made on the device
        bsac.SAC(5, Box(33), args)
