"""MBPO's SAC update on the device (``mbrl_lib_b200.SAC``, csrc/sac.cu) against float64 and against the reference.

Stated tolerances (from the deviations these tests print as ``DEVIATION <name> <value>``, measured on an H100):
  * one update against oracle/sac_f64.py (torch autograd + torch.optim.Adam in float64, same draws), Adam state
    pre-filled (step 9, non-zero moments) so that the update is a smooth function of the gradient:
      parameter update       |du32 - du64| <= 2e-4 * max |du64| + half an fp32 ulp of p, per tensor (measured 6e-8 ..
                             4e-7)
      exp_avg / exp_avg_sq   max |x32 - x64| <= 1e-5 * max |x64|, per tensor (measured <= 1.6e-6)
    except (45, 17, 512, 37) with entropy tuning, an ill-conditioned update: there torch's own fp32 autograd of the same
    update (checked on CPU) deviates from float64 by 2.6e-4 of the update and up to 6.9e-4 on the moments, so the bounds
    are 1e-3 and 2e-3 (measured 2.56e-4 on the update, 2.4e-4 on the first moments compared), and 1e-4 on the
    statistics (measured 1.8e-5 on the policy loss)
      statistics             1e-5 relative (1e-5 absolute below 1)
    from a fresh state (step 0) the first Adam step is lr * sign(g) wherever |g| >> eps, so the moments are compared
    (1e-5 of max) and the update only where |g64| > 1e-3 max |g64|
  * the soft target update: bit-equal to torch's t * (1 - tau) + p * tau on the device's updated critic
  * 300 updates against the reference's fp32 SAC.update_parameters on cuda, same batches and draws, from a fresh Adam
    state: ||p_dev - p_ref|| <= 0.25 ||p_ref - p_0|| per tensor (Frobenius norms; measured 4.6e-5 after 1 update,
    2.5e-4 after 10, 3.7e-2 after 100, 0.129 after 300; log_alpha within 4.6e-7).  The element-wise maximum,
    max |p_dev - p_ref| / max |p_ref - p_0|, is reported but not bounded: Adam's first steps move an element by
    lr * g / (|g| + eps), so elements whose gradient is near zero take different steps under any two fp32 summation
    orders (6.3e-3 after one update), and the difference compounds (0.42 after 300 updates)
"""
import os
import sys
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from baseline import reference_arm as ra  # noqa: E402
from mbrl_lib_b200 import replay, sac as bsac  # noqa: E402
from oracle import sac_f64  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
mbrl, REF_SRC = ra.import_reference()
needs_ref = pytest.mark.skipif(mbrl is None, reason=f"reference not importable here: {REF_SRC}")
M32 = np.uint64(0xFFFFFFFF)
RNG_STREAM_SAC = 0x70000


def _report(name, value):
    print(f"DEVIATION {name} {value:.3e}")


class Box:
    def __init__(self, A, lo=-1.0, hi=1.0):
        self.low = np.full(A, lo, np.float32) if np.isscalar(lo) else np.asarray(lo, np.float32)
        self.high = np.full(A, hi, np.float32) if np.isscalar(hi) else np.asarray(hi, np.float32)
        self.shape = (A,)


def _args(hidden, tuning=False, interval=1, lr=3e-4, alpha=0.2, device=DEV):
    return types.SimpleNamespace(gamma=0.99, tau=0.005, alpha=alpha, policy="Gaussian", target_update_interval=interval,
                                 automatic_entropy_tuning=tuning, target_entropy=None, hidden_size=hidden, device=device,
                                 lr=lr)


class Memory:
    """A replay buffer stand-in: sample() hands out the given batches in turn."""

    def __init__(self, batches):
        self.batches, self.i = batches, 0

    def sample(self, batch_size):
        b = self.batches[self.i % len(self.batches)]
        self.i += 1
        return b


def _batch(B, D, A, seed, terminated=0.3):
    rng = np.random.default_rng(seed)
    return replay.TransitionBatch(rng.standard_normal((B, D)), rng.uniform(-1, 1, (B, A)), rng.standard_normal((B, D)),
                                  rng.standard_normal(B), rng.random(B) < terminated, np.zeros(B, bool))


def _agent(D, A, H, seed, tuning=False, interval=1, box=None):
    torch.manual_seed(seed)
    agent = bsac.SAC(D, box or Box(A), _args(H, tuning, interval))
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():  # non-zero biases, so that no layer starts at an exact symmetry
        for p in list(agent.critic.parameters()) + list(agent.policy.parameters()):
            if p.dim() == 1:
                p.copy_(torch.randn(p.shape, generator=g) * 0.05)
        for t, p in zip(agent.critic_target.parameters(), agent.critic.parameters()):
            t.copy_(p + torch.randn(p.shape, generator=g).to(p.device) * 0.01)
    return agent


def _prefill(agent, seed):
    g = torch.Generator().manual_seed(seed)
    opts = [(agent.critic_optim, agent.critic.parameters()), (agent.policy_optim, agent.policy.parameters())]
    if agent.automatic_entropy_tuning:
        opts.append((agent.alpha_optim, [agent.log_alpha]))
        with torch.no_grad():
            agent.log_alpha.fill_(-0.7)
        agent.alpha = float(np.exp(-0.7))
    for opt, ps in opts:
        for p in ps:
            opt.state[p] = {"step": torch.tensor(9.0),
                            "exp_avg": (torch.randn(p.shape, generator=g) * 1e-2).to(p.device),
                            "exp_avg_sq": (torch.rand(p.shape, generator=g) * 1e-4 + 1e-6).to(p.device)}


def _snapshot(agent):
    sd = lambda m: {k: v.detach().double().cpu().clone() for k, v in m.state_dict().items()}  # noqa: E731
    st = lambda opt, mod: {k: (int(float(opt.state[p]["step"])) if p in opt.state else 0,  # noqa: E731
                               opt.state[p]["exp_avg"].double().cpu().clone() if p in opt.state else torch.zeros(p.shape, dtype=torch.float64),
                               opt.state[p]["exp_avg_sq"].double().cpu().clone() if p in opt.state else torch.zeros(p.shape, dtype=torch.float64))
                           for k, p in mod.named_parameters()}
    out = dict(critic=sd(agent.critic), target=sd(agent.critic_target), policy=sd(agent.policy),
               critic_state=st(agent.critic_optim, agent.critic), policy_state=st(agent.policy_optim, agent.policy))
    if agent.automatic_entropy_tuning:
        p = agent.log_alpha
        s = agent.alpha_optim.state
        out["log_alpha"] = p.detach().double().cpu().clone()
        out["alpha_state"] = (int(float(s[p]["step"])) if p in s else 0,
                              s[p]["exp_avg"].double().cpu().clone() if p in s else torch.zeros(1, dtype=torch.float64),
                              s[p]["exp_avg_sq"].double().cpu().clone() if p in s else torch.zeros(1, dtype=torch.float64))
    return out


def _oracle(agent, before, batch, eps, updates, reverse_mask):
    D = batch.obs.shape[1]
    cfg = dict(gamma=agent.gamma, tau=agent.tau, lr=agent.args.lr, alpha=float(agent.alpha),
               tuning=bool(agent.automatic_entropy_tuning), target_entropy=getattr(agent, "target_entropy", 0.0),
               target_update_interval=agent.target_update_interval, updates=updates, reverse_mask=reverse_mask,
               scale=agent.policy.action_scale.cpu(), bias=agent.policy.action_bias.cpu())
    f32 = lambda x: torch.from_numpy(np.asarray(x, np.float32)).double()  # noqa: E731  the rows the kernel reads
    b = (f32(batch.obs), f32(batch.act), f32(batch.next_obs), f32(batch.rewards), f32(batch.terminateds))
    assert b[0].shape[1] == D
    return sac_f64.sac_update(before["critic"], before["target"], before["policy"], before["critic_state"],
                              before["policy_state"], b, eps.double().cpu(), cfg, before.get("log_alpha"),
                              before.get("alpha_state"))


def _compare(name, before, after, want, fresh, bound=2e-4, moment_bound=1e-5):
    worst = {"update": 0.0, "moment": 0.0}
    for net, st in (("critic", "critic_state"), ("policy", "policy_state")):
        for k, p0 in before[net].items():
            p, q = after[net][k], want[net][k]
            du, du64 = p - p0, q - p0
            half_ulp = torch.from_numpy(np.spacing(np.abs(p.float().numpy()))).double() / 2
            m, v = after[st][k][1], after[st][k][2]
            m64, v64 = want[st][k][1], want[st][k][2]
            em = float((m - m64).abs().max() / m64.abs().max().clamp_min(1e-30))
            ev = float((v - v64).abs().max() / v64.abs().max().clamp_min(1e-30))
            if fresh:
                g64 = m64 / 0.1
                sel = g64.abs() > 1e-3 * g64.abs().max()
                err = float(((du - du64).abs() - half_ulp).clamp_min(0)[sel].max() / du64.abs().max()) if sel.any() else 0.0
            else:
                err = float(((du - du64).abs() - half_ulp).clamp_min(0).max() / du64.abs().max().clamp_min(1e-30))
            worst["update"] = max(worst["update"], err)
            worst["moment"] = max(worst["moment"], em, ev)
            assert err <= bound, f"{name} {net}.{k}: update off by {err:.3e} of its max"
            assert em <= moment_bound and ev <= moment_bound, f"{name} {net}.{k}: moments off by {em:.3e} / {ev:.3e}"
            assert after[st][k][0] == want[st][k][0]
    for k, v in want["target"].items():
        err = float((after["target"][k] - v).abs().max() / max(1e-30, float(v.abs().max())))
        assert err <= 1e-5, f"{name} target {k}: {err:.3e}"
    _report(f"update[{name}]", worst["update"])
    _report(f"moments[{name}]", worst["moment"])


UPDATE_CASES = [  # D, A, hidden, batch, tuning, reverse_mask, fresh
    (4, 1, 256, 256, True, True, False),
    (11, 3, 512, 37, False, True, False),
    (17, 6, 512, 256, True, False, False),
    (27, 8, 1024, 256, False, True, False),
    (45, 17, 1024, 300, False, False, False),
    (4, 1, 1024, 1, False, True, False),
    (11, 3, 256, 300, True, True, True),
    (17, 6, 1024, 37, False, True, True),
    (27, 8, 256, 1, True, False, False),
    (45, 17, 512, 37, True, True, False),
]


@pytest.mark.parametrize("D,A,H,B,tuning,reverse,fresh", UPDATE_CASES)
def test_one_update_matches_float64(D, A, H, B, tuning, reverse, fresh):
    agent = _agent(D, A, H, seed=D * 100 + H + B, tuning=tuning, box=Box(A, -np.linspace(1, 2, A), np.linspace(1, 3, A)))
    if not fresh:
        _prefill(agent, seed=B)
    batch = _batch(B, D, A, seed=B + D)
    eps = torch.randn(2, B, A, generator=torch.Generator().manual_seed(5)).to(DEV)
    before = _snapshot(agent)
    want = _oracle(agent, before, batch, eps, 0, reverse)
    out = agent.update_parameters(Memory([batch]), B, 0, reverse_mask=reverse, _eps=eps)
    after = _snapshot(agent)
    ill = (D, A, H, B, tuning) == (45, 17, 512, 37, True)
    _compare(f"{D},{A},{H},{B},{tuning},{reverse},{fresh}", before, after, want, fresh, 1e-3 if ill else 2e-4,
             2e-3 if ill else 1e-5)
    stats = list(out[:5])
    for got, w in zip(stats, want["stats"][:5]):
        assert abs(got - w) <= (1e-4 if ill else 1e-5) * max(1.0, abs(w)), (stats, want["stats"])
    if tuning:
        assert abs(float(agent.log_alpha) - float(want["log_alpha"])) <= 1e-6
        assert abs(float(agent.alpha) - want["alpha"]) <= 1e-6


@pytest.mark.parametrize("case", ["clamp", "ties"])
def test_clamp_bounds_and_min_ties(case):
    D, A, H, B = 17, 6, 256, 64
    agent = _agent(D, A, H, seed=3)
    _prefill(agent, seed=4)
    with torch.no_grad():
        if case == "clamp":  # log_std past the upper bound for the first half of the actions, past the lower for the rest
            agent.policy.log_std_linear.bias.copy_(torch.tensor([8.0, 8.0, 8.0, -30.0, -30.0, -30.0]))
            # At log_std = -20 the draw's std * eps (~2e-9) lies below an fp32 ulp of the mean, so x - mean is 0 in fp32
            # (in the reference as here) and log_prob differs from float64 by eps^2 / 2.  With alpha = 0 the
            # log-probability leaves the losses, and the clamp's zero gradient is checked through the reparameterisation.
            agent.alpha = 0.0
        else:  # identical twins: every min(Q1, Q2) is a tie
            for i in (1, 2, 3):
                for which in ("weight", "bias"):
                    for net in (agent.critic, agent.critic_target):
                        getattr(getattr(net, f"linear{i + 3}"), which).copy_(getattr(getattr(net, f"linear{i}"), which))
    batch = _batch(B, D, A, seed=9)
    eps = torch.randn(2, B, A, generator=torch.Generator().manual_seed(6)).to(DEV)
    before = _snapshot(agent)
    want = _oracle(agent, before, batch, eps, 0, True)
    agent.update_parameters(Memory([batch]), B, 0, reverse_mask=True, _eps=eps)
    after = _snapshot(agent)
    _compare(case, before, after, want, fresh=False)


@pytest.mark.parametrize("interval,updates", [(1, 0), (2, 3), (2, 4), (4, 8)])
def test_soft_update_is_torchs_formula(interval, updates):
    D, A, H, B = 11, 3, 256, 256
    agent = _agent(D, A, H, seed=11, interval=interval)
    _prefill(agent, seed=12)
    t0 = [p.detach().clone() for p in agent.critic_target.parameters()]
    agent.update_parameters(Memory([_batch(B, D, A, seed=13)]), B, updates, reverse_mask=True)
    due = updates % interval == 0
    for t, t_old, p in zip(agent.critic_target.parameters(), t0, agent.critic.parameters()):
        want = t_old * (1.0 - agent.tau) + p.detach() * agent.tau if due else t_old
        assert torch.equal(t.detach(), want)


def _workspace_eps(agent, B):
    """The draws on s of the last update, which the kernel keeps in its workspace (sac.cu SacWs.eps)."""
    H, A = agent._desc.hidden, agent._desc.act_dim
    r64 = lambda n: (n + 63) // 64 * 64  # noqa: E731
    off = 8 * r64(2 * B * H) + 2 * r64(B * H) + r64(2 * B * A) + r64(B * A)
    return agent._ws.view(torch.float32)[off:off + B * A].reshape(B, A).double().cpu().numpy()


def _workspace_act(agent, B):
    H, A = agent._desc.hidden, agent._desc.act_dim
    r64 = lambda n: (n + 63) // 64 * 64  # noqa: E731
    off = 8 * r64(2 * B * H) + 2 * r64(B * H)
    return agent._ws.view(torch.float32)[off:off + 2 * B * A].reshape(2, B, A).double().cpu().numpy()


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    c0, c1, c2, c3 = np.broadcast_arrays(*(np.asarray(c, np.uint64) for c in (c0, c1, c2, c3)))
    k0, k1 = int(k0), int(k1)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c0, np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ np.uint64(k0), p1 & M32, (p0 >> np.uint64(32)) ^ c3 ^ np.uint64(k1), p0 & M32
        k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
    return c0, c1, c2, c3


def sac_draws64(B, A, smp, seed, offset):
    """[B, A] draws of sample smp as common.cuh documents them: lane j & 3 of the Box-Muller block at counter (row, smp,
    RNG_STREAM_SAC | j >> 2, low word of offset) under key seed ^ (high word of offset)."""
    key = (seed ^ (offset & 0xFFFFFFFF00000000)) & 0xFFFFFFFFFFFFFFFF
    rows, j = np.arange(B)[:, None], np.arange(A)[None, :]
    r = philox4x32_10(rows, smp, RNG_STREAM_SAC | (j >> 2), offset & 0xFFFFFFFF, key & 0xFFFFFFFF, key >> 32)
    u = [((x >> np.uint64(8)).astype(np.float64) + 0.5) / 16777216.0 for x in r]
    lane = np.broadcast_to(j & 3, (B, A))
    ur, ua = np.where(lane < 2, u[0], u[2]), np.where(lane < 2, u[1], u[3])
    rad, ang = np.sqrt(-2.0 * np.log(ur)), 2.0 * np.pi * ua
    return np.where(lane & 1, rad * np.sin(ang), rad * np.cos(ang))


def test_draws_known_answer_and_statistics():
    from scipy import stats

    D, A, H, B = 11, 17, 256, 4000
    agent = _agent(D, A, H, seed=21)
    with torch.no_grad():  # mean 0 and log_std 0: the action is tanh(draw) on the unit box
        for lin in (agent.policy.mean_linear, agent.policy.log_std_linear):
            lin.weight.zero_()
            lin.bias.zero_()
    mem = Memory([_batch(B, D, A, seed=22)])
    draws = []
    for u in range(3):
        agent.update_parameters(mem, B, u, reverse_mask=True)
        got = _workspace_eps(agent, B)
        want = sac_draws64(B, A, 1, agent._seed, u)
        err = float(np.abs(got - want).max())
        _report(f"draws_known_answer[{u}]", err)
        assert err <= 1e-4
        a0 = _workspace_act(agent, B)[0]
        want0 = np.tanh(sac_draws64(B, A, 0, agent._seed, u))
        assert float(np.abs(a0 - want0).max()) <= 1e-4
        draws.append(got)
        with torch.no_grad():  # keep the heads at zero for the next update's check
            for lin in (agent.policy.mean_linear, agent.policy.log_std_linear):
                lin.weight.zero_()
                lin.bias.zero_()
    z = np.stack(draws)  # [update][row][action]
    p = stats.kstest(z.ravel(), "norm").pvalue
    _report("draws_ks_pvalue", p)
    assert p > 1e-3
    flat = lambda x: x.reshape(-1)  # noqa: E731
    for name, x, y in (("rows", z[0, :-1], z[0, 1:]), ("actions", z[0, :, :-1], z[0, :, 1:]), ("updates", z[0], z[1]),
                       ("samples", z[2], np.arctanh(np.clip(_workspace_act(agent, B)[0], -1 + 1e-6, 1 - 1e-6)))):
        c = abs(float(np.corrcoef(flat(x), flat(y))[0, 1]))
        _report(f"draws_corr_{name}", c)
        assert c < 0.03, name


def test_two_runs_are_bit_identical():
    D, A, H, B = 17, 6, 512, 256
    runs = []
    for _ in range(2):
        agent = _agent(D, A, H, seed=31, tuning=True)
        mem = Memory([_batch(B, D, A, seed=s) for s in range(3)])
        outs = [agent.update_parameters(mem, B, u, reverse_mask=True) for u in range(4)]
        runs.append((outs, [p.detach().clone() for p in list(agent.critic.parameters()) + list(agent.policy.parameters())
                            + list(agent.critic_target.parameters())], float(agent.log_alpha)))
    assert runs[0][0] == runs[1][0] and runs[0][2] == runs[1][2]
    assert all(torch.equal(a, b) for a, b in zip(runs[0][1], runs[1][1]))


# ---- against the reference --------------------------------------------------------------------------------------------
def _ref_sac(agent):
    from mbrl.third_party.pytorch_sac_pranz24.sac import SAC as RefSAC

    ref = RefSAC(agent._desc.obs_dim, Box(agent._desc.act_dim), agent.args)
    ref.critic.load_state_dict(agent.critic.state_dict())
    ref.critic_target.load_state_dict(agent.critic_target.state_dict())
    ref.policy.load_state_dict(agent.policy.state_dict())
    return ref


class _Eps:
    """Normal.rsample patched to consume recorded draws: loc + eps * scale."""

    def __init__(self, monkeypatch, queue):
        self.queue = queue
        monkeypatch.setattr(torch.distributions.Normal, "rsample", lambda d, sample_shape=torch.Size(): d.loc + self.queue.pop(0) * d.scale)


@needs_ref
def test_drift_against_the_reference_over_300_updates(monkeypatch):
    D, A, H, B, n = 11, 3, 256, 256, 300
    agent = _agent(D, A, H, seed=41, tuning=True, interval=2)
    ref = _ref_sac(agent)
    p0 = [p.detach().clone() for p in ref.policy.parameters()] + [p.detach().clone() for p in ref.critic.parameters()]
    batches = [_batch(B, D, A, seed=100 + i) for i in range(n)]
    g = torch.Generator().manual_seed(42)
    eps = [torch.randn(2, B, A, generator=g).to(DEV) for _ in range(n)]
    queue = []
    _Eps(monkeypatch, queue)
    mem_d, mem_r = Memory(batches), Memory(batches)
    names = [f"policy.{k}" for k, _ in ref.policy.named_parameters()] + [f"critic.{k}" for k, _ in ref.critic.named_parameters()]
    for u in range(n):
        agent.update_parameters(mem_d, B, u, reverse_mask=True, _eps=eps[u])
        queue.extend([eps[u][0], eps[u][1]])
        ref.update_parameters(mem_r, B, u, reverse_mask=True)
        if u + 1 in (1, 10, 100, n):
            mine = list(agent.policy.parameters()) + list(agent.critic.parameters())
            theirs = list(ref.policy.parameters()) + list(ref.critic.parameters())
            dev = [(float((p - q).abs().max() / (q - z).abs().max()), k) for p, q, z, k in zip(mine, theirs, p0, names)]
            rel = [(float((p - q).norm() / (q - z).norm()), k) for p, q, z, k in zip(mine, theirs, p0, names)]
            worst, where = max(dev)
            worst_norm, where_norm = max(rel)
            _report(f"drift_{u + 1}_elementwise[{where}]", worst)
            _report(f"drift_{u + 1}_norm[{where_norm}]", worst_norm)
            _report(f"drift_{u + 1}_log_alpha", abs(float(agent.log_alpha) - float(ref.log_alpha)))
    assert worst_norm <= 0.25
    assert abs(float(agent.log_alpha) - float(ref.log_alpha)) <= 2e-2 * abs(float(ref.log_alpha))


@needs_ref
def test_drop_in_with_the_reference_buffer_logger_and_checkpoints(tmp_path):
    from mbrl.util.replay_buffer import ReplayBuffer

    D, A, H, B = 17, 6, 256, 64
    rb = ReplayBuffer(1000, (D,), (A,), rng=np.random.default_rng(7))
    twin = ReplayBuffer(1000, (D,), (A,), rng=np.random.default_rng(7))
    b = _batch(500, D, A, seed=51)
    for buf in (rb, twin):
        buf.add_batch(b.obs, b.act, b.next_obs, b.rewards, b.terminateds, b.truncateds)
    agent = _agent(D, A, H, seed=52, tuning=True)

    class Log:
        def __init__(self):
            self.keys = []

        def log(self, key, value, step):
            self.keys.append(key)
            float(value)

    log = Log()
    seen = []
    orig = rb.sample
    rb.sample = lambda n: seen.append(orig(n)) or seen[-1]
    agent.update_parameters(rb, B, 0, logger=log, reverse_mask=True)
    want = twin.sample(B)
    np.testing.assert_array_equal(seen[0].obs, want.obs)
    assert log.keys == ["train/batch_reward", "train_critic/loss", "train_actor/loss", "train_actor/target_entropy",
                        "train_actor/entropy", "train_alpha/loss", "train_alpha/value"]
    assert all(float(agent.critic_optim.state[p]["step"]) == 1 for p in agent.critic.parameters())
    assert all(float(agent.policy_optim.state[p]["step"]) == 1 for p in agent.policy.parameters())
    assert float(agent.alpha_optim.state[agent.log_alpha]["step"]) == 1

    ref = _ref_sac(agent)
    path = str(tmp_path / "sac.pth")
    agent.save_checkpoint(ckpt_path=path)
    ref.load_checkpoint(path)
    for a, r in ((agent.policy, ref.policy), (agent.critic, ref.critic), (agent.critic_target, ref.critic_target)):
        assert a.state_dict().keys() == r.state_dict().keys()
        assert all(torch.equal(x, y) for x, y in zip(a.state_dict().values(), r.state_dict().values()))
    # and back: the reference's checkpoint into a fresh agent, which keeps training from the loaded Adam state
    path2 = str(tmp_path / "ref.pth")
    ref.save_checkpoint(ckpt_path=path2)
    other = _agent(D, A, H, seed=53, tuning=True)
    other.load_checkpoint(path2)
    assert all(torch.equal(x, y) for x, y in zip(other.policy.state_dict().values(), ref.policy.state_dict().values()))
    other.update_parameters(rb, B, 1, reverse_mask=True)
    assert all(float(other.critic_optim.state[p]["step"]) == 2 for p in other.critic.parameters())


@needs_ref
def test_sac_agent_runs_the_device_rollout():
    from mbrl.planning.sac_wrapper import SACAgent
    from mbrl.util.replay_buffer import ReplayBuffer

    import mbrl_lib_b200 as bp
    from mbrl_lib_b200 import functions, mbpo, synthetic as syn

    spec = syn.CASES["halfcheetah_small"]
    arrays = syn.make_model_arrays(spec)
    model = bp.model_from_arrays(spec, arrays, DEV)
    D, A = spec.obs_dim, spec.act_dim

    class Env:
        observation_space = Box(D, -np.inf, np.inf)
        action_space = Box(A)

    env = bp.ModelEnv(Env(), model, functions.no_termination, functions.reward_halfcheetah,
                      generator=torch.Generator(device=DEV))
    agent = SACAgent(_agent(D, A, 256, seed=61))
    rb = ReplayBuffer(1000, (D,), (A,), rng=np.random.default_rng(0))
    b = _batch(200, D, A, seed=62)
    rb.add_batch(b.obs.astype(np.float32), b.act.astype(np.float32), b.next_obs.astype(np.float32), b.rewards.astype(np.float32),
                 b.terminateds, b.truncateds)
    sac_buf = ReplayBuffer(10000, (D,), (A,), rng=np.random.default_rng(1))
    mbpo.rollout_model_and_populate_sac_buffer(env, rb, agent, sac_buf, True, 3, 50)
    assert len(sac_buf) == 150
    out = agent.sac_agent.update_parameters(sac_buf, 64, 0, reverse_mask=True)
    assert all(np.isfinite(out))
