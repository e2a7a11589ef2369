"""MBPO's SAC agent with its update on the device: ``SAC`` has the constructor, attributes and methods of mbrl-lib's
``mbrl.third_party.pytorch_sac_pranz24.SAC`` (sac.py), so ``mbpo.train`` runs it with
``algorithm.agent._target_=mbrl_lib_b200.SAC``.

``update_parameters`` samples the replay buffer once (its generator advances exactly as in the reference), packs the rows
as float32 into a pinned staging buffer, and makes one host-to-device copy, one launch of ``b200pets_sac_update`` (the
critic step, the policy step, the temperature step and the soft target update, csrc/sac.cu) and one device-to-host copy
of the statistics.  The networks, ``torch.optim.Adam`` optimizers and ``log_alpha`` are ordinary torch objects: the kernel
updates their tensors and the optimizers' ``exp_avg`` / ``exp_avg_sq`` in place, and this class advances each
optimizer's ``step``, so ``state_dict()`` and checkpoints stay truthful and move both ways with the reference.

Draws.  The reparameterisation noise of an update comes from Philox inside the kernel, keyed by a seed drawn from torch's
default generator at construction (``torch.manual_seed`` makes a run reproducible) and by the object's update counter.
It is not the stream ``Normal.rsample`` would draw from torch's generator, so the agent trains with other noise than the
reference does; given the same noise (``_eps``) it computes the reference's update.

Refused with ``NotImplementedError`` at construction: ``policy != "Gaussian"``, a device other than CUDA, and sizes the
kernel does not cover (more than 32 actions).  ``select_action`` is the reference's PyTorch code.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.distributions import Normal
from torch.optim import Adam

from . import _lib

LOG_SIG_MAX = 2
LOG_SIG_MIN = -20
EPSILON = 1e-6


def _xavier(m):
    if isinstance(m, nn.Linear):
        nn.init.xavier_uniform_(m.weight, gain=1)
        nn.init.constant_(m.bias, 0)


class QNetwork(nn.Module):
    """Twin Q networks on ``cat(state, action)``; parameter names as the reference's (linear1 .. linear6)."""

    def __init__(self, num_inputs, num_actions, hidden_dim):
        super().__init__()
        for first in (1, 4):
            setattr(self, f"linear{first}", nn.Linear(num_inputs + num_actions, hidden_dim))
            setattr(self, f"linear{first + 1}", nn.Linear(hidden_dim, hidden_dim))
            setattr(self, f"linear{first + 2}", nn.Linear(hidden_dim, 1))
        self.apply(_xavier)

    def _q(self, xu, first):
        layers = [getattr(self, f"linear{first + i}") for i in range(3)]
        return layers[2](F.relu(layers[1](F.relu(layers[0](xu)))))

    def forward(self, state, action):
        xu = torch.cat([state, action], 1)
        return self._q(xu, 1), self._q(xu, 4)


class GaussianPolicy(nn.Module):
    """tanh-squashed Gaussian policy; parameter names as the reference's (linear1, linear2, mean_linear, log_std_linear)."""

    def __init__(self, num_inputs, num_actions, hidden_dim, action_space=None):
        super().__init__()
        self.linear1 = nn.Linear(num_inputs, hidden_dim)
        self.linear2 = nn.Linear(hidden_dim, hidden_dim)
        self.mean_linear = nn.Linear(hidden_dim, num_actions)
        self.log_std_linear = nn.Linear(hidden_dim, num_actions)
        self.apply(_xavier)
        if action_space is None:
            self.action_scale, self.action_bias = torch.tensor(1.0), torch.tensor(0.0)
        else:
            high, low = np.array(action_space.high), np.array(action_space.low)
            self.action_scale = torch.FloatTensor((high - low) / 2.0)
            self.action_bias = torch.FloatTensor((high + low) / 2.0)

    def forward(self, state):
        x = F.relu(self.linear2(F.relu(self.linear1(state))))
        return self.mean_linear(x), torch.clamp(self.log_std_linear(x), min=LOG_SIG_MIN, max=LOG_SIG_MAX)

    def sample(self, state):
        mean, log_std = self.forward(state)
        normal = Normal(mean, log_std.exp())
        x_t = normal.rsample()
        y_t = torch.tanh(x_t)
        action = y_t * self.action_scale + self.action_bias
        log_prob = normal.log_prob(x_t) - torch.log(self.action_scale * (1 - y_t.pow(2)) + EPSILON)
        return action, log_prob.sum(1, keepdim=True), torch.tanh(mean) * self.action_scale + self.action_bias

    def to(self, device):
        self.action_scale = self.action_scale.to(device)
        self.action_bias = self.action_bias.to(device)
        return super().to(device)


def hard_update(target, source):
    for t, p in zip(target.parameters(), source.parameters()):
        t.data.copy_(p.data)


def sac_desc(num_inputs, action_space, args, target_entropy):
    A = int(action_space.shape[0])
    d = _lib.SacDesc()
    d.obs_dim, d.act_dim, d.hidden = int(num_inputs), A, int(args.hidden_size)
    if A <= _lib.SAC_MAX_ACTIONS:
        high, low = np.array(action_space.high, dtype=np.float64), np.array(action_space.low, dtype=np.float64)
        scale, bias = ((high - low) / 2.0).astype(np.float32), ((high + low) / 2.0).astype(np.float32)
        for j in range(A):
            d.action_scale[j], d.action_bias[j] = float(scale[j]), float(bias[j])
    d.gamma, d.tau, d.lr = float(args.gamma), float(args.tau), float(args.lr)
    d.beta1, d.beta2, d.eps = 0.9, 0.999, 1e-8  # torch.optim.Adam's defaults, which the reference uses
    d.automatic_entropy_tuning = 1 if args.automatic_entropy_tuning is True else 0
    d.target_entropy = float(target_entropy) if d.automatic_entropy_tuning else 0.0
    d.target_update_interval = int(args.target_update_interval)
    return d


class SAC:
    """Drop-in for ``mbrl.third_party.pytorch_sac_pranz24.SAC`` whose ``update_parameters`` is one device launch."""

    def __init__(self, num_inputs, action_space, args):
        self.args = args
        self.gamma = args.gamma
        self.tau = args.tau
        self.alpha = args.alpha
        self.policy_type = args.policy
        self.target_update_interval = args.target_update_interval
        self.automatic_entropy_tuning = args.automatic_entropy_tuning
        self.device = torch.device(args.device)
        if self.policy_type != "Gaussian":
            raise NotImplementedError(f"mbrl_lib_b200.SAC trains the Gaussian policy only, not {self.policy_type!r}")
        if self.device.type != "cuda":
            raise NotImplementedError(f"mbrl_lib_b200.SAC updates on a CUDA device, not {self.device}")
        A = int(action_space.shape[0])
        te = 0.0
        if self.automatic_entropy_tuning is True:
            te = -float(np.prod(action_space.shape)) if args.target_entropy is None else args.target_entropy
        desc = sac_desc(num_inputs, action_space, args, te)
        lib = _lib.load()
        if lib.b200pets_sac_supported(C.byref(desc)) != 0:
            raise NotImplementedError(lib.b200pets_last_error().decode())
        self._desc = desc
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())

        self.critic = QNetwork(num_inputs, A, args.hidden_size).to(device=self.device)
        self.critic_optim = Adam(self.critic.parameters(), lr=args.lr)
        self.critic_target = QNetwork(num_inputs, A, args.hidden_size).to(self.device)
        hard_update(self.critic_target, self.critic)
        if self.automatic_entropy_tuning is True:
            self.target_entropy = te
            self.log_alpha = torch.zeros(1, requires_grad=True, device=self.device)
            self.alpha_optim = Adam([self.log_alpha], lr=args.lr)
        self.policy = GaussianPolicy(num_inputs, A, args.hidden_size, action_space).to(self.device)
        self.policy_optim = Adam(self.policy.parameters(), lr=args.lr)

        self._seed = int(torch.randint(0, 2**62, (1,)).item())
        self._updates_done = 0
        self._alpha_dev = torch.full((1,), float(args.alpha), dtype=torch.float32, device=self.device)
        self._stats_dev = torch.zeros(8, dtype=torch.float32, device=self.device)
        self._stats_host = torch.zeros(8, dtype=torch.float32).pin_memory()
        self._rows = 0
        self._handle = None
        self._handle_key = None

    # ---- reference methods ------------------------------------------------------------------------------------------
    def select_action(self, state, batched=False, evaluate=False):
        state = torch.FloatTensor(state)
        if not batched:
            state = state.unsqueeze(0)
        state = state.to(self.device)
        if evaluate is False:
            action, _, _ = self.policy.sample(state)
        else:
            _, _, action = self.policy.sample(state)
        if batched:
            return action.detach().cpu().numpy()
        return action.detach().cpu().numpy()[0]

    def save_checkpoint(self, env_name=None, suffix="", ckpt_path=None):
        if ckpt_path is None:
            assert env_name is not None
            os.makedirs("checkpoints/", exist_ok=True)
            ckpt_path = "checkpoints/sac_checkpoint_{}_{}".format(env_name, suffix)
        print("Saving models to {}".format(ckpt_path))
        torch.save({"policy_state_dict": self.policy.state_dict(),
                    "critic_state_dict": self.critic.state_dict(),
                    "critic_target_state_dict": self.critic_target.state_dict(),
                    "critic_optimizer_state_dict": self.critic_optim.state_dict(),
                    "policy_optimizer_state_dict": self.policy_optim.state_dict()}, ckpt_path)

    def load_checkpoint(self, ckpt_path, evaluate=False):
        print("Loading models from {}".format(ckpt_path))
        if ckpt_path is not None:
            checkpoint = torch.load(ckpt_path)
            self.policy.load_state_dict(checkpoint["policy_state_dict"])
            self.critic.load_state_dict(checkpoint["critic_state_dict"])
            self.critic_target.load_state_dict(checkpoint["critic_target_state_dict"])
            self.critic_optim.load_state_dict(checkpoint["critic_optimizer_state_dict"])
            self.policy_optim.load_state_dict(checkpoint["policy_optimizer_state_dict"])
            for m in (self.policy, self.critic, self.critic_target):
                m.train(not evaluate)

    # ---- the device update ------------------------------------------------------------------------------------------
    def _optimizers(self):
        opts = [(self.critic_optim, list(self.critic.parameters())), (self.policy_optim, list(self.policy.parameters()))]
        if self.automatic_entropy_tuning is True:
            opts.append((self.alpha_optim, [self.log_alpha]))
        return opts

    @staticmethod
    def _adam_state(opt, params):
        """The optimizer's state of each parameter, created as torch.optim.Adam creates it at the first step; returns the
        common step count."""
        for p in params:
            st = opt.state[p]
            if len(st) == 0:
                scalar = torch.float64 if torch.get_default_dtype() == torch.float64 else torch.float32
                st["step"] = torch.tensor(0.0, dtype=scalar)
                st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        steps = {float(opt.state[p]["step"]) for p in params}
        if len(steps) != 1:
            raise RuntimeError(f"the parameters' Adam step counts differ ({sorted(steps)}); one fused step updates all")
        return int(steps.pop())

    def _sac_handle(self, opts):
        """The C handle over the current tensors (re-made when a load_state_dict replaced one of them)."""
        params = [p for _, ps in opts[:2] for p in ps]
        state = [(self.critic_optim if i < _lib.SAC_NUM_CRITIC_PARAMS else self.policy_optim).state[p]
                 for i, p in enumerate(params)]
        la = [None, None, None]
        if self.automatic_entropy_tuning is True:
            st = self.alpha_optim.state[self.log_alpha]
            la = [self.log_alpha.data_ptr(), st["exp_avg"].data_ptr(), st["exp_avg_sq"].data_ptr()]
        P = [p.data_ptr() for p in params]
        T = [p.data_ptr() for p in self.critic_target.parameters()]
        M = [s["exp_avg"].data_ptr() for s in state]
        V = [s["exp_avg_sq"].data_ptr() for s in state]
        key = (tuple(P), tuple(T), tuple(M), tuple(V), tuple(la))
        if key != self._handle_key:
            self._close()
            lib = _lib.load()
            arr = lambda xs: (C.c_void_p * len(xs))(*xs)
            h = C.c_void_p()
            _lib.check(lib.b200pets_sac_create(C.byref(self._desc), arr(P), arr(T), arr(M), arr(V), *la, C.byref(h)),
                       "sac_create")
            self._handle, self._handle_key = h, key
        return self._handle

    def _buffers(self, B):
        if B > self._rows:
            W = 2 * self._desc.obs_dim + self._desc.act_dim + 2
            self._stage_host = torch.empty(B, W, dtype=torch.float32).pin_memory()
            self._stage_dev = torch.empty(B, W, dtype=torch.float32, device=self.device)
            self._rows = B
        need = _lib.load().b200pets_sac_workspace_bytes(self._handle, B)
        if getattr(self, "_ws", None) is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)

    def update_parameters(self, memory, batch_size, updates, logger=None, reverse_mask=False, _eps=None):
        """One SAC update (sac.py:76-173).  ``_eps``: a [2][B][A] device tensor of reparameterisation draws (on s', then
        on s) used instead of the in-kernel ones, for tests."""
        state_batch, action_batch, next_state_batch, reward_batch, mask_batch, _ = memory.sample(batch_size).astuple()
        B = len(state_batch)
        D, A = self._desc.obs_dim, self._desc.act_dim
        lib = _lib.load()
        opts = self._optimizers()
        steps = [self._adam_state(o, ps) for o, ps in opts] + ([] if len(opts) == 3 else [0])
        h = self._sac_handle(opts)
        self._buffers(B)
        if self.alpha is not self._alpha_dev:  # args.alpha, or a temperature the caller set
            self._alpha_dev.fill_(float(self.alpha))
        stage = self._stage_host[:B].numpy()
        stage[:, :D] = state_batch
        stage[:, D:D + A] = action_batch
        stage[:, D + A:2 * D + A] = next_state_batch
        stage[:, 2 * D + A] = reward_batch
        stage[:, 2 * D + A + 1] = mask_batch
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream()
            self._stage_dev[:B].copy_(self._stage_host[:B], non_blocking=True)
            eps = None if _eps is None else _eps.contiguous()
            _lib.check(lib.b200pets_sac_update(h, B, int(updates), 1 if reverse_mask else 0, (C.c_int64 * 3)(*steps),
                                               _lib.ptr(self._stage_dev), _lib.ptr(eps), self._seed, self._updates_done,
                                               _lib.ptr(self._alpha_dev), _lib.ptr(self._stats_dev), _lib.ptr(self._ws),
                                               self._ws.numel(), C.c_void_p(stream.cuda_stream)), "sac_update")
            self._stats_host.copy_(self._stats_dev, non_blocking=True)
            stream.synchronize()
        self._updates_done += 1
        for o, ps in opts:
            for p in ps:
                o.state[p]["step"] += 1
        qf1, qf2, pol, alpha_loss, alpha, reward_mean, entropy, _ = self._stats_host.tolist()
        if self.automatic_entropy_tuning is True:
            self.alpha = self._alpha_dev
        if logger is not None:
            logger.log("train/batch_reward", reward_mean, updates)
            logger.log("train_critic/loss", qf1 + qf2, updates)
            logger.log("train_actor/loss", pol, updates)
            logger.log("train_actor/target_entropy",
                       self.target_entropy if self.automatic_entropy_tuning else 0, updates)
            logger.log("train_actor/entropy", entropy, updates)
            logger.log("train_alpha/loss", alpha_loss, updates)
            logger.log("train_alpha/value", alpha, updates)
        return qf1, qf2, pol, alpha_loss, alpha

    def _close(self):
        if self._handle is not None:
            _lib.load().b200pets_sac_destroy(self._handle)
            self._handle, self._handle_key = None, None

    def __del__(self):
        try:
            self._close()
        except Exception:
            pass
