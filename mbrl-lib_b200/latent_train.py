"""Training PlaNet's latent model on the device: ``PlaNetModel.loss`` / ``update`` (mbrl/models/planet.py:406-519)
with the recurrence as two kernels.

The reference walks the sequence one step at a time, running the conv encoder, the belief GRU, both transition models,
two draws, the conv decoder and the reward model on a batch of rows per step.  Only the recurrence is sequential in
time, so :func:`loss` runs

1. ``model.encoder`` once over all B x T frames and the posterior's encoding half ``P = enc W_q1e^T + b_q1``;
2. the recurrence (belief GRU, posterior, prior and both draws, all T steps) as one ``b200pets_latent_seq_forward``;
3. ``model.decoder`` and ``model.reward_model`` once over all B x T states, and the KL with free nats, the observation
   loss and the reward loss as one batched expression each.

``loss.backward()`` reaches the recurrence through :class:`Recurrence`, whose backward is one
``b200pets_latent_seq_backward`` launch followed by the weight gradients: those do not depend on the order in time, so
they are matrix products over all B x T rows of the stored layer inputs and the pre-activation gradients the kernel
wrote (torch matmuls, under the caller's matmul precision settings like the reference's own backward).  The
convolutions stay in the caller's modules under the caller's cuDNN settings, and :func:`update` ends with the
reference's ``clip_grad_norm_`` and the optimizer's own ``step()``.

Draws.  In-kernel Philox on ``RNG_STREAM_LATENT_TRAIN`` (csrc/common.cuh), keyed by the model's ``rng``: its
``initial_seed()`` and, for a CUDA generator, its Philox offset, which each call advances by 4, so ``rng.manual_seed``
makes a run reproducible.  The draws are not the reference's ``torch.randn`` stream, and the ``rng`` is not advanced the
way the reference's per-step ``torch.randn`` calls advance it.  ``eps=(eps_q, eps_p)``, each ``[T, B, L]``, replaces
them (tests).
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

from . import _lib

_TAPE_FWD = ("e", "gates", "q1", "p1", "pre_std", "eps")
_TAPE_BWD = ("de", "dgi", "dghn", "dq", "dv", "dp")


def is_trainable_latent_model(model) -> bool:
    """Whether ``model`` has the modules PlaNet's loss needs (``encoder``, ``posterior_transition_model``, ``decoder``
    beside the planning half)."""
    return all(hasattr(model, n) for n in ("belief_model", "prior_transition_model", "reward_model", "encoder",
                                           "posterior_transition_model", "decoder", "free_nats"))


def recurrence_params(model) -> List[torch.Tensor]:
    """The recurrence's parameters in the order ``b200pets_latent_seq_forward`` takes them (include/b200pets.h)."""
    emb, rnn = model.belief_model.embedding_layer[0], model.belief_model.rnn
    q1, q2 = model.posterior_transition_model[0], model.posterior_transition_model[2]
    p1, p2 = model.prior_transition_model[0], model.prior_transition_model[2]
    return [emb.weight, emb.bias, rnn.weight_ih, rnn.weight_hh, rnn.bias_ih, rnn.bias_hh, q1.weight, q2.weight, q2.bias,
            p1.weight, p1.bias, p2.weight, p2.bias]


def train_desc(model) -> _lib.LatentTrainDesc:
    """The C descriptor of a PlaNet model's recurrence; ValueError when its layers do not chain as PlaNet's do."""
    emb, rnn = model.belief_model.embedding_layer[0], model.belief_model.rnn
    q1, q2 = model.posterior_transition_model[0], model.posterior_transition_model[2]
    p1, p2 = model.prior_transition_model[0], model.prior_transition_model[2]
    Hb, L, Hf = int(rnn.hidden_size), int(p2.out_features) // 2, int(p1.out_features)
    A, E = int(emb.in_features) - L, int(q1.in_features) - Hb
    for mod, name in ((model.belief_model.embedding_layer[1], "belief_model.embedding_layer[1]"),
                      (model.prior_transition_model[1], "prior_transition_model[1]"),
                      (model.posterior_transition_model[1], "posterior_transition_model[1]")):
        if type(mod).__name__ != "ReLU":
            raise ValueError(f"{name} is {type(mod).__name__}; the recurrence kernels implement PlaNet's ReLU")
    if (int(emb.out_features), int(rnn.input_size), int(p1.in_features), int(q1.out_features), int(q2.in_features),
            int(q2.out_features)) != (Hb, Hb, Hb, Hf, Hf, 2 * L) or A < 1 or E < 1 or not getattr(rnn, "bias", True):
        raise ValueError("the latent model's layer sizes do not chain as PlaNet's do (planet.py:82-114, 225-252)")
    d = _lib.LatentTrainDesc()
    d.action_size, d.latent_size, d.belief_size, d.hidden_size, d.encoding_size = A, L, Hb, Hf, E
    d.min_std = float(model.min_std)
    return d


def supported(model) -> bool:
    """Whether the device path takes ``model``: PlaNet's layout, fp32 contiguous CUDA parameters on one device and sizes
    ``b200pets_latent_train_supported`` accepts (asked before anything is touched)."""
    if not is_trainable_latent_model(model):
        return False
    try:
        desc = train_desc(model)
    except ValueError:
        return False
    params = list(model.parameters())
    dev = params[0].device
    if dev.type != "cuda" or any(p.dtype != torch.float32 or p.device != dev for p in params) or \
            not all(p.is_contiguous() for p in recurrence_params(model)):
        return False
    with torch.cuda.device(dev):
        return _lib.load().b200pets_latent_train_supported(C.byref(desc)) == 0


def draw_key(model) -> Tuple[int, int]:
    """(seed, offset) of one call's Philox draws from the model's ``rng`` (see the module docstring)."""
    rng = getattr(model, "rng", None)
    if rng is None:
        rng = torch.default_generator
    seed = int(rng.initial_seed()) & 0xFFFFFFFFFFFFFFFF
    if rng.device.type == "cuda":
        offset = int(rng.get_offset())
        rng.set_offset(offset + 4)
        return seed, offset
    n = getattr(model, "_latent_train_calls", 0)
    model._latent_train_calls = n + 1
    return seed, n


class _Call:
    """What one recurrence call needs besides tensors."""

    def __init__(self, desc, B: int, T: int, eps, seed: int, offset: int):
        self.desc, self.B, self.T, self.eps, self.seed, self.offset = desc, B, T, eps, seed, offset


class Recurrence(torch.autograd.Function):
    """The RSSM over T steps: ``(beliefs [B,T,Hb], post_params [B,T,2L], post_samples [B,T,L], prior_params [B,T,2L],
    prior_samples [B,T,L])`` from ``P [B,T,Hf]``, ``act [B,T,A]`` and :func:`recurrence_params`."""

    @staticmethod
    def forward(ctx, call: _Call, P, act, *params):
        lib = _lib.load()
        d, B, T = call.desc, call.B, call.T
        L, Hb, Hf = d.latent_size, d.belief_size, d.hidden_size
        dev = P.device
        out = [torch.empty(B, T, w, device=dev) for w in (Hb, 2 * L, L, 2 * L, L)]
        keep = any(ctx.needs_input_grad[1:])
        tape = _lib.LatentTape()
        bufs = {}
        if keep:
            widths = {"e": Hb, "gates": 4 * Hb, "q1": Hf, "p1": Hf, "pre_std": 2 * L, "eps": 2 * L}
            bufs = {k: torch.empty(B, T, w, device=dev) for k, w in widths.items()}
            for k, v in bufs.items():
                setattr(tape, k, v.data_ptr())
        ws = torch.empty(lib.b200pets_latent_train_workspace_bytes(C.byref(d), B, T), dtype=torch.uint8, device=dev)
        ptrs = (C.c_void_p * len(params))(*[p.data_ptr() for p in params])
        eps_q, eps_p = call.eps if call.eps is not None else (None, None)
        with torch.cuda.device(dev):
            _lib.check(lib.b200pets_latent_seq_forward(
                C.byref(d), ptrs, B, T, _lib.ptr(P), _lib.ptr(act), _lib.ptr(eps_q), _lib.ptr(eps_p), call.seed,
                call.offset, *[_lib.ptr(o) for o in out], C.byref(tape) if keep else None, _lib.ptr(ws), ws.numel(),
                _lib.stream_ptr()), "latent_seq_forward")
        if keep:
            ctx.call = call
            ctx.bufs = bufs
            ctx.save_for_backward(act, out[0], out[2], *params)
        return tuple(out)

    @staticmethod
    def backward(ctx, g_bel, g_qp, g_qs, g_pp, g_ps):
        lib = _lib.load()
        call = ctx.call
        d, B, T = call.desc, call.B, call.T
        L, Hb, Hf = d.latent_size, d.belief_size, d.hidden_size
        act, beliefs, post_samples, *params = ctx.saved_tensors
        dev = beliefs.device
        bufs = ctx.bufs
        widths = {"de": Hb, "dgi": 3 * Hb, "dghn": Hb, "dq": 2 * L, "dv": Hf, "dp": 2 * L}
        bufs.update({k: torch.empty(B, T, w, device=dev) for k, w in widths.items()})
        tape = _lib.LatentTape(*[bufs[k].data_ptr() for k in _TAPE_FWD + _TAPE_BWD])
        dP = torch.empty(B, T, Hf, device=dev)
        grads = [None if g is None else g.contiguous() for g in (g_bel, g_qp, g_qs, g_pp, g_ps)]
        ptrs = (C.c_void_p * len(params))(*[p.data_ptr() for p in params])
        with torch.cuda.device(dev):
            _lib.check(lib.b200pets_latent_seq_backward(
                C.byref(d), ptrs, B, T, _lib.ptr(beliefs), *[_lib.ptr(g) for g in grads], C.byref(tape), _lib.ptr(dP),
                _lib.stream_ptr()), "latent_seq_backward")
        g = weight_grads(bufs, dP, act, beliefs, post_samples, params[6])
        ctx.bufs = None
        return (None, dP, None, *g)


def weight_grads(tape: Dict[str, torch.Tensor], dP, act, beliefs, post_samples, W_q1) -> List[torch.Tensor]:
    """The gradients of :func:`recurrence_params` from the backward kernel's tape: products over all B x T rows of the
    layers' stored inputs and pre-activation gradients (the order in time does not enter)."""
    B, T, Hb = beliefs.shape
    L, Hf = post_samples.shape[2], dP.shape[2]
    N, dev = B * T, beliefs.device
    rows = {k: v.view(N, -1) for k, v in tape.items()}
    # the layer inputs of step t: the state after step t - 1 (zeros before the first step)
    h_prev = torch.zeros(B, T, Hb, device=dev)
    h_prev[:, 1:] = beliefs[:, :-1]
    s_prev = torch.zeros(B, T, L, device=dev)
    s_prev[:, 1:] = post_samples[:, :-1]
    h, x = beliefs.reshape(N, Hb), torch.cat([s_prev, act], -1).view(N, -1)
    de, dgi, dq, dv, dp, du = rows["de"], rows["dgi"], rows["dq"], rows["dv"], rows["dp"], dP.view(N, Hf)
    dgh = torch.cat([dgi[:, :2 * Hb], rows["dghn"]], 1)
    g_wq1 = torch.zeros_like(W_q1)
    g_wq1[:, :Hb] = du.t() @ h
    return [de.t() @ x, de.sum(0), dgi.t() @ rows["e"], dgh.t() @ h_prev.view(N, Hb), dgi.sum(0), dgh.sum(0), g_wq1,
            dq.t() @ rows["q1"], dq.sum(0), dv.t() @ h, dv.sum(0), dp.t() @ rows["p1"], dp.sum(0)]


def recurrence(model, P: torch.Tensor, act: torch.Tensor, eps=None):
    """:class:`Recurrence` over the model's parameters, with the draws keyed by :func:`draw_key` unless ``eps``."""
    B, T = int(P.shape[0]), int(P.shape[1])
    desc = train_desc(model)
    seed, offset = (0, 0) if eps is not None else draw_key(model)
    if eps is not None:
        eps = tuple(e.to(P.device, torch.float32).contiguous() for e in eps)
    call = _Call(desc, B, T, eps, seed, offset)
    return Recurrence.apply(call, P.contiguous(), act.contiguous(), *recurrence_params(model))


def _process_batch(model, batch):
    """``PlaNetModel._process_batch(batch, pixel_obs=True)`` (planet.py:274-287, model.py:50-68)."""
    dev = next(model.parameters()).device
    obs, act, rew = (torch.as_tensor(x).to(dev).float() for x in (batch.obs, batch.act, batch.rewards))
    return obs / 256.0 - 0.5, act, rew


def _loss_terms(model, batch, eps=None):
    """Per-(b, t) observation, reward and KL losses and the reconstruction, as planet.py:429-462 computes them."""
    obs, action, rewards = _process_batch(model, batch)
    next_obs, act, rew = obs[:, 1:], action[:, :-1], rewards[:, :-1]
    B, T = int(next_obs.shape[0]), int(next_obs.shape[1])
    Hb, L = model.belief_size, model.latent_state_size
    q1 = model.posterior_transition_model[0]
    enc = model.encoder(next_obs.reshape(B * T, *next_obs.shape[2:]))
    P = F.linear(enc, q1.weight[:, Hb:], q1.bias).view(B, T, -1)
    beliefs, post_params, post_samples, prior_params, _ = recurrence(model, P, act, eps)
    pred_next_obs = model.decoder(torch.cat([post_samples, beliefs], -1).view(B * T, -1)).view(next_obs.shape)
    pred_rewards = model.reward_model(torch.cat([beliefs, post_samples], -1)).view(B, T)
    obs_loss = F.mse_loss(pred_next_obs, next_obs, reduction="none").sum((2, 3, 4))
    reward_loss = F.mse_loss(pred_rewards, rew, reduction="none")
    kl_loss = torch.distributions.kl_divergence(
        torch.distributions.Normal(post_params[..., :L], post_params[..., L:]),
        torch.distributions.Normal(prior_params[..., :L], prior_params[..., L:])).sum(2).max(model.free_nats)
    return obs_loss, reward_loss, kl_loss, pred_next_obs


def loss(model, batch, reduce: bool = True, *, eps=None) -> Tuple[torch.Tensor, Dict]:
    """``PlaNetModel.loss(batch, reduce=reduce)``: the same loss and meta dict (``reconstruction``,
    ``observations_loss``, ``reward_loss``, ``kl_loss``)."""
    obs_loss, reward_loss, kl_loss, recon = _loss_terms(model, batch, eps)
    if reduce:
        obs_loss, reward_loss, kl_loss = obs_loss.mean(), reward_loss.mean(), kl_loss.mean()
    o, r, k = torch.stack([obs_loss.detach().mean(), reward_loss.detach().mean(), kl_loss.detach().mean()]).tolist()
    meta = {"reconstruction": recon.detach(), "observations_loss": o, "reward_loss": r, "kl_loss": k}
    return obs_loss + reward_loss + model.kl_scale * kl_loss, meta


def update(model, batch, optimizer, *, eps=None) -> Tuple[float, Dict]:
    """``PlaNetModel.update(batch, optimizer)`` (planet.py:484-519): returns ``(loss, meta)`` with ``grad_norm``, the
    sum of the parameters' gradient 2-norms after clipping.  The meta scalars, the loss and ``grad_norm`` come to the
    host in one device-to-host copy."""
    model.train()
    optimizer.zero_grad()
    obs_loss, reward_loss, kl_loss, recon = _loss_terms(model, batch, eps)
    obs_loss, reward_loss, kl_loss = obs_loss.mean(), reward_loss.mean(), kl_loss.mean()
    total = obs_loss + reward_loss + model.kl_scale * kl_loss
    total.backward()
    torch.nn.utils.clip_grad_norm_(model.parameters(), model.grad_clip_norm, norm_type=2)
    with torch.no_grad():
        grads = [p.grad for p in model.parameters() if p.grad is not None]
        grad_norm = torch.stack(torch._foreach_norm(grads, 2)).sum()
        stats = torch.stack([total.detach(), obs_loss.detach(), reward_loss.detach(), kl_loss.detach(), grad_norm])
    optimizer.step()
    lv, o, r, k, gn = stats.tolist()
    return lv, {"reconstruction": recon.detach(), "observations_loss": o, "reward_loss": r, "kl_loss": k,
                "grad_norm": gn}


def eval_score(model, batch) -> Tuple[torch.Tensor, Dict]:
    """``PlaNetModel.eval_score(batch)``: ``loss(batch, reduce=False)`` under ``no_grad`` (the forward kernel keeps no
    tape)."""
    with torch.no_grad():
        return loss(model, batch, reduce=False)
