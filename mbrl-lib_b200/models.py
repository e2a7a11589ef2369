"""Parameter containers with the attribute layout the staging code reads.

The drop-in use case hands *mbrl-lib's own* ``OneDTransitionRewardModel(GaussianMLP)`` objects to
:class:`mbrl_lib_b200.ModelEnv` (duck typed, SURVEY.md section 8b "Model (read-only by the fast path)").
These classes exist so that tests, ``bench.py`` and users without mbrl-lib installed can build the same
structure: ``.model.hidden_layers[i][0].{weight[E,K,N], bias[E,1,N]}``, ``.model.mean_and_logvar``,
``.model.{min,max}_logvar``, ``.model.elite_models``, ``.input_normalizer.{mean,std}`` ...
(mbrl/models/gaussian_mlp.py:86-127, mbrl/models/one_dim_tr_model.py:84-101).  They also carry the reference's
PyTorch training interface (``loss`` / ``update`` / ``eval_score`` without propagation, ``_process_batch``): the loop
:class:`mbrl_lib_b200.ModelTrainer` falls back to, and the yardstick its device path is tested against.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

_ACT = {"relu": nn.ReLU, "silu": nn.SiLU, "leaky_relu": lambda: nn.LeakyReLU(0.01)}


class EnsembleLinearLayer(nn.Module):
    """weight [E, in, out], bias [E, 1, out]   (layout of mbrl/models/util.py:41-45)."""

    def __init__(self, num_members: int, in_size: int, out_size: int):
        super().__init__()
        self.num_members, self.in_size, self.out_size = num_members, in_size, out_size
        self.weight = nn.Parameter(torch.zeros(num_members, in_size, out_size))
        self.bias = nn.Parameter(torch.zeros(num_members, 1, out_size))

    def forward(self, x):  # every member (no elite selection): [E or 1, B, in] -> [E, B, out]
        return x.matmul(self.weight) + self.bias


class GaussianMLP(nn.Module):
    def __init__(self, in_size: int, out_size: int, device, num_layers: int = 4, ensemble_size: int = 1,
                 hid_size: int = 200, deterministic: bool = False, propagation_method: Optional[str] = None,
                 activation: str = "relu"):
        super().__init__()
        self.in_size, self.out_size, self.num_members = in_size, out_size, ensemble_size
        self.deterministic = deterministic
        self.propagation_method = propagation_method
        self.device = torch.device(device)
        layers = [nn.Sequential(EnsembleLinearLayer(ensemble_size, in_size, hid_size), _ACT[activation]())]
        for _ in range(num_layers - 1):
            layers.append(nn.Sequential(EnsembleLinearLayer(ensemble_size, hid_size, hid_size), _ACT[activation]()))
        self.hidden_layers = nn.Sequential(*layers)
        self.mean_and_logvar = EnsembleLinearLayer(ensemble_size, hid_size, out_size * (1 if deterministic else 2))
        if not deterministic:
            self.min_logvar = nn.Parameter(-10 * torch.ones(1, out_size), requires_grad=False)
            self.max_logvar = nn.Parameter(0.5 * torch.ones(1, out_size), requires_grad=False)
        self.elite_models: Optional[List[int]] = None
        self.to(self.device)

    def __len__(self):
        return self.num_members

    def set_elite(self, elite_indices: Sequence[int]):  # gaussian_mlp.py:377-379
        if len(elite_indices) != self.num_members:
            self.elite_models = list(elite_indices)

    def set_propagation_method(self, propagation_method: Optional[str] = None):
        self.propagation_method = propagation_method

    # ---- PyTorch training interface (gaussian_mlp.py:140-154, 283-361; model.py:129-167) --------------------------
    def forward(self, x, use_propagation: bool = False):
        """Every member's mean and (soft-bounded) logvar: [E, B, in] or [B, in] -> [E, B, out] each.  Only the
        ``use_propagation=False`` form of the reference, the one training and evaluation use."""
        ml = self.mean_and_logvar(self.hidden_layers(x))
        if self.deterministic:
            return ml, None
        mean, logvar = ml[..., :self.out_size], ml[..., self.out_size:]
        logvar = self.max_logvar - F.softplus(self.max_logvar - logvar)
        logvar = self.min_logvar + F.softplus(logvar - self.min_logvar)
        return mean, logvar

    def loss(self, model_in, target):
        if model_in.ndim == 2:
            model_in, target = model_in.unsqueeze(0), target.unsqueeze(0)
        mean, logvar = self.forward(model_in)
        if self.deterministic:  # _mse_loss: summed squared error
            return F.mse_loss(mean, target, reduction="none").sum((1, 2)).sum(), {}
        if target.shape[0] != self.num_members:
            target = target.repeat(self.num_members, 1, 1)
        # gaussian_nll(reduce=False) averaged per member, summed over members, plus the bound penalty (_nll_loss)
        nll = F.mse_loss(mean, target, reduction="none") * (-logvar).exp() + logvar
        loss = nll.mean((1, 2)).sum()
        return loss + 0.01 * (self.max_logvar.sum() - self.min_logvar.sum()), {}

    def update(self, model_in, optimizer, target=None):
        self.train()
        optimizer.zero_grad()
        loss, meta = self.loss(model_in, target)
        loss.backward()
        with torch.no_grad():  # the reference logs the gradient norm of every update
            meta["grad_norm"] = sum(p.grad.norm(2).item() ** 2 for p in self.parameters() if p.grad is not None)
        optimizer.step()
        return loss.item(), meta

    def eval_score(self, model_in, target):
        """Squared error per member, row and output column: [E, B, out]."""
        with torch.no_grad():
            mean, _ = self.forward(model_in)
            return F.mse_loss(mean, target.repeat((self.num_members, 1, 1)), reduction="none"), {}


class Normalizer:
    """mean / std of the model input, [1, in]   (mbrl/util/math.py:95-143)."""

    def __init__(self, in_size: int, device, dtype=torch.float32):
        self.mean = torch.zeros((1, in_size), device=device, dtype=dtype)
        self.std = torch.ones((1, in_size), device=device, dtype=dtype)
        self.eps = 1e-12 if dtype == torch.double else 1e-5
        self.device = device

    def update_stats(self, data):
        if isinstance(data, np.ndarray):
            data = torch.from_numpy(data).to(self.device)
        self.mean = data.mean(0, keepdim=True)
        self.std = data.std(0, keepdim=True)
        self.std[self.std < self.eps] = 1.0

    def normalize(self, val):
        if isinstance(val, np.ndarray):
            val = torch.from_numpy(val).to(self.device)
        return (val - self.mean) / self.std


class BasicEnsemble(nn.Module):
    """mbrl-lib's ``BasicEnsemble`` (mbrl/models/basic_ensemble.py) as the kernels read it: ``members``, E one-member
    GaussianMLPs of one shape, all of them used (``set_elite`` changes nothing, basic_ensemble.py:262-266).  Under
    ``random_model`` every forward draws each row's member with ``torch.randint(E, (B,))``; under ``fixed_model`` the
    rows keep the members of :meth:`sample_propagation_indices` for a whole rollout."""

    def __init__(self, members: Sequence[GaussianMLP], propagation_method: Optional[str] = None):
        super().__init__()
        self.members = nn.ModuleList(members)
        m0 = self.members[0]
        self.in_size, self.out_size = m0.in_size, m0.out_size
        self.num_members = len(self.members)
        self.deterministic = m0.deterministic
        self.propagation_method = propagation_method
        self.device = m0.device

    def __len__(self):
        return len(self.members)

    def set_elite(self, elite_indices: Sequence[int]):
        pass  # every member is used (basic_ensemble.py:262-266)

    def set_propagation_method(self, propagation_method: Optional[str] = None):
        self.propagation_method = propagation_method

    def sample_propagation_indices(self, batch_size: int, rng: torch.Generator) -> torch.Tensor:
        return torch.randint(len(self), (batch_size,), generator=rng, device=self.device)  # basic_ensemble.py:255-260


class OneDTransitionRewardModel:
    def __init__(self, model: GaussianMLP, target_is_delta: bool = True, normalize: bool = False,
                 normalize_double_precision: bool = False, learned_rewards: bool = True,
                 obs_process_fn: Optional[Callable] = None, no_delta_list: Optional[List[int]] = None,
                 num_elites: Optional[int] = None):
        self.model = model
        self.device = model.device
        self.input_normalizer: Optional[Normalizer] = None
        if normalize:
            self.input_normalizer = Normalizer(model.in_size, self.device,
                                               dtype=torch.double if normalize_double_precision else torch.float)
        self.learned_rewards = learned_rewards
        self.target_is_delta = target_is_delta
        self.no_delta_list = no_delta_list if no_delta_list else []
        self.obs_process_fn = obs_process_fn
        self.num_elites = num_elites or model.num_members

    def set_elite(self, elite_indices: Sequence[int]):
        self.model.set_elite(elite_indices)

    def set_propagation_method(self, propagation_method: Optional[str] = None):
        self.model.set_propagation_method(propagation_method)

    def __len__(self):
        return len(self.model)

    # ---- PyTorch training interface (one_dim_tr_model.py:103-223) -------------------------------------------------
    def parameters(self):
        return self.model.parameters()

    def state_dict(self):
        return {f"model.{k}": v for k, v in self.model.state_dict().items()}

    def load_state_dict(self, state_dict):
        return self.model.load_state_dict({k[len("model."):]: v for k, v in state_dict.items()})

    def update_normalizer(self, batch):
        if self.input_normalizer is None:
            return
        obs, act = torch.as_tensor(batch.obs), torch.as_tensor(batch.act)
        if obs.ndim == 1:
            obs, act = obs[None], act[None]
        if self.obs_process_fn:
            obs = self.obs_process_fn(obs)
        self.input_normalizer.update_stats(torch.cat([obs, act], dim=obs.ndim - 1).numpy())

    def _process_batch(self, batch):
        """Model input and target of a transition batch ([B, ...] or [E, B, ...] numpy arrays)."""
        obs, act, next_obs, reward = (torch.as_tensor(x).to(self.device) for x in
                                      (batch.obs, batch.act, batch.next_obs, batch.rewards))
        target = next_obs
        if self.target_is_delta:
            target = next_obs - obs
            for dim in self.no_delta_list:
                target[..., dim] = next_obs[..., dim]
        proc = self.obs_process_fn(obs) if self.obs_process_fn else obs
        model_in = torch.cat([proc, act], dim=obs.ndim - 1)
        if self.input_normalizer:
            model_in = self.input_normalizer.normalize(model_in).float()
        if self.learned_rewards:
            target = torch.cat([target, reward.unsqueeze(reward.ndim)], dim=obs.ndim - 1)
        return model_in.float(), target.float()

    def update(self, batch, optimizer, target=None):
        model_in, target = self._process_batch(batch)
        return self.model.update(model_in, optimizer, target=target)

    def eval_score(self, batch, target=None):
        with torch.no_grad():
            model_in, target = self._process_batch(batch)
            return self.model.eval_score(model_in, target=target)


def basic_ensemble_from_arrays(spec, arrays, device) -> OneDTransitionRewardModel:
    """The model of :func:`model_from_arrays` with its stacked ensemble split into a :class:`BasicEnsemble` of
    ``spec.ensemble_size`` one-member GaussianMLPs: member e holds slice e of every layer and the shared logvar bounds."""
    from . import functions

    members = []
    for e in range(spec.ensemble_size):
        mlp = GaussianMLP(spec.in_size, spec.out_size, device, num_layers=spec.num_layers, ensemble_size=1,
                          hid_size=spec.hid_size, deterministic=spec.deterministic, activation=spec.activation)
        with torch.no_grad():
            for li, layer in enumerate(list(mlp.hidden_layers) + [None]):
                lin = layer[0] if layer is not None else mlp.mean_and_logvar
                lin.weight.copy_(torch.from_numpy(arrays["weights"][li][e:e + 1]))
                lin.bias.copy_(torch.from_numpy(arrays["biases"][li][e:e + 1]))
            if not spec.deterministic:
                mlp.min_logvar.copy_(torch.from_numpy(arrays["min_logvar"]))
                mlp.max_logvar.copy_(torch.from_numpy(arrays["max_logvar"]))
        members.append(mlp)
    wrapper = OneDTransitionRewardModel(
        BasicEnsemble(members, spec.propagation), target_is_delta=spec.target_is_delta, normalize=spec.normalize is not None,
        normalize_double_precision=spec.normalize == "float64", learned_rewards=spec.learned_rewards,
        obs_process_fn=functions.OBS_PROCESS_FNS.get(spec.obs_process), no_delta_list=list(spec.no_delta_list))
    if spec.normalize is not None:
        wrapper.input_normalizer.mean = torch.from_numpy(arrays["norm_mean"]).to(device)
        wrapper.input_normalizer.std = torch.from_numpy(arrays["norm_std"]).to(device)
    return wrapper


def model_from_arrays(spec, arrays, device) -> OneDTransitionRewardModel:
    """Build the container for a ``synthetic.CaseSpec`` and its seeded arrays on ``device``."""
    from . import functions

    mlp = GaussianMLP(spec.in_size, spec.out_size, device, num_layers=spec.num_layers, ensemble_size=spec.ensemble_size,
                      hid_size=spec.hid_size, deterministic=spec.deterministic, propagation_method=spec.propagation,
                      activation=spec.activation)
    with torch.no_grad():
        for li, layer in enumerate(mlp.hidden_layers):
            layer[0].weight.copy_(torch.from_numpy(arrays["weights"][li]))
            layer[0].bias.copy_(torch.from_numpy(arrays["biases"][li]))
        mlp.mean_and_logvar.weight.copy_(torch.from_numpy(arrays["weights"][-1]))
        mlp.mean_and_logvar.bias.copy_(torch.from_numpy(arrays["biases"][-1]))
        if not spec.deterministic:
            mlp.min_logvar.copy_(torch.from_numpy(arrays["min_logvar"]))
            mlp.max_logvar.copy_(torch.from_numpy(arrays["max_logvar"]))
    wrapper = OneDTransitionRewardModel(
        mlp, target_is_delta=spec.target_is_delta, normalize=spec.normalize is not None,
        normalize_double_precision=spec.normalize == "float64", learned_rewards=spec.learned_rewards,
        obs_process_fn=functions.OBS_PROCESS_FNS.get(spec.obs_process), no_delta_list=list(spec.no_delta_list),
        num_elites=spec.num_models)
    if spec.normalize is not None:
        wrapper.input_normalizer.mean = torch.from_numpy(arrays["norm_mean"]).to(device)
        wrapper.input_normalizer.std = torch.from_numpy(arrays["norm_std"]).to(device)
    if spec.elites is not None:
        wrapper.set_elite(list(spec.elites))
    return wrapper


class _BeliefModel(nn.Module):  # mbrl/models/planet.py:82-101
    def __init__(self, latent_state_size: int, action_size: int, belief_size: int):
        super().__init__()
        self.embedding_layer = nn.Sequential(nn.Linear(latent_state_size + action_size, belief_size), nn.ReLU())
        self.rnn = nn.GRUCell(belief_size, belief_size)


class _Conv2dEncoder(nn.Module):  # mbrl/models/util.py:101-157
    def __init__(self, layers_config, image_shape, encoding_size: int):
        super().__init__()
        self.convs = nn.ModuleList([nn.Sequential(nn.Conv2d(c[0], c[1], c[2], stride=c[3]), nn.ReLU())
                                    for c in layers_config])
        with torch.no_grad():
            out = self.convs_forward(torch.zeros(1, layers_config[0][0], *image_shape))
        cnn_out_size = int(np.prod(out.shape[1:]))
        self.fc = nn.Identity() if cnn_out_size == encoding_size else nn.Linear(cnn_out_size, encoding_size)

    def convs_forward(self, obs):
        for conv in self.convs:
            obs = conv(obs)
        return obs

    def forward(self, obs):
        conv = self.convs_forward(obs)
        return self.fc(conv.view(conv.size(0), -1))


class _Conv2dDecoder(nn.Module):  # mbrl/models/util.py:162-212
    def __init__(self, encoding_size: int, deconv_input_shape, layers_config):
        super().__init__()
        self.encoding_size = encoding_size
        self.deconv_input_shape = tuple(deconv_input_shape)
        self.fc = nn.Linear(encoding_size, int(np.prod(self.deconv_input_shape)))
        mods = []
        for i, c in enumerate(layers_config):
            layer = nn.ConvTranspose2d(c[0], c[1], c[2], stride=c[3])
            mods.append(layer if i == len(layers_config) - 1 else nn.Sequential(layer, nn.ReLU()))
        self.deconvs = nn.ModuleList(mods)

    def forward(self, x):
        deconv = self.fc(x).view(-1, *self.deconv_input_shape)
        for layer in self.deconvs:
            deconv = layer(deconv)
        return deconv


class _MeanStdCat(nn.Module):  # mbrl/models/planet.py:103-114
    def __init__(self, latent_state_size: int, min_std: float):
        super().__init__()
        self.min_std = min_std
        self.latent_state_size = latent_state_size

    def forward(self, params):
        mean = params[:, : self.latent_state_size]
        std = F.softplus(params[:, self.latent_state_size:]) + self.min_std
        return torch.cat([mean, std], dim=1)


class PlaNetModel(nn.Module):
    """mbrl-lib's ``PlaNetModel`` (planet.py:121-306) with its attribute layout: ``belief_model.{embedding_layer, rnn}``,
    ``prior_transition_model[0, 2]``, ``reward_model[0, 2, 4]``, ``min_std`` and the posterior
    ``_current_posterior_sample [1, L]`` / ``_current_belief [1, Hb]`` that planning starts from.

    Without ``obs_shape`` it is the planning half only: no encoder, decoder or posterior model, and :meth:`set_posterior`
    stands in for ``update_posterior``.  With ``obs_shape``, ``obs_encoding_size``, ``encoder_config`` and
    ``decoder_config`` it also has ``encoder``, ``posterior_transition_model`` and ``decoder`` with the reference's
    layout and ``state_dict`` keys, and ``free_nats``, ``kl_scale``, ``grad_clip_norm`` and ``rng``: what
    :mod:`mbrl_lib_b200.latent_train` trains.  Weights start as torch's default initialisation unless ``seed`` is
    given, in which case every parameter is drawn from N(0, scale^2) with that numpy seed, in the order of
    ``latent.latent_params`` and then of the encoder, the posterior and the decoder."""

    def __init__(self, action_size: int, latent_state_size: int = 30, belief_size: int = 200, hidden_size_fcs: int = 200,
                 device="cpu", min_std: float = 0.1, seed: Optional[int] = None, scale: float = 0.1, *,
                 obs_shape=None, obs_encoding_size: Optional[int] = None, encoder_config=None, decoder_config=None,
                 free_nats: float = 3, kl_scale: float = 1.0, grad_clip_norm: float = 1000.0,
                 rng: Optional[torch.Generator] = None):
        super().__init__()
        self.action_size, self.latent_state_size, self.belief_size = action_size, latent_state_size, belief_size
        self.min_std = min_std
        self.device = torch.device(device)
        self.belief_model = _BeliefModel(latent_state_size, action_size, belief_size)
        self.prior_transition_model = nn.Sequential(nn.Linear(belief_size, hidden_size_fcs), nn.ReLU(),
                                                    nn.Linear(hidden_size_fcs, 2 * latent_state_size))
        if obs_shape is not None:  # the reference's module order (planet.py:227-265)
            self.obs_shape = tuple(obs_shape)
            self.free_nats = free_nats * torch.ones(1).to(device)
            self.kl_scale = kl_scale
            self.grad_clip_norm = grad_clip_norm
            self.rng = torch.Generator(device=self.device) if rng is None else rng
            self.encoder = _Conv2dEncoder(encoder_config, self.obs_shape[1:], obs_encoding_size)
            self.posterior_transition_model = nn.Sequential(
                nn.Linear(obs_encoding_size + belief_size, hidden_size_fcs), nn.ReLU(),
                nn.Linear(hidden_size_fcs, 2 * latent_state_size), _MeanStdCat(latent_state_size, min_std))
            self.decoder = _Conv2dDecoder(latent_state_size + belief_size, decoder_config[0], decoder_config[1])
        self.reward_model = nn.Sequential(nn.Linear(belief_size + latent_state_size, hidden_size_fcs), nn.ReLU(),
                                          nn.Linear(hidden_size_fcs, hidden_size_fcs), nn.ReLU(),
                                          nn.Linear(hidden_size_fcs, 1))
        if seed is not None:
            from .latent import latent_params

            rng_np = np.random.default_rng(seed)
            first = latent_params(self)
            rest = [] if obs_shape is None else \
                [p for mod in (self.encoder, self.posterior_transition_model, self.decoder) for p in mod.parameters()]
            with torch.no_grad():
                for p in first + rest:
                    p.copy_(torch.from_numpy(rng_np.normal(0.0, scale, tuple(p.shape)).astype(np.float32)))
        self._current_posterior_sample: Optional[torch.Tensor] = None
        self._current_belief: Optional[torch.Tensor] = None
        self.to(self.device)

    def set_posterior(self, latent, belief):
        """Set the state planning starts from: ``latent [L]`` / ``belief [Hb]`` (or ``[1, .]``)."""
        self._current_posterior_sample = torch.as_tensor(latent, dtype=torch.float32).reshape(1, -1).to(self.device)
        self._current_belief = torch.as_tensor(belief, dtype=torch.float32).reshape(1, -1).to(self.device)

    def reset_posterior(self):
        self._current_posterior_sample = None
        self._current_belief = None

    def reset(self, obs, rng=None):  # planet.py:662-677
        return {"latent": self._current_posterior_sample.repeat(obs.shape[0], 1),
                "belief": self._current_belief.repeat(obs.shape[0], 1)}
