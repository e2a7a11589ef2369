"""``ModelTrainer`` with the reference's interface (mbrl/models/model_trainer.py:31-296) that trains a
``OneDTransitionRewardModel(GaussianMLP)`` on the device.

Per ``train()`` call the dataset goes to the device once and one kernel turns it into model inputs and targets (the
normaliser is fixed during ``train()``).  Per epoch the iterator's own minibatch order is read from the iterator (so the
minibatches are the ones the reference would draw, its random generator advanced the same way), uploaded as one index
array, and one launch runs every Adam step of the epoch; evaluation is one launch over the whole evaluation set.  The
host synchronises once per epoch, to read the losses and scores the early-stopping rule needs.

``self.optimizer`` is a real ``torch.optim.Adam`` over the model's parameters: the kernels update its ``exp_avg`` /
``exp_avg_sq`` tensors and its ``step`` counts in place, so ``optimizer.state_dict()`` and checkpoints keep working, and a
later reference-style ``model.update(batch, trainer.optimizer)`` continues from the same state.

What runs where:
  * the device path: the model is a ``OneDTransitionRewardModel(GaussianMLP)`` (mbrl-lib's or :mod:`models`') with fp32
    CUDA parameters, a known ``obs_process_fn`` and no ``batch_callback``; datasets that are a ``TransitionIterator`` /
    ``BootstrapIterator`` (mbrl-lib's or :mod:`replay`'s, recognised by their attributes) train an epoch per launch, any
    other iterable of transition batches takes one fused Adam step per yielded batch.  Transitions may be float32 or
    float64 (mbrl-lib's PETS / MBPO replay buffers are float64 with ``normalize_double_precision``); float64 ones are
    processed in double, as the reference's numpy / torch code processes them, and rounded to float32 at the end;
  * the latent path: a ``PlaNetModel`` (mbrl-lib's or :mod:`models`' with the encoder and decoder) whose recurrence
    ``b200pets_latent_train_supported`` accepts, with fp32 CUDA parameters and one Adam param group over
    ``model.parameters()``: the reference's loop below, with each batch through :func:`latent_train.update` and each
    evaluation batch through :func:`latent_train.eval_score` in place of the model's own methods.  ``batch_callback`` is
    called per batch with the reference's arguments, as ``mbrl/algorithms/planet.py`` needs;
  * otherwise (a ``batch_callback`` on a GaussianMLP, which needs every batch's loss as it happens, another model, a
    model the kernels refuse -- more than 7 hidden layers, or layers too wide for the evaluation kernel's shared memory
    -- or transitions of another element type) the reference's PyTorch loop runs unchanged: ``model.update(batch,
    optimizer)`` / ``model.eval_score(batch)``.  A refused model runs the whole ``train()`` / ``evaluate()`` call that way.
"""
from __future__ import annotations

import copy
import ctypes as C
import functools
import itertools
from typing import Callable, Dict, List, Optional, Tuple

import numpy as np
import torch

from . import _lib, functions, latent_train, staging

MODEL_LOG_FORMAT = [
    ("train_iteration", "I", "int"),
    ("epoch", "E", "int"),
    ("train_dataset_size", "TD", "int"),
    ("val_dataset_size", "VD", "int"),
    ("model_loss", "MLOSS", "float"),
    ("model_val_score", "MVSCORE", "float"),
    ("model_best_val_score", "MBVSCORE", "float"),
]

_ITER_METHODS = ("__iter__", "__next__", "__getitem__", "_get_indices_next_batch")


def _iterator_kind(ds) -> Optional[str]:
    """"plain" / "bootstrap" for a TransitionIterator / BootstrapIterator whose iteration methods are the base classes'
    (a subclass that overrides how batches are formed, e.g. SequenceTransitionIterator, is not one), else None."""
    cls = type(ds)
    if not all(hasattr(ds, a) for a in ("transitions", "_order", "batch_size", "num_stored", "_current_batch")):
        return None
    owners = {getattr(getattr(cls, m, None), "__qualname__", "").split(".")[0] for m in _ITER_METHODS}
    if not owners <= {"TransitionIterator", "BootstrapIterator"}:
        return None
    if cls.__name__ == "BootstrapIterator" and hasattr(ds, "member_indices") and hasattr(ds, "_bootstrap_iter"):
        return "bootstrap"
    if cls.__name__ == "TransitionIterator":
        return "plain"
    return None


class _DeviceModel:
    """The C trainer handle over the model's live parameters and the optimizer's state, for one ``train()`` call."""

    def __init__(self, model, optimizer):
        self.lib = _lib.load()
        self.model, self.optimizer = model, optimizer
        self.mlp = mlp = model.model
        self.layers = [seq[0] for seq in mlp.hidden_layers] + [mlp.mean_and_logvar]
        self.device = mlp.mean_and_logvar.weight.device
        params = [p for layer in self.layers for p in (layer.weight, layer.bias)]
        self.bounds = [] if mlp.deterministic else [mlp.min_logvar, mlp.max_logvar]
        self.learn_bounds = bool(self.bounds) and all(p.requires_grad for p in self.bounds)
        self.trained = params + (self.bounds if self.learn_bounds else [])
        group = optimizer.param_groups[0]
        for p in self.trained:
            st = optimizer.state[p]
            if len(st) == 0:  # the state torch.optim.Adam creates at a parameter's first step
                scalar = torch.float64 if torch.get_default_dtype() == torch.float64 else torch.float32
                st["step"] = torch.tensor(0.0, dtype=scalar)
                st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        steps = {float(optimizer.state[p]["step"]) for p in self.trained}
        if len(steps) != 1:
            raise RuntimeError(f"the parameters' Adam step counts differ ({sorted(steps)}); one fused step updates all")
        allp = params + self.bounds
        n = len(allp)
        P = (C.c_void_p * n)(*[p.data_ptr() for p in allp])
        M = (C.c_void_p * n)(*[optimizer.state[p]["exp_avg"].data_ptr() if p in optimizer.state else None for p in allp])
        V = (C.c_void_p * n)(*[optimizer.state[p]["exp_avg_sq"].data_ptr() if p in optimizer.state else None for p in allp])
        d = train_desc(mlp, group)
        self.E = d.ensemble_size
        h = C.c_void_p()
        _lib.check(self.lib.b200pets_trainer_create(C.byref(d), P, M, V, C.byref(h)), "trainer_create")
        self.handle = h
        self._data: Dict[int, tuple] = {}

    @property
    def adam_step(self) -> int:
        return int(float(self.optimizer.state[self.trained[0]]["step"]))

    def advance(self, steps: int):
        for p in self.trained:
            self.optimizer.state[p]["step"] += steps

    def stream(self):
        with torch.cuda.device(self.device):
            return _lib.stream_ptr()

    # ---- data ----------------------------------------------------------------------------------------------------
    def stage(self, batch):
        """Model inputs [n, in] and targets [n, out] of a TransitionBatch of n rows (b200pets_train_preprocess)."""
        w = self.model
        dev = self.device
        dtype = transition_dtype(batch)
        if dtype is None:
            raise TypeError("the training kernels read float32 or float64 transitions; got "
                            f"{[str(getattr(x, 'dtype', type(x))) for x in (batch.obs, batch.act, batch.next_obs, batch.rewards)]}")
        check_model_sizes(w, int(np.shape(batch.obs)[-1]), int(np.shape(batch.act)[-1]))
        obs, act, next_obs, reward = (torch.as_tensor(x).to(dev, dtype).contiguous()
                                      for x in (batch.obs, batch.act, batch.next_obs, batch.rewards))
        rows = int(obs.shape[0])
        d = _lib.PrepDesc()
        d.dtype = _lib.DTYPE["float64" if dtype == torch.float64 else "float32"]
        d.obs_dim, d.act_dim = int(obs.shape[-1]), int(act.shape[-1])
        d.obs_process = functions.resolve_obs_process(getattr(w, "obs_process_fn", None))
        norm = getattr(w, "input_normalizer", None)
        nm = ns = None
        if norm is not None:
            dt = torch.float64 if norm.mean.dtype == torch.float64 else torch.float32
            nm = norm.mean.to(dev, dt).contiguous()
            ns = norm.std.to(dev, dt).contiguous()
            d.norm_mode = 2 if dt == torch.float64 else 1
        d.target_is_delta, d.learned_rewards = int(bool(w.target_is_delta)), int(bool(w.learned_rewards))
        nd = [int(i) % d.obs_dim for i in (getattr(w, "no_delta_list", None) or [])]
        nd_arr = (C.c_int32 * max(len(nd), 1))(*nd)
        X = torch.empty(rows, int(self.mlp.in_size), device=dev)
        Y = torch.empty(rows, int(self.mlp.out_size), device=dev)
        _lib.check(self.lib.b200pets_train_preprocess(C.byref(d), rows, _lib.ptr(obs), _lib.ptr(act), _lib.ptr(next_obs),
                                                      _lib.ptr(reward), _lib.ptr(nm), _lib.ptr(ns), nd_arr, len(nd),
                                                      _lib.ptr(X), _lib.ptr(Y), self.stream()), "train_preprocess")
        return X, Y, (obs, act, next_obs, reward, nm, ns)

    def dataset(self, ds):
        """Staged inputs / targets of an iterator's whole store, once per train() call."""
        key = id(ds)
        got = self._data.get(key)
        if got is None or got[0] is not ds.transitions or got[1] != ds.num_stored:
            X, Y, _ = self.stage(ds.transitions)
            got = (ds.transitions, ds.num_stored, X, Y)
            self._data[key] = got
        return got[2], got[3]

    # ---- kernels -------------------------------------------------------------------------------------------------
    def run_steps(self, X, Y, idx: np.ndarray, last_batch: int) -> np.ndarray:
        """idx int32 [E, steps, batch]: Adam steps over rows of (X, Y); returns the per-step losses."""
        E, steps, batch = idx.shape
        idx_dev = torch.from_numpy(np.ascontiguousarray(idx, dtype=np.int32)).to(self.device)
        losses = torch.empty(steps, device=self.device)
        nbytes = self.lib.b200pets_train_workspace_bytes(self.handle, batch)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        _lib.check(self.lib.b200pets_train_epoch(self.handle, int(X.shape[0]), _lib.ptr(X), _lib.ptr(Y), _lib.ptr(idx_dev), steps,
                                                 batch, last_batch, self.adam_step, _lib.ptr(losses), _lib.ptr(ws), nbytes,
                                                 self.stream()), "train_epoch")
        self.advance(steps)
        staging.mark_trained(self.mlp)
        return losses.cpu().numpy()

    def eval_score(self, X, Y) -> torch.Tensor:
        rows = int(X.shape[0])
        scores = torch.empty(self.E, device=self.device)
        nbytes = self.lib.b200pets_eval_score_workspace_bytes(self.handle, rows)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        _lib.check(self.lib.b200pets_eval_score(self.handle, rows, _lib.ptr(X), _lib.ptr(Y), _lib.ptr(scores), _lib.ptr(ws),
                                                nbytes, self.stream()), "eval_score")
        return scores

    def close(self):
        if self.handle is not None:
            self.lib.b200pets_trainer_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def train_desc(mlp, group) -> _lib.TrainDesc:
    """The C descriptor of a GaussianMLP trained with the Adam hyper-parameters of ``group``."""
    layers = [seq[0] for seq in mlp.hidden_layers] + [mlp.mean_and_logvar]
    act, slope = staging._activation_of(mlp.hidden_layers[0][1])
    learn_bounds = not mlp.deterministic and mlp.min_logvar.requires_grad and mlp.max_logvar.requires_grad
    d = _lib.TrainDesc()
    d.ensemble_size = int(layers[0].weight.shape[0])
    d.in_size, d.out_size = int(mlp.in_size), int(mlp.out_size)
    d.hid_size, d.num_hidden = int(layers[0].weight.shape[2]), len(layers) - 1
    d.activation, d.leaky_slope = act, slope
    d.deterministic, d.learn_logvar_bounds = int(bool(mlp.deterministic)), int(learn_bounds)
    d.lr, (d.beta1, d.beta2), d.eps, d.weight_decay = group["lr"], group["betas"], group["eps"], group["weight_decay"]
    return d


def check_model_sizes(model, obs_dim: int, act_dim: int):
    """Raise ValueError unless the model's ``in_size`` / ``out_size`` are the widths ``_process_batch`` makes of
    transitions with ``obs_dim`` / ``act_dim`` columns: ``obs_process_fn``'s output plus the action, and the observation
    plus the reward when it is learned.  The preprocessing kernel writes those widths whatever the model says, so a model
    built for other data (the cartpole ``obs_process_fn`` adds a column) would have it write past the staged arrays; the
    reference raises a shape error there too."""
    proc = functions.resolve_obs_process(getattr(model, "obs_process_fn", None))
    want_in = obs_dim + (1 if proc == _lib.PROC["cartpole"] else 0) + act_dim
    want_out = obs_dim + int(bool(model.learned_rewards))
    mlp = model.model
    if (int(mlp.in_size), int(mlp.out_size)) != (want_in, want_out):
        raise ValueError(f"transitions with {obs_dim} observation and {act_dim} action columns make model inputs of "
                         f"{want_in} and targets of {want_out} columns; the model has in_size {mlp.in_size} and "
                         f"out_size {mlp.out_size}")


def transition_dtype(batch) -> Optional[torch.dtype]:
    """The precision the reference's ``_process_batch`` computes a batch in: float64 when obs, act or next_obs is float64
    (numpy / torch promote the others), float32 when all are float32 (the reward column is rounded to float32 either way:
    bootstrap batches store it as float32 and ``.float()`` ends the computation).  None for any other element type:
    the kernels do not read it."""
    dts = [torch.as_tensor(x[:0] if hasattr(x, "__getitem__") else x).dtype
           for x in (batch.obs, batch.act, batch.next_obs, batch.rewards)]
    if any(dt not in (torch.float32, torch.float64) for dt in dts):
        return None
    return torch.float64 if torch.float64 in dts[:3] else torch.float32


def epoch_indices(ds, kind: str, num_members: int) -> Tuple[np.ndarray, int]:
    """Start one pass over a TransitionIterator / BootstrapIterator exactly as ``for batch in ds`` does and return its
    minibatches as rows ``[E, steps, batch_size]`` (the last step's first ``last_batch`` entries are used) without forming
    them; the iterator is left exhausted, as after the loop."""
    iter(ds)
    n, bs = int(ds.num_stored), int(ds.batch_size)
    steps = (n - 1) // bs + 1
    order = np.asarray(ds._order)
    rows = np.asarray(ds.member_indices)[:, order] if kind == "bootstrap" and ds._bootstrap_iter \
        else np.broadcast_to(order, (num_members, n))
    idx = np.zeros((num_members, steps * bs), dtype=np.int32)
    idx[:, :n] = rows
    ds._current_batch = steps
    return idx.reshape(num_members, steps, bs), n - (steps - 1) * bs


class ModelTrainer:
    """Drop-in for ``mbrl.models.ModelTrainer`` (same constructor, ``train`` / ``evaluate`` / ``maybe_get_best_weights``)."""

    _LOG_GROUP_NAME = "model_train"

    def __init__(self, model, optim_lr: float = 1e-4, weight_decay: float = 1e-5, optim_eps: float = 1e-8, logger=None):
        self.model = model
        self._train_iteration = 0
        self.logger = logger
        if self.logger:
            self.logger.register_group(self._LOG_GROUP_NAME, MODEL_LOG_FORMAT, color="blue", dump_frequency=1)
        self.optimizer = torch.optim.Adam(self.model.parameters(), lr=optim_lr, weight_decay=weight_decay, eps=optim_eps)
        self._dev: Optional[_DeviceModel] = None
        self._latent = False

    # ---- which path ----------------------------------------------------------------------------------------------
    def _device_supported(self) -> bool:
        mlp = getattr(self.model, "model", None)
        if mlp is None or not hasattr(mlp, "hidden_layers") or not hasattr(mlp, "mean_and_logvar"):
            return False
        try:
            staging._activation_of(mlp.hidden_layers[0][1])
            functions.resolve_obs_process(getattr(self.model, "obs_process_fn", None))
        except NotImplementedError:
            return False
        layers = [seq[0] for seq in mlp.hidden_layers] + [mlp.mean_and_logvar]
        params = [p for layer in layers for p in (layer.weight, layer.bias)]
        if not mlp.deterministic:
            params += [mlp.min_logvar, mlp.max_logvar]
        dev = layers[0].weight.device
        if dev.type != "cuda" or any(p.dtype != torch.float32 or not p.is_contiguous() or p.device != dev for p in params):
            return False
        if len(self.optimizer.param_groups) != 1:
            return False
        g = self.optimizer.param_groups[0]
        if g.get("amsgrad") or g.get("maximize") or g.get("capturable") or g.get("differentiable") or g.get("fused") or \
                g.get("decoupled_weight_decay") or isinstance(g["lr"], torch.Tensor):
            return False
        if {id(p) for p in g["params"]} != {id(p) for p in params}:
            return False
        # the kernels' own limits (more than 7 hidden layers; layers too wide for the evaluation kernel's shared memory),
        # asked before anything is touched, so that the reference loop runs from the same state
        with torch.cuda.device(dev):
            return _lib.load().b200pets_trainer_supported(C.byref(train_desc(mlp, g))) == 0

    def _latent_supported(self) -> bool:
        """The latent path (see the module docstring), asked before anything is touched."""
        if not latent_train.is_trainable_latent_model(self.model) or len(self.optimizer.param_groups) != 1:
            return False
        if {id(p) for p in self.optimizer.param_groups[0]["params"]} != {id(p) for p in self.model.parameters()}:
            return False
        return latent_train.supported(self.model)

    def _model_update(self, batch):
        if self._latent:
            return latent_train.update(self.model, batch, self.optimizer)
        return self.model.update(batch, self.optimizer)

    def _model_eval_score(self, batch):
        if self._latent:
            return latent_train.eval_score(self.model, batch)
        return self.model.eval_score(batch)

    @staticmethod
    def _store_supported(ds) -> bool:
        return transition_dtype(ds.transitions) is not None

    def _device(self) -> _DeviceModel:
        if self._dev is None:
            self._dev = _DeviceModel(self.model, self.optimizer)
        return self._dev

    # ---- the reference's interface -------------------------------------------------------------------------------
    def train(self, dataset_train, dataset_val=None, num_epochs: Optional[int] = None, patience: Optional[int] = None,
              improvement_threshold: float = 0.01, callback: Optional[Callable] = None,
              batch_callback: Optional[Callable] = None, evaluate: bool = True, silent: bool = False
              ) -> Tuple[List[float], List[float]]:
        """Trains the model for some number of epochs (model_trainer.py:70-214): returns the per-epoch mean training
        losses and evaluation scores; keeps the weights of the best evaluation score (relative improvement of any member
        above ``improvement_threshold``), stops after ``patience`` epochs without one and sets the elite members."""
        self._latent = self._latent_supported()
        device = not self._latent and batch_callback is None and self._device_supported()
        self._dev = None
        try:
            return self._train(dataset_train, dataset_val, num_epochs, patience, improvement_threshold, callback,
                               batch_callback, evaluate, silent, device)
        finally:
            if self._dev is not None:
                self._dev.close()
                self._dev = None

    def _train(self, dataset_train, dataset_val, num_epochs, patience, improvement_threshold, callback, batch_callback,
               evaluate, silent, device):
        eval_dataset = dataset_train if dataset_val is None else dataset_val
        training_losses, val_scores = [], []
        best_weights: Optional[Dict] = None
        epoch_iter = range(num_epochs) if num_epochs else itertools.count()
        epochs_since_update = 0
        best_val_score = self._evaluate(eval_dataset, None, device) if evaluate else None
        for epoch in epoch_iter:
            batch_callback_epoch = functools.partial(batch_callback, epoch) if batch_callback else None
            if device:
                batch_losses = self._device_epoch(dataset_train)
            else:
                batch_losses = []
                for batch in dataset_train:
                    loss, meta = self._model_update(batch)
                    batch_losses.append(loss)
                    if batch_callback_epoch:
                        batch_callback_epoch(loss, meta, "train")
            total_avg_loss = np.mean(batch_losses).mean().item()
            training_losses.append(total_avg_loss)

            eval_score = None
            model_val_score = 0
            if evaluate:
                eval_score = self._evaluate(eval_dataset, batch_callback_epoch, device)
                val_scores.append(eval_score.mean().item())
                maybe_best_weights = self.maybe_get_best_weights(best_val_score, eval_score, improvement_threshold)
                if maybe_best_weights:
                    best_val_score = torch.minimum(best_val_score, eval_score)
                    best_weights = maybe_best_weights
                    epochs_since_update = 0
                else:
                    epochs_since_update += 1
                model_val_score = eval_score.mean()

            if self.logger and not silent:
                self.logger.log_data(self._LOG_GROUP_NAME, {
                    "iteration": self._train_iteration, "epoch": epoch, "train_dataset_size": dataset_train.num_stored,
                    "val_dataset_size": dataset_val.num_stored if dataset_val is not None else 0,
                    "model_loss": total_avg_loss, "model_val_score": model_val_score,
                    "model_best_val_score": best_val_score.mean() if best_val_score is not None else 0})
            if callback:
                callback(self.model, self._train_iteration, epoch, total_avg_loss, eval_score, best_val_score)
            if patience and epochs_since_update >= patience:
                break

        if evaluate:
            self._maybe_set_best_weights_and_elite(best_weights, best_val_score)
        if device:
            staging.mark_trained(self.model.model)
        self._train_iteration += 1
        return training_losses, val_scores

    def _device_epoch(self, ds) -> List[float]:
        dm = self._device()
        kind = _iterator_kind(ds)
        if kind is not None and self._store_supported(ds) and \
                (kind == "plain" or not ds._bootstrap_iter or ds.ensemble_size == dm.E):
            X, Y = dm.dataset(ds)
            idx, last = epoch_indices(ds, kind, dm.E)
            return [float(v) for v in dm.run_steps(X, Y, idx, last)]
        losses = []  # any other iterable: one fused step per yielded batch
        for batch in ds:
            if transition_dtype(batch) is None:  # not float32 / float64: the reference's update for this batch
                losses.append(self.model.update(batch, self.optimizer)[0])
                continue
            X, Y, _ = dm.stage(_flatten_members(batch))
            b = int(np.shape(batch.obs)[-2]) if np.ndim(batch.obs) == 3 else int(np.shape(batch.obs)[0])
            if np.ndim(batch.obs) == 3:
                if np.shape(batch.obs)[0] != dm.E:
                    raise ValueError(f"a batch of {np.shape(batch.obs)[0]} member slices for an ensemble of {dm.E}")
                idx = np.arange(dm.E * b, dtype=np.int32).reshape(dm.E, 1, b)
            else:
                idx = np.broadcast_to(np.arange(b, dtype=np.int32), (dm.E, 1, b))
            losses.append(float(dm.run_steps(X, Y, idx, b)[0]))
        return losses

    def _evaluate(self, dataset, batch_callback, device) -> torch.Tensor:
        if device and batch_callback is None:
            kind = _iterator_kind(dataset)
            if kind is not None and self._store_supported(dataset):
                dm = self._device()
                if kind == "bootstrap":
                    dataset.toggle_bootstrap()
                iter(dataset)  # the pass the reference makes (a shuffling iterator draws its permutation)
                dataset._current_batch = len(dataset)
                if kind == "bootstrap":
                    dataset.toggle_bootstrap()
                X, Y = dm.dataset(dataset)
                return dm.eval_score(X, Y)
        return self._evaluate_reference(dataset, batch_callback)

    def evaluate(self, dataset, batch_callback: Optional[Callable] = None) -> torch.Tensor:
        """Mean score of the model over the dataset, per ensemble member (model_trainer.py:216-262)."""
        if self._dev is None:
            self._latent = self._latent_supported()
        if batch_callback is None and self._dev is None and self._device_supported():
            try:
                return self._evaluate(dataset, None, True)
            finally:
                if self._dev is not None:
                    self._dev.close()
                    self._dev = None
        return self._evaluate(dataset, batch_callback, self._dev is not None)

    def _evaluate_reference(self, dataset, batch_callback=None) -> torch.Tensor:
        bootstrap = hasattr(dataset, "toggle_bootstrap")
        if bootstrap:
            dataset.toggle_bootstrap()
        batch_scores_list = []
        for batch in dataset:
            batch_score, meta = self._model_eval_score(batch)
            batch_scores_list.append(batch_score)
            if batch_callback:
                batch_callback(batch_score.mean(), meta, "eval")
        batch_scores = torch.cat(batch_scores_list, dim=batch_scores_list[0].ndim - 2)
        if bootstrap:
            dataset.toggle_bootstrap()
        mean_axis = 1 if batch_scores.ndim == 2 else (1, 2)
        return batch_scores.mean(dim=mean_axis)

    def maybe_get_best_weights(self, best_val_score: torch.Tensor, val_score: torch.Tensor,
                               threshold: float = 0.01) -> Optional[Dict]:
        improvement = (best_val_score - val_score) / torch.abs(best_val_score)
        improved = (improvement > threshold).any().item()
        return copy.deepcopy(self.model.state_dict()) if improved else None

    def _maybe_set_best_weights_and_elite(self, best_weights: Optional[Dict], best_val_score: torch.Tensor):
        if best_weights is not None:
            self.model.load_state_dict(best_weights)
        if len(best_val_score) > 1 and hasattr(self.model, "num_elites"):
            sorted_indices = np.argsort(best_val_score.tolist())
            elite_models = sorted_indices[: self.model.num_elites]
            self.model.set_elite(elite_models)


def _flatten_members(batch):
    """A [E, B, ...] transition batch as E * B rows (member-major); [B, ...] unchanged."""
    if np.ndim(batch.obs) != 3:
        return batch
    t = batch.astuple()
    flat = [np.reshape(x, (-1,) + np.shape(x)[2:]) for x in t]
    return type("_Rows", (), {"obs": flat[0], "act": flat[1], "next_obs": flat[2], "rewards": flat[3]})
