"""b200pets: an H100-native PETS planning inner loop behind mbrl-lib's Agent / Optimizer / ModelEnv API.

Sub-modules are imported lazily so that the seeded synthetic-input helpers (``synthetic``) can be used
without the CUDA library; every compute entry point fails loudly when ``libb200pets.so`` is missing.
"""
__version__ = "0.1.0"

_LAZY = {
    "ModelEnv": "model_env", "StagedModel": "staging", "LatentModelEnv": "latent", "StagedLatentModel": "latent",
    "Agent": "planning", "Optimizer": "planning", "CEMOptimizer": "planning", "ICEMOptimizer": "planning", "MPPIOptimizer": "planning",
    "TrajectoryOptimizer": "planning", "TrajectoryOptimizerAgent": "planning",
    "create_trajectory_optim_agent_for_model": "planning", "complete_agent_cfg": "planning", "rollout_model_env": "planning",
    "GaussianMLP": "models", "OneDTransitionRewardModel": "models", "EnsembleLinearLayer": "models", "BasicEnsemble": "models",
    "Normalizer": "models", "model_from_arrays": "models", "PlaNetModel": "models", "ModelTrainer": "trainer",
    "TransitionBatch": "replay", "TransitionIterator": "replay", "BootstrapIterator": "replay", "SAC": "sac",
}


def __getattr__(name):
    import importlib

    if name in _LAZY:
        return getattr(importlib.import_module(f"{__name__}.{_LAZY[name]}"), name)
    if name in ("synthetic", "functions", "planning", "models", "model_env", "staging", "_lib", "build", "dist", "mbpo",
                "trainer", "replay", "latent", "sac"):
        return importlib.import_module(f"{__name__}.{name}")
    raise AttributeError(name)
