"""Model training at the pets_halfcheetah config: the reference-shaped PyTorch trainer against the device trainer, and one
agent.act, timed in the same process so that a PETS trial's breakdown comes from one run.

Model: ensemble 7 (5 elites), 4 x 200 SiLU, HalfCheetah dimensions (obs 18 -> processed 18, act 6, out 18, no learned
reward, no_delta_list [0], fp64 normaliser).  Training as the shipped overrides run it after every 1 000-step trial:
batch 32, lr 2.8e-4, weight decay 1e-4, 12 epochs, validation_ratio 0 (every epoch is also evaluated over the whole
training set), patience 12.  Synthetic transitions, --sizes of them, stored as float64 (the replay buffer pets.train
builds with normalize_double_precision; --store-dtype float32 for a float32 store), BootstrapIterator with shuffling.

Per size, --rounds rounds alternate the two trainers (each from the same initial weights and Adam state) and the medians
are reported.  The PyTorch trainer is ModelTrainer's reference loop (``model.update`` / ``model.eval_score`` per batch,
the batch copied to the device per step, as mbrl-lib does); at sizes above --full-torch-rows it runs --torch-epochs
epochs per round and its 12-epoch time is extrapolated from the measured per-epoch cost (marked "x" in the table).  The
trial share assumes one train() per 1 000 agent.act calls (bench.py's HalfCheetah CEM agent, host clock).

    python tests/prof_train.py [--sizes 10000,100000,300000] [--rounds 3] [--torch-epochs 1] [--full-torch-rows 10000]
                               [--store-dtype float64]
"""
import argparse
import copy
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from prof_callables import gpu_description  # noqa: E402

E, ELITES, HID, LAYERS, D, A = 7, 5, 200, 4, 18, 6
LR, WD, BATCH, EPOCHS = 2.8e-4, 1e-4, 32, 12


def make_model(dev):
    from mbrl_lib_b200 import functions, models

    torch.manual_seed(0)
    mlp = models.GaussianMLP(D + A, D, dev, num_layers=LAYERS, ensemble_size=E, hid_size=HID, activation="silu")
    with torch.no_grad():
        for layer in [s[0] for s in mlp.hidden_layers] + [mlp.mean_and_logvar]:
            layer.weight.normal_(0.0, 1.0 / (2.0 * np.sqrt(layer.weight.shape[1])))
    m = models.OneDTransitionRewardModel(mlp, normalize=True, normalize_double_precision=True, learned_rewards=False,
                                         obs_process_fn=functions.OBS_PROCESS_FNS["halfcheetah"], no_delta_list=[0],
                                         num_elites=ELITES)
    return m


def make_store(n, seed=0, dtype=np.float64):
    from mbrl_lib_b200 import replay

    rng = np.random.default_rng(seed)
    obs = rng.standard_normal((n, D)).astype(dtype)
    act = rng.uniform(-1, 1, (n, A)).astype(dtype)
    nxt = (obs + 0.1 * np.tanh(obs @ rng.standard_normal((D, D)) * 0.3) + 0.05 * act.sum(1, keepdims=True)).astype(dtype)
    rew = rng.standard_normal(n).astype(dtype)
    return replay.TransitionBatch(obs, act, nxt, rew, np.zeros(n, bool), np.zeros(n, bool))


def run(model, store, device, epochs):
    from mbrl_lib_b200 import replay, trainer as tr

    m = copy.deepcopy(model)
    t = tr.ModelTrainer(m, optim_lr=LR, weight_decay=WD)
    if not device:
        t._device_supported = lambda: False
    ds = replay.BootstrapIterator(store, BATCH, E, shuffle_each_epoch=True, rng=np.random.default_rng(1))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    losses, scores = t.train(ds, num_epochs=epochs, patience=12, silent=True)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, losses, scores


def time_act(dev, reps=30):
    import mbrl_lib_b200 as bp

    spec, _, env = bench.build_problem(dev)
    cfg = {"_target_": "mbrl_lib_b200.TrajectoryOptimizerAgent", "planning_horizon": spec.horizon, "replan_freq": 1,
           "verbose": False,
           "optimizer_cfg": {"_target_": "mbrl_lib_b200.CEMOptimizer", "num_iterations": bench.CEM_ITERS,
                             "elite_ratio": bench.ELITE_RATIO, "population_size": spec.population, "alpha": bench.ALPHA,
                             "device": dev, "return_mean_elites": True}}
    agent = bp.create_trajectory_optim_agent_for_model(env, cfg, num_particles=spec.particles)
    obs0 = np.zeros(spec.obs_dim, np.float32)
    for _ in range(5):
        agent.act(obs0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        agent.act(obs0)
    return (time.perf_counter() - t0) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="10000,100000,300000")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--torch-epochs", type=int, default=1)
    ap.add_argument("--full-torch-rows", type=int, default=10000)
    ap.add_argument("--store-dtype", default="float64", choices=["float64", "float32"])
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    args = ap.parse_args()
    dev = "cuda:0"
    assert torch.cuda.is_available(), "prof_train needs a GPU"
    print(gpu_description())
    print(f"store: {args.store_dtype}; PyTorch trainer: 12 epochs up to {args.full_torch_rows} transitions, "
          f"{args.torch_epochs} scaled to 12 above")
    act_s = time_act(dev)
    print(f"agent.act (HalfCheetah CEM, bench.py's agent): {act_s * 1e3:.2f} ms per call, "
          f"{act_s * 1e3:.2f} s of planning per 1 000-step trial")
    model = make_model(dev)
    rows = []
    print(f"{'transitions':>11} {'PyTorch s':>10} {'device s':>9} {'speed-up':>8} {'train share':>11} "
          f"{'loss dev/torch':>15}")
    for n in [int(s) for s in args.sizes.split(",")]:
        dtype = np.dtype(args.store_dtype)
        store = make_store(n, dtype=dtype)
        m = copy.deepcopy(model)
        x = np.concatenate([store.obs[:, 1:2], np.sin(store.obs[:, 2:3]), np.cos(store.obs[:, 2:3]), store.obs[:, 3:],
                            store.act], 1).astype(np.float64)
        m.input_normalizer.mean = torch.tensor(x.mean(0, keepdims=True), device=dev)
        m.input_normalizer.std = torch.tensor(x.std(0, ddof=1, keepdims=True), device=dev)
        run(m, make_store(2048, 5, dtype), True, 1)  # warm-up of every kernel and allocation
        run(m, make_store(2048, 5, dtype), False, 1)
        t_dev, t_torch = [], []
        torch_epochs = EPOCHS if n <= args.full_torch_rows else args.torch_epochs
        for _ in range(args.rounds):
            td, ld, _ = run(m, store, True, EPOCHS)
            tt, lt, _ = run(m, store, False, torch_epochs)
            t_dev.append(td)
            t_torch.append(tt * EPOCHS / torch_epochs if torch_epochs != EPOCHS else tt)
        md, mt = float(np.median(t_dev)), float(np.median(t_torch))
        k = min(len(ld), len(lt))
        agree = float(np.max(np.abs(np.array(ld[:k]) - lt[:k]) / np.abs(lt[:k])))
        share = md / (md + 1000 * act_s)
        share_torch = mt / (mt + 1000 * act_s)
        mark = "" if torch_epochs == EPOCHS else "x"
        print(f"{n:>11} {mt:>9.2f}{mark:1} {md:>9.3f} {mt / md:>8.1f} {share * 100:>10.1f}% {agree:>15.2e}"
              f"   (PyTorch trainer: training is {share_torch * 100:.1f}% of the trial)")
        rows.append({"transitions": n, "torch_s": mt, "torch_extrapolated_from_epochs": torch_epochs,
                     "device_s": md, "speedup": mt / md, "trial_share_device": share, "trial_share_torch": share_torch,
                     "loss_rel_diff_first_epochs": agree, "device_runs_s": t_dev, "torch_runs_s": t_torch})
    result = {"gpu": gpu_description(), "act_ms": act_s * 1e3, "store_dtype": args.store_dtype, "rows": rows}
    print(json.dumps(result))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
