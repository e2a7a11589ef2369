"""Diagnostics: the worst per-element errors behind the bars of tests/test_gpu_transitions.py.

For every case, kernel and member draw (trajectories as one window and as single-step windows, ModelEnv.step at its
batches, the unregistered model options) prints the worst error of next_obs and of the reward against the float64 step,
relative to max(1, |ref|) per element, the number of done flags that differ, and the negative controls' errors.
"""
import os
import sys
import traceback

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_transitions as tt  # noqa: E402

worst = {"f32": {}, "bf16_tc": {}}


def show(tag, precision, err):
    print(f"{tag:58s} {precision:8s} next_obs {err['next_obs']:.2e}  reward {err['reward']:.2e}  done {err['done']}"
          + (f"  link {err['link_rows_differ']}" if "link_rows_differ" in err else "")
          + f"  median row {np.median(err['rows']):.1e}, rows above bar {(err['rows'] > tt.BAR[precision]).mean():.4f}",
          flush=True)
    w = worst[precision]
    for k in ("next_obs", "reward"):
        if err[k] > w.get(k, (0, ""))[0]:
            w[k] = (err[k], tag)


def guarded(fn):
    try:
        fn()
    except Exception:  # report and go on: one failure should not hide the other measurements
        traceback.print_exc()


for name, precision, mode in tt.TRAJ:
    for windows in ("one", "steps"):
        guarded(lambda: show(f"trajectory {name} {mode} {windows}", precision,
                             tt.trajectory_errors(name, precision, mode, windows, link=windows == "one")[0]))
for name, precision, mode in tt.STEP:
    guarded(lambda: show(f"step {name} {mode}", precision, tt.step_errors(name, precision, mode)))
for opt in tt.OPTIONS:
    for precision in ("f32", "bf16_tc"):
        guarded(lambda: show(f"option {opt}", precision, tt.option_errors(opt, precision)[0]))
for kind in ("slope", "no_delta", "member", "eps"):
    for precision in ("f32", "bf16_tc"):
        guarded(lambda: print(f"control {kind:10s} {precision:8s} {tt._control_error(kind, precision):.2e} "
                              f"(bar {tt.BAR[precision]:.0e})", flush=True))
for precision, w in worst.items():
    for k, (v, tag) in w.items():
        print(f"worst {precision} {k}: {v:.3e} ({tag})")
