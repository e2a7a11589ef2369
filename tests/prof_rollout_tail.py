"""What is left of the tensor-core rollout's per-step tail: the step's Gaussian draws and the next step's action loads.

Times the rollout (evaluate_action_sequences at bench.py's build_problem config: PETS HalfCheetah, ensemble 7 / 5 elites,
4 x 200 SiLU, 20 particles, H 30, tile shuffle, in-kernel noise) against two throwaway builds of the same library:

  * no_noise:  rollout_tc.cu with the per-step Philox draws removed (the noise words stay zero);
  * const_act: rollout_tc.cu with every action word after a tile's first step set to a constant instead of loaded.

The variants are compiled into a temporary directory from the committed source (text substitutions that must each match
once) and linked with the other objects of the in-tree build, so build() must have run first.  Each library is timed in
its own process; the three alternate for --rounds rounds, and the medians are reported.  Their results are wrong on
purpose: they only bound how much time the draws and the loads still take.

    python tests/prof_rollout_tail.py [--rounds 3] [--pops 1,32] [--libs name=path,...]

--pops are multiples of the 500-sequence population (1: bench.py's value, 32: pop 16 000); --libs times prebuilt
libraries instead of building the variants.
"""
import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "mbrl-lib_b200")
CSRC = os.path.join(PKG, "csrc")

# (variant, [(text in rollout_tc.cu, replacement), ...]); every text must occur exactly once
VARIANTS = [
    ("no_noise", [
        ("philox_normal4((uint32_t)rid_glob, (uint32_t)t, RNG_STREAM_EPS | (uint32_t)gq, (uint32_t)prob_offset<BATCH>(a, bt, kp),\n"
         "                               prob_seed<BATCH>(a, bt, kp), z);",
         ""),
    ]),
    ("const_act", [
        ("v[j] = (j < m.A && valid) ? ap[j] : 0.f;", "v[j] = (j < m.A && valid) ? (t == a.t0 ? ap[j] : 0.25f) : 0.f;"),
        ("for (int j = 0; j < m.A; ++j) my_act[j] = valid ? ap[j] : 0.f;",
         "for (int j = 0; j < m.A; ++j) my_act[j] = valid ? (t == a.t0 ? ap[j] : 0.25f) : 0.f;"),
    ]),
]


def gpu_description():
    import torch

    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as exc:  # pragma: no cover - depends on the box
        out = f"nvidia-smi unavailable ({type(exc).__name__})"
    return f"{name}, power limit / max SM clock / SM clock: {out}"


def worker(lib, pops):
    """ms per evaluate_action_sequences call at each population multiple, with the library at `lib`."""
    sys.path.insert(0, ROOT)
    from mbrl_lib_b200 import _lib

    _lib.LIB_PATH = lib
    import torch

    import bench
    from mbrl_lib_b200 import synthetic as syn

    spec, _, env = bench.build_problem("cuda:0")
    inp = syn.make_rollout_inputs(spec, with_noise=False)
    out = {}
    for scale in pops:
        acts = torch.from_numpy(inp["actions"]).to("cuda:0").repeat(scale, 1, 1)
        calls = max(5, 40 // scale)
        for _ in range(6):
            env.evaluate_action_sequences(acts, inp["obs0"], spec.particles)
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        blocks = []
        for _ in range(5):
            s.record()
            for _ in range(calls):
                env.evaluate_action_sequences(acts, inp["obs0"], spec.particles)
            e.record()
            torch.cuda.synchronize()
            blocks.append(s.elapsed_time(e) / calls)
        out[str(acts.shape[0])] = statistics.median(blocks)
    print("RESULT " + json.dumps(out), flush=True)


def build_variants(tmp):
    src = open(os.path.join(CSRC, "rollout_tc.cu")).read()
    others = [os.path.join(CSRC, f) for f in ("api.o", "rollout_f32.o", "cem.o", "mbpo.o", "train.o")]
    missing = [o for o in others if not os.path.exists(o)]
    if missing:
        sys.exit(f"in-tree objects missing ({', '.join(missing)}): run build() first")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    sys.path.insert(0, PKG)
    from build import NVCC_FLAGS

    procs, libs = [], {}
    for name, subs in VARIANTS:
        text = src
        for old, new in subs:
            assert text.count(old) == 1, f"{name}: expected one occurrence of {old!r} in rollout_tc.cu"
            text = text.replace(old, new)
        d = os.path.join(tmp, name)
        os.makedirs(d)
        cu = os.path.join(d, "rollout_tc.cu")
        open(cu, "w").write(text)
        obj, lib = os.path.join(d, "rollout_tc.o"), os.path.join(d, "libb200pets.so")
        cmd = (f"{nvcc} {' '.join(NVCC_FLAGS)} -I{CSRC} -c {cu} -o {obj} && "
               f"{nvcc} -shared -o {lib} {obj} {' '.join(others)} -gencode arch=compute_90a,code=sm_90a -lcudart")
        procs.append(subprocess.Popen(cmd, shell=True))
        libs[name] = lib
    for p in procs:
        if p.wait() != 0:
            sys.exit("variant build failed")
    return libs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--pops", default="1,32")
    ap.add_argument("--libs", help="name=path,... prebuilt libraries to time (the first is the baseline)")
    ap.add_argument("--worker", help=argparse.SUPPRESS)
    args = ap.parse_args()
    pops = [int(x) for x in args.pops.split(",")]
    if args.worker:
        return worker(args.worker, pops)

    tmp = tempfile.mkdtemp(prefix="b200pets_tail_")
    try:
        if args.libs:
            libs = dict(kv.split("=", 1) for kv in args.libs.split(","))
        else:
            libs = {"committed": os.path.join(PKG, "libb200pets.so"), **build_variants(tmp)}
        import torch  # noqa: F401  (device description only)

        print(gpu_description(), flush=True)
        times = {n: [] for n in libs}
        for rnd in range(args.rounds):
            for name, lib in libs.items():
                out = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", lib, "--pops", args.pops],
                                     capture_output=True, text=True, cwd=ROOT)
                line = [ln for ln in out.stdout.splitlines() if ln.startswith("RESULT ")]
                if out.returncode or not line:
                    sys.exit(f"{name} worker failed:\n{out.stdout}\n{out.stderr}")
                res = json.loads(line[0][7:])
                times[name].append(res)
                print(f"round {rnd} {name}: " + ", ".join(f"pop {k}: {v:.4f} ms" for k, v in res.items()), flush=True)
        base = next(iter(libs))
        for pop in times[base][0]:
            b = statistics.median(r[pop] for r in times[base])
            print(f"pop {pop}: {base} {b:.4f} ms per evaluation (median of {args.rounds})")
            for name in list(libs)[1:]:
                v = statistics.median(r[pop] for r in times[name])
                print(f"  {name}: {v:.4f} ms, {100 * (b - v) / b:+.1f} % of {base}")
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
