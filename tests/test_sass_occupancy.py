"""CPU-only check of the register and stack use of the tensor-core rollout's 64-row CTA (160 threads): the plan sizes
its shared memory for two CTAs per SM, so the registers must allow two as well (65 536 per SM, allocated per warp in
units of 256).  The launcher sizes its grid for two resident CTAs per SM without asking the occupancy API, so this is
where a register regression shows."""
import importlib.util
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CUOBJDUMP = shutil.which("cuobjdump") or os.path.join(os.path.dirname(NVCC), "cuobjdump")


def _resources():
    """{kernel name: (registers, stack bytes, static shared memory bytes)} of the library as build.py builds it."""
    if not (os.path.exists(NVCC) and os.path.exists(CUOBJDUMP)):
        pytest.skip("needs nvcc and cuobjdump")
    spec = importlib.util.spec_from_file_location("b200pets_build_occ", os.path.join(ROOT, "mbrl-lib_b200", "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    lib = mod.build()
    out = subprocess.run([CUOBJDUMP, "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    res, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+) SHARED:(\d+)", line)
        if m and name:
            res[name] = tuple(int(g) for g in m.groups())
            name = None
    return res


def test_64_row_variants_fit_twice_per_sm():
    res = _resources()
    # trailing template argument NWG = 1 (rollout_tc.cu): the 64-row, 160-thread variants
    small = {n: r for n, r in res.items() if "rollout_tc_kernel" in n and re.search(r"ELi1EEEv", n)}
    assert len(small) == 12, sorted(small)  # 3 activations x (plain, expectation, 2 trajectory variants)
    # the launcher budgets every 64-row launch, batched or not, with the plain SiLU kernel's static shared memory
    batch = {n: r for n, r in res.items() if "rollout_tc_batch_kernel" in n and re.search(r"ELi1EEEv", n)}
    assert len(batch) == 6, sorted(batch)  # 3 activations x (plain, expectation)
    assert len({r[2] for r in (*small.values(), *batch.values())}) == 1, {n: r[2] for n, r in {**small, **batch}.items()}
    warps = 2 * 160 // 32
    for name, (regs, stack, _) in small.items():
        per_warp = -(-regs * 32 // 256) * 256
        assert warps * per_warp <= 65536, f"{name}: {regs} registers leave room for one 160-thread CTA per SM"
        assert stack <= 112, f"{name}: {stack} B stack frame"
