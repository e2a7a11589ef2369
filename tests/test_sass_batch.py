"""CPU-only checks of the batched tensor-core rollout (rollout_tc_batch_kernel) in the library as build.py builds it: the
64-row variants leave room for two CTAs per SM, their stack frames stay small, and every variant issues each full K
slice of a 200-wide hidden layer as one chain of HGMMAs with no wait between them (the checks test_sass_occupancy.py and
test_sass_wgmma.py make of the single-problem kernels)."""
import importlib.util
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CUOBJDUMP = shutil.which("cuobjdump") or os.path.join(os.path.dirname(NVCC), "cuobjdump")
SLICE_K16 = 4  # K steps per full ring slot (kSliceK16 in rollout_tc.cu)
NAME = "rollout_tc_batch_kernel"


@pytest.fixture(scope="module")
def library():
    if not (os.path.exists(NVCC) and os.path.exists(CUOBJDUMP)):
        pytest.skip("needs nvcc and cuobjdump")
    spec = importlib.util.spec_from_file_location("b200pets_build_batch", os.path.join(ROOT, "mbrl-lib_b200", "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.build()


def _resources(lib):
    out = subprocess.run([CUOBJDUMP, "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    res, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+)", line)
        if m and name:
            res[name] = (int(m.group(1)), int(m.group(2)))
            name = None
    return {n: r for n, r in res.items() if NAME in n}


def test_batch_variants_fit_twice_per_sm(library):
    res = _resources(library)
    assert len(res) == 12, sorted(res)  # 3 activations x (plain, expectation) x 2 CTA shapes
    small = {n: r for n, r in res.items() if re.search(r"ELi1EEEv", n)}  # trailing NWG = 1: 64-row, 160-thread CTAs
    assert len(small) == 6, sorted(small)
    warps = 2 * 160 // 32
    for name, (regs, _) in small.items():
        per_warp = -(-regs * 32 // 256) * 256
        assert warps * per_warp <= 65536, f"{name}: {regs} registers leave room for one 160-thread CTA per SM"
    for name, (_, stack) in res.items():
        assert stack <= 112, f"{name}: {stack} B stack frame"


def test_batch_wgmma_slices_issue_back_to_back(library):
    sass = subprocess.run([CUOBJDUMP, "-sass", library], capture_output=True, text=True, check=True).stdout
    kernels, name = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1) if NAME in m.group(1) else None
            if name:
                kernels[name] = []
        elif name and ("HGMMA" in line or "WARPGROUP" in line):
            kernels[name].append(line.split("*/", 1)[1].split(";")[0].strip())
    assert len(kernels) == 12, sorted(kernels)
    for name, instrs in kernels.items():
        groups, cur = [], None
        for ins in instrs:  # the instructions between one WARPGROUP.ARRIVE (wgmma.fence) and the next
            if ins.startswith("WARPGROUP.ARRIVE"):
                cur = []
                groups.append(cur)
            elif cur is not None:
                cur.append(ins)
        assert groups, name
        for g in groups:
            hg = [i for i, ins in enumerate(g) if ins.startswith("HGMMA")]
            between = g[hg[0]:hg[-1]] if hg else []
            assert not any(ins.startswith("WARPGROUP.DEPBAR") for ins in between), (name, g)
        shapes = [[int(m.group(1)) for m in (re.match(r"HGMMA\.64x(\d+)x16\.F32\.BF16", i) for i in g) if m] for g in groups]
        assert [128, 80] * SLICE_K16 in shapes, f"{name}: no {SLICE_K16}-step slice of 64x128 + 64x80 MMAs issued back to back"
