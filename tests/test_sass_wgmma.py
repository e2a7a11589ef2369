"""CPU-only check of the code ptxas makes of the tensor-core rollout: every layer's K slice must be one asynchronous
chain of wgmma (HGMMA) instructions.  When ptxas cannot prove that a chain is safe to keep in flight it inserts a wait
after each MMA (WARPGROUP.DEPBAR.LE gsb0, 0x0) and reports C7510 / C7520; the kernel still computes the same result,
only several times slower, so nothing but the compiled code shows it."""
import importlib.util
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "mbrl-lib_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CUOBJDUMP = shutil.which("cuobjdump") or os.path.join(os.path.dirname(NVCC), "cuobjdump")
SLICE_K16 = 4  # K steps per full ring slot (kSliceK16 in rollout_tc.cu)


def _nvcc_flags():
    spec = importlib.util.spec_from_file_location("b200pets_build_flags", os.path.join(ROOT, "mbrl-lib_b200", "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.NVCC_FLAGS


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    """(ptxas -v log, {kernel name: [HGMMA / WARPGROUP instruction, ...]}) of rollout_tc.cu as build.py compiles it."""
    if not (os.path.exists(NVCC) and os.path.exists(CUOBJDUMP)):
        pytest.skip("needs nvcc and cuobjdump")
    obj = str(tmp_path_factory.mktemp("sass") / "rollout_tc.o")
    res = subprocess.run([NVCC, *_nvcc_flags(), "-Xptxas=-v", "-c", os.path.join(CSRC, "rollout_tc.cu"), "-o", obj],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    sass = subprocess.run([CUOBJDUMP, "-sass", obj], capture_output=True, text=True, check=True).stdout
    kernels, name = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            kernels[name] = []
        elif name and ("HGMMA" in line or "WARPGROUP" in line):
            kernels[name].append(line.split("*/", 1)[1].split(";")[0].strip())
    return res.stdout + res.stderr, kernels


def _groups(instrs):
    """The HGMMA / WARPGROUP.DEPBAR instructions between one WARPGROUP.ARRIVE (wgmma.fence) and the next."""
    groups, cur = [], None
    for ins in instrs:
        if ins.startswith("WARPGROUP.ARRIVE"):
            cur = []
            groups.append(cur)
        elif cur is not None:
            cur.append(ins)
    return groups


def _hgmma_shape(ins):
    m = re.match(r"HGMMA\.64x(\d+)x16\.F32\.BF16", ins)
    return int(m.group(1)) if m else None


def test_ptxas_does_not_serialise_wgmma(compiled):
    log, _ = compiled
    bad = [line for line in log.splitlines() if re.search(r"\(C75(10|20)\)", line)]
    assert not bad, "ptxas serialises wgmma chains:\n" + "\n".join(bad[:10])


def test_wgmma_slices_issue_back_to_back(compiled):
    _, kernels = compiled
    act_silu = re.search(r"#define B200PETS_ACT_SILU (\d+)", open(os.path.join(ROOT, "include", "b200pets.h")).read())
    # <SILU, no expectation, no trajectory, NWG = 1>: the benched one (500 x 20 rows are 80 tiles: 64-row CTAs)
    flagship = f"17rollout_tc_kernelILi{act_silu.group(1)}ELb0ELb0ELi1EEEv8ModelDev11RolloutArgs6TcPlanx"
    names = [n for n in kernels if "rollout_tc_kernel" in n or "wgmma_selftest_kernel" in n]
    assert any(n.endswith(flagship) for n in names), names
    for name in names:
        groups = _groups(kernels[name])
        assert groups, name
        for g in groups:  # once issued, a slice's MMAs are not waited for one at a time
            hg = [i for i, ins in enumerate(g) if ins.startswith("HGMMA")]
            between = g[hg[0]:hg[-1]] if hg else []
            assert not any(ins.startswith("WARPGROUP.DEPBAR") for ins in between), (name, g)
        # a full slice of a 200-wide hidden layer (Np 208 = 128 + 80 columns): 4 K steps x 2 MMAs in one group
        full = [[128, 80] * SLICE_K16 == [_hgmma_shape(ins) for ins in g if ins.startswith("HGMMA")] for g in groups]
        assert any(full), f"{name}: no {SLICE_K16}-step slice of 64x128 + 64x80 MMAs issued back to back"
