"""Code-size guard for the K1 kernels with per-instance frame placement (no GPU needed: nvcc cross-compiles for sm_90a).

k1p_kernel is the collision instantiation of K1 with each frame task's pose in its node read per instance (bik_step_placed,
bik_converge_placed), in track mode (bik_track_placed), and in track mode with held targets.  Its fp32 instantiations must
keep the register budget of the fp32 k1_kernel (__launch_bounds__(128, 4): 128 registers), and no instantiation may spill.
"""

import os
import re
import subprocess

import pytest

from mink_b200 import build as b

MAX_REGISTERS_F32 = 128
GS = [1, 2, 4, 8, 16, 32]
MODES = [(0, 0), (1, 0), (1, 1)]   # (TR, HO): step / converge, track, track with held targets
KERNELS = [f"_Z10k1p_kernelI{t}Li{g}ELb{tr}ELb{ho}EEvPKjiiN3bik7K1PArgsE" for t in "fd" for g in GS for tr, ho in MODES]


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    try:
        nvcc = b._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    obj = str(tmp_path_factory.mktemp("k1p") / "bik_k1.o")
    r = subprocess.run([nvcc, *b.NVCC_FLAGS, "-Xptxas", "-v", "-c", "-o", obj, os.path.join(b.CSRC, "bik_k1.cu")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stderr


def _props(log):
    out = {}
    for m in re.finditer(r"Function properties for (_Z10k1p_kernel\S+)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads\n[^\n]*Used (\d+) registers", log):
        out[m.group(1)] = {"spill_stores": int(m.group(2)), "spill_loads": int(m.group(3)), "registers": int(m.group(4))}
    return out


def test_every_instantiation_is_compiled(ptxas_log):
    """fp32 and fp64, every lane count, step / converge, track and track with held targets (36 kernels)."""
    assert set(_props(ptxas_log)) == set(KERNELS), sorted(set(_props(ptxas_log)) ^ set(KERNELS))


@pytest.mark.parametrize("fn", KERNELS)
def test_k1p_kernel_has_no_spills(ptxas_log, fn):
    p = _props(ptxas_log)[fn]
    assert p["spill_stores"] == 0 and p["spill_loads"] == 0, p
    if "IfLi" in fn:
        assert p["registers"] <= MAX_REGISTERS_F32, p
