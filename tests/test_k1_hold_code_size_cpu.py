"""Code-size guard for the K1 kernels with held targets (no GPU needed: nvcc cross-compiles for sm_90a).

k1h_kernel is track mode's k1_kernel with each task's hold mask read, and the held values captured on the first pass of a
run (bik_track_hold), with and without per-instance collision arguments.  Its fp32 instantiations must keep the register
budget of the fp32 k1_kernel (__launch_bounds__(128, 4): 128 registers), and no instantiation may spill.
"""

import os
import re
import subprocess

import pytest

from mink_b200 import build as b

MAX_REGISTERS_F32 = 128
GS = [1, 2, 4, 8, 16, 32]
KERNELS = [f"_Z10k1h_kernelI{t}Li{g}ELb{co}EEvPKjiiN3bik7K1HArgsE" for t in "fd" for g in GS for co in (0, 1)]


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    try:
        nvcc = b._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    obj = str(tmp_path_factory.mktemp("k1h") / "bik_k1.o")
    r = subprocess.run([nvcc, *b.NVCC_FLAGS, "-Xptxas", "-v", "-c", "-o", obj, os.path.join(b.CSRC, "bik_k1.cu")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stderr


def _props(log):
    out = {}
    for m in re.finditer(r"Function properties for (_Z10k1h_kernel\S+)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads\n[^\n]*Used (\d+) registers", log):
        out[m.group(1)] = {"spill_stores": int(m.group(2)), "spill_loads": int(m.group(3)), "registers": int(m.group(4))}
    return out


def test_every_instantiation_is_compiled(ptxas_log):
    """fp32 and fp64, every lane count, with and without collision arguments (24 kernels)."""
    assert set(_props(ptxas_log)) == set(KERNELS), sorted(set(_props(ptxas_log)) ^ set(KERNELS))


@pytest.mark.parametrize("fn", KERNELS)
def test_k1h_kernel_has_no_spills(ptxas_log, fn):
    p = _props(ptxas_log)[fn]
    assert p["spill_stores"] == 0 and p["spill_loads"] == 0, p
    if "IfLi" in fn:
        assert p["registers"] <= MAX_REGISTERS_F32, p
