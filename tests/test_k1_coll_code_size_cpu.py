"""Code-size guard for the K1 kernels with per-instance collision pairs and distances (no GPU needed: nvcc cross-compiles for
sm_90a).

k1c_kernel is the packed k1_kernel with each instance's pair mask and distances read in the collision rows
(bik_step_coll, bik_converge_coll, bik_track_coll).  Its fp32 instantiations (BIK_K1_PRECISION=f32) must keep the
register budget of the fp32 k1_kernel (__launch_bounds__(128, 4): 128 registers), and no instantiation may spill.
"""

import os
import re
import shutil
import subprocess

import pytest

from mink_b200 import build as b

MAX_REGISTERS_F32 = 128
GS = [1, 2, 4, 8, 16, 32]
KERNELS = [f"_Z10k1c_kernelI{t}Li{g}ELb{tr}EEvPKjiiN3bik7K1CArgsE" for t in "fd" for g in GS for tr in (0, 1)]


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    try:
        nvcc = b._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    if not os.path.exists(cuobjdump):
        cuobjdump = shutil.which("cuobjdump")
    if not cuobjdump:
        pytest.skip("cuobjdump not found")
    obj = str(tmp_path_factory.mktemp("k1c") / "bik_k1.o")
    r = subprocess.run([nvcc, *b.NVCC_FLAGS, "-Xptxas", "-v", "-c", "-o", obj, os.path.join(b.CSRC, "bik_k1.cu")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    return r.stderr, sass


def _ptxas_props(log, fn):
    m = re.search(r"Function properties for " + re.escape(fn) + r"\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads\n[^\n]*Used (\d+) registers", log)
    assert m, f"no ptxas report for {fn}"
    return {"spill_stores": int(m.group(2)), "spill_loads": int(m.group(3)), "registers": int(m.group(4))}


def test_every_instantiation_is_compiled(compiled):
    """Packed form only: fp32 and fp64, every lane count, step / converge and track mode (24 kernels)."""
    _, sass = compiled
    found = set(re.findall(r"Function : (_Z10k1c_kernel\S+)", sass))
    assert found == set(KERNELS), sorted(found ^ set(KERNELS))


@pytest.mark.parametrize("fn", KERNELS)
def test_k1c_kernel_has_no_spills(compiled, fn):
    log, _ = compiled
    p = _ptxas_props(log, fn)
    assert p["spill_stores"] == 0 and p["spill_loads"] == 0, p
    if "IfLi" in fn:
        assert p["registers"] <= MAX_REGISTERS_F32, p
