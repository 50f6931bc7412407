"""Code-size guard for the small-group K2 kernel that bik_step runs (no GPU needed: nvcc cross-compiles for sm_90a).

The fp64 step instantiation k2t_kernel<double, G, 256, M, F32IO=true, STEP=true> is bound by instruction issue and
instruction fetch: at 17.6 k SASS instructions, K2 in the G1 step took 0.78 ms on one H100 80GB HBM3 (SXM, 700 W power
limit), and 0.60 ms at 9.2 k (DESIGN.md §3).  This test fails when its code grows back, spills, or needs more registers
than two 256-thread CTAs per SM allow.
"""

import os
import re
import shutil
import subprocess

import pytest

from mink_b200 import build as b

# SASS instructions of k2t_kernel<double, 8, 256, uint32_t, true, true> (the G1 headline): 9 216 measured with CUDA 12.9.
K2_STEP_SASS_BUDGET = 9_300
MAX_REGISTERS = 128   # __launch_bounds__(256, 2)

STEP_KERNELS = {
    "_Z10k2t_kernelIdLi8ELi256EjLb1ELb1EEvPKjiN3bik6K2ArgsEPj": "G=8, 32-bit masks",
    "_Z10k2t_kernelIdLi4ELi256EjLb1ELb1EEvPKjiN3bik6K2ArgsEPj": "G=4, 32-bit masks",
    "_Z10k2t_kernelIdLi8ELi256EmLb1ELb1EEvPKjiN3bik6K2ArgsEPj": "G=8, 64-bit masks",
}
HEADLINE = "_Z10k2t_kernelIdLi8ELi256EjLb1ELb1EEvPKjiN3bik6K2ArgsEPj"


def _nvcc():
    try:
        return b._nvcc()
    except RuntimeError:
        return None


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    if not os.path.exists(cuobjdump):
        cuobjdump = shutil.which("cuobjdump")
    if not cuobjdump:
        pytest.skip("cuobjdump not found")
    obj = str(tmp_path_factory.mktemp("k2t") / "bik_k2t.o")
    r = subprocess.run([nvcc, *b.NVCC_FLAGS, "-Xptxas", "-v", "-c", "-o", obj, os.path.join(b.CSRC, "bik_k2t.cu")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    return r.stderr, sass


def _ptxas_props(log, fn):
    m = re.search(r"Function properties for " + re.escape(fn) + r"\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads\n[^\n]*Used (\d+) registers", log)
    assert m, f"no ptxas report for {fn}"
    return {"spill_stores": int(m.group(2)), "spill_loads": int(m.group(3)), "registers": int(m.group(4))}


def _sass_count(sass, fn):
    n, cur = 0, None
    for line in sass.splitlines():
        if "Function :" in line:
            cur = line.split("Function :", 1)[1].strip()
        elif cur == fn and re.match(r"\s+/\*[0-9a-f]{4,}\*/\s", line):
            n += 1
    return n


@pytest.mark.parametrize("fn", sorted(STEP_KERNELS), ids=lambda fn: STEP_KERNELS[fn])
def test_k2_step_kernel_has_no_spills_and_fits_two_ctas(compiled, fn):
    log, _ = compiled
    p = _ptxas_props(log, fn)
    assert p["spill_stores"] == 0 and p["spill_loads"] == 0, p
    assert p["registers"] <= MAX_REGISTERS, p


def test_k2_step_kernel_sass_within_budget(compiled):
    _, sass = compiled
    n = _sass_count(sass, HEADLINE)
    assert n > 0, "step instantiation missing from the object"
    assert n <= K2_STEP_SASS_BUDGET, f"{n} SASS instructions, budget {K2_STEP_SASS_BUDGET}"
