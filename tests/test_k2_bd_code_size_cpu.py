"""Code-size guard for the small-group K2 kernels with per-instance bounds (no GPU needed: nvcc cross-compiles for sm_90a).

k2t_bd_kernel is k2t_pw_kernel (posture weights, here possibly null) with each dof's box narrowed by the instance's bounds
(bik_step_bounded, bik_converge_bounded, bik_track_bounded).  The kernel is bound by instruction issue and fetch like the
others (tests/test_k2_code_size_cpu.py), so its step instantiations must not spill, must fit two 256-thread CTAs per SM, and
must stay within 3 % of the SASS of the posture-weighted step instantiation they extend.
"""

import os
import re
import shutil
import subprocess

import pytest

from mink_b200 import build as b

MAX_REGISTERS = 128   # __launch_bounds__(256, 2)
SASS_GROWTH = 0.03

# bounded step instantiation -> the posture-weighted one it extends
STEP_KERNELS = {
    "_Z13k2t_bd_kernelIdLi8ELi256EjLb1ELb1EEvPKjiN3bik8K2BdArgsEPj": "_Z13k2t_pw_kernelIdLi8ELi256EjLb1ELb1EEvPKjiN3bik8K2PwArgsEPj",
    "_Z13k2t_bd_kernelIdLi4ELi256EjLb1ELb1EEvPKjiN3bik8K2BdArgsEPj": "_Z13k2t_pw_kernelIdLi4ELi256EjLb1ELb1EEvPKjiN3bik8K2PwArgsEPj",
    "_Z13k2t_bd_kernelIdLi8ELi256EmLb1ELb1EEvPKjiN3bik8K2BdArgsEPj": "_Z13k2t_pw_kernelIdLi8ELi256EmLb1ELb1EEvPKjiN3bik8K2PwArgsEPj",
}
# the run-time-I/O form the fp64 entry points (and fp32 callers whose K1 runs in fp64) launch
IO_KERNELS = [
    "_Z13k2t_bd_kernelIdLi8ELi256EjLb0ELb0EEvPKjiN3bik8K2BdArgsEPj",
    "_Z13k2t_bd_kernelIdLi4ELi256EjLb0ELb0EEvPKjiN3bik8K2BdArgsEPj",
    "_Z13k2t_bd_kernelIdLi8ELi256EmLb0ELb0EEvPKjiN3bik8K2BdArgsEPj",
]


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
    obj = str(tmp_path_factory.mktemp("k2t_bd") / "bik_k2t.o")
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


@pytest.mark.parametrize("fn", sorted(STEP_KERNELS) + IO_KERNELS)
def test_bd_kernel_has_no_spills_and_fits_two_ctas(compiled, fn):
    log, _ = compiled
    p = _ptxas_props(log, fn)
    assert p["spill_stores"] == 0 and p["spill_loads"] == 0, p
    assert p["registers"] <= MAX_REGISTERS, p


@pytest.mark.parametrize("fn", sorted(STEP_KERNELS))
def test_bd_step_kernel_sass_within_3_percent_of_posture_weighted(compiled, fn):
    _, sass = compiled
    n, n0 = _sass_count(sass, fn), _sass_count(sass, STEP_KERNELS[fn])
    assert n > 0 and n0 > 0, "step instantiation missing from the object"
    assert n <= n0 * (1 + SASS_GROWTH), f"{n} SASS instructions against {n0} posture-weighted (+{100 * (n / n0 - 1):.1f} %)"
