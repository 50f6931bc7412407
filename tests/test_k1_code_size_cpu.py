"""Register guard for K1 (no GPU needed: nvcc cross-compiles for sm_90a).

The fp32 instantiations of k1_kernel are built for 4 CTAs of 128 threads per SM (BIK_K1_MINBLOCKS): 128 registers.  The packed
ones -- what bik_step, bik_converge and bik_track run -- must fit that budget without spilling: a spill costs K1 of the step
about 4 % (bik_k1.cu).  The track-mode instantiations (per-instance frame cursor) are held to the same bar.
"""

import os
import re
import subprocess

import pytest

from mink_b200 import build as b

MAX_REGISTERS = 128


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    try:
        nvcc = b._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    obj = str(tmp_path_factory.mktemp("k1") / "bik_k1.o")
    r = subprocess.run([nvcc, *b.NVCC_FLAGS, "-Xptxas", "-v", "-c", "-o", obj, os.path.join(b.CSRC, "bik_k1.cu")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stderr


def _packed_fp32(log):
    """{mangled name: (spill store bytes, spill load bytes, registers)} of k1_kernel<float, G, PK = true, TR>."""
    out = {}
    for m in re.finditer(r"Function properties for (_Z9k1_kernelIfLi\d+ELb1ELb[01]E\S*)\n\s*\d+ bytes stack frame, (\d+) bytes spill "
                         r"stores, (\d+) bytes spill loads\n[^\n]*Used (\d+) registers", log):
        out[m.group(1)] = (int(m.group(2)), int(m.group(3)), int(m.group(4)))
    return out


def test_k1_packed_fp32_kernels_do_not_spill(ptxas_log):
    props = _packed_fp32(ptxas_log)
    assert len(props) == 12, sorted(props)   # G = 1..32, converge / step form and track form
    for fn, (st, ld, regs) in props.items():
        assert st == 0 and ld == 0 and regs <= MAX_REGISTERS, (fn, st, ld, regs)
