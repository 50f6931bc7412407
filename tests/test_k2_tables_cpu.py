"""The small-group K2's build-time tables (bik_build.h: K2TaskRec, the packed-record weights, K2DofRec, K2PostRec, the
quaternion-joint list) against what the kernel derived per tile before they existed, from the other sections of the same
problem image.  Exact comparisons: the kernel's results stay bit-identical only if every table entry is.

The image is built by the same host code bik_problem_create runs (bik_build.h, compiled here with g++); the expected values
are recomputed in numpy from the image's fp32 records."""

import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from mink_b200._abi import (LIMIT_CONFIGURATION, LIMIT_VELOCITY, TASK_COM, TASK_FRAME, TASK_POSTURE, TASK_RELATIVE_FRAME,
                            LimitSpec, ProblemSpec, TaskSpec, spec_from_workload)
from mink_b200.flatten import Frame
from mink_b200.workloads import MODELS_DIR, WORKLOADS, load_flat

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "mink_b200", "csrc")

SHIM = r'''
#include <stddef.h>
#include "bik_build.h"
using namespace bik;
static std::string g_err;
extern "C" const char* k2tab_error() { return g_err.c_str(); }
// image words into out[cap] (returns the word count, -1 on a build error); hdr: the header fields the test reads
extern "C" int k2tab_image(const void* blob, size_t n, const bik_task_desc* t, int nt, const bik_limit_desc* l, int nl, uint32_t* out, int cap,
                           int32_t* hdr) {
  HostModel m; std::vector<uint32_t> img;
  if (!parse_model_blob(blob, n, &m, &g_err) || !build_image(m, t, nt, l, nl, 0, &img, &g_err)) return -1;
  if ((int)img.size() > cap) return -2;
  memcpy(out, img.data(), img.size() * 4);
  const PHeader& h = *reinterpret_cast<const PHeader*>(img.data());
  const K2Header& k = *reinterpret_cast<const K2Header*>(img.data() + h.words64);
  const int32_t v[] = {h.nv, h.nnode, h.F, h.C, h.P, h.ncfg, h.off_nodes, h.off_frames, h.off_cols, h.off_com, h.com_cols_off, h.com_ncols,
                       h.off_posture, h.off_cfg, h.off_vmax, h.off_dofqadr, h.off_umap, h.pk_stride, h.words32, h.words64,
                       k.tasks, k.w, k.dofs, k.post, k.quat, k.nquat, h.words};
  memcpy(hdr, v, sizeof v);
  return (int)img.size();
}
'''
HDR = ("nv nnode F C P ncfg off_nodes off_frames off_cols off_com com_cols_off com_ncols off_posture off_cfg off_vmax off_dofqadr "
       "off_umap pk_stride words32 words64 off_k2tasks off_k2w off_k2dofs off_k2post off_quat nquat words").split()   # K2Header fields as off_k2*
NODE_WORDS, FRAME_WORDS = 20, 36   # bik_layout.h
JNT_FREE, JNT_BALL = 0, 1


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("k2tab")
    src, so = d / "k2tab.cpp", d / "k2tab.so"
    src.write_text(SHIM)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", CSRC, "-o", str(so), str(src)])
    lib = C.CDLL(str(so))
    lib.k2tab_error.restype = C.c_char_p
    return lib


def _image(shim, fm, spec, may_fail=False):
    blob = fm.to_blob()
    t, nt, l, nl, _keep = spec.to_c()
    out = np.zeros(1 << 20, np.uint32)
    hdr = np.zeros(len(HDR), np.int32)
    n = shim.k2tab_image(blob, len(blob), t, nt, l, nl, out.ctypes.data_as(C.POINTER(C.c_uint32)), out.size,
                         hdr.ctypes.data_as(C.POINTER(C.c_int32)))
    if may_fail and n == -1:
        return None, shim.k2tab_error().decode()
    assert n > 0, shim.k2tab_error().decode()
    return out[:n].copy(), dict(zip(HDR, (int(v) for v in hdr)))


def _check(img, h):
    f32, i32 = img.view(np.float32), img.view(np.int32)
    nv, F, C_, P = h["nv"], h["F"], h["C"], h["P"]
    assert h["words32"] <= h["words64"] < h["off_k2tasks"] < h["words"] == len(img)
    umap = i32[h["off_umap"]:h["off_umap"] + nv]
    cols = i32[h["off_cols"]:]
    tri = lambda i: i * (i + 1) // 2
    w = img[h["off_k2w"]:h["off_k2w"] + 2 * h["pk_stride"]].view(np.float64)
    covered = np.zeros(h["pk_stride"], bool)
    # ---- tasks: record, weights of the packed elements, pair schedule ----
    for t in range(F + C_):
        rec = i32[h["off_k2tasks"] + 8 * t:h["off_k2tasks"] + 8 * t + 8]
        nr, nc, coff, row0, pk_off, pairs_off, ucol_off = (int(x) for x in rec[:7])
        lm = f32[h["off_k2tasks"] + 8 * t + 7]
        if t < F:   # k2_task: FrameRec
            fo = h["off_frames"] + FRAME_WORDS * t
            exp = (6, i32[fo + 16], i32[fo + 17], i32[fo + 18], i32[fo + 31])
            cost, gain, elm = f32[fo + 8:fo + 14], f32[fo + 14], f32[fo + 15]
        else:       # k2_task: the CoM record { cost[3], gain, lm, row0, pk_off, pad }
            co = h["off_com"] + 8 * (t - F)
            exp = (3, h["com_ncols"], h["com_cols_off"], i32[co + 5], i32[co + 6])
            cost, gain, elm = f32[co:co + 3], f32[co + 3], f32[co + 4]
        assert (nr, nc, coff, row0, pk_off) == exp and lm == elm
        # k2t_stage_task: element k of the block is weighted by cost[k % nr] (Jacobian) or cost[r] * -gain (error)
        nj = nr * nc
        k = np.arange(nj + nr)
        we = np.where(k < nj, cost.astype(np.float64)[k % nr], cost.astype(np.float64)[(k - nj) % nr] * np.float64(-gain))
        assert np.array_equal(w[pk_off:pk_off + nj + nr], we)
        covered[pk_off:pk_off + nj + nr] = True
        # k2t_task_accumulate_nr: H entry (ia, ib) at tri(max(ua, ub)) + min(ua, ub), ua = umap[cols[coff + ia] & 0xffff]
        ua = umap[cols[coff:coff + nc] & 0xffff]
        assert (ua >= 0).all()
        ucol = img[ucol_off:].view(np.int16)[:nc]
        assert np.array_equal(ucol, ua)
        pairs = img[pairs_off:].view(np.int16)[:tri(nc)]
        exp_pairs = [tri(max(ua[ia], ua[ib])) + min(ua[ia], ua[ib]) for ia in range(nc) for ib in range(ia + 1)]
        assert np.array_equal(pairs, np.array(exp_pairs, np.int16))
    assert not w[~covered].any()   # the record's alignment padding weighs nothing
    # ---- per dof: qpos address, coupled index, box inputs (box_dof) ----
    qadr = i32[h["off_dofqadr"]:h["off_dofqadr"] + nv]
    vmax = f32[h["off_vmax"]:h["off_vmax"] + nv]
    for d in range(nv):
        o = h["off_k2dofs"] + 12 * d
        assert (i32[o], i32[o + 1]) == (qadr[d], umap[d])
        assert f32[o + 8].tobytes() == vmax[d].tobytes()
        for c in range(h["ncfg"]):
            cf = f32[h["off_cfg"] + c * (2 + 2 * nv):]
            got = f32[o + 2 + 3 * c:o + 5 + 3 * c]
            assert got.tobytes() == np.array([cf[0], cf[2 + d], cf[2 + nv + d]], np.float32).tobytes()
    # ---- posture: w^2, (gain w) w and w gain of every (task, dof), in double from the fp32 record ----
    post = img[h["off_k2post"]:h["off_k2post"] + 8 * P * nv].view(np.float64).reshape(P, nv, 4)
    for p in range(P):
        pr = f32[h["off_posture"] + p * (2 + nv):h["off_posture"] + (p + 1) * (2 + nv)].astype(np.float64)
        g, wd = pr[0], pr[2:]
        assert np.array_equal(post[p, :, 0], wd * wd)
        assert np.array_equal(post[p, :, 1], (g * wd) * wd)
        assert np.array_equal(post[p, :, 2], wd * g)
    # ---- free and ball joints, in node order ----
    types = i32[h["off_nodes"] + 1:h["off_nodes"] + NODE_WORDS * h["nnode"]:NODE_WORDS]
    exp_q = np.nonzero((types == JNT_FREE) | (types == JNT_BALL))[0]
    assert h["nquat"] == len(exp_q) and np.array_equal(i32[h["off_quat"]:h["off_quat"] + h["nquat"]], exp_q)


@pytest.mark.parametrize("name", sorted(WORKLOADS))
def test_k2_tables_of_every_workload(shim, name):
    wl = WORKLOADS[name]
    fm = load_flat(wl["robot"])
    _check(*_image(shim, fm, spec_from_workload(fm, wl)))


def _rich_spec(fm, com=True):
    """Two frame tasks, a relative frame task, two posture tasks with uneven dof costs and LM damping, a CoM task and both
    kinds of box limit: every table is populated."""
    n = fm.nnode
    fr = lambda node: Frame(node, np.array([0.01, -0.02, 0.03]), np.array([1.0, 0.0, 0.0, 0.0]))
    nonfree = np.array([d for d in range(fm.nv) if fm.node_type[fm.dof_node[d]] != JNT_FREE], np.int32)
    limited = np.nonzero(fm.dof_limited)[0].astype(np.int32)
    rng = np.random.default_rng(n)
    tasks = [TaskSpec(TASK_FRAME, frame=fr(n - 1), cost=np.array([3.0, 3.0, 3.0, 0.7, 0.7, 0.7]), gain=0.9, lm_damping=0.3),
             TaskSpec(TASK_FRAME, frame=fr(n // 2), cost=np.array([1.0, 2.0, 0.0, 0.1, 0.2, 0.3]), gain=0.37),
             TaskSpec(TASK_RELATIVE_FRAME, frame=fr(n - 1), root=fr(max(n // 3, 0)), cost=np.full(6, 0.3), gain=0.61),
             TaskSpec(TASK_POSTURE, dof_cost=rng.uniform(0.01, 2.0, fm.nv), gain=0.77, lm_damping=0.25),
             TaskSpec(TASK_POSTURE, dof_cost=rng.uniform(0.01, 2.0, fm.nv), gain=0.0)]
    if com:
        tasks.append(TaskSpec(TASK_COM, cost=np.array([200.0, 150.0, 10.0, 0, 0, 0]), gain=0.83, lm_damping=0.1))
    limits = [LimitSpec(LIMIT_VELOCITY, dof=nonfree, vmax=rng.uniform(0.5, 3.0, len(nonfree)))]
    if len(limited):
        limits += [LimitSpec(LIMIT_CONFIGURATION, dof=limited, lower=fm.dof_lo[limited] + 0.01, upper=fm.dof_hi[limited] - 0.01, gain=0.95),
                   LimitSpec(LIMIT_CONFIGURATION, dof=limited[::2], lower=fm.dof_lo[limited[::2]], upper=fm.dof_hi[limited[::2]], gain=0.5)]
    return ProblemSpec(tasks, limits)


@pytest.mark.parametrize("robot", sorted(f[:-5] for f in os.listdir(MODELS_DIR) if f.endswith(".bikm")))
def test_k2_tables_of_every_model(shim, robot):
    fm = load_flat(robot)
    img, h = _image(shim, fm, _rich_spec(fm), may_fail=True)
    if img is None:   # a model without mass below its root body takes no CoM task
        assert "ComTask" in h
        img, h = _image(shim, fm, _rich_spec(fm, com=False))
    assert h["P"] == 2 and h["F"] == 3
    _check(img, h)
