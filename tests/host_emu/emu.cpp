// TEST INFRASTRUCTURE -- compiles the kernel headers (mink_b200/csrc/bik_k1.h, bik_k2.h, bik_k2t.h) for the host
// with one lane per instance (G = W = 1) so the device math can be checked against the oracle on a
// machine without a GPU.  Never shipped, never loaded by mink_b200/: the product path is CUDA only.
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include "../../mink_b200/csrc/bik_build.h"
#include "../../mink_b200/csrc/bik_k2t.h"

using namespace bik;

static std::string g_err;
extern "C" const char* emu_last_error() { return g_err.c_str(); }

struct EmuProblem {
  std::vector<uint32_t> image;        // problem image (tasks + limits; FK visits only the nodes they need)
  std::vector<uint32_t> model_image;  // model-only image, as bik_model_create builds it (FK visits every node)
};

extern "C" void* emu_problem_create(const void* blob, size_t nbytes, const bik_task_desc* tasks, int ntasks, const bik_limit_desc* limits, int nlimits) {
  HostModel m;
  if (!parse_model_blob(blob, nbytes, &m, &g_err)) return nullptr;
  EmuProblem* p = new EmuProblem;
  if (!build_image(m, tasks, ntasks, limits, nlimits, 1, &p->image, &g_err)) { delete p; return nullptr; }
  if (!build_image(m, nullptr, 0, nullptr, 0, 1, &p->model_image, &g_err)) { delete p; return nullptr; }
  return p;
}
// header fields of the problem image the CPU tests pin: nv, nu, nfree, nnode, nneeded, nslots, G, nsteps, pk_stride, words32, words
extern "C" void emu_header(void* prob, int32_t* out) {
  const PHeader& h = PView{static_cast<EmuProblem*>(prob)->image.data()}.h();
  out[0] = h.nv; out[1] = h.nu; out[2] = h.nfree; out[3] = h.nnode; out[4] = h.nneeded; out[5] = h.nslots; out[6] = h.G; out[7] = h.nsteps;
  out[8] = h.pk_stride; out[9] = h.words32; out[10] = h.words;
}
extern "C" void emu_set_knobs(void* prob, int sweeps) {   // what BIK_K2_SWEEPS does in bik_problem_create
  PHeader* h = reinterpret_cast<PHeader*>(static_cast<EmuProblem*>(prob)->image.data());
  h->k2_sweeps = sweeps < 1 ? 1 : (sweeps > 16 ? 16 : sweeps);
}
extern "C" void emu_problem_destroy(void* p) { delete static_cast<EmuProblem*>(p); }

extern "C" int emu_lane_program(const void* blob, size_t nbytes, int G, int32_t* out, int cap) {
  HostModel m;
  if (!parse_model_blob(blob, nbytes, &m, &g_err)) return -1;
  std::vector<int32_t> prog; int nsteps;
  lane_program(m, G, &prog, &nsteps);
  if ((int)prog.size() > cap) return -2;
  memcpy(out, prog.data(), prog.size() * 4);
  return nsteps;
}

// K1.  f64 = 0: fp32 instantiation, fp32 buffers.  f64 = 1: fp64 instantiation, fp64 inputs and outputs.
// f64 = 2: fp64 instantiation on fp32 inputs (what bik_step runs for ill-conditioned problems of fp32 callers), fp64 outputs.
// pk != null: packed hand-off instead of dense J / e / ep.  status != null: fused check_limits.
extern "C" int emu_fk_jac(void* prob, int B, int f64, const void* q, const void* ftgt, const void* ptgt, int pbatched, const void* ctgt, double dt,
                          void* J, void* e, void* ep, void* Gc, void* hc, void* pk, int32_t* status) {
  EmuProblem* p = static_cast<EmuProblem*>(prob);
  PView P{p->image.data()};
  K1Args a;
  memset(&a, 0, sizeof a);
  a.B = B; a.q = q; a.ftgt = ftgt; a.ptgt = ptgt; a.ctgt = ctgt; a.in64 = f64 == 1; a.pbatched = pbatched; a.dt = dt;
  a.J = J; a.e = e; a.ep = ep; a.Gc = Gc; a.hc = hc; a.pk = pk; a.status = status; a.tol = 1e-6f;
  std::vector<double> wsm(k1_warp_words(P.h(), 1) + 16);
  for (int b = 0; b < B; ++b) {
    if (f64) { if (pk) k1_warp_tile<double, 1, 1, true>(P, a, b, wsm.data(), 0); else k1_warp_tile<double, 1, 1, false>(P, a, b, wsm.data(), 0); }
    else if (pk) k1_warp_tile<float, 1, 1, true>(P, a, b, reinterpret_cast<float*>(wsm.data()), 0);
    else k1_warp_tile<float, 1, 1, false>(P, a, b, reinterpret_cast<float*>(wsm.data()), 0);
  }
  return 0;
}

// K2 (fp64 solve).  path: 1 general, 3 small-group, 8 small-group with 64-bit masks.
// Task rows: packed (pk, pk64) or dense (J, e, ep fp32; ep may be null with ptgt set).  io64: q / ptgt / dq are fp64.
// Packed fp32 rows with fp32 I/O take the small-group step instantiation, as in bik_step.
template <typename M>
static void emu_k2t(const PView& P, const K2Args& a, int B, double* tw) {
  const bool step = a.pk && !a.pk64 && !a.io64;
  for (int b = 0; b < B; ++b) {
    if (step) k2t_warp_tile<double, 1, 1, M, true, true>(P, a, b, tw, 0);
    else k2t_warp_tile<double, 1, 1, M>(P, a, b, tw, 0);
  }
}
extern "C" int emu_solve(void* prob, int B, int path, int io64, const void* q, const void* pk, int pk64, const float* J, const float* e, const float* ep,
                         const void* ptgt, int pbatched, const void* Gc, const void* hc, int gc64, double dt, double damping, void* dq,
                         int integrate, int32_t* status, int32_t* iters, double* H, double* c, void* lo, void* hi, signed char* warm,
                         const int32_t* skip) {
  EmuProblem* p = static_cast<EmuProblem*>(prob);
  PView P{p->image.data()};
  K2Args a;
  memset(&a, 0, sizeof a);
  a.B = B; a.q = q; a.io64 = io64; a.pk = pk; a.pk64 = pk64; a.J = J; a.e = e; a.ep = ep; a.dense64 = 0; a.ptgt = ptgt; a.pbatched = pbatched;
  a.Gc = Gc; a.hc = hc; a.gc64 = gc64; a.dt = dt; a.damping = damping; a.dq = dq; a.integrate = integrate; a.status = status; a.iters = iters;
  a.Hout = H; a.cout = c; a.lo_out = lo; a.hi_out = hi; a.warm = warm; a.skip = skip;
  if (path == 3 || path == 8) {
    const int nmax = path == 8 ? K2T_NMAX_WIDE : K2T_NMAX;
    if (P.h().npairs != 0 || P.h().nu < 1 || P.h().nu > nmax) { g_err = "small-group path not applicable"; return -1; }
    std::vector<double> tw(k2t_warp_bytes(P, 8, 1) / 8 + 16);
    if (path == 3) emu_k2t<uint32_t>(P, a, B, tw.data());
    else emu_k2t<uint64_t>(P, a, B, tw.data());
    return 0;
  }
  if (path != 1) { g_err = "unknown K2 path " + std::to_string(path); return -1; }
  std::vector<double> wsm(k2_warp_bytes(P.h(), 8) / 8 + 16);
  for (int b = 0; b < B; ++b) k2_warp<double, 1, 65>(P, a, b, wsm.data(), 0);
  return 0;
}

extern "C" int emu_fk(void* prob, int B, int f64, const void* q, const bik_frame* frames, int nframes, void* poses, void* com, void* J) {
  EmuProblem* p = static_cast<EmuProblem*>(prob);
  PView P{p->model_image.data()};
  if (nframes > 16) return -1;
  FkArgs a; memset(&a, 0, sizeof a);
  a.B = B; a.nframes = nframes; a.q = q; a.poses = poses; a.com = com; a.J = J; a.io64 = f64;
  for (int f = 0; f < nframes; ++f) { a.frames[f].node = frames[f].node; put_frame64(frames[f], a.frames[f].lpos, a.frames[f].lquat); }
  std::vector<double> wsm(fk_warp_words(P.h(), 1) + 16);
  for (int b = 0; b < B; ++b) {
    if (f64) fk_warp_tile<double, 1, 1>(P, a, b, wsm.data(), 0);
    else fk_warp_tile<float, 1, 1>(P, a, b, reinterpret_cast<float*>(wsm.data()), 0);
  }
  return 0;
}

extern "C" int emu_integrate(void* prob, int B, float* q, const float* dq) {
  EmuProblem* p = static_cast<EmuProblem*>(prob);
  PView P{p->image.data()};
  for (int b = 0; b < B; ++b) integrate_instance<float>(P, q + (size_t)b * P.h().nq, dq + (size_t)b * P.h().nv);
  return 0;
}
extern "C" int emu_check_limits(void* prob, int B, const float* q, float tol, int32_t* status) {
  EmuProblem* p = static_cast<EmuProblem*>(prob);
  PView P{p->image.data()};
  for (int b = 0; b < B; ++b) status[b] = check_limits_instance<float>(P, q + (size_t)b * P.h().nq, tol);
  return 0;
}
