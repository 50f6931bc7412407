// TEST INFRASTRUCTURE -- the pass loops of bik_converge64 and bik_track64 with the kernel headers (mink_b200/csrc/bik_k1.h,
// bik_k2.h, bik_k2t.h) compiled for the host, one lane per instance (G = W = 1), so that the fp64 loops can be checked
// against the goldens, the per-frame converge loop and the oracle on a machine without a GPU.  The fp32 loops are in
// track_emu.cpp.  Never shipped, never loaded by mink_b200/: the product path is CUDA only.
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../mink_b200/csrc/bik_build.h"
#include "../../mink_b200/csrc/bik_k2t.h"

using namespace bik;

static std::string g_err;
extern "C" const char* track64_emu_last_error() { return g_err.c_str(); }

struct EmuProblem {
  std::vector<uint32_t> image;   // problem image, as bik_problem_create builds it with one lane per instance
};

extern "C" void* track64_emu_problem_create(const void* blob, size_t nbytes, const bik_task_desc* tasks, int ntasks, const bik_limit_desc* limits,
                                            int nlimits) {
  HostModel m;
  if (!parse_model_blob(blob, nbytes, &m, &g_err)) return nullptr;
  EmuProblem* p = new EmuProblem;
  if (!build_image(m, tasks, ntasks, limits, nlimits, 1, &p->image, &g_err)) { delete p; return nullptr; }
  return p;
}
extern "C" void track64_emu_problem_destroy(void* p) { delete static_cast<EmuProblem*>(p); }

// The pass loops of bik_converge64 and bik_track64 (bik_api.cu: converge_pass and the bookkeeping kernels): fp64 buffers, the
// fp64 K1 with its packed and collision rows in fp64 (pk64, gc64), and K2's fp64-I/O small-group form where the device takes
// the small-group path (box limits only, nu <= K2T_NMAX_WIDE), else the general path.  Each loop runs its passes like the
// WHILE node: tick, K1, condition, K2 when the condition says go, and another pass while it does.
struct EmuLoop64 {
  const PView P;
  std::vector<double> wsm, k2w, pk, dq, Gc, hc;
  std::vector<int32_t> done, st;
  std::vector<signed char> warm;
  int count[3] = {0, 0, 0};
  K2Args a2;
  EmuLoop64(EmuProblem* p, int B, const double* ptgt, int pbatched, double* q, double dt, double damping) : P{p->image.data()} {
    const PHeader& h = P.h();
    const int nw = h.nu > 0 ? h.nu : 1, np = h.npairs > 0 ? h.npairs : 1;
    wsm.assign(k1_warp_words(h, 1) + 16, 0.0);
    k2w.assign(std::max((size_t)k2t_warp_bytes(P, 8, 1), (size_t)k2_warp_bytes(h, 8)) / 8 + 16, 0.0);
    pk.assign((size_t)B * (size_t)std::max((int)h.pk_stride, 4), 0.0); dq.assign((size_t)B * h.nv, 0.0);
    Gc.assign((size_t)B * np * h.nv, 0.0); hc.assign((size_t)B * np, 0.0);
    done.assign(B, 0); st.assign(B, 0); warm.assign((size_t)B * nw, 0);
    memset(&a2, 0, sizeof a2);
    a2.B = B; a2.q = q; a2.io64 = 1; a2.pk = pk.data(); a2.pk64 = 1; a2.ptgt = ptgt; a2.pbatched = pbatched; a2.dt = dt; a2.damping = damping;
    a2.Gc = Gc.data(); a2.hc = hc.data(); a2.gc64 = 1; a2.dq = dq.data(); a2.integrate = 1; a2.warm = warm.data(); a2.skip = done.data();
  }
  void k2() {
    const PHeader& h = P.h();
    const bool group = h.npairs == 0 && h.nu >= 1 && h.nu <= K2T_NMAX_WIDE;
    for (int b = 0; b < a2.B; ++b) {
      if (!group) k2_warp<double, 1, 65>(P, a2, b, k2w.data(), 0);
      else if (h.nu <= K2T_NMAX) k2t_warp_tile<double, 1, 1, uint32_t>(P, a2, b, k2w.data(), 0);
      else k2t_warp_tile<double, 1, 1, uint64_t>(P, a2, b, k2w.data(), 0);
    }
  }
  template <bool TR>
  void k1(const K1Args& a) { for (int b = 0; b < a.B; ++b) k1_warp_tile<double, 1, 1, true, TR>(P, a, b, wsm.data(), 0); }
  K1Args args(int B, const double* q, const double* ftgt, const double* ptgt, int pbatched, const double* ctgt, double dt, int max_iters,
              double pos, double ori) {
    K1Args a;
    memset(&a, 0, sizeof a);
    a.B = B; a.q = q; a.ftgt = ftgt; a.ptgt = ptgt; a.ctgt = ctgt; a.in64 = 1; a.pbatched = pbatched; a.dt = dt; a.pk = pk.data(); a.tol = 1e-6f;
    a.Gc = Gc.data(); a.hc = hc.data();
    a.done = done.data(); a.not_done = count + 1; a.conv_it = count; a.conv_max = max_iters;
    a.pos_thr = (float)pos; a.ori_thr = (float)ori; a.pos_thr64 = pos; a.ori_thr64 = ori;   // as the driver fills them
    return a;
  }
};

extern "C" int track64_emu_converge(void* prob, int B, double* q, const double* ftgt, const double* ptgt, int pbatched, const double* ctgt,
                                    double dt, double damping, int max_iters, double pos, double ori, int32_t* iters, int32_t* status) {
  EmuLoop64 L(static_cast<EmuProblem*>(prob), B, ptgt, pbatched, q, dt, damping);
  K1Args a = L.args(B, q, ftgt, ptgt, pbatched, ctgt, dt, max_iters, pos, ori);
  a.iters = iters; a.status = status; L.a2.status = status;
  L.count[0] = -1;
  for (int go = 1; go;) {
    L.count[0] += 1; L.count[1] = 0;
    L.k1<false>(a);
    const int it = L.count[0];
    go = it < max_iters && (it == 0 || L.count[1] > 0);
    if (go) L.k2();
  }
  for (int b = 0; b < B; ++b) if (!L.done[b]) { iters[b] = max_iters; status[b] |= 16; }
  return 0;
}

extern "C" int track64_emu_track(void* prob, int B, int T, double* q, const double* ftgt, const double* ptgt, int pbatched, const double* ctgt,
                                 const int32_t* lengths, double dt, double damping, int max_iters, double pos, double ori, double* q_traj,
                                 int32_t* iters, int32_t* status, int32_t* passes) {
  EmuLoop64 L(static_cast<EmuProblem*>(prob), B, ptgt, pbatched, q, dt, damping);
  std::vector<int32_t> cursor(B, 0), step(B);
  for (int b = 0; b < B; ++b) step[b] = (lengths ? lengths[b] : T) > 0 ? 0 : -1;
  K1Args a = L.args(B, q, ftgt, ptgt, pbatched, ctgt, dt, max_iters, pos, ori);
  a.iters = iters; a.status = L.st.data(); L.a2.status = L.st.data();
  a.cursor = cursor.data(); a.tstep = step.data(); a.lengths = lengths; a.T = T; a.q_traj = q_traj; a.traj_status = status; a.warm = L.warm.data();
  L.count[0] = 0; L.count[2] = 1;
  for (int go = 1; go;) {
    L.count[0] += L.count[2]; L.count[1] = 0;
    L.k1<true>(a);
    go = L.count[2] = L.count[1] > 0;
    if (go) L.k2();
  }
  *passes = L.count[0];
  return 0;
}
