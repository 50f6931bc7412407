// TEST INFRASTRUCTURE -- the pass loops of bik_converge and bik_track with the kernel headers (mink_b200/csrc/bik_k1.h,
// bik_k2.h, bik_k2t.h) compiled for the host, one lane per instance (G = W = 1), so that bik_track's bookkeeping can be
// checked against the per-frame converge loop and the oracle on a machine without a GPU.  Never shipped, never loaded by
// mink_b200/: the product path is CUDA only.
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../mink_b200/csrc/bik_build.h"
#include "../../mink_b200/csrc/bik_k2t.h"

using namespace bik;

static std::string g_err;
extern "C" const char* track_emu_last_error() { return g_err.c_str(); }

struct EmuProblem {
  std::vector<uint32_t> image;   // problem image, as bik_problem_create builds it with one lane per instance
};

extern "C" void* track_emu_problem_create(const void* blob, size_t nbytes, const bik_task_desc* tasks, int ntasks, const bik_limit_desc* limits,
                                          int nlimits) {
  HostModel m;
  if (!parse_model_blob(blob, nbytes, &m, &g_err)) return nullptr;
  EmuProblem* p = new EmuProblem;
  if (!build_image(m, tasks, ntasks, limits, nlimits, 1, &p->image, &g_err)) { delete p; return nullptr; }
  return p;
}
extern "C" void track_emu_problem_destroy(void* p) { delete static_cast<EmuProblem*>(p); }

// The pass loops of bik_converge and bik_track (bik_api.cu: converge_pass and the bookkeeping kernels), fp32 buffers and the
// fp32 K1, one instance per tile.  K2 takes the small-group step instantiation where bik_step would (box limits only,
// nu <= K2T_NMAX_WIDE), else the general path.  Each loop runs its passes like the WHILE node: tick, K1, condition, K2 when the
// condition says go, and another pass while it does.
struct EmuLoop {
  const PView P;
  std::vector<double> wsm, k2w;
  std::vector<float> pk, dq;
  std::vector<int32_t> done, st;
  std::vector<signed char> warm;
  int count[3] = {0, 0, 0};
  K2Args a2;
  EmuLoop(EmuProblem* p, int B, const float* ptgt, int pbatched, float* q, double dt, double damping) : P{p->image.data()} {
    const PHeader& h = P.h();
    const int nw = h.nu > 0 ? h.nu : 1;
    wsm.assign(k1_warp_words(h, 1) + 16, 0.0);
    k2w.assign(std::max((size_t)k2t_warp_bytes(P, 8, 1), (size_t)k2_warp_bytes(h, 8)) / 8 + 16, 0.0);
    pk.assign((size_t)B * (size_t)std::max((int)h.pk_stride, 4), 0.f); dq.assign((size_t)B * h.nv, 0.f);
    done.assign(B, 0); st.assign(B, 0); warm.assign((size_t)B * nw, 0);
    memset(&a2, 0, sizeof a2);
    a2.B = B; a2.q = q; a2.pk = pk.data(); a2.ptgt = ptgt; a2.pbatched = pbatched; a2.dt = dt; a2.damping = damping; a2.dq = dq.data();
    a2.integrate = 1; a2.warm = warm.data(); a2.skip = done.data();
  }
  void k2() {
    const PHeader& h = P.h();
    const bool group = h.npairs == 0 && h.nu >= 1 && h.nu <= K2T_NMAX_WIDE;
    for (int b = 0; b < a2.B; ++b) {
      if (!group) k2_warp<double, 1, 65>(P, a2, b, k2w.data(), 0);
      else if (h.nu <= K2T_NMAX) k2t_warp_tile<double, 1, 1, uint32_t, true, true>(P, a2, b, k2w.data(), 0);
      else k2t_warp_tile<double, 1, 1, uint64_t, true, true>(P, a2, b, k2w.data(), 0);
    }
  }
  template <bool TR>
  void k1(const K1Args& a) { for (int b = 0; b < a.B; ++b) k1_warp_tile<float, 1, 1, true, TR>(P, a, b, reinterpret_cast<float*>(wsm.data()), 0); }
  K1Args args(int B, const float* q, const float* ftgt, const float* ptgt, int pbatched, const float* ctgt, double dt, int max_iters, float pos, float ori) {
    K1Args a;
    memset(&a, 0, sizeof a);
    a.B = B; a.q = q; a.ftgt = ftgt; a.ptgt = ptgt; a.ctgt = ctgt; a.pbatched = pbatched; a.dt = dt; a.pk = pk.data(); a.tol = 1e-6f;
    a.done = done.data(); a.not_done = count + 1; a.conv_it = count; a.conv_max = max_iters; a.pos_thr = pos; a.ori_thr = ori;
    return a;
  }
};

// Collision rows would need the K1 -> K2 collision hand-off (and the fp64 K1 bik_step picks for them): not emulated here.
static bool loop_supported(EmuProblem* p) {
  if (PView{p->image.data()}.h().npairs == 0) return true;
  g_err = "the emulated pass loops take problems without collision rows";
  return false;
}

extern "C" int track_emu_converge(void* prob, int B, float* q, const float* ftgt, const float* ptgt, int pbatched, const float* ctgt, double dt,
                            double damping, int max_iters, float pos, float ori, int32_t* iters, int32_t* status) {
  EmuProblem* p = static_cast<EmuProblem*>(prob);
  if (!loop_supported(p)) return -1;
  EmuLoop L(p, B, ptgt, pbatched, q, dt, damping);
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

extern "C" int track_emu_track(void* prob, int B, int T, float* q, const float* ftgt, const float* ptgt, int pbatched, const float* ctgt,
                         const int32_t* lengths, double dt, double damping, int max_iters, float pos, float ori, float* q_traj, int32_t* iters,
                         int32_t* status, int32_t* passes) {
  EmuProblem* p = static_cast<EmuProblem*>(prob);
  if (!loop_supported(p)) return -1;
  EmuLoop L(p, B, ptgt, pbatched, q, dt, damping);
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
