// TEST INFRASTRUCTURE -- compiles the kernel headers (mink_b200/csrc/bik_k1.h, bik_k2.h, bik_k2t.h) and the pass loop of
// bik_converge / bik_track (bik_loop.h) for the host with one lane per instance (G = W = 1) so the device math can be checked
// against the oracle on a machine without a GPU.  Never shipped, never loaded by mink_b200/: the product path is CUDA only.
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include "../../mink_b200/csrc/bik_build.h"
#include "../../mink_b200/csrc/bik_k2t.h"
#include "../../mink_b200/csrc/bik_loop.h"

using namespace bik;

static std::string g_err;
extern "C" const char* emu_last_error() { return g_err.c_str(); }

struct EmuProblem {
  std::vector<uint32_t> image;        // problem image (tasks + limits; FK visits only the nodes they need)
  std::vector<uint32_t> model_image;  // model-only image, as bik_model_create builds it (FK visits every node)
  K1Conditioning k1cond;              // what the driver's automatic choice of K1's precision rests on
};

extern "C" void* emu_problem_create(const void* blob, size_t nbytes, const bik_task_desc* tasks, int ntasks, const bik_limit_desc* limits, int nlimits) {
  HostModel m;
  if (!parse_model_blob(blob, nbytes, &m, &g_err)) return nullptr;
  EmuProblem* p = new EmuProblem;
  if (!build_image(m, tasks, ntasks, limits, nlimits, 1, &p->image, &g_err)) { delete p; return nullptr; }
  if (!build_image(m, nullptr, 0, nullptr, 0, 1, &p->model_image, &g_err)) { delete p; return nullptr; }
  p->k1cond = k1_conditioning(m, p->image, tasks, ntasks);
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

// K2 (fp64 solve), one instance per tile.  path: 1 general, 3 small-group, 8 small-group with 64-bit masks.  The small-group
// instantiation follows launch_k2t: fp64 I/O or fp64 rows take the generic form, packed fp32 rows with fp32 I/O the step form.
template <typename M>
static void emu_k2t(const PView& P, const K2Args& a, double* tw) {
  const bool step = a.pk && !a.pk64 && !a.io64;
  for (int b = 0; b < a.B; ++b) {
    if (step) k2t_warp_tile<double, 1, 1, M, true, true>(P, a, b, tw, 0);
    else k2t_warp_tile<double, 1, 1, M>(P, a, b, tw, 0);
  }
}
static int emu_k2(const PView& P, const K2Args& a, int path) {
  if (path == 3 || path == 8) {
    const int nmax = path == 8 ? K2T_NMAX_WIDE : K2T_NMAX;
    if (P.h().npairs != 0 || P.h().nu < 1 || P.h().nu > nmax) { g_err = "small-group path not applicable"; return -1; }
    std::vector<double> tw(k2t_warp_bytes(P, 8, 1) / 8 + 16);
    if (path == 3) emu_k2t<uint32_t>(P, a, tw.data());
    else emu_k2t<uint64_t>(P, a, tw.data());
    return 0;
  }
  if (path != 1) { g_err = "unknown K2 path " + std::to_string(path); return -1; }
  std::vector<double> wsm(k2_warp_bytes(P.h(), 8) / 8 + 16);
  for (int b = 0; b < a.B; ++b) k2_warp<double, 1, 65>(P, a, b, wsm.data(), 0);
  return 0;
}
// the path a solving launch takes on the device (bik_k2_group_applies, shared memory and BIK_K2_PATH aside)
static int emu_k2_path(const PHeader& h) {
  if (h.npairs != 0 || h.nu < 1 || h.nu > K2T_NMAX_WIDE) return 1;
  return h.nu <= K2T_NMAX ? 3 : 8;
}

// Task rows: packed (pk, pk64) or dense (J, e, ep fp32; ep may be null with ptgt set).  io64: q / ptgt / dq are fp64.
extern "C" int emu_solve(void* prob, int B, int path, int io64, const void* q, const void* pk, int pk64, const float* J, const float* e, const float* ep,
                         const void* ptgt, int pbatched, const void* Gc, const void* hc, int gc64, double dt, double damping, void* dq,
                         int integrate, int32_t* status, int32_t* iters, double* H, double* c, void* lo, void* hi, signed char* warm,
                         const int32_t* skip) {
  EmuProblem* p = static_cast<EmuProblem*>(prob);
  K2Args a;
  memset(&a, 0, sizeof a);
  a.B = B; a.q = q; a.io64 = io64; a.pk = pk; a.pk64 = pk64; a.J = J; a.e = e; a.ep = ep; a.dense64 = 0; a.ptgt = ptgt; a.pbatched = pbatched;
  a.Gc = Gc; a.hc = hc; a.gc64 = gc64; a.dt = dt; a.damping = damping; a.dq = dq; a.integrate = integrate; a.status = status; a.iters = iters;
  a.Hout = H; a.cout = c; a.lo_out = lo; a.hi_out = hi; a.warm = warm; a.skip = skip;
  return emu_k2(PView{p->image.data()}, a, path);
}

// The pass loop of bik_converge / bik_track (bik_loop.h) on host buffers: the reset, then passes as the WHILE node runs them
// (tick, K1, condition, K2 when the condition says go) while the condition says go.  K1 runs in fp64 exactly when the driver's
// would (BIK_K1_PRECISION aside), K2 takes the path the device takes.
template <typename T>
static void emu_k1_pass(const PView& P, const K1Args& a, bool track, double* wsm) {
  for (int b = 0; b < a.B; ++b) {
    if (track) k1_warp_tile<T, 1, 1, true, true>(P, a, b, reinterpret_cast<T*>(wsm), 0);
    else k1_warp_tile<T, 1, 1, true, false>(P, a, b, reinterpret_cast<T*>(wsm), 0);
  }
}
static int emu_loop(EmuProblem* p, ConvCall c, int32_t* passes) {
  const PView P{p->image.data()};
  const PHeader& h = P.h();
  const size_t B = c.B;
  const HandoffSizes n = handoff_sizes(h);
  c.k1d = c.io64 || k1_auto_double(h, p->k1cond, c.damping);
  // hand-off rows and dq sized for fp64 elements whatever the precision
  std::vector<double> pk(B * n.pk), Gc(B * n.Gc), hc(B * n.hc), dq(B * h.nv), wsm(k1_warp_words(h, 1) + 16);
  std::vector<signed char> warm(B * n.warm);
  std::vector<int32_t> done(B), cursor(B), step(B), status(B);
  int count[3];
  const ConvBufs s{pk.data(), Gc.data(), hc.data(), dq.data(), warm.data(), done.data(), cursor.data(), step.data(), status.data(), count};
  for (int b = 0; b < c.B; ++b) conv_reset(c.track, c.T, c.lengths, s, b);
  const K1Args a1 = conv_k1_args(c, s, c.status);
  const K2Args a2 = conv_k2_args(c, s, c.status);
  const int path = emu_k2_path(h);
  for (int go = 1; go;) {
    conv_tick(c.track, count);
    if (c.k1d) emu_k1_pass<double>(P, a1, c.track, wsm.data());
    else emu_k1_pass<float>(P, a1, c.track, wsm.data());
    go = conv_cond(c.track, c.max_iters, count);
    if (go && emu_k2(P, a2, path)) return -1;
  }
  if (c.track) *passes = count[0];
  else for (int b = 0; b < c.B; ++b) conv_finish(c.max_iters, done.data(), c.iters, c.status, b);
  return 0;
}
// f64 = 0: bik_converge / bik_track on fp32 buffers (dt and the thresholds are rounded to float, as their parameters are);
// f64 = 1: bik_converge64 / bik_track64 on fp64 buffers.
static int emu_call(void* prob, int f64, bool track, int B, int T, void* q, const void* ftgt, const void* ptgt, int pbatched, const void* ctgt,
                    const int32_t* lengths, double dt, double damping, int max_iters, double pos, double ori, void* q_traj, int32_t* iters,
                    int32_t* status, int32_t* passes) {
  if (!f64) { dt = (float)dt; pos = (float)pos; ori = (float)ori; }
  bik_inputs in;
  memset(&in, 0, sizeof in);
  in.q = q; in.frame_targets = ftgt; in.posture_targets = ptgt; in.com_targets = ctgt; in.posture_batched = pbatched; in.f64 = f64;
  ConvCall c;
  memset(&c, 0, sizeof c);
  c.B = B; c.T = T; c.max_iters = max_iters; c.dt = dt; c.pos = pos; c.ori = ori; c.damping = damping; c.q = q; c.in = &in;
  c.lengths = lengths; c.q_traj = q_traj; c.iters = iters; c.status = status; c.track = track; c.io64 = f64 != 0;
  return emu_loop(static_cast<EmuProblem*>(prob), c, passes);
}
extern "C" int emu_converge(void* prob, int f64, int B, void* q, const void* ftgt, const void* ptgt, int pbatched, const void* ctgt, double dt,
                            double damping, int max_iters, double pos, double ori, int32_t* iters, int32_t* status) {
  return emu_call(prob, f64, false, B, 1, q, ftgt, ptgt, pbatched, ctgt, nullptr, dt, damping, max_iters, pos, ori, nullptr, iters, status, nullptr);
}
extern "C" int emu_track(void* prob, int f64, int B, int T, void* q, const void* ftgt, const void* ptgt, int pbatched, const void* ctgt,
                         const int32_t* lengths, double dt, double damping, int max_iters, double pos, double ori, void* q_traj, int32_t* iters,
                         int32_t* status, int32_t* passes) {
  return emu_call(prob, f64, true, B, T, q, ftgt, ptgt, pbatched, ctgt, lengths, dt, damping, max_iters, pos, ori, q_traj, iters, status, passes);
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

// f64 = 0: integrate_instance<float> on fp32 q / dq; f64 = 1: integrate_instance<double> on fp64 q / dq.
template <typename T>
static void emu_integrate_t(const PView& P, int B, T* q, const T* dq) {
  for (int b = 0; b < B; ++b) integrate_instance<T>(P, q + (size_t)b * P.h().nq, dq + (size_t)b * P.h().nv);
}
extern "C" int emu_integrate(void* prob, int f64, int B, void* q, const void* dq) {
  PView P{static_cast<EmuProblem*>(prob)->image.data()};
  if (f64) emu_integrate_t<double>(P, B, static_cast<double*>(q), static_cast<const double*>(dq));
  else emu_integrate_t<float>(P, B, static_cast<float*>(q), static_cast<const float*>(dq));
  return 0;
}
extern "C" int emu_check_limits(void* prob, int B, const float* q, float tol, int32_t* status) {
  EmuProblem* p = static_cast<EmuProblem*>(prob);
  PView P{p->image.data()};
  for (int b = 0; b < B; ++b) status[b] = check_limits_instance<float>(P, q + (size_t)b * P.h().nq, tol);
  return 0;
}

// bik_math.h's Lie layer, one function on n inputs, in float (f64 = 0) or double (f64 = 1).  Inputs and outputs are fp64
// arrays: inputs are rounded to T on the way in (exact when the caller rounded them to T already), results widened on the way out.
template <typename T> static Q4<T> ld_q4(const double* a) { return q4<T>(T(a[0]), T(a[1]), T(a[2]), T(a[3])); }
template <typename T> static V3<T> ld_v3(const double* a) { return v3<T>(T(a[0]), T(a[1]), T(a[2])); }
template <typename T> static void st_v3(V3<T> v, double* a) { a[0] = v.x; a[1] = v.y; a[2] = v.z; }
template <typename T> static void st_m3(const M3<T>& m, double* a) { for (int i = 0; i < 9; ++i) a[i] = m.m[i]; }

template <typename T>
static void lie_t(int fn, int n, const double* a, const double* b, double* out, double* out2) {
  for (int i = 0; i < n; ++i) {
    if (fn == 0) {          // coefficients at theta^2 = a[i]: out[4i..] = A, B, C, D
      T B, C, D;
      coef_BCD<T>(T(a[i]), &B, &C, &D);
      out[4 * i] = coef_A<T>(T(a[i])); out[4 * i + 1] = B; out[4 * i + 2] = C; out[4 * i + 3] = D;
    } else if (fn == 1) {   // so3_log(q = a[4i..])
      st_v3(so3_log<T>(ld_q4<T>(a + 4 * i)), out + 3 * i);
    } else if (fn == 2) {   // se3_log(q = a[4i..], t = b[3i..]) -> (v, w)
      V3<T> v, w;
      se3_log<T>(ld_q4<T>(a + 4 * i), ld_v3<T>(b + 3 * i), &v, &w);
      st_v3(v, out + 6 * i); st_v3(w, out + 6 * i + 3);
    } else if (fn == 3) {   // se3_ljacinv_blocks(v = a[6i..], w = a[6i+3..]) -> Ji (out), Mi (out2), row major
      M3<T> Ji, Mi;
      se3_ljacinv_blocks<T>(ld_v3<T>(a + 6 * i), ld_v3<T>(a + 6 * i + 3), &Ji, &Mi);
      st_m3(Ji, out + 9 * i); st_m3(Mi, out2 + 9 * i);
    } else if (fn == 4) {   // quat_sub(qa = a[4i..], qb = b[4i..])
      st_v3(quat_sub<T>(ld_q4<T>(a + 4 * i), ld_q4<T>(b + 4 * i)), out + 3 * i);
    } else {                // quat_integrate(q = a[4i..], w = b[3i..])
      Q4<T> o = quat_integrate<T>(ld_q4<T>(a + 4 * i), ld_v3<T>(b + 3 * i));
      out[4 * i] = o.w; out[4 * i + 1] = o.x; out[4 * i + 2] = o.y; out[4 * i + 3] = o.z;
    }
  }
}
extern "C" int emu_lie(int fn, int f64, int n, const double* a, const double* b, double* out, double* out2) {
  if (fn < 0 || fn > 5) { g_err = "unknown Lie function " + std::to_string(fn); return -1; }
  if (f64) lie_t<double>(fn, n, a, b, out, out2);
  else lie_t<float>(fn, n, a, b, out, out2);
  return 0;
}
