// bik_k1.h -- K1: forward kinematics + task errors + task Jacobians (+ collision rows, + check_limits).
//
// Mapping: G lanes cooperate on one robot instance (G in {1,2,4,8,16,32}); a warp of W lanes
// therefore carries IPW = W/G consecutive instances.  The tree is walked by a host-compiled lane
// program (bik_build.h: lane_program): at step s lane g composes node prog[s][g] from its parent's
// pose, which an earlier step left in the per-instance shared-memory state.
//
// Scalar type T: float is the default (the Jacobian sweep is bandwidth / issue bound); double is the
// instantiation for ill-conditioned problems and for fp64 callers (the reference is fp64 end to end,
// mink/solve_ik.py:13-22): it reads the fp64 side tables of the image (kinematic constants at full
// precision), takes fp32 or fp64 inputs and writes fp64 rows.
//
// Outputs, two forms:
//   dense   J[B][K][nv], e[B][K], e_posture, collision rows -- what Task.compute_jacobian returns (bik_fk_jac);
//   packed  pk[B][pk_stride]: per task only the non-zero (ancestor-dof) columns, column-major [ncols][6] followed by
//           e[6] -- the K1 -> K2 hand-off inside bik_step (G1: 792 B instead of 3 168 B per instance, no zero-fill).
//
// The same source is compiled for the host with W = G = 1 (tests/host_emu) -- every cross-lane
// primitive degenerates to a no-op there.
//
// Reference semantics: mujoco mj_kinematics / mj_jac via mink/configuration.py:63-64,144-153;
// FrameTask mink/tasks/frame_task.py:95-146; ComTask mink/tasks/com_task.py:71-97;
// PostureTask.compute_error mink/tasks/posture_task.py:87-118;
// CollisionAvoidanceLimit mink/limits/collision_avoidance_limit.py:59-72,187-210;
// Configuration.check_limits mink/configuration.py:77-110.
#pragma once
#include "bik_layout.h"
#include "bik_math.h"
#if defined(__CUDACC__)
#include "bik_ptx.cuh"
#endif

#if defined(__CUDA_ARCH__)
#define BIK_SYNCWARP() __syncwarp()
#else
#define BIK_SYNCWARP() ((void)0)
#endif

#define BIK_INF_F (bik::bik_inf())

namespace bik {

// plain 8/16-byte carriers for vectorised shared/global moves (float2/float4 only exist under nvcc)
struct alignas(8) F2 { float x, y; };
struct alignas(16) F4 { float x, y, z, w; };
struct alignas(16) D2 { double x, y; };

BIK_HD float bik_inf() {
#if defined(__CUDA_ARCH__)
  return __int_as_float(0x7f800000);
#else
  return INFINITY;
#endif
}

// input element i of a caller buffer that holds fp32 or fp64 values (warp-uniform flag)
// The fp32 instantiations only ever see fp32 buffers (the launchers refuse anything else), so for them the flag is ignored
// at compile time: no branch, no fp64 load path in the fp32 kernels.
template <typename T> BIK_HD T ldin(const void* p, long long i, int is64) {
  if (sizeof(T) == 4) return T(reinterpret_cast<const float*>(p)[i]);
  return is64 ? T(reinterpret_cast<const double*>(p)[i]) : T(reinterpret_cast<const float*>(p)[i]);
}
template <typename T> BIK_HD void stout(void* p, long long i, int is64, T v) {
  if (sizeof(T) == 4) { reinterpret_cast<float*>(p)[i] = float(v); return; }
  if (is64) reinterpret_cast<double*>(p)[i] = double(v); else reinterpret_cast<float*>(p)[i] = float(v);
}

struct PView {
  const uint32_t* base;
  BIK_HD const PHeader& h() const { return *reinterpret_cast<const PHeader*>(base); }
  BIK_HD const NodeRec& node(int n) const { return *reinterpret_cast<const NodeRec*>(base + h().off_nodes + NODE_WORDS * n); }
  BIK_HD const FrameRec& frame(int f) const { return *reinterpret_cast<const FrameRec*>(base + h().off_frames + FRAME_WORDS * f); }
  BIK_HD const ComNodeRec& comnode(int n) const { return *reinterpret_cast<const ComNodeRec*>(base + h().off_comnodes + COMNODE_WORDS * n); }
  BIK_HD const GeomRec& geom(int g) const { return *reinterpret_cast<const GeomRec*>(base + h().off_geoms + GEOM_WORDS * g); }
  BIK_HD const NodeRec64& node64(int n) const { return *reinterpret_cast<const NodeRec64*>(base + h().off_nodes64 + NODE64_WORDS * n); }
  BIK_HD const FrameRec64& frame64(int f) const { return *reinterpret_cast<const FrameRec64*>(base + h().off_frames64 + FRAME64_WORDS * f); }
  BIK_HD const ComNodeRec64& comnode64(int n) const { return *reinterpret_cast<const ComNodeRec64*>(base + h().off_comnodes64 + COMNODE64_WORDS * n); }
  BIK_HD const GeomRec64& geom64(int g) const { return *reinterpret_cast<const GeomRec64*>(base + h().off_geoms64 + GEOM64_WORDS * g); }
  BIK_HD const float* f(int off) const { return reinterpret_cast<const float*>(base + off); }
  BIK_HD const int32_t* i(int off) const { return reinterpret_cast<const int32_t*>(base + off); }
  BIK_HD const double* d(int off) const { return reinterpret_cast<const double*>(base + off); }
};

// ---- kinematic constants at the precision of the instantiation -------------------------------------------
template <typename T> struct KC;
template <> struct KC<float> {
  // (the caller's NodeRec reference is used as is: re-deriving it from the image header costs a dependent shared-memory load each time)
  static BIK_HD V3<float> npos(const PView&, int, const NodeRec& r) { return v3<float>(r.pos[0], r.pos[1], r.pos[2]); }
  static BIK_HD Q4<float> nquat(const PView&, int, const NodeRec& r) { return q4<float>(r.quat[0], r.quat[1], r.quat[2], r.quat[3]); }
  static BIK_HD V3<float> naxis(const PView&, int, const NodeRec& r) { return v3<float>(r.axis[0], r.axis[1], r.axis[2]); }
  static BIK_HD V3<float> njpos(const PView&, int, const NodeRec& r) { return v3<float>(r.jpos[0], r.jpos[1], r.jpos[2]); }
  static BIK_HD float qpos0(const PView& P, int k) { return P.f(P.h().off_qpos0)[k]; }
  static BIK_HD V3<float> flpos(const PView& P, int f) { const FrameRec& r = P.frame(f); return v3<float>(r.lpos[0], r.lpos[1], r.lpos[2]); }
  static BIK_HD Q4<float> flquat(const PView& P, int f) { const FrameRec& r = P.frame(f); return q4<float>(r.lquat[0], r.lquat[1], r.lquat[2], r.lquat[3]); }
  static BIK_HD V3<float> frlpos(const PView& P, int f) { const FrameRec& r = P.frame(f); return v3<float>(r.rlpos[0], r.rlpos[1], r.rlpos[2]); }
  static BIK_HD Q4<float> frlquat(const PView& P, int f) { const FrameRec& r = P.frame(f); return q4<float>(r.rlquat[0], r.rlquat[1], r.rlquat[2], r.rlquat[3]); }
  static BIK_HD float own_m(const PView& P, int n) { return P.comnode(n).own_m; }
  static BIK_HD float sub_m(const PView& P, int n) { return P.comnode(n).sub_m; }
  static BIK_HD V3<float> own_c(const PView& P, int n) { const ComNodeRec& r = P.comnode(n); return v3<float>(r.own_c[0], r.own_c[1], r.own_c[2]); }
  static BIK_HD float com_mass(const PView& P) { return P.h().com_total_mass; }
  static BIK_HD V3<float> com_fixed(const PView& P) { const PHeader& h = P.h(); return v3<float>(h.com_fixed[0], h.com_fixed[1], h.com_fixed[2]); }
  static BIK_HD V3<float> glpos(const PView& P, int g) { const GeomRec& r = P.geom(g); return v3<float>(r.lpos[0], r.lpos[1], r.lpos[2]); }
  static BIK_HD Q4<float> glquat(const PView& P, int g) { const GeomRec& r = P.geom(g); return q4<float>(r.lquat[0], r.lquat[1], r.lquat[2], r.lquat[3]); }
  static BIK_HD float gsize(const PView& P, int g, int k) { return P.geom(g).size[k]; }
  static BIK_HD float coll(const PView& P, int k) { const PHeader& h = P.h(); return k == 0 ? h.coll_gain : (k == 1 ? h.coll_dmin : (k == 2 ? h.coll_ddet : h.coll_relax)); }
};
template <> struct KC<double> {
  static BIK_HD V3<double> npos(const PView& P, int n, const NodeRec&) { const NodeRec64& r = P.node64(n); return v3<double>(r.pos[0], r.pos[1], r.pos[2]); }
  static BIK_HD Q4<double> nquat(const PView& P, int n, const NodeRec&) { const NodeRec64& r = P.node64(n); return q4<double>(r.quat[0], r.quat[1], r.quat[2], r.quat[3]); }
  static BIK_HD V3<double> naxis(const PView& P, int n, const NodeRec&) { const NodeRec64& r = P.node64(n); return v3<double>(r.axis[0], r.axis[1], r.axis[2]); }
  static BIK_HD V3<double> njpos(const PView& P, int n, const NodeRec&) { const NodeRec64& r = P.node64(n); return v3<double>(r.jpos[0], r.jpos[1], r.jpos[2]); }
  static BIK_HD double qpos0(const PView& P, int k) { return P.d(P.h().off_qpos064)[k]; }
  static BIK_HD V3<double> flpos(const PView& P, int f) { const FrameRec64& r = P.frame64(f); return v3<double>(r.lpos[0], r.lpos[1], r.lpos[2]); }
  static BIK_HD Q4<double> flquat(const PView& P, int f) { const FrameRec64& r = P.frame64(f); return q4<double>(r.lquat[0], r.lquat[1], r.lquat[2], r.lquat[3]); }
  static BIK_HD V3<double> frlpos(const PView& P, int f) { const FrameRec64& r = P.frame64(f); return v3<double>(r.rlpos[0], r.rlpos[1], r.rlpos[2]); }
  static BIK_HD Q4<double> frlquat(const PView& P, int f) { const FrameRec64& r = P.frame64(f); return q4<double>(r.rlquat[0], r.rlquat[1], r.rlquat[2], r.rlquat[3]); }
  static BIK_HD double own_m(const PView& P, int n) { return P.comnode64(n).own_m; }
  static BIK_HD double sub_m(const PView& P, int n) { return P.comnode64(n).sub_m; }
  static BIK_HD V3<double> own_c(const PView& P, int n) { const ComNodeRec64& r = P.comnode64(n); return v3<double>(r.own_c[0], r.own_c[1], r.own_c[2]); }
  static BIK_HD double com_mass(const PView& P) { return P.d(P.h().off_com64)[0]; }
  static BIK_HD V3<double> com_fixed(const PView& P) { const double* c = P.d(P.h().off_com64); return v3<double>(c[1], c[2], c[3]); }
  static BIK_HD V3<double> glpos(const PView& P, int g) { const GeomRec64& r = P.geom64(g); return v3<double>(r.lpos[0], r.lpos[1], r.lpos[2]); }
  static BIK_HD Q4<double> glquat(const PView& P, int g) { const GeomRec64& r = P.geom64(g); return q4<double>(r.lquat[0], r.lquat[1], r.lquat[2], r.lquat[3]); }
  static BIK_HD double gsize(const PView& P, int g, int k) { return P.geom64(g).size[k]; }
  static BIK_HD double coll(const PView& P, int k) { return P.d(P.h().off_com64)[4 + k]; }
};

struct K1Args {
  int B;
  const void* q;         // [B][nq]          fp32, or fp64 when in64
  const void* ftgt;      // [B][F][7]
  const void* ptgt;      // [B or 1][P][nq]; track mode with ptcur set: the sequence, [T][P][nq] (pbatched 2) or [B][T][P][nq] (3)
  const void* ctgt;      // [B][C][3]
  int in64;
  int pbatched;
  double dt;
  // dense outputs (element type = T of the instantiation); any of them may be null when pk is set
  void* J;               // [B][K][nv]
  void* e;               // [B][K]
  void* ep;              // [B][P][nv]
  void* Gc;              // [B][npairs][nv]
  void* hc;              // [B][npairs]
  void* pk;              // [B][pk_stride] packed hand-off (then J / e / ep are not written)
  // fused Configuration.check_limits (null: skipped)
  int32_t* status;       // [B]
  int accumulate;        // 0: status = bits, 1: status |= bits
  float tol;
  // fused convergence test of bik_converge (done == null: skipped): instances whose frame-task errors are under the
  // thresholds are marked done (iters = conv_it), the others are counted in *not_done
  int32_t* done;
  int32_t* iters;
  int* not_done;
  const int* conv_it;    // device counter: steps taken so far (0: nothing is tested yet)
  int conv_max;          // max_iters: at step conv_max nothing is solved any more, so the limits are not checked either
  float pos_thr, ori_thr;
  // track mode of bik_track (the TR instantiation): the same test, but every instance walks its own sequence of frames.
  // The step index is per instance; a test that ends a frame writes iters / traj_status / q_traj at row b*T + cursor[b],
  // clears b's warm-start bytes and moves the cursor on.  done[] is rewritten on every pass: 1 = K2 leaves b alone in this
  // pass (its frame just ended, or it has no frames left); *not_done counts the instances with frames left; status is
  // the [B] status of the frame in progress.  iters is [B][T] here.
  int32_t* cursor;       // [B] frame each instance is on
  int32_t* tstep;        // [B] steps taken in that frame; -1: no frames left (nothing is computed for the instance)
  const int32_t* lengths;   // [B] frames per instance, or null: all T
  int T;
  void* q_traj;          // [B][T][nq], q's element type
  int32_t* traj_status;  // [B][T] or null
  signed char* warm;     // [B][max(nu,1)] K2's warm-start bytes
  // the thresholds as the fp64 instantiation compares them (the reference tests np.linalg.norm(err[:3]) <= pos_threshold in
  // double); fp32 callers store (double)(float) threshold here, so that the fp64 K1 they may run decides as the fp32 one
  double pos_thr64, ori_thr64;
  // per-instance task weights of the packed form (null: all ones): [B][K], track mode [B][T][K] (row b*T + cursor[b]), in the
  // inputs' element type.  Row r of the packed J and e is multiplied by the weight clamped to [0, 1] (NaN: 0), so that K2's
  // cost_r becomes cost_r * w_r; the errors K1 tests stay unweighted.
  const void* weights;
  // track mode with a posture target sequence (null: none): [B][P][nq] in the inputs' element type.  On the first pass of each
  // of b's frames K1 copies that frame's posture rows of ptgt into row b; K2 reads this buffer as its per-instance targets.
  void* ptcur;
};
// The arguments of the per-instance collision instantiation (k1c_kernel, k1_warp_tile<..., CO = true>): the ..._coll entry
// points.  Row r of the buffers is instance b's (b*T + cursor[b] in track mode); each may be null.  enabled [rows][npairs]:
// pair k is computed iff its byte is != 0, else it hands K2 what a pair beyond the detection distance hands it (a zero G row,
// h = +inf) without its distance being computed.  dmin / ddet [rows], in the inputs' element type: the instance's
// minimum_distance_from_collisions / collision_detection_distance; a non-finite value falls back to the problem's and sets
// BIK_STATUS_NONFINITE on the instance.
struct K1CArgs : K1Args {
  const uint8_t* enabled;
  const void* dmin;
  const void* ddet;
};
// The arguments of the held-target instantiation (k1h_kernel, k1_warp_tile<..., TR, CO, HO = true>): the bik_track_hold entry
// points, track mode only; the collision members as in K1CArgs, each may be null.  hold [B][T][H], H = F + C + P: byte k of
// row b*T + t is != 0 iff instance b holds task k on frame t (frame-like tasks, then CoM tasks, then posture-type tasks, each
// in the order of its target buffer).  On the first pass of the frame a run of held frames starts on, K1 captures the task's
// value at q in the caller's precision: into held ([B][7F + 3C], frame tasks then CoM tasks) for frame and CoM tasks, into b's
// row of ptcur for posture-type tasks.  Every pass of the run then takes that value as the task's target.  ptcur is set, and
// filled from ptgt on the first pass of every frame that does not hold the task, whatever pbatched says.
struct K1HArgs : K1CArgs {
  const uint8_t* hold;
  void* held;
};
// Task k of instance b on its current frame: 0 not held, 1 held (the target is the held value), 2 held and its run starts on
// this frame, whose first pass this is (capture the value now).  Read before track mode's test moves the cursor on.
BIK_HD int k1h_hold(const K1Args& a, const PHeader& h, int b, int k) {
  const uint8_t* hold = static_cast<const K1HArgs&>(a).hold;
  const long long H = h.F + h.C + h.P, row = (long long)b * a.T + a.cursor[b];
  if (!hold[row * H + k]) return 0;
  return a.tstep[b] == 0 && (a.cursor[b] == 0 || !hold[(row - 1) * H + k]) ? 2 : 1;
}
// The arguments of the placement instantiation (k1p_kernel, k1_warp_tile<..., CO = true, HO, PL = true>): the ..._placed entry
// points; the collision and hold members as in K1CArgs / K1HArgs, each may be null (HO: hold and held set).  placement [B][F][7],
// in the inputs' element type: row b*F + f is the pose (wxyz, xyz) of frame task f's frame in its tree node for instance b, in
// place of the problem's (KC<T>::flpos / flquat), on every frame in track mode.  It is used as given (a quaternion is not
// renormalised); a row with a non-finite element falls back to the problem's and sets BIK_STATUS_NONFINITE on the instance.
// A RELATIVE_FRAME task's root keeps the problem's placement.
struct K1PArgs : K1HArgs {
  const void* placement;
};
// v as the caller's precision holds it (a captured target is stored there, as a target the caller passed would be)
template <typename T> BIK_HD T k1h_round(T v, int is64) { return sizeof(T) == 8 && !is64 ? T(float(v)) : v; }
// row of instance b in the K1CArgs buffers: b, or in track mode that of its current frame
template <bool TR>
BIK_HD long long k1c_row(const K1Args& a, int b) { return TR ? (long long)b * a.T + a.cursor[b] : (long long)b; }
// row `row` of a distance buffer is finite (or the buffer is null)
template <typename T>
BIK_HD bool k1c_finite(const void* buf, long long row, int is64) {
  if (!buf) return true;
  const T v = ldin<T>(buf, row, is64);
  return v - v == T(0);
}
// collision constant k of KC<T>::coll; CO: for k = 1 (minimum distance) and 2 (detection distance) the instance's value in row
// `row` of the K1CArgs buffer instead, where the lane is valid and the buffer gives a finite one
template <typename T, bool CO>
BIK_HD T k1c_coll(const PView& P, const K1Args& a, bool valid, long long row, int k) {
  if constexpr (CO) {
    const K1CArgs& ca = static_cast<const K1CArgs&>(a);
    const void* buf = k == 1 ? ca.dmin : (k == 2 ? ca.ddet : nullptr);
    if (valid && buf && k1c_finite<T>(buf, row, a.in64)) return ldin<T>(buf, row, a.in64);
  }
  return KC<T>::coll(P, k);
}
// the thresholds of the convergence test in the instantiation's precision
template <typename T>
BIK_HD T k1_pos_thr(const K1Args& a) { if constexpr (sizeof(T) == 8) return a.pos_thr64; else return T(a.pos_thr); }
template <typename T>
BIK_HD T k1_ori_thr(const K1Args& a) { if constexpr (sizeof(T) == 8) return a.ori_thr64; else return T(a.ori_thr); }
// first weight of instance b's rows (a.weights set): the instance's row of [B][K], or in track mode that of its current frame
template <bool TR>
BIK_HD long long k1_wbase(const K1Args& a, const PHeader& h, int b) { return (TR ? (long long)b * a.T + a.cursor[b] : (long long)b) * h.K; }
// weight i of a.weights clamped to [0, 1], NaN to 0
template <typename T>
BIK_HD T k1_weight(const K1Args& a, long long i) {
  const T w = ldin<T>(a.weights, i, a.in64);
  return w >= T(0) ? (w <= T(1) ? w : T(1)) : T(0);
}
template <typename T>
BIK_HD V3<T> k1_weight3(const K1Args& a, long long i) { return v3<T>(k1_weight<T>(a, i), k1_weight<T>(a, i + 1), k1_weight<T>(a, i + 2)); }
// the convergence test skips a frame task's position (orientation) error when all three of its weights are 0
template <typename T>
BIK_HD bool k1_tested(const K1Args& a, long long i) { return !a.weights || k1_weight<T>(a, i) > T(0) || k1_weight<T>(a, i + 1) > T(0) || k1_weight<T>(a, i + 2) > T(0); }
template <typename T> BIK_HD V3<T> vmul(V3<T> a, V3<T> b) { return v3<T>(a.x * b.x, a.y * b.y, a.z * b.z); }

// ---- per-warp scratch layout (elements of T) --------------------------------------------------
BIK_HD int k1_state_stride(const PHeader& h) {  // pose (7) + CoM first moment (3) per node, odd stride
  int s = 7 * h.nslots + (h.C > 0 ? 3 * h.nnode : 0);
  return s | 1;
}
BIK_HD int k1_state_words(const PHeader& h, int ipw) { return (ipw * k1_state_stride(h) + 3) & ~3; }  // keeps the stage 16-byte aligned
BIK_HD int k1_fsc_stride(const PHeader& h) { return h.nrel > 0 ? 32 : 24; }
// Frame-task rows go straight to global memory when J holds nothing else (k1_frames_direct); the staging tile (6 rows
// per instance) is only needed for CoM rows, collision rows, and frame rows that share a dense J with CoM rows.
BIK_HD bool k1_frames_direct(const PHeader& h) { return h.C == 0; }
BIK_HD int k1_stage_words(const PHeader& h, int ipw) {
  if (k1_frames_direct(h) && h.npairs == 0) return 0;
  return (ipw * 6 * h.nv + 3) & ~3;
}
BIK_HD int k1_tgt_words(const PHeader& h) { return 7 * h.F + 3 * h.C; }   // frame + CoM targets of one instance
BIK_HD int k1_e_words(const PHeader& h, int ipw) { return (ipw * (h.K > 0 ? h.K : 1) + 3) & ~3; }
BIK_HD int k1_qtile_offset(const PHeader& h, int ipw) {   // where the tile's inputs (q rows, then targets) sit in the warp's scratch (16-byte aligned)
  return k1_state_words(h, ipw) + k1_stage_words(h, ipw) + k1_e_words(h, ipw) + ipw * (h.F > 0 ? h.F : 1) * k1_fsc_stride(h);
}
BIK_HD int k1_warp_words(const PHeader& h, int ipw) {
  int w = k1_qtile_offset(h, ipw) + ((ipw * h.nq + 3) & ~3) + ((ipw * k1_tgt_words(h) + 3) & ~3) + ((ipw + 3) & ~3);
  return (w + 3) & ~3;
}

// Per-warp input pipeline (device): the q rows and the targets of a tile are contiguous runs of global memory, so the NEXT
// tile's travel into shared memory as 1-D bulk async copies (cp.async.bulk + mbarrier) while the current tile computes its
// Jacobian columns -- the inputs are dead by then.  `armed` is the first instance of the tile whose copies are in flight or
// have landed (-1: none; the tile then loads its inputs itself).
struct K1Pipe {
  uint64_t* bar;
  uint32_t phase;
  int armed;
};
// Bulk copies need 16-byte sizes and addresses, and the buffers must hold the kernel's scalar type (fp32 kernel, fp32 inputs).
// TR (track mode): only the q rows travel this way; a tile's targets are rows of different frames, loaded per instance.
template <typename T, bool TR = false>
BIK_HD bool k1_tile_bulk_ok(const PHeader& h, const K1Args& a, int inst0, int ipw) {
  if (sizeof(T) != 4 || a.in64 || inst0 < 0 || inst0 >= a.B) return false;
  const int nvalid = (a.B - inst0) < ipw ? (a.B - inst0) : ipw;
  const size_t qb = (size_t)nvalid * h.nq * 4, fb = (size_t)nvalid * h.F * 7 * 4, cb = (size_t)nvalid * h.C * 3 * 4;
  const size_t qa = reinterpret_cast<size_t>(a.q) + (size_t)inst0 * h.nq * 4, fa = reinterpret_cast<size_t>(a.ftgt) + (size_t)inst0 * h.F * 7 * 4,
               ca = reinterpret_cast<size_t>(a.ctgt) + (size_t)inst0 * h.C * 3 * 4;
  if ((qb | qa) & 15) return false;
  if (TR) return true;
  if (h.F > 0 && ((fb | fa | ((size_t)ipw * h.F * 7 * 4)) & 15)) return false;   // (the CoM targets sit behind a full tile of frame targets)
  if (h.C > 0 && ((cb | ca) & 15)) return false;
  return true;
}
#if defined(__CUDACC__)
// lane 0 of the warp: arm the barrier with the byte count and issue the copies of the tile starting at inst0
template <typename T, bool TR = false>
__device__ __forceinline__ void k1_pipe_arm(const PHeader& h, const K1Args& a, int inst0, int ipw, K1Pipe* pipe, T* qtile, T* ttile) {
  const int nvalid = (a.B - inst0) < ipw ? (a.B - inst0) : ipw;
  const uint32_t qb = (uint32_t)nvalid * h.nq * 4, fb = TR ? 0u : (uint32_t)nvalid * h.F * 7 * 4, cb = TR ? 0u : (uint32_t)nvalid * h.C * 3 * 4;
  mbar_expect_tx(pipe->bar, qb + fb + cb);
  bulk_g2s(qtile, reinterpret_cast<const float*>(a.q) + (size_t)inst0 * h.nq, qb, pipe->bar);
  if (fb) bulk_g2s(ttile, reinterpret_cast<const float*>(a.ftgt) + (size_t)inst0 * h.F * 7, fb, pipe->bar);
  if (cb) bulk_g2s(ttile + ipw * h.F * 7, reinterpret_cast<const float*>(a.ctgt) + (size_t)inst0 * h.C * 3, cb, pipe->bar);
}
#endif

template <typename T> BIK_HD Q4<T> ld_q(const T* p) { return q4<T>(p[0], p[1], p[2], p[3]); }
template <typename T> BIK_HD V3<T> ld_v(const T* p) { return v3<T>(p[0], p[1], p[2]); }
template <typename T> BIK_HD V3<T> unit_axis(int c) { return v3<T>(c == 0 ? T(1) : T(0), c == 1 ? T(1) : T(0), c == 2 ? T(1) : T(0)); }

// One node of the tree: pose of the node frame after its joint (mj_kinematics, one joint per node).
template <typename T>
BIK_HD void fk_node(const PView& P, int n, const T* q, T* xs) {
  const NodeRec& r = P.node(n);
  Q4<T> quat;
  V3<T> pos;
  if (r.type == JNT_FREE) {
    pos = ld_v(q + r.qadr);
    quat = ld_q(q + r.qadr + 3);
  } else {
    if (r.parent >= 0) {
      Q4<T> pq = ld_q(xs + 7 * r.pslot);
      pos = ld_v(xs + 7 * r.pslot + 4) + qrot(pq, KC<T>::npos(P, n, r));
      quat = qmul(pq, KC<T>::nquat(P, n, r));
    } else {
      pos = KC<T>::npos(P, n, r);
      quat = KC<T>::nquat(P, n, r);
    }
    if (r.type == JNT_SLIDE) {
      pos = pos + (q[r.qadr] - KC<T>::qpos0(P, r.qadr)) * qrot(quat, KC<T>::naxis(P, n, r));
    } else {
      V3<T> jp = KC<T>::njpos(P, n, r);
      bool off_centre = (jp.x != T(0)) || (jp.y != T(0)) || (jp.z != T(0));
      V3<T> anchor = pos;
      if (off_centre) anchor = pos + qrot(quat, jp);
      Q4<T> ql;
      if (r.type == JNT_HINGE) {
        T s, c;
        bik_sincos<T>(T(0.5) * (q[r.qadr] - KC<T>::qpos0(P, r.qadr)), &s, &c);
        V3<T> ax = KC<T>::naxis(P, n, r);
        ql = q4<T>(c, s * ax.x, s * ax.y, s * ax.z);
      } else {
        ql = qnormalize(ld_q(q + r.qadr));
      }
      quat = qmul(quat, ql);
      if (off_centre) pos = anchor - qrot(quat, jp);
    }
  }
  // mj_kinematics renormalises every body quaternion.  A product of unit quaternions leaves the unit sphere by ~1e-7
  // per level in fp32 (1e-6 at the deepest node of the BASELINE robots, against a 1e-4 parity budget), so the fp32
  // instantiation only renormalises quaternions that come straight from q (free / ball joints: callers may pass them
  // unnormalised); the fp64 instantiation follows the reference literally.
  if (sizeof(T) == 8 || r.type == JNT_FREE) quat = qnormalize(quat);
  T* o = xs + 7 * r.slot;
  o[0] = quat.w; o[1] = quat.x; o[2] = quat.y; o[3] = quat.z; o[4] = pos.x; o[5] = pos.y; o[6] = pos.z;
}

// `node` is the STATE ROW of the frame's node (FrameRec::slot; the node id itself where slots are the identity), -1 = world
template <typename T>
BIK_HD void frame_pose(int node, V3<T> lpos, Q4<T> lquat, const T* xs, Q4<T>* qf, V3<T>* pf) {
  if (node < 0) { *qf = lquat; *pf = lpos; return; }
  Q4<T> nq = ld_q(xs + 7 * node);
  *qf = qnormalize(qmul(nq, lquat));
  *pf = ld_v(xs + 7 * node + 4) + qrot(nq, lpos);
}
// frame_pose of frame task f's frame (tree state row `slot`) for instance b of a K1PArgs call: at the instance's placement row
// where all seven values are finite, else at the problem's
template <typename T>
BIK_HD void k1p_frame_pose(const PView& P, const K1Args& a, int b, int f, int slot, const T* xs, Q4<T>* qf, V3<T>* pf) {
  const long long r = ((long long)b * P.h().F + f) * 7;
  const void* pl = static_cast<const K1PArgs&>(a).placement;
  T v[7];
  bool fin = true;
  for (int k = 0; k < 7; ++k) { v[k] = ldin<T>(pl, r + k, a.in64); fin = fin && v[k] - v[k] == T(0); }
  if (fin) frame_pose<T>(slot, v3<T>(v[4], v[5], v[6]), q4<T>(v[0], v[1], v[2], v[3]), xs, qf, pf);
  else frame_pose<T>(slot, KC<T>::flpos(P, f), KC<T>::flquat(P, f), xs, qf, pf);
}
// root^-1 * frame for two world poses as bik_fk reports them, composed as mink's SE3 does (root.inverse() @ frame): the pose a
// held RELATIVE_FRAME task captures (RelativeFrameTask.set_target_from_configuration)
template <typename T>
BIK_HD void held_relative(Q4<T> qr, V3<T> pr, Q4<T> qf, V3<T> pf, Q4<T>* q, V3<T>* p) {
  const Q4<T> r = qconj(qr);
  *q = qmul(r, qf);
  *p = qrot(r, pf) - qrot(r, pr);
}
// The pose a held frame task captures from the frame's world pose (qf, pf) and, for a RELATIVE_FRAME, its root's (qr, pr), as
// frame_pose gives them: the world pose as bik_fk reports it (FrameTask.set_target_from_configuration), or held_relative.
template <typename T>
BIK_HD void held_frame_value(bool relative, Q4<T> qf, V3<T> pf, Q4<T> qr, V3<T> pr, Q4<T>* q, V3<T>* p) {
  *q = mat2quat(q2mat(qf)); *p = pf;
  if (relative) held_relative<T>(mat2quat(q2mat(qr)), pr, *q, pf, q, p);
}
// The model's CoM at the node poses xs (mj_comPos's subtree_com of body 1), summed as bik_fk sums it (fk_warp_tile), over the
// nodes with mass below them: K1 does not pose the others, whose terms in bik_fk's sum are exact zeros.
template <typename T>
BIK_HD V3<T> model_com(const PView& P, const T* xs) {
  const PHeader& h = P.h();
  V3<T> tot = KC<T>::com_fixed(P);
  for (int n = 0; n < h.nnode; ++n) {
    if (!(KC<T>::sub_m(P, n) > T(0))) continue;
    tot = tot + KC<T>::own_m(P, n) * ld_v(xs + 7 * n + 4) + qrot(ld_q(xs + 7 * n), KC<T>::own_c(P, n));
  }
  T M = KC<T>::com_mass(P);
  T invM = M > T(0) ? T(1) / M : T(0);
  return v3<T>(tot.x * invM, tot.y * invM, tot.z * invM);
}

// World-aligned point-Jacobian column of dof `d` (owned by node n) for a point p moving with a
// descendant of n: jp = linear part, jr = angular part (mj_jac restated per column).
template <typename T>
BIK_HD void jac_column(const PView& P, int d, int n, const T* xs, V3<T> p, V3<T>* jp, V3<T>* jr) {
  const NodeRec& r = P.node(n);
  Q4<T> nq = ld_q(xs + 7 * r.slot);
  V3<T> np = ld_v(xs + 7 * r.slot + 4);
  int k = d - r.dadr;
  if (r.type == JNT_HINGE) {
    V3<T> ax = qrot(nq, KC<T>::naxis(P, n, r));
    V3<T> anchor = np + qrot(nq, KC<T>::njpos(P, n, r));
    *jr = ax; *jp = cross(ax, p - anchor);
  } else if (r.type == JNT_SLIDE) {
    *jr = v3<T>(T(0), T(0), T(0)); *jp = qrot(nq, KC<T>::naxis(P, n, r));
  } else if (r.type == JNT_FREE && k < 3) {
    *jr = v3<T>(T(0), T(0), T(0)); *jp = unit_axis<T>(k);
  } else {  // rotational dof of a free or ball joint: body-frame axis k
    int c = (r.type == JNT_FREE) ? k - 3 : k;
    V3<T> ax = qrot(nq, unit_axis<T>(c));
    V3<T> anchor = (r.type == JNT_FREE) ? np : np + qrot(nq, KC<T>::njpos(P, n, r));
    *jr = ax; *jp = cross(ax, p - anchor);
  }
}

// FrameTask error and the two 3x3 blocks that map world-aligned (jp, jr) columns to task-Jacobian
// columns:  J[:,d] = [A1 jp + A2 jr ; A1 jr]   with A1 = -Ji R^T, A2 = -Mi R^T.
template <typename T>
BIK_HD void frame_task(Q4<T> qf, V3<T> pf, Q4<T> tq, V3<T> tp, V3<T>* ev, V3<T>* ew, M3<T>* A1, M3<T>* A2) {
  tq = qnormalize(tq);
  // e = log(T_wb^-1 T_wt)                                (frame_task.py:119-122)
  se3_log<T>(qmul(qconj(qf), tq), qrot_inv(qf, tp - pf), ev, ew);
  // jlog(T_wt^-1 T_wb) = ljacinv(-log(T_tb))            (frame_task.py:145-146, lie/base.py:151-156)
  // and log(T_tb) = log(T_bt^-1) = -e, so the argument of ljacinv is e itself: no second logarithm.
  M3<T> Ji, Mi;
  se3_ljacinv_blocks<T>(*ev, *ew, &Ji, &Mi);
  M3<T> Rt = mtrans(q2mat(qf));
  *A1 = mmul(Ji, Rt);
  *A2 = mmul(Mi, Rt);
  for (int i = 0; i < 9; ++i) { A1->m[i] = -A1->m[i]; A2->m[i] = -A2->m[i]; }
}

// RelativeFrameTask (reference mink/tasks/relative_frame_task.py:106-142): pose of frame f in root r,
//   e = log(T_rt^-1 T_rf),   J = jlog(T_tf) (J_f - Ad(T_rf^-1) J_r),   T_tf = T_rt^-1 T_rf.
// Returns e and the blocks (Ji, Mi) of jlog(T_tf) = ljacinv(-log T_tf).
template <typename T>
BIK_HD void relative_frame_task(Q4<T> qf, V3<T> pf, Q4<T> qr, V3<T> pr, Q4<T> tq, V3<T> tp, V3<T>* ev, V3<T>* ew, M3<T>* Ji, M3<T>* Mi) {
  Q4<T> q_rf = qmul(qconj(qr), qf);
  V3<T> t_rf = qrot_inv(qr, pf - pr);
  tq = qnormalize(tq);
  se3_log<T>(qmul(qconj(tq), q_rf), qrot_inv(tq, t_rf - tp), ev, ew);
  se3_ljacinv_blocks<T>(v3<T>(-ev->x, -ev->y, -ev->z), v3<T>(-ew->x, -ew->y, -ew->z), Ji, Mi);
}

// Posture error of dof d:  e = q* (-) q with free-joint dofs zeroed (posture_task.py:107-118, mj_differentiatePos).
// tg(i) / qq(i) return element i of the posture target / of q as T.
template <typename T, typename FT, typename FQ>
BIK_HD T posture_err_dof(const PView& P, int d, FT tg, FQ qq) {
  const PHeader& h = P.h();
  const int qa = P.i(h.off_dofqadr)[d];
  if (qa >= 0) return tg(qa) - qq(qa);
  const NodeRec& r = P.node(P.i(h.off_dofnode)[d]);
  if (r.type != JNT_BALL) return T(0);
  V3<T> w = quat_sub<T>(qnormalize(q4<T>(tg(r.qadr), tg(r.qadr + 1), tg(r.qadr + 2), tg(r.qadr + 3))),
                        qnormalize(q4<T>(qq(r.qadr), qq(r.qadr + 1), qq(r.qadr + 2), qq(r.qadr + 3))));
  const int c = d - r.dadr;
  return c == 0 ? w.x : (c == 1 ? w.y : w.z);
}

// ---- primitive geom distance (plane / sphere / capsule / box) ------------------------------
template <typename T>
BIK_HD void seg_closest(V3<T> p1, V3<T> d1, V3<T> p2, V3<T> d2, V3<T>* a, V3<T>* b) {
  V3<T> r = p1 - p2;
  T A = dot(d1, d1), E = dot(d2, d2), Bq = dot(d1, d2), C = dot(d1, r), F = dot(d2, r);
  T den = A * E - Bq * Bq, s = T(0), t = T(0);
  const T tiny = sizeof(T) == 8 ? T(1e-24) : T(1e-12);
  if (den > tiny) s = bik_min(bik_max((Bq * F - C * E) / den, T(-1)), T(1));
  if (E > tiny) t = (Bq * s + F) / E;
  if (t < T(-1) || t > T(1)) {
    t = t < T(-1) ? T(-1) : T(1);
    s = (A > tiny) ? bik_min(bik_max((Bq * t - C) / A, T(-1)), T(1)) : T(0);
  }
  *a = p1 + s * d1; *b = p2 + t * d2;
}
// Parameter t in [-1, 1] of the point of the segment c + t d nearest to the box |x_k| <= s_k (everything in the box frame).
// f(t) = sum_k max(|c_k + t d_k| - s_k, 0)^2 is convex and C1 with a piecewise-linear derivative: bisect f' and finish with
// one secant step, which lands on the root of the linear piece the bracket has shrunk into.
template <typename T>
BIK_HD T seg_box_slope(V3<T> c, V3<T> d, V3<T> s, T t) {
  const T px = c.x + t * d.x, py = c.y + t * d.y, pz = c.z + t * d.z;
  const T ex = px > s.x ? px - s.x : (px < -s.x ? px + s.x : T(0));
  const T ey = py > s.y ? py - s.y : (py < -s.y ? py + s.y : T(0));
  const T ez = pz > s.z ? pz - s.z : (pz < -s.z ? pz + s.z : T(0));
  return d.x * ex + d.y * ey + d.z * ez;
}
// If the segment passes through the box the distance is zero on a whole interval of t: take the middle of the part inside
// (slab clipping), so that the penetrating branch of the caller sees one well-defined core point.
template <typename T>
BIK_HD bool seg_box_clip(T c, T d, T s, T* t0, T* t1) {
  if (d == T(0)) return c >= -s && c <= s;
  T a = (-s - c) / d, b = (s - c) / d;
  if (a > b) { T x = a; a = b; b = x; }
  *t0 = bik_max(*t0, a); *t1 = bik_min(*t1, b);
  return *t0 <= *t1;
}
template <typename T>
BIK_HD T seg_box_param(V3<T> c, V3<T> d, V3<T> s) {
  T t0 = T(-1), t1 = T(1);
  if (seg_box_clip<T>(c.x, d.x, s.x, &t0, &t1) && seg_box_clip<T>(c.y, d.y, s.y, &t0, &t1) && seg_box_clip<T>(c.z, d.z, s.z, &t0, &t1))
    return T(0.5) * (t0 + t1);
  T lo = T(-1), hi = T(1);
  T flo = seg_box_slope<T>(c, d, s, lo), fhi = seg_box_slope<T>(c, d, s, hi);
  if (flo >= T(0)) return lo;
  if (fhi <= T(0)) return hi;
  const int iters = sizeof(T) == 8 ? 48 : 22;
  for (int it = 0; it < iters; ++it) {
    T mid = T(0.5) * (lo + hi), fm = seg_box_slope<T>(c, d, s, mid);
    if (fm == T(0)) return mid;
    if (fm < T(0)) { lo = mid; flo = fm; } else { hi = mid; fhi = fm; }
  }
  return lo + (hi - lo) * (-flo / (fhi - flo));
}
template <typename T>
BIK_HD T geom_distance(const PView& P, int i1, int i2, const T* xs, T distmax, V3<T>* on1, V3<T>* on2) {
  int ia = i1, ib = i2;
  bool swap = false;
  // canonical order: a plane first, else a box first (plane-plane and box-box pairs are refused when the problem is built)
  if (P.geom(i2).type == 0 || (P.geom(i2).type == 6 && P.geom(i1).type != 0)) { ia = i2; ib = i1; swap = true; }
  const GeomRec& A = P.geom(ia); const GeomRec& Bg = P.geom(ib);
  Q4<T> qa, qb; V3<T> pa, pb;
  frame_pose<T>(A.node, KC<T>::glpos(P, ia), KC<T>::glquat(P, ia), xs, &qa, &pa);
  frame_pose<T>(Bg.node, KC<T>::glpos(P, ib), KC<T>::glquat(P, ib), xs, &qb, &pb);
  const T ra = KC<T>::gsize(P, ia, 0), rb = KC<T>::gsize(P, ib, 0), ha = KC<T>::gsize(P, ia, 1), hb = KC<T>::gsize(P, ib, 1);
  V3<T> oa, ob; T dist;
  V3<T> zb = qrot(qb, unit_axis<T>(2));
  if (A.type == 0 && Bg.type == 6) {  // plane vs box: the lowest corner
    V3<T> n = qrot(qa, unit_axis<T>(2));
    V3<T> end = pb;
    for (int k = 0; k < 3; ++k) {
      V3<T> ax = KC<T>::gsize(P, ib, k) * qrot(qb, unit_axis<T>(k));
      end = dot(ax, n) >= T(0) ? end - ax : end + ax;
    }
    T hgt = dot(end - pa, n);
    dist = hgt;
    ob = end; oa = end - hgt * n;
  } else if (A.type == 0) {  // plane vs sphere/capsule
    V3<T> n = qrot(qa, unit_axis<T>(2));
    V3<T> end = pb;
    if (Bg.type == 3) {
      V3<T> e1 = pb + hb * zb, e2 = pb - hb * zb;
      end = dot(e1 - pa, n) <= dot(e2 - pa, n) ? e1 : e2;
    }
    T hgt = dot(end - pa, n);
    dist = hgt - rb;
    ob = end - rb * n; oa = end - hgt * n;
  } else if (A.type == 6) {  // box vs sphere/capsule: nearest point of the core segment, in the box frame
    const V3<T> s = v3<T>(ra, ha, KC<T>::gsize(P, ia, 2));
    const V3<T> c = qrot_inv(qa, pb - pa);
    const V3<T> d = Bg.type == 3 ? hb * qrot_inv(qa, zb) : v3<T>(T(0), T(0), T(0));
    const T t = Bg.type == 3 ? seg_box_param<T>(c, d, s) : T(0);
    const V3<T> p = c + t * d;
    V3<T> qc = v3<T>(bik_min(bik_max(p.x, -s.x), s.x), bik_min(bik_max(p.y, -s.y), s.y), bik_min(bik_max(p.z, -s.z), s.z));
    V3<T> v = p - qc, nl;
    T L = bik_sqrt<T>(dot(v, v));
    if (L > T(1e-15)) {
      nl = (T(1) / L) * v;
    } else {  // the core point is inside the box: leave through the nearest face (depth is signed, L < 0)
      const T gx = s.x - (p.x < T(0) ? -p.x : p.x), gy = s.y - (p.y < T(0) ? -p.y : p.y), gz = s.z - (p.z < T(0) ? -p.z : p.z);
      nl = v3<T>(T(0), T(0), T(0));
      if (gx <= gy && gx <= gz) { nl.x = p.x < T(0) ? T(-1) : T(1); L = -gx; }
      else if (gy <= gz) { nl.y = p.y < T(0) ? T(-1) : T(1); L = -gy; }
      else { nl.z = p.z < T(0) ? T(-1) : T(1); L = -gz; }
      qc = p - L * nl;
    }
    dist = L - rb;
    oa = pa + qrot(qa, qc); ob = pa + qrot(qa, p - rb * nl);
  } else {
    V3<T> d1 = v3<T>(T(0), T(0), T(0)), d2 = d1, a, b;
    if (A.type == 3) d1 = ha * qrot(qa, unit_axis<T>(2));
    if (Bg.type == 3) d2 = hb * zb;
    seg_closest<T>(pa, d1, pb, d2, &a, &b);
    V3<T> v = b - a;
    T L = bik_sqrt<T>(dot(v, v));
    V3<T> nr = L > T(1e-15) ? (T(1) / L) * v : v3<T>(T(1), T(0), T(0));
    dist = L - ra - rb;
    oa = a + ra * nr; ob = b - rb * nr;
  }
  if (dist >= distmax) return distmax;
  if (swap) { *on1 = ob; *on2 = oa; } else { *on1 = oa; *on2 = ob; }
  return dist;
}

// ---- staging flush: IPW x (R*nv) elements -> global rows [inst][row0 .. row0+R) ----------------
template <int W, typename T>
BIK_HD void flush_rows(const T* stage, int chunk, int nvalid, T* out, long long inst_stride, int lane) {
  const bool vec2 = sizeof(T) == 4 && ((chunk | (int)(inst_stride & 1)) & 1) == 0 && ((reinterpret_cast<size_t>(out) | reinterpret_cast<size_t>(stage)) & 7) == 0;
  if (vec2) {  // 8-byte stores: every run starts on an 8-byte boundary
    const int c2 = chunk >> 1;
    for (int li = 0; li < nvalid; ++li) {
      F2* o = reinterpret_cast<F2*>(out + li * inst_stride);
      const F2* s = reinterpret_cast<const F2*>(stage + li * chunk);
      for (int k = lane; k < c2; k += W) o[k] = s[k];
    }
    return;
  }
  for (int li = 0; li < nvalid; ++li) {
    T* o = out + li * inst_stride;
    const T* s = stage + li * chunk;
    for (int k = lane; k < chunk; k += W) o[k] = s[k];
  }
}
template <int W, typename T>
BIK_HD void zero_words(T* p, int count, int lane) {  // 16-byte stores where p is 16-byte aligned
  constexpr int V = 16 / (int)sizeof(T);
  if ((reinterpret_cast<size_t>(p) & 15) == 0) {
    F4* p4 = reinterpret_cast<F4*>(p);
    const int c4 = count / V;
    const F4 z = {0.f, 0.f, 0.f, 0.f};
    for (int k = lane; k < c4; k += W) p4[k] = z;
    for (int k = c4 * V + lane; k < count; k += W) p[k] = T(0);
  } else {
    for (int k = lane; k < count; k += W) p[k] = T(0);
  }
}
// six consecutive elements (one packed Jacobian column), destination 8-byte (fp32) / 16-byte (fp64) aligned
template <typename T> BIK_HD void store6(T* o, V3<T> top, V3<T> bot);
template <> BIK_HD void store6<float>(float* o, V3<float> top, V3<float> bot) {
  F2* o2 = reinterpret_cast<F2*>(o);
  o2[0] = F2{top.x, top.y}; o2[1] = F2{top.z, bot.x}; o2[2] = F2{bot.y, bot.z};
}
template <> BIK_HD void store6<double>(double* o, V3<double> top, V3<double> bot) {
  D2* o2 = reinterpret_cast<D2*>(o);
  o2[0] = D2{top.x, top.y}; o2[1] = D2{top.z, bot.x}; o2[2] = D2{bot.y, bot.z};
}

// One warp tile: instances [inst0, inst0 + IPW) clipped to B.
// PK (compile time): packed hand-off with the fused check_limits / convergence test (bik_step, bik_converge), else the dense
// API form (bik_fk_jac) -- two instantiations so that neither carries the other's registers and code.
// TR (compile time, with PK): track mode of bik_track (see K1Args); a third instantiation, so the other two are unchanged.
// CO (compile time, with PK): `a` is a K1CArgs, per-instance collision pairs and distances (the ..._coll entry points).
// HO (compile time, with TR): `a` is a K1HArgs, held targets (the bik_track_hold entry points).
// PL (compile time, with CO): `a` is a K1PArgs, per-instance frame placement (the ..._placed entry points).
template <typename T, int G, int W, bool PK, bool TR = false, bool CO = false, bool HO = false, bool PL = false>
BIK_HD void k1_warp_tile(const PView& P, const K1Args& a, int inst0, T* wsm, int lane, K1Pipe* pipe = nullptr, int next_inst0 = -1) {
  static_assert(!TR || PK, "track mode writes the packed hand-off");
  static_assert(!CO || PK, "per-instance collision pairs write the packed hand-off");
  static_assert(!HO || TR, "held targets are a track-mode feature");
  static_assert(!PL || CO, "frame placement runs with the collision arguments");
  const PHeader& h = P.h();
  constexpr int IPW = W / G;
  const int nv = h.nv, nq = h.nq, K = h.K;
  const int li = lane / G, g = lane % G;
  const int b = inst0 + li;
  const int nvalid = (a.B - inst0) < IPW ? (a.B - inst0) : IPW;
  const bool valid = li < nvalid && (!TR || a.tstep[b] >= 0);   // track mode: an instance without frames left does no work
  long long crow = 0;   // CO: the instance's row of the K1CArgs buffers, taken before track mode's test moves the cursor on
  if constexpr (CO) crow = valid ? k1c_row<TR>(a, b) : 0;
  const int SS = k1_state_stride(h);
  constexpr bool packed = PK;
  const long long PKS = h.pk_stride;
  T* const Jg = reinterpret_cast<T*>(a.J);
  T* const pkg = reinterpret_cast<T*>(a.pk);
  T* state = wsm;
  T* stage = wsm + k1_state_words(h, IPW);
  T* estage = stage + k1_stage_words(h, IPW);
  T* fsc = estage + k1_e_words(h, IPW);     // per (instance, frame): per-frame SE(3) results
  const int FS = k1_fsc_stride(h);
  T* qtile = wsm + k1_qtile_offset(h, IPW);          // q of this tile: one contiguous, coalesced run of global memory
  T* ttile = qtile + ((IPW * nq + 3) & ~3);         // targets of this tile: [IPW][F][7] frame targets, then [IPW][C][3] CoM targets
  int32_t* sflag = reinterpret_cast<int32_t*>(ttile + ((IPW * k1_tgt_words(h) + 3) & ~3));   // check_limits bits per instance
  T* xs = state + li * SS;
  const bool direct = !packed && k1_frames_direct(h);
  {
    bool landed = false;
#if defined(__CUDA_ARCH__)
    if (pipe && pipe->armed == inst0) {   // this tile's inputs were sent ahead by the previous tile (or the kernel prologue)
      mbar_wait(pipe->bar, pipe->phase);
      pipe->phase ^= 1u;
      pipe->armed = -1;
      landed = true;
    }
#endif
    if (!landed) {
      const long long q0 = (long long)inst0 * nq, f0 = (long long)inst0 * h.F * 7, c0 = (long long)inst0 * h.C * 3;
      for (int k = lane; k < nvalid * nq; k += W) qtile[k] = ldin<T>(a.q, q0 + k, a.in64);
      if (!TR) {
        for (int k = lane; k < nvalid * h.F * 7; k += W) ttile[k] = ldin<T>(a.ftgt, f0 + k, a.in64);
        for (int k = lane; k < nvalid * h.C * 3; k += W) ttile[IPW * h.F * 7 + k] = ldin<T>(a.ctgt, c0 + k, a.in64);
      }
    }
    if (TR) {   // the targets of each instance's current frame: row b*T + cursor[b] of the [B][T] sequences
      const int FW = h.F * 7, CW = h.C * 3;
      for (int i = 0; i < nvalid; ++i) {
        if (a.tstep[inst0 + i] < 0) continue;
        const long long row = (long long)(inst0 + i) * a.T + a.cursor[inst0 + i];
        for (int k = lane; k < FW; k += W) ttile[i * FW + k] = ldin<T>(a.ftgt, row * FW + k, a.in64);
        for (int k = lane; k < CW; k += W) ttile[IPW * FW + i * CW + k] = ldin<T>(a.ctgt, row * CW + k, a.in64);
      }
    }
    if constexpr (HO) {   // first pass of a frame: each posture-type task's row of ptcur, which this pass's K2 reads
      const int PW = h.P * nq;
      for (int i = 0; i < nvalid; ++i) {
        const int bi = inst0 + i;
        if (a.tstep[bi] != 0) continue;
        const long long r0 = a.pbatched == 3 ? (long long)bi * a.T + a.cursor[bi] : (a.pbatched == 2 ? a.cursor[bi] : (a.pbatched == 1 ? bi : 0));
        for (int p = 0; p < h.P; ++p) {
          const int s = k1h_hold(a, h, bi, h.F + h.C + p);
          if (s == 1) continue;   // held since an earlier frame: the captured q stays
          // the run starts here: q itself; not held: the frame's row of the posture targets
          const void* src = s == 2 ? a.q : a.ptgt;
          const long long so = s == 2 ? (long long)bi * nq : (r0 * h.P + p) * nq, dst = (long long)bi * PW + (long long)p * nq;
          if constexpr (sizeof(T) == 8) {
            if (a.in64)
              for (int k = lane; k < nq; k += W) static_cast<double*>(a.ptcur)[dst + k] = static_cast<const double*>(src)[so + k];
          }
          if (sizeof(T) == 4 || !a.in64)
            for (int k = lane; k < nq; k += W) static_cast<float*>(a.ptcur)[dst + k] = static_cast<const float*>(src)[so + k];
        }
      }
    } else if constexpr (TR) {   // first pass of a frame: its posture rows become the instance's row of ptcur, which this pass's K2 reads
      if (a.ptcur) {
        const int PW = h.P * nq;
        for (int i = 0; i < nvalid; ++i) {
          const int bi = inst0 + i;
          if (a.tstep[bi] != 0) continue;
          const long long src = ((a.pbatched == 3 ? (long long)bi * a.T : 0) + a.cursor[bi]) * PW, dst = (long long)bi * PW;
          // (as for q_traj below: the fp32 instantiations only ever copy fp32 rows)
          if constexpr (sizeof(T) == 8) {
            if (a.in64)
              for (int k = lane; k < PW; k += W) static_cast<double*>(a.ptcur)[dst + k] = static_cast<const double*>(a.ptgt)[src + k];
          }
          if (sizeof(T) == 4 || !a.in64)
            for (int k = lane; k < PW; k += W) static_cast<float*>(a.ptcur)[dst + k] = static_cast<const float*>(a.ptgt)[src + k];
        }
      }
    }
    if (PK && a.status && lane < IPW) sflag[lane] = 0;
  }
  BIK_SYNCWARP();
  const T* qb = qtile + (valid ? li : 0) * nq;

  // ---- Configuration.check_limits (configuration.py:77-110), fused: every lane tests a few dofs of the tile ----
  // inside bik_converge the step index lives on the device (the loop may be a CUDA-graph WHILE node: no host in between)
  // (track mode: the same rules with each instance's own step index)
  const int conv_step = (PK && !TR && a.done) ? *a.conv_it : 0;
  const bool do_check = PK && a.status && !(!TR && a.done && conv_step >= a.conv_max);
  const bool accumulate = a.done ? conv_step > 0 : a.accumulate != 0;
  if (do_check) {
    const int32_t* dofqadr = P.i(h.off_dofqadr);
    const float* rng = P.f(h.off_range);
    for (int i = 0; i < nvalid; ++i) {
      if (TR) { const int s = a.tstep[inst0 + i]; if (s < 0 || s >= a.conv_max) continue; }
      int bad = 0;
      for (int d = lane; d < nv; d += W) {
        const int qa = dofqadr[d];
        if (qa < 0) continue;
        const T v = qtile[i * nq + qa];
        if (v < T(rng[d]) - T(a.tol) || v > T(rng[nv + d]) + T(a.tol)) bad |= 1;
        if (!(v == v)) bad |= 4;
      }
      if (a.weights) {   // weights outside [0, 1] or NaN: BIK_STATUS_BAD_WEIGHT (they are clamped where they are applied)
        const long long w0 = k1_wbase<TR>(a, h, inst0 + i);
        for (int k = lane; k < K; k += W) {
          const T w = ldin<T>(a.weights, w0 + k, a.in64);
          if (!(w >= T(0) && w <= T(1))) bad |= 32;
        }
      }
      if constexpr (CO) {   // a non-finite collision distance: BIK_STATUS_NONFINITE (the problem's value is used)
        const K1CArgs& ca = static_cast<const K1CArgs&>(a);
        if (lane == 0) {
          const long long r = k1c_row<TR>(a, inst0 + i);
          if (!k1c_finite<T>(ca.dmin, r, a.in64) || !k1c_finite<T>(ca.ddet, r, a.in64)) bad |= 4;
        }
      }
      if constexpr (PL) {   // a non-finite placement: BIK_STATUS_NONFINITE (the problem's placement is used)
        const void* pl = static_cast<const K1PArgs&>(a).placement;
        const long long r0 = (long long)(inst0 + i) * h.F * 7;
        for (int k = lane; k < h.F * 7; k += W) {
          const T v = ldin<T>(pl, r0 + k, a.in64);
          if (!(v - v == T(0))) bad |= 4;
        }
      }
      if (bad) {
#if defined(__CUDA_ARCH__)
        atomicOr(&sflag[i], bad);
#else
        sflag[i] |= bad;
#endif
      }
    }
    BIK_SYNCWARP();
    if (TR) {
      const int s = lane < nvalid ? a.tstep[inst0 + lane] : -1;
      if (s >= 0 && s < a.conv_max) a.status[inst0 + lane] = s > 0 ? (a.status[inst0 + lane] | sflag[lane]) : sflag[lane];
    } else if (lane < nvalid) {
      a.status[inst0 + lane] = accumulate ? (a.status[inst0 + lane] | sflag[lane]) : sflag[lane];
    }
  }

  // ---- forward kinematics over the lane program --------------------------------------------
  const int32_t* prog = P.i(h.off_prog);
  for (int s = 0; s < h.nsteps; ++s) {
    int n = prog[s * G + g];
    if (valid && n >= 0) fk_node<T>(P, n, qb, xs);
    BIK_SYNCWARP();
  }

  // ---- held targets: a task held on this frame takes the held value in place of its sequence row; on the first pass of a
  // run, the value is captured first, from q, into the held buffer (in the caller's precision), so that this pass's errors
  // are taken against it.  A phase of its own after FK (the input loads and the frame loop keep their registers: fp32 spills
  // otherwise); each lane handles the frames the frame loop gives it, and the CoM tasks the CoM phase's lane.
  if constexpr (HO) {
    if (valid) {
      void* const held = static_cast<const K1HArgs&>(a).held;
      const long long h0 = (long long)b * k1_tgt_words(h);
      for (int f = g; f < h.F; f += G) {
        const int s = k1h_hold(a, h, b, f);
        if (s == 0) continue;
        T* tg = ttile + (li * h.F + f) * 7;
        if (s == 1) {
          for (int k = 0; k < 7; ++k) tg[k] = ldin<T>(held, h0 + 7 * f + k, a.in64);
          continue;
        }
        const FrameRec& fr = P.frame(f);
        Q4<T> qf, qr, tq; V3<T> pf, pr, tp;
        if constexpr (PL) k1p_frame_pose<T>(P, a, b, f, fr.slot, xs, &qf, &pf);
        else frame_pose<T>(fr.slot, KC<T>::flpos(P, f), KC<T>::flquat(P, f), xs, &qf, &pf);
        qr = qf; pr = pf;
        if (fr.relative) frame_pose<T>(fr.rslot, KC<T>::frlpos(P, f), KC<T>::frlquat(P, f), xs, &qr, &pr);
        held_frame_value<T>(fr.relative, qf, pf, qr, pr, &tq, &tp);
        const T v[7] = {tq.w, tq.x, tq.y, tq.z, tp.x, tp.y, tp.z};
        for (int k = 0; k < 7; ++k) { tg[k] = k1h_round<T>(v[k], a.in64); stout<T>(held, h0 + 7 * f + k, a.in64, tg[k]); }
      }
      if (g == 0)
        for (int c = 0; c < h.C; ++c) {
          const int s = k1h_hold(a, h, b, h.F + c);
          if (s == 0) continue;
          T* tg = ttile + IPW * h.F * 7 + (li * h.C + c) * 3;
          if (s == 1) {
            for (int k = 0; k < 3; ++k) tg[k] = ldin<T>(held, h0 + 7 * h.F + 3 * c + k, a.in64);
            continue;
          }
          const V3<T> cv = model_com<T>(P, xs);
          const T v[3] = {cv.x, cv.y, cv.z};
          for (int k = 0; k < 3; ++k) { tg[k] = k1h_round<T>(v[k], a.in64); stout<T>(held, h0 + 7 * h.F + 3 * c + k, a.in64, tg[k]); }
        }
    }
    BIK_SYNCWARP();
  }

  // ---- frame tasks -------------------------------------------------------------------------
  // (1) the G lanes of an instance evaluate different frames' SE(3) algebra (error, jlog blocks) in parallel
  const int32_t* cols = P.i(h.off_cols);
  if (valid) {
    for (int f = g; f < h.F; f += G) {
      const FrameRec& fr = P.frame(f);
      Q4<T> qf; V3<T> pf, ev, ew; M3<T> A1, A2;
      if constexpr (PL) k1p_frame_pose<T>(P, a, b, f, fr.slot, xs, &qf, &pf);
      else frame_pose<T>(fr.slot, KC<T>::flpos(P, f), KC<T>::flquat(P, f), xs, &qf, &pf);
      T* sc = fsc + (li * h.F + f) * FS;
      const T* tg = ttile + (li * h.F + f) * 7;
      Q4<T> tq = q4<T>(tg[0], tg[1], tg[2], tg[3]);
      V3<T> tp = v3<T>(tg[4], tg[5], tg[6]);
      if (!fr.relative) {
        frame_task<T>(qf, pf, tq, tp, &ev, &ew, &A1, &A2);
        sc[0] = pf.x; sc[1] = pf.y; sc[2] = pf.z;
      } else {   // A1 = Ji, A2 = Mi of jlog(T_tf); plus both frames' poses for the column phase
        Q4<T> qr; V3<T> pr;
        frame_pose<T>(fr.rslot, KC<T>::frlpos(P, f), KC<T>::frlquat(P, f), xs, &qr, &pr);
        relative_frame_task<T>(qf, pf, qr, pr, tq, tp, &ev, &ew, &A1, &A2);
        sc[0] = pf.x; sc[1] = pf.y; sc[2] = pf.z;
        sc[21] = qf.w; sc[22] = qf.x; sc[23] = qf.y; sc[24] = qf.z;
        sc[25] = qr.w; sc[26] = qr.x; sc[27] = qr.y; sc[28] = qr.z;
        sc[29] = pr.x; sc[30] = pr.y; sc[31] = pr.z;
      }
      T* eo = estage + li * K + fr.row0;
      eo[0] = ev.x; eo[1] = ev.y; eo[2] = ev.z; eo[3] = ew.x; eo[4] = ew.y; eo[5] = ew.z;
      if (packed) {   // e rides behind the task's columns
        T* po = pkg + (long long)b * PKS + fr.pk_off + 6 * fr.ncols;
        if (a.weights) {
          const long long w0 = k1_wbase<TR>(a, h, b) + fr.row0;
          ev = vmul(ev, k1_weight3<T>(a, w0)); ew = vmul(ew, k1_weight3<T>(a, w0 + 3));
        }
        store6<T>(po, ev, ew);
      }
      for (int k = 0; k < 9; ++k) { sc[3 + k] = A1.m[k]; sc[12 + k] = A2.m[k]; }
    }
  }
  if (valid && g == 0)   // CoM targets wait in the error slots until the CoM phase turns them into e = com - target
    for (int c = 0; c < h.C; ++c) {
      const int row0 = reinterpret_cast<const int32_t*>(P.f(h.off_com) + 8 * c)[5];
      for (int k = 0; k < 3; ++k) estage[li * K + row0 + k] = ttile[IPW * h.F * 7 + (li * h.C + c) * 3 + k];
    }
  // ---- posture errors: e = q* (-) q, free-joint dofs zeroed (posture_task.py:107-118) ------------
  // (the packed hand-off carries none: K2 recomputes them from q and the target it reads anyway)
  if (h.P > 0 && !packed) {
    T* epg = reinterpret_cast<T*>(a.ep);
    const int per = h.P * nv;
    const uint32_t mper = ((1u << 20) + per - 1) / per, mnv = ((1u << 20) + nv - 1) / nv;   // k / per, r / nv by multiplication (exact below 2^20 / divisor)
    for (int k = lane; k < nvalid * per; k += W) {   // the tile's posture rows are one contiguous run of global memory
      const int l2 = (int)(((uint32_t)k * mper) >> 20), r = k - l2 * per, p = (int)(((uint32_t)r * mnv) >> 20), d = r - p * nv;
      const T* qq = qtile + l2 * nq;
      const long long t0 = ((long long)(a.pbatched ? (inst0 + l2) : 0) * h.P + p) * nq;
      epg[(long long)inst0 * per + k] = posture_err_dof<T>(P, d, [&](int i) { return ldin<T>(a.ptgt, t0 + i, a.in64); }, [&](int i) { return qq[i]; });
    }
  }
  // Dense direct form (J holds frame rows only): the tile's K x nv blocks are one contiguous run of global memory; it is
  // zero-filled with 16-byte stores straight from registers, then each lane scatters the columns it computes (a frame
  // touches 12 of G1's 43 columns).  Zero-fill and scatter are ordered by the warp barrier; the partial sectors merge in L2.
  // (Alternatives: zero-fill at the top of the tile -- by plain stores or by bulk async stores from a block of zeros -- lets
  //  the zeros be written back to DRAM before the scatter reaches L2, so every line goes out twice; "write once" -- non-zero
  //  columns parked in a compact [6][max_cols] block per instance, then every element of the 6 x nv blocks produced from an
  //  inverse column table and stored as contiguous runs, no zero-fill -- makes the kernel issue-bound.)
  if (direct && h.F > 0) zero_words<W, T>(Jg + (long long)inst0 * K * nv, nvalid * K * nv, lane);
  BIK_SYNCWARP();
  // ---- the tile's inputs are dead from here on: send the next tile's ahead (bulk async copies into the same buffers) ----
#if defined(__CUDA_ARCH__)
  if (pipe && k1_tile_bulk_ok<T, TR>(h, a, next_inst0, IPW)) {
    if (lane == 0) k1_pipe_arm<T, TR>(h, a, next_inst0, IPW, pipe, qtile, ttile);
    pipe->armed = next_inst0;
  }
#endif
  // (2) per frame: Jacobian columns.
  // Packed form: each lane writes the six entries of every column it computes as one 24-byte (fp32) run of the task's
  // block -- nothing else is written, nothing is zero-filled.  Dense direct form: scatter into the zero-filled run (see
  // the top of the tile).  Dense staged form (CoM rows share J): per frame through the staging tile, flushed as contiguous runs.
  for (int f = 0; f < h.F; ++f) {
    const FrameRec& fr = P.frame(f);
    const bool staged = !packed && !direct;
    if (staged) {
      zero_words<W, T>(stage, IPW * 6 * nv, lane);
      BIK_SYNCWARP();
    }
    if (valid) {
      const T* sc = fsc + (li * h.F + f) * FS;
      V3<T> pf = ld_v(sc);
      M3<T> A1, A2;
      for (int k = 0; k < 9; ++k) { A1.m[k] = sc[3 + k]; A2.m[k] = sc[12 + k]; }
      T* st = packed ? pkg + (long long)b * PKS + fr.pk_off : (direct ? Jg + ((long long)b * K + fr.row0) * nv : stage + li * 6 * nv);
      Q4<T> qf, qr, q_fr; V3<T> pr, t_fr;
      if (fr.relative) {
        qf = ld_q(sc + 21); qr = ld_q(sc + 25); pr = ld_v(sc + 29);
        q_fr = qmul(qconj(qf), qr);          // rotation of T_rf^-1 = T_fr
        t_fr = qrot_inv(qf, pr - pf);        // translation of T_fr
      }
      const bool weighted = packed && a.weights;
      for (int c = g; c < fr.ncols; c += G) {
        int ent = cols[fr.col_off + c], d = ent & 0xffff, n = (ent >> 16) & 0x7fff;
        V3<T> jp, jr, tv, tw;
        if (!fr.relative) {
          jac_column<T>(P, d, n, xs, pf, &tv, &tw);
        } else if (ent >= 0) {                  // column of J_f (body frame of f)
          jac_column<T>(P, d, n, xs, pf, &jp, &jr);
          tv = qrot_inv(qf, jp); tw = qrot_inv(qf, jr);
        } else {                                // minus Ad(T_fr) applied to the column of J_r
          jac_column<T>(P, d, n, xs, pr, &jp, &jr);
          V3<T> bv = qrot(q_fr, qrot_inv(qr, jp)), bw = qrot(q_fr, qrot_inv(qr, jr));
          V3<T> x = cross(t_fr, bw);
          tv = v3<T>(-(bv.x + x.x), -(bv.y + x.y), -(bv.z + x.z));
          tw = v3<T>(-bw.x, -bw.y, -bw.z);
        }
        V3<T> top = mmul(A1, tv) + mmul(A2, tw), bot = mmul(A1, tw);
        if (weighted) {   // (fetched per column: six weights held across the loop make the track-mode kernels spill)
          const long long w0 = k1_wbase<TR>(a, h, b) + fr.row0;
          top = vmul(top, k1_weight3<T>(a, w0)); bot = vmul(bot, k1_weight3<T>(a, w0 + 3));
        }
        if (packed) store6<T>(st + 6 * c, top, bot);
        else {
          st[d] = top.x; st[nv + d] = top.y; st[2 * nv + d] = top.z;
          st[3 * nv + d] = bot.x; st[4 * nv + d] = bot.y; st[5 * nv + d] = bot.z;
        }
      }
    }
    if (staged) {
      BIK_SYNCWARP();
      flush_rows<W, T>(stage, 6 * nv, nvalid, Jg + ((long long)inst0 * K + fr.row0) * nv, (long long)K * nv, lane);
      BIK_SYNCWARP();
    }
  }

  // ---- centre-of-mass tasks (mj_comPos + mj_jacSubtreeCom for body 1) -------------------------
  if (h.C > 0) {
    T* S = xs + 7 * h.nslots;  // first moments per node (a CoM task keeps slots == node ids)
    if (valid && g == 0) {
      for (int n = 0; n < h.nnode; ++n) {
        V3<T> m = v3<T>(T(0), T(0), T(0));   // nodes without mass below them are not visited by the lane program
        if (KC<T>::sub_m(P, n) > T(0)) m = KC<T>::own_m(P, n) * ld_v(xs + 7 * n + 4) + qrot(ld_q(xs + 7 * n), KC<T>::own_c(P, n));
        S[3 * n] = m.x; S[3 * n + 1] = m.y; S[3 * n + 2] = m.z;
      }
      for (int n = h.nnode - 1; n >= 0; --n) {
        int p = P.node(n).parent;
        if (p >= 0) { S[3 * p] += S[3 * n]; S[3 * p + 1] += S[3 * n + 1]; S[3 * p + 2] += S[3 * n + 2]; }
      }
    }
    BIK_SYNCWARP();
    const T invM = T(1) / KC<T>::com_mass(P);
    for (int c = 0; c < h.C; ++c) {
      const float* cr = P.f(h.off_com) + 8 * c;
      const int row0 = reinterpret_cast<const int32_t*>(cr)[5], pk_off = reinterpret_cast<const int32_t*>(cr)[6];
      if (!packed) {
        zero_words<W, T>(stage, IPW * 3 * nv, lane);
        BIK_SYNCWARP();
      }
      if (valid) {
        const bool weighted = packed && a.weights;
        V3<T> wc;
        if (weighted) wc = k1_weight3<T>(a, k1_wbase<TR>(a, h, b) + row0);
        if (g == 0) {
          V3<T> tot = KC<T>::com_fixed(P);
          for (int n = 0; n < h.nnode; ++n) if (P.node(n).parent < 0) tot = tot + ld_v(S + 3 * n);
          T* eo = estage + li * K + row0;  // e = com - target (com_task.py:82); the target was parked here
          eo[0] = tot.x * invM - eo[0]; eo[1] = tot.y * invM - eo[1]; eo[2] = tot.z * invM - eo[2];
          if (packed) {
            V3<T> ec = ld_v(eo);
            if (weighted) ec = vmul(ec, wc);
            T* po = pkg + (long long)b * PKS + pk_off + 3 * h.com_ncols; po[0] = ec.x; po[1] = ec.y; po[2] = ec.z;
          }
        }
        T* st = packed ? pkg + (long long)b * PKS + pk_off : stage + li * 3 * nv;
        for (int ci = g; ci < h.com_ncols; ci += G) {
          int ent = cols[h.com_cols_off + ci], d = ent & 0xffff, n = (ent >> 16) & 0x7fff;
          const NodeRec& r = P.node(n);
          T Ms = KC<T>::sub_m(P, n);
          Q4<T> nq_ = ld_q(xs + 7 * n); V3<T> np = ld_v(xs + 7 * n + 4), Sn = ld_v(S + 3 * n), col;
          int k = d - r.dadr;
          if (r.type == JNT_SLIDE) col = (Ms * invM) * qrot(nq_, KC<T>::naxis(P, n, r));
          else if (r.type == JNT_FREE && k < 3) col = (Ms * invM) * unit_axis<T>(k);
          else {
            V3<T> ax, anchor;
            if (r.type == JNT_HINGE) { ax = qrot(nq_, KC<T>::naxis(P, n, r)); anchor = np + qrot(nq_, KC<T>::njpos(P, n, r)); }
            else {
              int cc = (r.type == JNT_FREE) ? k - 3 : k;
              ax = qrot(nq_, unit_axis<T>(cc));
              anchor = (r.type == JNT_FREE) ? np : np + qrot(nq_, KC<T>::njpos(P, n, r));
            }
            col = invM * cross(ax, Sn - Ms * anchor);
          }
          if (weighted) col = vmul(col, wc);
          if (packed) { st[3 * ci] = col.x; st[3 * ci + 1] = col.y; st[3 * ci + 2] = col.z; }
          else { st[d] = col.x; st[nv + d] = col.y; st[2 * nv + d] = col.z; }
        }
      }
      if (!packed) {
        BIK_SYNCWARP();
        flush_rows<W, T>(stage, 3 * nv, nvalid, Jg + ((long long)inst0 * K + row0) * nv, (long long)K * nv, lane);
        BIK_SYNCWARP();
      }
    }
  }

  // ---- convergence test of the examples' inner loop (bik_converge), on the unweighted frame errors --------
  if (PK && !TR && a.done) {
    BIK_SYNCWARP();
    const int it = conv_step;
    if (it > 0 && lane < nvalid && !a.done[inst0 + lane]) {
      bool ok = true;
      for (int f = 0; f < h.F; ++f) {
        const T* eb = estage + lane * K + P.frame(f).row0;
        const T pos = bik_sqrt<T>(eb[0] * eb[0] + eb[1] * eb[1] + eb[2] * eb[2]), ori = bik_sqrt<T>(eb[3] * eb[3] + eb[4] * eb[4] + eb[5] * eb[5]);
        const long long w0 = a.weights ? k1_wbase<false>(a, h, inst0 + lane) + P.frame(f).row0 : 0;
        ok = ok && (pos <= k1_pos_thr<T>(a) || !k1_tested<T>(a, w0)) && (ori <= k1_ori_thr<T>(a) || !k1_tested<T>(a, w0 + 3));
      }
      if (ok) { a.done[inst0 + lane] = 1; a.iters[inst0 + lane] = it; }
      else {
#if defined(__CUDA_ARCH__)
        atomicAdd(a.not_done, 1);
#else
        *a.not_done += 1;
#endif
      }
    }
  }
  // ---- track mode (bik_track): the same test ends the instance's frame instead of the call -----------------------------
  // A frame ends when its errors pass after at least one step, or after max_iters steps (then with BIK_STATUS_NOT_CONVERGED);
  // its results are those of a bik_converge call on that frame.  The next pass starts the next frame at step 0 with a cold
  // warm start, exactly as a new bik_converge call does.
  if (TR) {
    BIK_SYNCWARP();
    int ended = -1;   // frame of instance inst0 + lane that ends in this pass
    if (lane < nvalid) {
      const int bi = inst0 + lane, s = a.tstep[bi];
      int skip = 1, left = 0;
      if (s >= 0) {
        bool ok = s > 0;
        for (int f = 0; ok && f < h.F; ++f) {
          const T* eb = estage + lane * K + P.frame(f).row0;
          const T pos = bik_sqrt<T>(eb[0] * eb[0] + eb[1] * eb[1] + eb[2] * eb[2]), ori = bik_sqrt<T>(eb[3] * eb[3] + eb[4] * eb[4] + eb[5] * eb[5]);
          const long long w0 = a.weights ? k1_wbase<true>(a, h, bi) + P.frame(f).row0 : 0;
          ok = (pos <= k1_pos_thr<T>(a) || !k1_tested<T>(a, w0)) && (ori <= k1_ori_thr<T>(a) || !k1_tested<T>(a, w0 + 3));
        }
        if (ok || s >= a.conv_max) {
          const int c = a.cursor[bi];
          const long long row = (long long)bi * a.T + c;
          a.iters[row] = s;
          if (a.traj_status) a.traj_status[row] = a.status[bi] | (ok ? 0 : 16);
          ended = c;
          left = c + 1 < (a.lengths ? a.lengths[bi] : a.T);
          a.cursor[bi] = c + 1;
          a.tstep[bi] = left ? 0 : -1;
        } else {
          a.tstep[bi] = s + 1;
          skip = 0; left = 1;
        }
      }
      a.done[bi] = skip;
      if (left) {
#if defined(__CUDA_ARCH__)
        atomicAdd(a.not_done, 1);
#else
        *a.not_done += 1;
#endif
      }
    }
    if (lane < IPW) sflag[lane] = ended;
    BIK_SYNCWARP();
    // q_traj rows of the frames that ended (from global q: the tile's copy may already hold the next tile's rows), and a cold
    // warm start for the next frame.  q and q_traj are fp64 only in the fp64 instantiation (bik_track64).
    // (two plain loops rather than one generic one: the fp32 instantiations then compile to the code they had before)
    if constexpr (sizeof(T) == 8) {
      if (a.in64) {
        const double* qg = static_cast<const double*>(a.q);
        for (int k = lane; k < nvalid * nq; k += W) {
          const int i = k / nq, c = sflag[i];
          if (c >= 0) static_cast<double*>(a.q_traj)[((long long)(inst0 + i) * a.T + c) * nq + (k - i * nq)] = qg[(long long)inst0 * nq + k];
        }
      }
    }
    if (sizeof(T) == 4 || !a.in64) {
      const float* qg = reinterpret_cast<const float*>(a.q);
      for (int k = lane; k < nvalid * nq; k += W) {
        const int i = k / nq, c = sflag[i];
        if (c >= 0) static_cast<float*>(a.q_traj)[((long long)(inst0 + i) * a.T + c) * nq + (k - i * nq)] = qg[(long long)inst0 * nq + k];
      }
    }
    const int nw = h.nu > 0 ? h.nu : 1;
    for (int k = lane; k < nvalid * nw; k += W)
      if (sflag[k / nw] >= 0) a.warm[(long long)inst0 * nw + k] = 0;
    BIK_SYNCWARP();
  }

  // ---- task errors out (contiguous IPW x K run) ------------------------------------------------
  if (K > 0 && !packed) {
    T* eg = reinterpret_cast<T*>(a.e);
    for (int k = lane; k < nvalid * K; k += W) eg[(long long)inst0 * K + k] = estage[k];
  }

  // ---- collision rows (collision_avoidance_limit.py:187-210), 6 pairs per staging pass -----------
  if (h.npairs > 0) {
    const int32_t* pairs = P.i(h.off_pairs);
    T* Gcg = reinterpret_cast<T*>(a.Gc);
    T* hcg = reinterpret_cast<T*>(a.hc);
    // CO: the instance's distances (the problem's for a null buffer, a non-finite value or an invalid lane) and its row of the
    // pair mask, or null (every pair)
    const T ddet = k1c_coll<T, CO>(P, a, valid, crow, 2), dmin = k1c_coll<T, CO>(P, a, valid, crow, 1), cgain = KC<T>::coll(P, 0), relax = KC<T>::coll(P, 3);
    const uint8_t* en = nullptr;
    if constexpr (CO) {
      const uint8_t* m = static_cast<const K1CArgs&>(a).enabled;
      if (valid && m) en = m + crow * h.npairs;
    }
    for (int p0 = 0; p0 < h.npairs; p0 += 6) {
      int np_ = h.npairs - p0 < 6 ? h.npairs - p0 : 6;
      zero_words<W, T>(stage, IPW * np_ * nv, lane);
      BIK_SYNCWARP();
      if (valid) {
        for (int pi = g; pi < np_; pi += G) {
          const int i1 = pairs[2 * (p0 + pi)], i2 = pairs[2 * (p0 + pi) + 1];
          V3<T> o1, o2;
          T dist = !en || en[p0 + pi] ? geom_distance<T>(P, i1, i2, xs, ddet, &o1, &o2) : ddet;   // a disabled pair: as one beyond ddet
          T hval = T(BIK_INF_F);
          if (dist != ddet) {
            hval = dist > dmin ? cgain * (dist - dmin) / T(a.dt) + relax : relax;
            V3<T> nr = o2 - o1;
            T L = bik_sqrt<T>(dot(nr, nr));
            nr = L > T(1e-15) ? (T(1) / L) * nr : v3<T>(T(1), T(0), T(0));
            T* st = stage + (li * np_ + pi) * nv;
            for (int side = 0; side < 2; ++side) {  // row = -n.(Jp2 - Jp1)
              V3<T> pt = side ? o2 : o1;
              T sgn = side ? T(-1) : T(1);
              for (int n = P.geom(side ? i2 : i1).node; n >= 0; n = P.node(n).parent) {
                const NodeRec& r = P.node(n);
                int nd = r.type == JNT_FREE ? 6 : (r.type == JNT_BALL ? 3 : 1);
                for (int k = 0; k < nd; ++k) {
                  V3<T> jp, jr;
                  jac_column<T>(P, r.dadr + k, n, xs, pt, &jp, &jr);
                  st[r.dadr + k] += sgn * dot(nr, jp);
                }
              }
            }
          }
          hcg[(long long)b * h.npairs + p0 + pi] = hval;
        }
      }
      BIK_SYNCWARP();
      flush_rows<W, T>(stage, np_ * nv, nvalid, Gcg + ((long long)inst0 * h.npairs + p0) * nv, (long long)h.npairs * nv, lane);
      BIK_SYNCWARP();
    }
  }
}

// ---- FK of arbitrary frames / body-frame Jacobians (Configuration API) -------------------------
struct FkFrame { int32_t node, pad; double lpos[3], lquat[4]; };   // 64 bytes; frames travel by value in the launch arguments
struct FkArgs {
  int B, nframes;
  const void* q;   // fp32, or fp64 when io64 (then the outputs are fp64 too and the fp64 instantiation runs)
  void* poses;     // [B][nframes][7] or null
  void* com;       // [B][3] or null
  void* J;         // [B][nframes][6][nv] or null
  int io64;
  FkFrame frames[16];
};

template <typename T, int G, int W>
BIK_HD void fk_warp_tile(const PView& P, const FkArgs& a, int inst0, T* wsm, int lane) {
  const PHeader& h = P.h();
  constexpr int IPW = W / G;
  const int li = lane / G, g = lane % G, b = inst0 + li, nv = h.nv, nq = h.nq;
  const int nvalid = (a.B - inst0) < IPW ? (a.B - inst0) : IPW;
  const bool valid = li < nvalid;
  const int SS = (7 * h.nnode + nq) | 1;
  T* xs = wsm + li * SS;
  T* qb = xs + 7 * h.nnode;
  if (valid) for (int k = g; k < nq; k += G) qb[k] = ldin<T>(a.q, (long long)b * nq + k, a.io64);
  BIK_SYNCWARP();
  const int32_t* prog = P.i(h.off_prog);
  for (int s = 0; s < h.nsteps; ++s) {
    int n = prog[s * G + g];
    if (valid && n >= 0) fk_node<T>(P, n, qb, xs);
    BIK_SYNCWARP();
  }
  if (!valid) return;
  for (int f = g; f < a.nframes; f += G) {
    const FkFrame& fr = a.frames[f];
    Q4<T> qf; V3<T> pf;
    frame_pose<T>(fr.node, v3<T>(T(fr.lpos[0]), T(fr.lpos[1]), T(fr.lpos[2])), q4<T>(T(fr.lquat[0]), T(fr.lquat[1]), T(fr.lquat[2]), T(fr.lquat[3])), xs, &qf, &pf);
    M3<T> R = q2mat(qf);
    if (a.poses) {
      Q4<T> qs = mat2quat(R);  // sign convention of SO3.from_matrix (configuration.py:182)
      const long long o = ((long long)b * a.nframes + f) * 7;
      stout<T>(a.poses, o, a.io64, qs.w); stout<T>(a.poses, o + 1, a.io64, qs.x); stout<T>(a.poses, o + 2, a.io64, qs.y); stout<T>(a.poses, o + 3, a.io64, qs.z);
      stout<T>(a.poses, o + 4, a.io64, pf.x); stout<T>(a.poses, o + 5, a.io64, pf.y); stout<T>(a.poses, o + 6, a.io64, pf.z);
    }
    if (a.J) {  // blockdiag(R^T, R^T) [jacp; jacr]  (configuration.py:143-153)
      const long long o = ((long long)b * a.nframes + f) * 6 * nv;
      for (int k = 0; k < 6 * nv; ++k) stout<T>(a.J, o + k, a.io64, T(0));
      M3<T> Rt = mtrans(R);
      for (int n = fr.node; n >= 0; n = P.node(n).parent) {
        const NodeRec& r = P.node(n);
        int nd = r.type == JNT_FREE ? 6 : (r.type == JNT_BALL ? 3 : 1);
        for (int k = 0; k < nd; ++k) {
          V3<T> jp, jr;
          int d = r.dadr + k;
          jac_column<T>(P, d, n, xs, pf, &jp, &jr);
          V3<T> top = mmul(Rt, jp), bot = mmul(Rt, jr);
          stout<T>(a.J, o + d, a.io64, top.x); stout<T>(a.J, o + nv + d, a.io64, top.y); stout<T>(a.J, o + 2 * nv + d, a.io64, top.z);
          stout<T>(a.J, o + 3 * nv + d, a.io64, bot.x); stout<T>(a.J, o + 4 * nv + d, a.io64, bot.y); stout<T>(a.J, o + 5 * nv + d, a.io64, bot.z);
        }
      }
    }
  }
  if (a.com && g == 0) {
    V3<T> tot = KC<T>::com_fixed(P);
    for (int n = 0; n < h.nnode; ++n) tot = tot + KC<T>::own_m(P, n) * ld_v(xs + 7 * n + 4) + qrot(ld_q(xs + 7 * n), KC<T>::own_c(P, n));
    T M = KC<T>::com_mass(P);
    T invM = M > T(0) ? T(1) / M : T(0);
    stout<T>(a.com, (long long)b * 3, a.io64, tot.x * invM); stout<T>(a.com, (long long)b * 3 + 1, a.io64, tot.y * invM); stout<T>(a.com, (long long)b * 3 + 2, a.io64, tot.z * invM);
  }
}
BIK_HD int fk_warp_words(const PHeader& h, int ipw) { return (ipw * ((7 * h.nnode + h.nq) | 1) + 3) & ~3; }

// ---- integrate / check_limits / box limits: per instance ----------------------------
// mj_integratePos of ONE node, dt folded into dq (configuration.py:228-236)
template <typename T>
BIK_HD void integrate_node(const NodeRec& r, T* q, const T* dq) {
  if (r.type == JNT_FREE) {
    for (int k = 0; k < 3; ++k) q[r.qadr + k] += dq[r.dadr + k];
    Q4<T> o = quat_integrate<T>(ld_q(q + r.qadr + 3), ld_v(dq + r.dadr + 3));
    q[r.qadr + 3] = o.w; q[r.qadr + 4] = o.x; q[r.qadr + 5] = o.y; q[r.qadr + 6] = o.z;
  } else if (r.type == JNT_BALL) {
    Q4<T> o = quat_integrate<T>(ld_q(q + r.qadr), ld_v(dq + r.dadr));
    q[r.qadr] = o.w; q[r.qadr + 1] = o.x; q[r.qadr + 2] = o.y; q[r.qadr + 3] = o.z;
  } else {
    q[r.qadr] += dq[r.dadr];
  }
}
template <typename T>
BIK_HD void integrate_instance(const PView& P, T* q, const T* dq) {
  const PHeader& h = P.h();
  for (int n = 0; n < h.nnode; ++n) integrate_node<T>(P.node(n), q, dq);
}
template <typename T>
BIK_HD int check_limits_instance(const PView& P, const T* q, float tol) {  // configuration.py:77-110
  const PHeader& h = P.h();
  const int32_t* dofqadr = P.i(h.off_dofqadr);
  const float* rng = P.f(h.off_range);
  int bad = 0;
  for (int d = 0; d < h.nv; ++d) {
    int qa = dofqadr[d];
    if (qa < 0) continue;
    T v = q[qa];
    if (v < T(rng[d]) - T(tol) || v > T(rng[h.nv + d]) + T(tol)) bad = 1;
    if (!(v == v)) bad |= 4;
  }
  return bad;
}
// ---- per-instance bounds (the ..._bounded entry points) ---------------------------------------------------------------
// One instance's rows of the caller's [B][nv] lower / upper / vmax buffers, each null when not given; element type by is64.
// A null row, or a BoundsRow of null rows, narrows nothing.
struct BoundsRow { const void *lo, *up, *vm; int is64; };
// The problem's bound `tab` of dof d narrowed by the instance's value in `row`: the larger of the two for a lower bound, the
// smaller for an upper bound or a cap.  `tab` itself for a null row, or for a NaN value, which sets BIK_STATUS_NONFINITE (4)
// in *st.  The callers narrow only the bounds the problem gives a dof, so the set of bounded dofs never changes.
template <typename T, bool UPPER>
BIK_HD T bd_narrow(T tab, const void* row, int d, int is64, int* st) {
  if (!row) return tab;
  const T v = ldin<T>(row, d, is64);
  if (!(v == v)) { *st |= 4; return tab; }
  return UPPER ? bik_min(tab, v) : bik_max(tab, v);
}
// ConfigurationLimit c lists the dof (gives it a finite bound): its bounds [lc, uc] are narrowed by the instance's
template <typename T>
BIK_HD void bd_narrow_cfg(const BoundsRow& bd, int d, T* lc, T* uc, int* st) {
  if (*lc > -T(BIK_INF_F) || *uc < T(BIK_INF_F)) {
    *lc = bd_narrow<T, false>(*lc, bd.lo, d, bd.is64, st);
    *uc = bd_narrow<T, true>(*uc, bd.up, d, bd.is64, st);
  }
}
// the VelocityLimit lists the dof (gives it a finite cap): the cap is narrowed by the instance's
template <typename T>
BIK_HD T bd_narrow_vmax(const BoundsRow& bd, int d, T vmax, int* st) {
  return vmax < T(BIK_INF_F) ? bd_narrow<T, true>(vmax, bd.vm, d, bd.is64, st) : vmax;
}

// lo <= dq <= hi from ConfigurationLimit(s) and VelocityLimit (configuration_limit.py:98-124, velocity_limit.py:99-101);
// qi = q of the dof (unused for free / ball dofs).  BD (compile time): the instance's bounds `bd` narrow the problem's before
// they enter the same products (NaN bounds set BIK_STATUS_NONFINITE in *st), so bounds equal to the problem's give its bits.
template <typename T, bool BD = false>
BIK_HD void box_dof(const PView& P, int d, T qi, T dt, T* lo, T* hi, const BoundsRow* bd = nullptr, int* st = nullptr) {
  const PHeader& h = P.h();
  T l = -T(BIK_INF_F), u = T(BIK_INF_F);
  if (P.i(h.off_dofqadr)[d] >= 0) {
    for (int c = 0; c < h.ncfg; ++c) {
      const float* p = P.f(h.off_cfg) + c * (2 + 2 * h.nv);
      T up, dn;
      if constexpr (BD) {
        T lc = T(p[2 + d]), uc = T(p[2 + h.nv + d]);
        bd_narrow_cfg<T>(*bd, d, &lc, &uc, st);
        up = T(p[0]) * (uc - qi); dn = T(p[0]) * (qi - lc);
      } else {
        up = T(p[0]) * (T(p[2 + h.nv + d]) - qi); dn = T(p[0]) * (qi - T(p[2 + d]));
      }
      u = bik_min(u, up); l = bik_max(l, -dn);
    }
  }
  if (h.has_vel) {
    T vm;
    if constexpr (BD) vm = dt * bd_narrow_vmax<T>(*bd, d, T(P.f(h.off_vmax)[d]), st);
    else vm = dt * T(P.f(h.off_vmax)[d]);
    u = bik_min(u, vm); l = bik_max(l, -vm);
  }
  *lo = l; *hi = u;
}

}  // namespace bik
