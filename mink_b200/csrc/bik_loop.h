// bik_loop.h -- one pass of the bik_converge / bik_track loop, defined once for the driver (bik_api.cu) and the host
// emulation (tests/host_emu).
//
// One pass = tick, K1 (which also tests the thresholds on the errors it has just computed), condition, K2 (gated by the
// condition).  The driver runs the passes as the body of a CUDA-graph WHILE node, or from a host-polled loop; the emulation
// runs them one after the other on the CPU.  Both fill K1Args / K2Args here and keep the bookkeeping rules here.
#pragma once
#include <string.h>

#include "../../include/bik.h"
#include "bik_k2.h"

namespace bik {

// The arguments of one bik_converge / bik_track call.  io64: fp64 buffers (bik_converge64 / bik_track64).  k1d: K1 runs in
// fp64 (k1_auto_double, or io64).  dt and the thresholds of fp32 calls are their float values.  weights: the ..._weighted entry
// points' per-instance task weights (K1Args::weights), or null.  posture_weights: the ..._weighted_ex entry points' per-instance
// posture weights (K2PwArgs), or null.  bounds: the ..._bounded entry points' per-instance bounds (K2BdArgs), all three null
// for none; held by value, so that the converge graph's key holds the three pointers.  coll: the ..._coll entry points'
// per-instance collision pairs and distances (K1CArgs), all three null for none; held by value for the same reason.  hold: the
// bik_track_hold entry points' [B][T][F + C + P] hold mask (K1HArgs), or null.  placement: the ..._placed entry points' [B][F][7]
// frame placements (K1PArgs), or null.
struct ConvCall {
  int B, T, max_iters; double dt, pos, ori; double damping; void* q; const bik_inputs* in; const int32_t* lengths;
  void* q_traj; int32_t *iters, *status; bool track, k1d, io64; const void* weights; const void* posture_weights; bik_bounds bounds;
  bik_collision coll; const uint8_t* hold; const void* placement;
};
inline bool has_bounds(const bik_bounds& bd) { return bd.lower || bd.upper || bd.vmax; }
inline bool has_coll(const bik_collision& co) { return co.enabled || co.minimum_distance || co.detection_distance; }

// The loop state.  pk / Gc / hc: K1 -> K2 hand-off rows, fp64 when k1d.  dq: K2's dq of the previous pass (its warm start), in
// the caller's precision.  warm: [B][max(nu,1)] active-set guess.  done: [B] K2 leaves the instance alone.  cursor / step /
// status: [B] frame each instance is on, steps taken in it (-1: no frames left) and its status (track only).
// count = { steps taken (converge) or passes run (track), instances left, go }.  ptcur: [B][P][nq] posture targets of each
// instance's current frame, in the caller's precision (uses_ptcur only, else unused).  held: [B][7F + 3C] the held frame and
// CoM targets, in the caller's precision (track with a hold mask only, else unused).
struct ConvBufs {
  void *pk, *Gc, *hc, *dq;
  signed char* warm;
  int32_t *done, *cursor, *step, *status;
  int* count;
  void* ptcur;
  void* held;
};
// bik_inputs.posture_batched names a posture target sequence (bik_track entry points only)
inline bool posture_seq(const bik_inputs* in) {
  return in->posture_batched == BIK_POSTURE_SEQ_SHARED || in->posture_batched == BIK_POSTURE_SEQ_BATCHED;
}
// K1 keeps each instance's posture targets of its current frame in ptcur, which K2 reads: track mode with a posture target
// sequence, or with a hold mask (a held posture target is the q its run started from)
inline bool uses_ptcur(const ConvCall& c) { return c.track && (posture_seq(c.in) || c.hold); }
// Per instance: elements of a pk / Gc / hc row (4 or 8 bytes each, by K1's precision) and bytes of warm.
struct HandoffSizes { size_t pk, Gc, hc, warm; };
inline HandoffSizes handoff_sizes(const PHeader& h) {
  const size_t np = h.npairs > 0 ? h.npairs : 1;
  return HandoffSizes{(size_t)(h.pk_stride > 4 ? h.pk_stride : 4), np * h.nv, np, (size_t)(h.nu > 0 ? h.nu : 1)};
}

// K1 of a pass.  `status` is the call's status buffer, or null (the driver's warm-up pass before a graph capture).
inline K1Args conv_k1_args(const ConvCall& c, const ConvBufs& s, int32_t* status) {
  const bik_inputs* in = c.in;
  K1Args a;
  memset(&a, 0, sizeof a);
  a.B = c.B; a.q = c.q; a.ftgt = in->frame_targets; a.ptgt = in->posture_targets; a.ctgt = in->com_targets; a.pbatched = in->posture_batched;
  a.in64 = c.io64; a.dt = c.dt; a.pk = s.pk; a.Gc = s.Gc; a.hc = s.hc;
  a.status = c.track ? s.status : status; a.tol = 1e-6f;
  a.done = s.done; a.iters = c.iters; a.not_done = s.count + 1; a.conv_it = s.count; a.conv_max = c.max_iters;
  a.pos_thr = (float)c.pos; a.ori_thr = (float)c.ori; a.pos_thr64 = c.pos; a.ori_thr64 = c.ori; a.weights = c.weights;
  if (c.track) {
    a.cursor = s.cursor; a.tstep = s.step; a.lengths = c.lengths; a.T = c.T;
    a.q_traj = c.q_traj; a.traj_status = status; a.warm = s.warm;
    if (uses_ptcur(c)) a.ptcur = s.ptcur;
  }
  return a;
}
// The same for the collision instantiation of K1 (has_coll(c.coll)).  Track mode reads row b*T + cursor[b].
inline K1CArgs conv_k1c_args(const ConvCall& c, const ConvBufs& s, int32_t* status) {
  K1CArgs a;
  memset(&a, 0, sizeof a);
  static_cast<K1Args&>(a) = conv_k1_args(c, s, status);
  a.enabled = c.coll.enabled; a.dmin = c.coll.minimum_distance; a.ddet = c.coll.detection_distance;
  return a;
}
// The same for the held-target instantiation of K1 (c.hold set, track mode); the collision arguments may be null.
inline K1HArgs conv_k1h_args(const ConvCall& c, const ConvBufs& s, int32_t* status) {
  K1HArgs a;
  memset(&a, 0, sizeof a);
  static_cast<K1CArgs&>(a) = conv_k1c_args(c, s, status);
  a.hold = c.hold; a.held = s.held;
  return a;
}
// The same for the placement instantiation of K1 (c.placement set); the collision arguments may be null, the hold members are
// set with a hold mask (track mode).
inline K1PArgs conv_k1p_args(const ConvCall& c, const ConvBufs& s, int32_t* status) {
  K1PArgs a;
  memset(&a, 0, sizeof a);
  static_cast<K1CArgs&>(a) = conv_k1c_args(c, s, status);
  if (c.hold) { a.hold = c.hold; a.held = s.held; }
  a.placement = c.placement;
  return a;
}
// K2 of a pass: solves and integrates the instances K1 left undone, and does nothing once the condition said stop.
inline K2Args conv_k2_args(const ConvCall& c, const ConvBufs& s, int32_t* status) {
  const bik_inputs* in = c.in;
  K2Args a;
  memset(&a, 0, sizeof a);
  a.B = c.B; a.q = c.q; a.io64 = c.io64; a.pk = s.pk; a.pk64 = c.k1d; a.ptgt = in->posture_targets; a.pbatched = in->posture_batched;
  a.Gc = s.Gc; a.hc = s.hc; a.gc64 = c.k1d; a.dt = c.dt; a.damping = c.damping; a.dq = s.dq; a.integrate = 1;
  a.status = c.track ? s.status : status;
  a.warm = s.warm; a.skip = s.done; a.gate = s.count + 2;
  if (uses_ptcur(c)) { a.ptgt = s.ptcur; a.pbatched = 1; }   // K1 keeps each instance's current frame there
  return a;
}
// The same for the posture-weighted K2 (c.posture_weights set).  Track mode reads the row of each instance's current frame.
inline K2PwArgs conv_k2_pw_args(const ConvCall& c, const ConvBufs& s, int32_t* status) {
  K2PwArgs a;
  memset(&a, 0, sizeof a);
  static_cast<K2Args&>(a) = conv_k2_args(c, s, status);
  a.pw = c.posture_weights;
  if (c.track) { a.pw_cursor = s.cursor; a.pw_T = c.T; }
  return a;
}
// The same for the bounded K2 (has_bounds(c.bounds)); the posture weights may be null.  Track mode reads row b on every frame.
inline K2BdArgs conv_k2_bd_args(const ConvCall& c, const ConvBufs& s, int32_t* status) {
  K2BdArgs a;
  memset(&a, 0, sizeof a);
  static_cast<K2PwArgs&>(a) = conv_k2_pw_args(c, s, status);
  a.lower = c.bounds.lower; a.upper = c.bounds.upper; a.vmax = c.bounds.vmax;
  return a;
}

// Before the first pass, per instance.  converge: nobody has converged, and the step counter is -1 so that the first tick
// makes it 0.  track: every instance starts at frame 0, step 0 (step -1: no frames at all).
BIK_HD void conv_reset(bool track, int T, const int32_t* lengths, const ConvBufs& s, int b) {
  if (track) { s.cursor[b] = 0; s.step[b] = (lengths ? lengths[b] : T) > 0 ? 0 : -1; }
  else s.done[b] = 0;
  if (b == 0) { s.count[0] = track ? 0 : -1; s.count[1] = 0; s.count[2] = 1; }
}
// Before K1: advance the step counter (track: count a pass only when the previous one left work, so that the extra passes of
// the host-polled loop are not counted) and rewind the count that K1's test rebuilds.
BIK_HD void conv_tick(bool track, int* count) { count[0] += track ? count[2] : 1; count[1] = 0; }
// After K1's test: go on iff somebody has frames left (track), or iff step `it` < max_iters and (nothing has been tested yet
// or somebody is still unconverged) (converge).  `go` gates this pass's K2 and the next pass.
BIK_HD int conv_cond(bool track, int max_iters, int* count) {
  const int it = count[0];
  const int go = track ? count[1] > 0 : it < max_iters && (it == 0 || count[1] > 0);
  count[2] = go;
  return go;
}
// After the last pass (converge): an instance that never met the thresholds gets iters = max_iters and status bit
// BIK_STATUS_NOT_CONVERGED.
BIK_HD void conv_finish(int max_iters, const int32_t* done, int32_t* iters, int32_t* status, int b) {
  if (!done[b]) { iters[b] = max_iters; if (status) status[b] |= 16; }
}
// Passes a host-polled loop runs at most: converge, steps 0..max_iters; track, T frames of max_iters + 1 passes each.
inline long long conv_pass_cap(const ConvCall& c) { return c.track ? (long long)c.T * (c.max_iters + 1) : (long long)c.max_iters + 1; }

}  // namespace bik
