// TEST INFRASTRUCTURE -- the host emulation (emu.cpp) plus the pass loops of bik_converge_weighted / bik_track_weighted
// (per-instance task weights, K1Args::weights).  Built as its own library so that emu.cpp keeps its entry points as they are;
// every emu_* function of emu.cpp is exported from it as well.  Never shipped, never loaded by mink_b200/.
#include "emu.cpp"

// f64 = 0: the fp32 loops (dt and the thresholds rounded to float, as their parameters are), f64 = 1: the ...64 ones.
// weights: [B][K] (converge) or [B][T][K] (track) in q's element type, or null (all ones).
static int emu_weighted_call(void* prob, int f64, bool track, int B, int T, void* q, const void* ftgt, const void* ptgt, int pbatched,
                             const void* ctgt, const void* weights, const int32_t* lengths, double dt, double damping, int max_iters, double pos,
                             double ori, void* q_traj, int32_t* iters, int32_t* status, int32_t* passes) {
  if (!f64) { dt = (float)dt; pos = (float)pos; ori = (float)ori; }
  bik_inputs in;
  memset(&in, 0, sizeof in);
  in.q = q; in.frame_targets = ftgt; in.posture_targets = ptgt; in.com_targets = ctgt; in.posture_batched = pbatched; in.f64 = f64;
  ConvCall c;
  memset(&c, 0, sizeof c);
  c.B = B; c.T = T; c.max_iters = max_iters; c.dt = dt; c.pos = pos; c.ori = ori; c.damping = damping; c.q = q; c.in = &in;
  c.lengths = lengths; c.q_traj = q_traj; c.iters = iters; c.status = status; c.track = track; c.io64 = f64 != 0; c.weights = weights;
  return emu_loop(static_cast<EmuProblem*>(prob), c, passes);
}
extern "C" int emu_converge_weighted(void* prob, int f64, int B, void* q, const void* ftgt, const void* ptgt, int pbatched, const void* ctgt,
                                     const void* weights, double dt, double damping, int max_iters, double pos, double ori, int32_t* iters,
                                     int32_t* status) {
  return emu_weighted_call(prob, f64, false, B, 1, q, ftgt, ptgt, pbatched, ctgt, weights, nullptr, dt, damping, max_iters, pos, ori, nullptr, iters,
                           status, nullptr);
}
extern "C" int emu_track_weighted(void* prob, int f64, int B, int T, void* q, const void* ftgt, const void* ptgt, int pbatched, const void* ctgt,
                                  const void* weights, const int32_t* lengths, double dt, double damping, int max_iters, double pos, double ori,
                                  void* q_traj, int32_t* iters, int32_t* status, int32_t* passes) {
  return emu_weighted_call(prob, f64, true, B, T, q, ftgt, ptgt, pbatched, ctgt, weights, lengths, dt, damping, max_iters, pos, ori, q_traj, iters,
                           status, passes);
}
