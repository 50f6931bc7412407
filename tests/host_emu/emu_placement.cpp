// TEST INFRASTRUCTURE -- the host emulation (emu.cpp, emu_bounds.cpp, emu_collision.cpp, emu_hold.cpp) plus the step and the pass
// loops of bik_step_placed / bik_converge_placed / bik_track_placed (per-instance frame placement, K1PArgs).  With a placement
// K1 runs the PL instantiation (k1_warp_tile<..., PK, TR, CO = true, HO, PL = true>, what k1p_kernel runs); K2 runs what the
// ..._coll / bik_track_hold loops run.  Built as its own library so that the other emulation units keep their entry points as
// they are; every emu_* function of theirs is exported from it as well.  Never shipped, never loaded by mink_b200/.
#include "emu_hold.cpp"

template <typename T, bool TR, bool HO>
static void emu_k1p_pass(const PView& P, const K1PArgs& a, double* wsm) {
  for (int b = 0; b < a.B; ++b) k1_warp_tile<T, 1, 1, true, TR, true, HO, true>(P, a, b, reinterpret_cast<T*>(wsm), 0);
}
template <typename T>
static void emu_k1p_pass(const PView& P, const K1PArgs& a, bool track, bool hold, double* wsm) {
  if (hold) emu_k1p_pass<T, true, true>(P, a, wsm);
  else if (track) emu_k1p_pass<T, true, false>(P, a, wsm);
  else emu_k1p_pass<T, false, false>(P, a, wsm);
}

// The bik_converge_placed / bik_track_placed loop; a null placement runs the bik_converge_coll / bik_track_hold loop.  f32k1 as
// in emu_coll_loop.
static int emu_placed_loop(EmuProblem* p, ConvCall c, int f32k1, int32_t* passes) {
  if (!c.placement) return c.hold ? emu_hold_loop(p, c, f32k1, passes) : emu_coll_loop(p, c, f32k1, passes);
  const PView P{p->image.data()};
  const PHeader& h = P.h();
  const size_t B = c.B;
  const HandoffSizes n = handoff_sizes(h);
  c.k1d = c.io64 || (!f32k1 && k1_auto_double(h, p->k1cond, c.damping, c.posture_weights != nullptr));
  std::vector<double> pk(B * n.pk), Gc(B * n.Gc), hc(B * n.hc), dq(B * h.nv), wsm(k1_warp_words(h, 1) + 16);
  std::vector<double> ptcur(B * (h.P > 0 ? h.P : 1) * h.nq), held(B * (k1_tgt_words(h) > 0 ? k1_tgt_words(h) : 1));
  std::vector<signed char> warm(B * n.warm);
  std::vector<int32_t> done(B), cursor(B), step(B), status(B);
  int count[3];
  const ConvBufs s{pk.data(), Gc.data(), hc.data(), dq.data(), warm.data(), done.data(), cursor.data(), step.data(), status.data(), count,
                   ptcur.data(), held.data()};
  for (int b = 0; b < c.B; ++b) conv_reset(c.track, c.T, c.lengths, s, b);
  const K1PArgs a1 = conv_k1p_args(c, s, c.status);
  const K2Args a2 = conv_k2_args(c, s, c.status);
  const K2PwArgs a2w = conv_k2_pw_args(c, s, c.status);
  const int path = emu_k2_path(h);
  for (int go = 1; go;) {
    conv_tick(c.track, count);
    if (c.k1d) emu_k1p_pass<double>(P, a1, c.track, c.hold != nullptr, wsm.data());
    else emu_k1p_pass<float>(P, a1, c.track, c.hold != nullptr, wsm.data());
    go = conv_cond(c.track, c.max_iters, count);
    if (!go) break;
    if (c.posture_weights) emu_k2_as<true, false>(P, a2w, path);
    else if (emu_k2(P, a2, path)) return -1;
  }
  if (c.track) *passes = count[0];
  else for (int b = 0; b < c.B; ++b) conv_finish(c.max_iters, done.data(), c.iters, c.status, b);
  return 0;
}

// f64 = 0: the fp32 loops (dt and the thresholds rounded to float), f64 = 1: the ...64 ones.  placement: [B][F][7] in q's element
// type, or null; hold: [B][T][F + C + P] bytes (track only), or null; enabled / dmin / ddet as in emu_coll_call.
extern "C" int emu_loop_placed(void* prob, int f64, int f32k1, int track, int B, int T, void* q, const void* ftgt, const void* ptgt, int pbatched,
                               const void* ctgt, const uint8_t* enabled, const void* dmin, const void* ddet, const uint8_t* hold,
                               const void* placement, const int32_t* lengths, double dt, double damping, int max_iters, double pos, double ori,
                               void* q_traj, int32_t* iters, int32_t* status, int32_t* passes) {
  if (!f64) { dt = (float)dt; pos = (float)pos; ori = (float)ori; }
  const PHeader& h = PView{static_cast<EmuProblem*>(prob)->image.data()}.h();
  if (placement && h.F == 0) { g_err = "placement given for a problem without a FrameTask or RelativeFrameTask"; return -1; }   // check_inputs
  bik_inputs in;
  memset(&in, 0, sizeof in);
  in.q = q; in.frame_targets = ftgt; in.posture_targets = ptgt; in.com_targets = ctgt; in.posture_batched = pbatched; in.f64 = f64;
  ConvCall c;
  memset(&c, 0, sizeof c);
  c.B = B; c.T = track ? T : 1; c.max_iters = max_iters; c.dt = dt; c.pos = pos; c.ori = ori; c.damping = damping; c.q = q; c.in = &in;
  c.iters = iters; c.status = status; c.track = track != 0; c.io64 = f64 != 0;
  if (track) { c.lengths = lengths; c.q_traj = q_traj; c.hold = hold; }
  c.coll.enabled = enabled; c.coll.minimum_distance = dmin; c.coll.detection_distance = ddet;
  c.placement = placement;
  return emu_placed_loop(static_cast<EmuProblem*>(prob), c, f32k1, passes);
}

// bik_step_placed / bik_step_coll (null placement) on host buffers, what the driver's step_core runs: nsteps of K1 (packed
// hand-off, fused check_limits) and K2 (solve, integrate into q when `integrate`).  dq [B][nv] in q's element type.
extern "C" int emu_step_placed(void* prob, int f64, int f32k1, int B, void* q, const void* ftgt, const void* ptgt, int pbatched, const void* ctgt,
                               const uint8_t* enabled, const void* dmin, const void* ddet, const void* placement, double dt, double damping,
                               int nsteps, int integrate, void* dq, int32_t* status) {
  EmuProblem* p = static_cast<EmuProblem*>(prob);
  const PView P{p->image.data()};
  const PHeader& h = P.h();
  if (placement && h.F == 0) { g_err = "placement given for a problem without a FrameTask or RelativeFrameTask"; return -1; }
  if (!f64) dt = (float)dt;
  const bool k1d = f64 || (!f32k1 && k1_auto_double(h, p->k1cond, damping));
  const HandoffSizes n = handoff_sizes(h);
  std::vector<double> pk((size_t)B * n.pk), Gc((size_t)B * n.Gc), hc((size_t)B * n.hc), wsm(k1_warp_words(h, 1) + 16);
  std::vector<signed char> warm((size_t)B * n.warm);
  const int path = emu_k2_path(h);
  for (int s = 0; s < nsteps; ++s) {
    K1PArgs a;
    memset(&a, 0, sizeof a);
    a.B = B; a.q = q; a.ftgt = ftgt; a.ptgt = ptgt; a.ctgt = ctgt; a.in64 = f64; a.pbatched = pbatched;
    a.dt = dt; a.pk = pk.data(); a.Gc = Gc.data(); a.hc = hc.data();
    a.status = status; a.accumulate = s > 0; a.tol = 1e-6f;
    a.enabled = enabled; a.dmin = dmin; a.ddet = ddet; a.placement = placement;
    if (placement) {
      if (k1d) emu_k1p_pass<double>(P, a, false, false, wsm.data());
      else emu_k1p_pass<float>(P, a, false, false, wsm.data());
    } else if (enabled || dmin || ddet) {
      if (k1d) emu_k1c_pass<double>(P, a, false, wsm.data());
      else emu_k1c_pass<float>(P, a, false, wsm.data());
    } else {
      if (k1d) emu_k1_pass<double>(P, a, false, wsm.data());
      else emu_k1_pass<float>(P, a, false, wsm.data());
    }
    K2Args a2;
    memset(&a2, 0, sizeof a2);
    a2.B = B; a2.q = q; a2.io64 = f64; a2.pk = pk.data(); a2.pk64 = k1d; a2.ptgt = ptgt; a2.pbatched = pbatched;
    a2.Gc = Gc.data(); a2.hc = hc.data(); a2.gc64 = k1d; a2.dt = dt; a2.damping = damping; a2.dq = dq; a2.integrate = integrate; a2.status = status;
    a2.warm = nsteps > 1 ? warm.data() : nullptr;
    if (emu_k2(P, a2, path)) return -1;
  }
  return 0;
}
