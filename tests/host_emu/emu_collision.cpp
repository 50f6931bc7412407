// TEST INFRASTRUCTURE -- the host emulation (emu.cpp) plus the pass loops of bik_converge_coll / bik_track_coll (per-instance
// collision pairs and distances, K1CArgs).  With collision arguments K1 runs the CO instantiation (k1_warp_tile<..., PK, TR,
// CO = true>, what k1c_kernel runs); K2 runs what the ..._bounded loops run, bounded, posture-weighted or not, as the driver's
// converge_pass picks.  Built as its own library so that emu.cpp and emu_bounds.cpp keep their entry points as they are; every
// emu_* function of both is exported from it as well.  Never shipped, never loaded by mink_b200/.
#include "emu_bounds.cpp"

template <typename T>
static void emu_k1c_pass(const PView& P, const K1CArgs& a, bool track, double* wsm) {
  for (int b = 0; b < a.B; ++b) {
    if (track) k1_warp_tile<T, 1, 1, true, true, true>(P, a, b, reinterpret_cast<T*>(wsm), 0);
    else k1_warp_tile<T, 1, 1, true, false, true>(P, a, b, reinterpret_cast<T*>(wsm), 0);
  }
}

// f32k1: K1 in fp32 for fp32 callers (what BIK_K1_PRECISION=f32 selects), else the driver's choice.
static int emu_coll_loop(EmuProblem* p, ConvCall c, int f32k1, int32_t* passes) {
  const PView P{p->image.data()};
  const PHeader& h = P.h();
  const size_t B = c.B;
  const HandoffSizes n = handoff_sizes(h);
  c.k1d = c.io64 || (!f32k1 && k1_auto_double(h, p->k1cond, c.damping, c.posture_weights != nullptr));
  std::vector<double> pk(B * n.pk), Gc(B * n.Gc), hc(B * n.hc), dq(B * h.nv), wsm(k1_warp_words(h, 1) + 16);
  std::vector<double> ptcur(posture_seq(c.in) ? B * h.P * h.nq : 0);
  std::vector<signed char> warm(B * n.warm);
  std::vector<int32_t> done(B), cursor(B), step(B), status(B);
  int count[3];
  const ConvBufs s{pk.data(), Gc.data(), hc.data(), dq.data(), warm.data(), done.data(), cursor.data(), step.data(), status.data(), count,
                   ptcur.data()};
  for (int b = 0; b < c.B; ++b) conv_reset(c.track, c.T, c.lengths, s, b);
  const K1Args a1 = conv_k1_args(c, s, c.status);
  const K1CArgs a1c = conv_k1c_args(c, s, c.status);
  const K2Args a2 = conv_k2_args(c, s, c.status);
  const K2PwArgs a2w = conv_k2_pw_args(c, s, c.status);
  const K2BdArgs a2b = conv_k2_bd_args(c, s, c.status);
  const int path = emu_k2_path(h);
  for (int go = 1; go;) {
    conv_tick(c.track, count);
    if (has_coll(c.coll)) {
      if (c.k1d) emu_k1c_pass<double>(P, a1c, c.track, wsm.data());
      else emu_k1c_pass<float>(P, a1c, c.track, wsm.data());
    } else {
      if (c.k1d) emu_k1_pass<double>(P, a1, c.track, wsm.data());
      else emu_k1_pass<float>(P, a1, c.track, wsm.data());
    }
    go = conv_cond(c.track, c.max_iters, count);
    if (!go) break;
    if (has_bounds(c.bounds)) emu_k2_as<true, true>(P, a2b, path);
    else if (c.posture_weights) emu_k2_as<true, false>(P, a2w, path);
    else if (emu_k2(P, a2, path)) return -1;
  }
  if (c.track) *passes = count[0];
  else for (int b = 0; b < c.B; ++b) conv_finish(c.max_iters, done.data(), c.iters, c.status, b);
  return 0;
}

// f64 = 0: the fp32 loops (dt and the thresholds rounded to float, as their parameters are), f64 = 1: the ...64 ones.
// enabled: [B][npairs] / [B][T][npairs] bytes; dmin / ddet: [B] / [B][T] in q's element type; each may be null.
static int emu_coll_call(void* prob, int f64, int f32k1, bool track, int B, int T, void* q, const void* ftgt, const void* ptgt, int pbatched,
                         const void* ctgt, const void* posture_weights, const uint8_t* enabled, const void* dmin, const void* ddet,
                         const int32_t* lengths, double dt, double damping, int max_iters, double pos, double ori, void* q_traj,
                         int32_t* iters, int32_t* status, int32_t* passes) {
  if (!f64) { dt = (float)dt; pos = (float)pos; ori = (float)ori; }
  const PHeader& h = PView{static_cast<EmuProblem*>(prob)->image.data()}.h();
  if ((enabled || dmin || ddet) && h.npairs == 0) { g_err = "coll given for a problem without a CollisionAvoidanceLimit"; return -1; }   // check_inputs
  bik_inputs in;
  memset(&in, 0, sizeof in);
  in.q = q; in.frame_targets = ftgt; in.posture_targets = ptgt; in.com_targets = ctgt; in.posture_batched = pbatched; in.f64 = f64;
  ConvCall c;
  memset(&c, 0, sizeof c);
  c.B = B; c.T = T; c.max_iters = max_iters; c.dt = dt; c.pos = pos; c.ori = ori; c.damping = damping; c.q = q; c.in = &in;
  c.lengths = lengths; c.q_traj = q_traj; c.iters = iters; c.status = status; c.track = track; c.io64 = f64 != 0;
  c.posture_weights = posture_weights;
  c.coll.enabled = enabled; c.coll.minimum_distance = dmin; c.coll.detection_distance = ddet;
  return emu_coll_loop(static_cast<EmuProblem*>(prob), c, f32k1, passes);
}
extern "C" int emu_converge_coll(void* prob, int f64, int f32k1, int B, void* q, const void* ftgt, const void* ptgt, int pbatched, const void* ctgt,
                                 const void* posture_weights, const uint8_t* enabled, const void* dmin, const void* ddet, double dt, double damping,
                                 int max_iters, double pos, double ori, int32_t* iters, int32_t* status) {
  return emu_coll_call(prob, f64, f32k1, false, B, 1, q, ftgt, ptgt, pbatched, ctgt, posture_weights, enabled, dmin, ddet, nullptr, dt, damping,
                       max_iters, pos, ori, nullptr, iters, status, nullptr);
}
extern "C" int emu_track_coll(void* prob, int f64, int f32k1, int B, int T, void* q, const void* ftgt, const void* ptgt, int pbatched,
                              const void* ctgt, const void* posture_weights, const uint8_t* enabled, const void* dmin, const void* ddet,
                              const int32_t* lengths, double dt, double damping, int max_iters, double pos, double ori, void* q_traj,
                              int32_t* iters, int32_t* status, int32_t* passes) {
  return emu_coll_call(prob, f64, f32k1, true, B, T, q, ftgt, ptgt, pbatched, ctgt, posture_weights, enabled, dmin, ddet, lengths, dt, damping,
                       max_iters, pos, ori, q_traj, iters, status, passes);
}

// One K1 of a step (packed hand-off, fused check_limits) with collision arguments: the collision rows it hands K2.
// f64 = 1: fp64 instantiation on fp64 inputs, 2: fp64 instantiation on fp32 inputs, 0: fp32.  Gc / hc: fp64 when f64, else fp32.
extern "C" int emu_k1_coll(void* prob, int B, int f64, const void* q, const void* ftgt, const void* ptgt, int pbatched, const void* ctgt, double dt,
                           const uint8_t* enabled, const void* dmin, const void* ddet, void* pk, void* Gc, void* hc, int32_t* status) {
  EmuProblem* p = static_cast<EmuProblem*>(prob);
  PView P{p->image.data()};
  K1CArgs a;
  memset(&a, 0, sizeof a);
  a.B = B; a.q = q; a.ftgt = ftgt; a.ptgt = ptgt; a.ctgt = ctgt; a.in64 = f64 == 1; a.pbatched = pbatched; a.dt = dt;
  a.Gc = Gc; a.hc = hc; a.pk = pk; a.status = status; a.tol = 1e-6f;
  a.enabled = enabled; a.dmin = dmin; a.ddet = ddet;
  std::vector<double> wsm(k1_warp_words(P.h(), 1) + 16);
  for (int b = 0; b < B; ++b) {
    if (f64) k1_warp_tile<double, 1, 1, true, false, true>(P, a, b, wsm.data(), 0);
    else k1_warp_tile<float, 1, 1, true, false, true>(P, a, b, reinterpret_cast<float*>(wsm.data()), 0);
  }
  return 0;
}
