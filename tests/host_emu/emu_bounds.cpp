// TEST INFRASTRUCTURE -- the host emulation (emu.cpp) plus the pass loops of bik_converge_bounded / bik_track_bounded
// (per-instance bounds, K2BdArgs).  With bounds K2 runs the BD instantiations of both paths (k2t_warp_tile<..., PW, BD = true>,
// k2_warp<..., PW, BD = true>); without them it runs what the ..._weighted_ex loops run, posture-weighted or not, as the driver's
// converge_pass picks.  Built as its own library so that emu.cpp keeps its entry points as they are; every emu_* function of
// emu.cpp is exported from it as well.  Never shipped, never loaded by mink_b200/.
#include "emu.cpp"

// K2 of one pass, the instantiation launch_k2t / launch_k2 picks for the argument type A (K2Args, K2PwArgs or K2BdArgs):
// run-time I/O form, or the fp32 step form.  path: 1 general, 3 small-group, 8 small-group with 64-bit masks.
template <typename M, bool PW, bool BD>
static void emu_k2t_as(const PView& P, const K2Args& a, double* tw) {
  const bool step = !a.pk64 && !a.io64;
  for (int b = 0; b < a.B; ++b) {
    if (step) k2t_warp_tile<double, 1, 1, M, true, true, PW, BD>(P, a, b, tw, 0);
    else k2t_warp_tile<double, 1, 1, M, false, false, PW, BD>(P, a, b, tw, 0);
  }
}
template <bool PW, bool BD>
static int emu_k2_as(const PView& P, const K2Args& a, int path) {
  if (path == 3 || path == 8) {
    std::vector<double> tw(k2t_warp_bytes(P, 8, 1) / 8 + 16);
    if (path == 3) emu_k2t_as<uint32_t, PW, BD>(P, a, tw.data());
    else emu_k2t_as<uint64_t, PW, BD>(P, a, tw.data());
    return 0;
  }
  std::vector<double> wsm(k2_warp_bytes(P.h(), 8) / 8 + 16);
  for (int b = 0; b < a.B; ++b) k2_warp<double, 1, 65, PW, BD>(P, a, b, wsm.data(), 0);
  return 0;
}

// path: 0 the device's choice (emu_k2_path), 1 the general path (what BIK_K2_PATH=dense selects).  K1's precision for fp32 callers
// follows the posture weights alone (k1_auto_double): bounds do not enter it.
static int emu_bd_loop(EmuProblem* p, ConvCall c, int path, int32_t* passes) {
  const PView P{p->image.data()};
  const PHeader& h = P.h();
  const size_t B = c.B;
  const HandoffSizes n = handoff_sizes(h);
  c.k1d = c.io64 || k1_auto_double(h, p->k1cond, c.damping, c.posture_weights != nullptr);
  std::vector<double> pk(B * n.pk), Gc(B * n.Gc), hc(B * n.hc), dq(B * h.nv), wsm(k1_warp_words(h, 1) + 16);
  std::vector<double> ptcur(posture_seq(c.in) ? B * h.P * h.nq : 0);
  std::vector<signed char> warm(B * n.warm);
  std::vector<int32_t> done(B), cursor(B), step(B), status(B);
  int count[3];
  const ConvBufs s{pk.data(), Gc.data(), hc.data(), dq.data(), warm.data(), done.data(), cursor.data(), step.data(), status.data(), count,
                   ptcur.data()};
  for (int b = 0; b < c.B; ++b) conv_reset(c.track, c.T, c.lengths, s, b);
  const K1Args a1 = conv_k1_args(c, s, c.status);
  const K2Args a2 = conv_k2_args(c, s, c.status);
  const K2PwArgs a2w = conv_k2_pw_args(c, s, c.status);
  const K2BdArgs a2b = conv_k2_bd_args(c, s, c.status);
  if (path == 0) path = emu_k2_path(h);
  for (int go = 1; go;) {
    conv_tick(c.track, count);
    if (c.k1d) emu_k1_pass<double>(P, a1, c.track, wsm.data());
    else emu_k1_pass<float>(P, a1, c.track, wsm.data());
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
// weights: [B][K] / [B][T][K], posture_weights: [B][P][nv] / [B][T][P][nv], lower / upper / vmax: [B][nv], all in q's element
// type or null.
static int emu_bd_call(void* prob, int f64, bool track, int path, int B, int T, void* q, const void* ftgt, const void* ptgt, int pbatched,
                       const void* ctgt, const void* weights, const void* posture_weights, const void* lower, const void* upper,
                       const void* vmax, const int32_t* lengths, double dt, double damping, int max_iters, double pos, double ori,
                       void* q_traj, int32_t* iters, int32_t* status, int32_t* passes) {
  if (!f64) { dt = (float)dt; pos = (float)pos; ori = (float)ori; }
  const PHeader& h = PView{static_cast<EmuProblem*>(prob)->image.data()}.h();
  if (((lower || upper) && h.ncfg == 0) || (vmax && !h.has_vel)) { g_err = "bounds without the matching limit"; return -1; }   // check_inputs
  bik_inputs in;
  memset(&in, 0, sizeof in);
  in.q = q; in.frame_targets = ftgt; in.posture_targets = ptgt; in.com_targets = ctgt; in.posture_batched = pbatched; in.f64 = f64;
  ConvCall c;
  memset(&c, 0, sizeof c);
  c.B = B; c.T = T; c.max_iters = max_iters; c.dt = dt; c.pos = pos; c.ori = ori; c.damping = damping; c.q = q; c.in = &in;
  c.lengths = lengths; c.q_traj = q_traj; c.iters = iters; c.status = status; c.track = track; c.io64 = f64 != 0; c.weights = weights;
  c.posture_weights = posture_weights;
  c.bounds.lower = lower; c.bounds.upper = upper; c.bounds.vmax = vmax;
  return emu_bd_loop(static_cast<EmuProblem*>(prob), c, path, passes);
}
extern "C" int emu_converge_bd(void* prob, int f64, int path, int B, void* q, const void* ftgt, const void* ptgt, int pbatched, const void* ctgt,
                               const void* weights, const void* posture_weights, const void* lower, const void* upper, const void* vmax,
                               double dt, double damping, int max_iters, double pos, double ori, int32_t* iters, int32_t* status) {
  return emu_bd_call(prob, f64, false, path, B, 1, q, ftgt, ptgt, pbatched, ctgt, weights, posture_weights, lower, upper, vmax, nullptr, dt, damping,
                     max_iters, pos, ori, nullptr, iters, status, nullptr);
}
extern "C" int emu_track_bd(void* prob, int f64, int path, int B, int T, void* q, const void* ftgt, const void* ptgt, int pbatched, const void* ctgt,
                            const void* weights, const void* posture_weights, const void* lower, const void* upper, const void* vmax,
                            const int32_t* lengths, double dt, double damping, int max_iters, double pos, double ori, void* q_traj,
                            int32_t* iters, int32_t* status, int32_t* passes) {
  return emu_bd_call(prob, f64, true, path, B, T, q, ftgt, ptgt, pbatched, ctgt, weights, posture_weights, lower, upper, vmax, lengths, dt, damping,
                     max_iters, pos, ori, q_traj, iters, status, passes);
}
