// TEST INFRASTRUCTURE -- the host emulation (emu.cpp) plus the pass loop of bik_track with a posture target sequence
// (bik_inputs.posture_batched = BIK_POSTURE_SEQ_SHARED / BIK_POSTURE_SEQ_BATCHED).  The loop is emu.cpp's with one more buffer,
// ConvBufs::ptcur, the [B][P][nq] posture targets of each instance's current frame that K1 fills and K2 reads.  Built as its own
// library so that emu.cpp keeps its entry points as they are; every emu_* function of emu.cpp is exported from it as well.
// Never shipped, never loaded by mink_b200/.
#include "emu.cpp"

static int emu_posture_loop(EmuProblem* p, ConvCall c, int32_t* passes) {
  const PView P{p->image.data()};
  const PHeader& h = P.h();
  const size_t B = c.B;
  const HandoffSizes n = handoff_sizes(h);
  c.k1d = c.io64 || k1_auto_double(h, p->k1cond, c.damping);
  // hand-off rows, dq and ptcur sized for fp64 elements whatever the precision
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
  const int path = emu_k2_path(h);
  for (int go = 1; go;) {
    conv_tick(c.track, count);
    if (c.k1d) emu_k1_pass<double>(P, a1, c.track, wsm.data());
    else emu_k1_pass<float>(P, a1, c.track, wsm.data());
    go = conv_cond(c.track, c.max_iters, count);
    if (go && emu_k2(P, a2, path)) return -1;
  }
  *passes = count[0];
  return 0;
}

// bik_track (f64 = 0: fp32 buffers, dt and the thresholds rounded to float as their parameters are) or bik_track64 (f64 = 1).
// pbatched: bik_inputs.posture_batched, the sequence forms 2 ([T][P][nq]) and 3 ([B][T][P][nq]) included.  weights: [B][T][K]
// in q's element type, or null.
extern "C" int emu_track_posture(void* prob, int f64, int B, int T, void* q, const void* ftgt, const void* ptgt, int pbatched, const void* ctgt,
                                 const void* weights, const int32_t* lengths, double dt, double damping, int max_iters, double pos, double ori,
                                 void* q_traj, int32_t* iters, int32_t* status, int32_t* passes) {
  if (!f64) { dt = (float)dt; pos = (float)pos; ori = (float)ori; }
  bik_inputs in;
  memset(&in, 0, sizeof in);
  in.q = q; in.frame_targets = ftgt; in.posture_targets = ptgt; in.com_targets = ctgt; in.posture_batched = pbatched; in.f64 = f64;
  ConvCall c;
  memset(&c, 0, sizeof c);
  c.B = B; c.T = T; c.max_iters = max_iters; c.dt = dt; c.pos = pos; c.ori = ori; c.damping = damping; c.q = q; c.in = &in;
  c.lengths = lengths; c.q_traj = q_traj; c.iters = iters; c.status = status; c.track = true; c.io64 = f64 != 0; c.weights = weights;
  return emu_posture_loop(static_cast<EmuProblem*>(prob), c, passes);
}
