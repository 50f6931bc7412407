// TEST INFRASTRUCTURE -- the host emulation (emu.cpp, emu_bounds.cpp, emu_collision.cpp) plus the pass loop of bik_track_hold
// (held targets, K1HArgs).  With a hold mask K1 runs the HO instantiation (k1_warp_tile<..., TR, CO, HO = true>, what
// k1h_kernel runs), with or without collision arguments; K2 reads each instance's posture targets from ptcur.  Built as its own
// library so that the other emulation units keep their entry points as they are; every emu_* function of theirs is exported
// from it as well.  Never shipped, never loaded by mink_b200/.
#include "emu_collision.cpp"

template <typename T, bool CO>
static void emu_k1h_pass(const PView& P, const K1HArgs& a, double* wsm) {
  for (int b = 0; b < a.B; ++b) k1_warp_tile<T, 1, 1, true, true, CO, true>(P, a, b, reinterpret_cast<T*>(wsm), 0);
}

// The bik_track_hold loop; a null hold runs the bik_track_coll loop (emu_collision.cpp).  f32k1 as in emu_coll_loop.
static int emu_hold_loop(EmuProblem* p, ConvCall c, int f32k1, int32_t* passes) {
  if (!c.hold) return emu_coll_loop(p, c, f32k1, passes);
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
  const K1HArgs a1 = conv_k1h_args(c, s, c.status);
  const K2Args a2 = conv_k2_args(c, s, c.status);
  const K2PwArgs a2w = conv_k2_pw_args(c, s, c.status);
  const int path = emu_k2_path(h);
  for (int go = 1; go;) {
    conv_tick(c.track, count);
    if (has_coll(c.coll)) {
      if (c.k1d) emu_k1h_pass<double, true>(P, a1, wsm.data());
      else emu_k1h_pass<float, true>(P, a1, wsm.data());
    } else {
      if (c.k1d) emu_k1h_pass<double, false>(P, a1, wsm.data());
      else emu_k1h_pass<float, false>(P, a1, wsm.data());
    }
    go = conv_cond(c.track, c.max_iters, count);
    if (!go) break;
    if (c.posture_weights) emu_k2_as<true, false>(P, a2w, path);
    else if (emu_k2(P, a2, path)) return -1;
  }
  *passes = count[0];
  return 0;
}

// bik_track_hold / bik_track_hold64 (f64) on host buffers: the arguments of emu_track_coll, plus hold [B][T][F + C + P] bytes
// (or null).  pbatched: bik_inputs.posture_batched (0 / 1, or a sequence: 2 / 3).
extern "C" int emu_track_hold(void* prob, int f64, int f32k1, int B, int T, void* q, const void* ftgt, const void* ptgt, int pbatched,
                              const void* ctgt, const void* posture_weights, const uint8_t* enabled, const void* dmin, const void* ddet,
                              const uint8_t* hold, const int32_t* lengths, double dt, double damping, int max_iters, double pos, double ori,
                              void* q_traj, int32_t* iters, int32_t* status, int32_t* passes) {
  if (!f64) { dt = (float)dt; pos = (float)pos; ori = (float)ori; }
  bik_inputs in;
  memset(&in, 0, sizeof in);
  in.q = q; in.frame_targets = ftgt; in.posture_targets = ptgt; in.com_targets = ctgt; in.posture_batched = pbatched; in.f64 = f64;
  ConvCall c;
  memset(&c, 0, sizeof c);
  c.B = B; c.T = T; c.max_iters = max_iters; c.dt = dt; c.pos = pos; c.ori = ori; c.damping = damping; c.q = q; c.in = &in;
  c.lengths = lengths; c.q_traj = q_traj; c.iters = iters; c.status = status; c.track = true; c.io64 = f64 != 0;
  c.posture_weights = posture_weights;
  c.coll.enabled = enabled; c.coll.minimum_distance = dmin; c.coll.detection_distance = ddet;
  c.hold = hold;
  return emu_hold_loop(static_cast<EmuProblem*>(prob), c, f32k1, passes);
}

// The pose of a frame in its root as a held RELATIVE_FRAME task captures it (held_relative), from the two world poses [B][7]
// (wxyz, xyz) that bik_fk reports; f64 selects the element type.
extern "C" void emu_relative_pose(int f64, int B, const void* root, const void* frame, void* out) {
  for (int b = 0; b < B; ++b) {
    auto run = [&](auto zero) {
      using T = decltype(zero);
      const T* r = static_cast<const T*>(root) + 7 * b;
      const T* f = static_cast<const T*>(frame) + 7 * b;
      Q4<T> q; V3<T> p;
      held_relative<T>(q4<T>(r[0], r[1], r[2], r[3]), v3<T>(r[4], r[5], r[6]), q4<T>(f[0], f[1], f[2], f[3]), v3<T>(f[4], f[5], f[6]), &q, &p);
      T* o = static_cast<T*>(out) + 7 * b;
      o[0] = q.w; o[1] = q.x; o[2] = q.y; o[3] = q.z; o[4] = p.x; o[5] = p.y; o[6] = p.z;
    };
    if (f64) run(0.0); else run(0.0f);
  }
}
