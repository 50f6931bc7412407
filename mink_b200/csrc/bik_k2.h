// bik_k2.h -- K2: per-instance QP assembly and exact solve, one warp per problem (the general path: collision rows,
// any number of coupled dofs; box-only problems with at most 64 coupled dofs take the small-group path of bik_k2t.h).
//
//   H = damping I + sum_t (W_t J_t)^T (W_t J_t) + mu_t I,   c = sum_t -(W_t(-gain_t e_t))^T W_t J_t
//       (reference mink/tasks/task.py:105-138, mink/solve_ik.py:13-22)
//   min 1/2 dq^T H dq + c^T dq   s.t.  lo <= dq <= hi  [+ general rows G dq <= h]
//       (reference mink/solve_ik.py:43-65,101 -> qpsolvers)
//
// Structure exploited (SURVEY.md 8): frame-task Jacobians only have their ancestor-dof columns
// non-zero, so each task adds a small dense block to H; the posture task is a diagonal; configuration
// and velocity limits share their index set and collapse to one box per dof.
//
// Task rows arrive either packed (K1's hand-off inside bik_step: per task the non-zero columns, [ncols][6] + e[6], fp32
// or fp64) or dense (bik_solve: what Task.compute_jacobian returns).
//
// Solver, two phases, same KKT point (the optimum quadprog / daqp return for the strictly convex QP):
//   1. block principal pivoting (Kunisch-Rendl infeasible active set): guess the active set -- inside a rollout the
//      previous step's --, solve the reduced system with a fresh packed Cholesky of the free block, flip every violated
//      index at once.  Usually 2-4 iterations, 1-2 when warm-started; it has no descent property and stalls on a few
//      instances per thousand once a rollout is under way.
//   2. when the number of infeasibilities has not improved for PATIENCE iterations: a primal active-set method from the
//      feasible point clip(0, lo, hi) (dq = 0 satisfies every limit of a configuration inside its limits: h >= 0 for the
//      collision rows, collision_avoidance_limit.py:203).  Each iteration solves for the minimiser of the current working
//      set, moves the feasible iterate towards it until the first bound or general row blocks (ratio test), adds that
//      constraint; at a feasible subspace minimiser it drops the constraint with the most negative multiplier or stops.
//      The objective decreases monotonically, so it terminates.
// General rows (collision) enter both phases through a Schur complement on the factor.
//
// Lanes own rows (row i -> lane i % W); reductions over lanes use shuffles.  W = 1 on the host.
#pragma once
#include "bik_k1.h"

#if defined(__CUDACC__)
#define BIK_NOINLINE __host__ __device__ __noinline__
// Out-of-line helpers receive generic pointers; telling the compiler they point into shared memory turns their LD.E/ST.E
// (two R2UR descriptor moves each) into LDS/STS.
#if defined(__CUDA_ARCH__)
#define BIK_IN_SHARED(p) __builtin_assume(__isShared(p))
#else
#define BIK_IN_SHARED(p) ((void)0)
#endif
#else
#define BIK_NOINLINE __attribute__((noinline))
#define BIK_IN_SHARED(p) ((void)0)
#endif

namespace bik {

struct K2Args {
  int B;
  const void* q;       // [B][nq]; fp64 when io64
  int io64;            // q, posture targets and dq are fp64 (else fp32)
  // task rows, one of two forms
  const void* pk;      // packed K1 hand-off [B][pk_stride] (fp64 when pk64), or null
  int pk64;
  const void* J;       // dense [B][K][nv]   (bik_solve / bik_qp_objective); fp64 when dense64
  const void* e;       // dense [B][K]
  const void* ep;      // dense [B][P][nv]; null: the posture error is computed from q and ptgt
  int dense64;
  const void* ptgt;    // [B or 1][P][nq] posture targets (dtype follows io64)
  int pbatched;
  const void* Gc;      // [B][npairs][nv], [B][npairs] collision rows (fp64 when gc64)
  const void* hc;
  int gc64;
  double dt;
  double damping;
  void* dq;            // [B][nv]
  int integrate;       // q <- q (+) dq in place after the solve (Configuration.integrate_inplace, configuration.py:228-236)
  int32_t* status;     // [B] or null (OR-ed into)
  int32_t* iters;      // [B] or null: factorisations per instance (diagnostics)
  double* Hout;        // [B][nv][nv] or null  (bik_qp_objective)
  double* cout;        // [B][nv] or null
  void* lo_out;        // [B][nv] or null      (bik_limits_box; dtype follows io64)
  void* hi_out;
  int skip_objective;  // bik_limits_box: task rows are not read
  int skip_box;        // bik_qp_objective: q is not read
  signed char* warm;   // [B][nu] or null: active-set guess in (0 free, 1 lower, 2 upper; +4 = dq still holds the previous step's result), read at entry, updated at exit
  const int32_t* skip; // [B] or null: instances marked here are neither solved nor integrated (bik_converge: already converged)
  const int* gate;     // device flag or null: the whole launch is a no-op when it reads 0 (bik_converge's last pass through the graph body)
};
// The arguments of the posture-weighted instantiations (PW; the ..._weighted_ex entry points): K2Args and the per-instance
// posture weights.  A struct of its own, so that the kernels without posture weights keep their parameter block as it is.
struct K2PwArgs : K2Args {
  // [B][P][nv], element type follows io64.  Track mode: [B][T][P][nv], row b*pw_T + pw_cursor[b] -- K1 ends a frame in the pass
  // that moves the cursor and leaves the instance out of that pass's K2, so whenever K2 solves b the cursor names the frame
  // being solved.
  const void* pw;
  const int32_t* pw_cursor;   // [B] or null (step / converge)
  int pw_T;
};
// The arguments of the bounded instantiations (BD; the ..._bounded entry points): K2PwArgs, whose posture weights may be null
// here, and the per-instance bounds.  Each is [B][nv] or null, element type follows io64; in track mode too, row b holds on
// every frame.  They narrow the problem's ConfigurationLimit bounds and VelocityLimit caps (box_dof).
struct K2BdArgs : K2PwArgs {
  const void* lower;
  const void* upper;
  const void* vmax;
};

enum { K2_MAX_GEN = 24 };  // general (collision) rows that may be active at once; more than that sets BIK_STATUS_QP_MAXITER

BIK_HD int tri(int i) { return (i * (i + 1)) >> 1; }

BIK_HD int k2_max_gen(const PHeader& h) { return h.npairs < K2_MAX_GEN ? h.npairs : K2_MAX_GEN; }
// General rows whose h is finite (pairs inside the detection distance) are gathered into a window of at most this many rows per
// problem; everything the solver keeps per row is sized by the window, not by the number of pairs (ALOHA: 1 104 pairs, a
// dozen inside the detection distance).  More finite rows than the window sets BIK_STATUS_QP_MAXITER.
enum { K2_ROW_WINDOW = 64 };
BIK_HD int k2_row_cap(const PHeader& h) { return h.npairs < K2_ROW_WINDOW ? h.npairs : K2_ROW_WINDOW; }
// per-warp scratch, in bytes, for scalar type of size `ts`.
// Layout: Hp | dinv c lo hi x xf xfull | [general-row block] | U | ints.   U is a union: during assembly it
// holds the weighted task blocks (packed layout), afterwards the packed factor augmented by the rhs row.
BIK_HD int k2_union_bytes(const PHeader& h, int ts) {
  int n = h.nu;
  int lp = tri(n + 1) * ts + 16;                       // (n+1) rows: factor + fused right-hand side
  int wj = (h.pk_stride > 0 ? h.pk_stride : 4) * ts + 16;
  return ((lp > wj ? lp : wj) + 15) & ~15;
}
BIK_HD int k2_warp_bytes(const PHeader& h, int ts) {
  int n = h.nu, np = h.npairs, mg = k2_max_gen(h), rc = k2_row_cap(h);
  int words_T = tri(n) + 6 * n + h.nv + (np > 0 ? (mg * n + mg * mg + 2 * mg + rc) : 0);
  int bytes = ((words_T * ts + 15) & ~15) + k2_union_bytes(h, ts) + 4 * (2 * n + 4 * rc + 20);
  return (bytes + 15) & ~15;
}

template <typename T> BIK_HD T bik_rsqrt(T x) {
#if defined(__CUDA_ARCH__)
  return rsqrt(x);
#else
  return T(1) / sqrt(x);
#endif
}

// The lanes of one problem are W consecutive lanes of a warp (W = 32: the whole warp; W = 1 on the host).  Sub-warp groups
// synchronise and shuffle among themselves only, so the groups of one warp may run different iteration counts.
template <int W> BIK_HD unsigned k2_gmask() {
#if defined(__CUDA_ARCH__)
  if (W >= 32) return 0xffffffffu;
  unsigned lane32;
  asm("mov.u32 %0, %%laneid;" : "=r"(lane32));
  return (W >= 32 ? 0u : ((1u << (W & 31)) - 1u)) << (lane32 & ~(unsigned)(W - 1));
#else
  return 0u;
#endif
}
template <int W> BIK_HD void k2_sync() {
#if defined(__CUDA_ARCH__)
  __syncwarp(k2_gmask<W>());
#endif
}
template <int W> BIK_HD int warp_sum_i(int v) {
#if defined(__CUDA_ARCH__)
  const unsigned m = k2_gmask<W>();
  for (int o = W / 2; o > 0; o >>= 1) v += __shfl_xor_sync(m, v, o);
#endif
  return v;
}
template <int W> BIK_HD int warp_max_i(int v) {
#if defined(__CUDA_ARCH__)
  const unsigned m = k2_gmask<W>();
  for (int o = W / 2; o > 0; o >>= 1) { int t = __shfl_xor_sync(m, v, o); v = t > v ? t : v; }
#endif
  return v;
}
template <int W> BIK_HD int warp_min_i(int v) { return -warp_max_i<W>(-v); }
template <int W, typename T> BIK_HD T warp_min_t(T v) {
#if defined(__CUDA_ARCH__)
  const unsigned m = k2_gmask<W>();
  for (int o = W / 2; o > 0; o >>= 1) { T t = __shfl_xor_sync(m, v, o); v = t < v ? t : v; }
#endif
  return v;
}
template <int W, typename T> BIK_HD T warp_sum_t(T v) {
#if defined(__CUDA_ARCH__)
  const unsigned m = k2_gmask<W>();
  for (int o = W / 2; o > 0; o >>= 1) v += __shfl_xor_sync(m, v, o);
#endif
  return v;
}
template <typename T, int W> BIK_HD T warp_bcast(T v, int src) {   // src: lane within the group
#if defined(__CUDA_ARCH__)
  return __shfl_sync(k2_gmask<W>(), v, src, W);
#else
  (void)src;
  return v;
#endif
}

template <typename T> struct K2Ws {
  T *Hp, *Lp, *dinv, *c, *lo, *hi, *x, *xf, *xfull;
  T *Y, *S, *lam, *rg, *hg;            // general rows: Y = L^-1 G_F^T (maxg x n), S Schur, lam, rhs, h of the window rows
  int *st, *idx, *gst, *gidx, *gnew, *frow;   // per window row: state, active list, proposed state, pair index of the row
  int nrows;                           // rows in the window (set by k2_solve)
  T *wpk;                              // weighted task blocks in the packed layout (aliases Lp)
};
template <typename T> BIK_HD K2Ws<T> k2_carve(const PHeader& h, void* mem) {
  K2Ws<T> w;
  int n = h.nu, np = h.npairs, mg = k2_max_gen(h), rc = k2_row_cap(h);
  w.nrows = 0;
  char* base = reinterpret_cast<char*>(mem);
  BIK_IN_SHARED(base);
  T* p = reinterpret_cast<T*>(base);
  w.Hp = p; p += tri(n);
  w.dinv = p; p += n; w.c = p; p += n; w.lo = p; p += n; w.hi = p; p += n; w.x = p; p += n; w.xf = p; p += n; w.xfull = p; p += h.nv;
  w.Y = w.S = w.lam = w.rg = w.hg = nullptr;
  if (np > 0) { w.Y = p; p += mg * n; w.S = p; p += mg * mg; w.lam = p; p += mg; w.rg = p; p += mg; w.hg = p; p += rc; }
  int words_T = (int)(p - reinterpret_cast<T*>(base));
  char* u = base + ((words_T * (int)sizeof(T) + 15) & ~15);
  w.Lp = reinterpret_cast<T*>(u);
  w.wpk = reinterpret_cast<T*>(u);
  int* ip = reinterpret_cast<int*>(u + k2_union_bytes(h, sizeof(T)));
  w.st = ip; ip += n; w.idx = ip; ip += n; w.gst = ip; ip += rc + 4; w.gidx = ip; ip += rc + 4; w.gnew = ip; ip += rc + 4; w.frow = ip; ip += rc + 4;
  return w;
}

template <typename T> BIK_HD T Hsym(const T* Hp, int i, int j) { return i >= j ? Hp[tri(i) + j] : Hp[tri(j) + i]; }

// ---- per-instance posture weights (K2PwArgs) ---------------------------------------------------------------------------
// instance b's posture weights: its [P][nv] block, or in track mode that of its current frame.  `a` is the K2PwArgs a PW
// instantiation was launched with.
BIK_HD const void* k2_pw_row(const K2Args& a, const PHeader& h, long long b, int is64) {
  const K2PwArgs& pa = static_cast<const K2PwArgs&>(a);
  const long long r = pa.pw_cursor ? b * pa.pw_T + pa.pw_cursor[b] : b;
  return reinterpret_cast<const char*>(pa.pw) + r * h.P * h.nv * (is64 ? 8 : 4);
}
// weight i of pw clamped to [0, 1], NaN to 0; a weight that needed it sets BIK_STATUS_BAD_WEIGHT (32) in *st
template <typename T>
BIK_HD T k2_pw(const void* pw, long long i, int is64, int* st) {
  const T w = ldin<T>(pw, i, is64);
  if (!(w >= T(0) && w <= T(1))) *st |= 32;
  return w >= T(0) ? (w <= T(1) ? w : T(1)) : T(0);
}
// ---- per-instance bounds (K2BdArgs) --------------------------------------------------------------------------------------
// instance b's rows of the bound buffers.  `a` is the K2BdArgs a BD instantiation was launched with.
BIK_HD BoundsRow k2_bd_row(const K2Args& a, int nv, long long b, int is64) {
  const K2BdArgs& ba = static_cast<const K2BdArgs&>(a);
  const long long off = b * nv * (is64 ? 8 : 4);
  auto row = [&](const void* p) -> const void* { return p ? reinterpret_cast<const char*>(p) + off : nullptr; };
  return BoundsRow{row(ba.lower), row(ba.upper), row(ba.vmax), is64};
}

// One task of the stacked objective: rows, non-zero columns and where its block sits in the packed record.
struct K2Task { int row0, nr, nc, coff, pk_off; const float* cost; float gain, lm; };
BIK_HD K2Task k2_task(const PView& P, int t) {
  const PHeader& h = P.h();
  K2Task k;
  if (t < h.F) { const FrameRec& fr = P.frame(t); k.row0 = fr.row0; k.nr = 6; k.nc = fr.ncols; k.coff = fr.col_off; k.pk_off = fr.pk_off; k.cost = fr.cost; k.gain = fr.gain; k.lm = fr.lm; }
  else {
    const float* cr = P.f(h.off_com) + 8 * (t - h.F);
    k.row0 = reinterpret_cast<const int32_t*>(cr)[5]; k.pk_off = reinterpret_cast<const int32_t*>(cr)[6];
    k.nr = 3; k.nc = h.com_ncols; k.coff = h.com_cols_off; k.cost = cr; k.gain = cr[3]; k.lm = cr[4];
  }
  return k;
}

// ---- assembly ------------------------------------------------------------------------------
// PW (compile time): per-instance posture weights (K2PwArgs, which `a` then is): the cost of posture task p on dof d is
// cost_eff[d] * w.
// BD (compile time, with PW): per-instance bounds (K2BdArgs, which `a` then is) narrow the box; the posture weights may be null.
template <typename T, int W, bool PW = false, bool BD = false>
BIK_HD int k2_assemble(const PView& P, const K2Args& a, int b, K2Ws<T>& w, int lane) {
  const PHeader& h = P.h();
  const int n = h.nv, nu = h.nu, K = h.K, nq = h.nq;
  const int32_t* cols = P.i(h.off_cols);
  const int32_t* umap = P.i(h.off_umap);
  const int32_t* dofqadr = P.i(h.off_dofqadr);
  auto qv = [&](int i) { return ldin<T>(a.q, (long long)b * nq + i, a.io64); };
  int status = 0;
  if (a.skip_objective) {  // bik_limits_box: only the box, for every dof
    for (int d = lane; d < n; d += W) {
      T lo, hi;
      const int qa = dofqadr[d];
      box_dof<T>(P, d, qa >= 0 ? qv(qa) : T(0), T(a.dt), &lo, &hi);
      stout<T>(a.lo_out, (long long)b * n + d, a.io64, lo); stout<T>(a.hi_out, (long long)b * n + d, a.io64, hi);
    }
    return 0;
  }
  for (int k = lane; k < tri(nu); k += W) w.Hp[k] = T(0);
  for (int k = lane; k < nu; k += W) w.c[k] = T(0);
  // weighted task blocks in the packed layout:  [ia][r] = cost_r J[row0+r][col_ia],  then  cost_r (-gain e[row0+r])
  for (int t = 0; t < h.F + h.C; ++t) {
    const K2Task tk = k2_task(P, t);
    const int nj = tk.nr * tk.nc;
    for (int k = lane; k < nj + tk.nr; k += W) {
      const int ia = k / tk.nr, r = k - ia * tk.nr;
      T v;
      if (a.pk) v = ldin<T>(a.pk, (long long)b * h.pk_stride + tk.pk_off + k, a.pk64);
      else if (k < nj) v = ldin<T>(a.J, ((long long)b * K + tk.row0 + r) * n + (cols[tk.coff + ia] & 0xffff), a.dense64);
      else v = ldin<T>(a.e, (long long)b * K + tk.row0 + r, a.dense64);
      w.wpk[tk.pk_off + k] = k < nj ? T(tk.cost[r]) * v : T(tk.cost[r]) * (T(-tk.gain) * v);
    }
  }
  k2_sync<W>();
  // block contributions (W J)^T (W J) and the linear term, lower triangle of the COUPLED block, per task over its non-zero columns
  for (int t = 0; t < h.F + h.C; ++t) {
    const K2Task tk = k2_task(P, t);
    const T* blk = w.wpk + tk.pk_off;
    const T* we = blk + tk.nr * tk.nc;
    for (int p = lane; p < tri(tk.nc); p += W) {   // p = tri(ia) + ib, ib <= ia
      int ia = (int)((bik_sqrt<float>(8.f * (float)p + 1.f) - 1.f) * 0.5f);
      if (tri(ia) > p) --ia; else if (tri(ia + 1) <= p) ++ia;
      const int ib = p - tri(ia);
      T s = T(0);
      for (int r = 0; r < tk.nr; ++r) s += blk[ia * tk.nr + r] * blk[ib * tk.nr + r];
      const int ua = umap[cols[tk.coff + ia] & 0xffff], ub = umap[cols[tk.coff + ib] & 0xffff];   // column lists are ascending: ua >= ub
      w.Hp[tri(ua) + ub] += s;
    }
    for (int ia = lane; ia < tk.nc; ia += W) {
      T cs = T(0);
      for (int r = 0; r < tk.nr; ++r) cs += we[r] * blk[ia * tk.nr + r];
      w.c[umap[cols[tk.coff + ia] & 0xffff]] -= cs;
    }
    k2_sync<W>();
  }
  // Levenberg-Marquardt terms mu_t = lm_t ||W(-gain e)||^2 (task.py:131) -- every lane, same order
  T mu = T(a.damping);
  for (int t = 0; t < h.F + h.C; ++t) {
    const K2Task tk = k2_task(P, t);
    if (tk.lm != 0.f) { const T* we = w.wpk + tk.pk_off + tk.nr * tk.nc; T s = T(0); for (int r = 0; r < tk.nr; ++r) s += we[r] * we[r]; mu += T(tk.lm) * s; }
  }
  auto eperr = [&](int p, int d) -> T {
    if (a.ep) return ldin<T>(a.ep, ((long long)b * h.P + p) * n + d, a.dense64);
    const long long t0 = ((long long)(a.pbatched ? b : 0) * h.P + p) * nq;
    return posture_err_dof<T>(P, d, [&](int i) { return ldin<T>(a.ptgt, t0 + i, a.io64); }, qv);
  };
  const void* pw = nullptr;
  if constexpr (PW) if (!BD || static_cast<const K2PwArgs&>(a).pw) pw = k2_pw_row(a, h, b, a.io64);
  for (int p = 0; p < h.P; ++p) {
    const float* pr = P.f(h.off_posture) + p * (2 + n);
    if (pr[1] != 0.f) {
      T s = T(0);
      for (int d = lane; d < n; d += W) {
        T wgt = T(pr[2 + d]);
        if constexpr (PW) if (!BD || pw) wgt *= k2_pw<T>(pw, p * n + d, a.io64, &status);
        T v = wgt * T(pr[0]) * eperr(p, d);
        s += v * v;
      }
      s = warp_sum_t<W, T>(s);
      mu += T(pr[1]) * s;
    }
  }
  // diagonal, posture part of the linear term and box.  A DECOUPLED dof (zero column in every task Jacobian) only sees
  // the diagonal: its optimum is the clamp of -c/h, written straight to xfull.
  BoundsRow bd{};
  if constexpr (BD) bd = k2_bd_row(a, n, b, a.io64);
  for (int d = lane; d < n; d += W) {
    const int u = umap[d];
    T cd = T(0), hd = mu;
    for (int p = 0; p < h.P; ++p) {
      const float* pr = P.f(h.off_posture) + p * (2 + n);
      T wgt = T(pr[2 + d]);
      if constexpr (PW) if (!BD || pw) wgt *= k2_pw<T>(pw, p * n + d, a.io64, &status);
      hd += wgt * wgt;                                  // (W J)^T (W J), J = -I
      if (wgt != T(0)) cd -= T(pr[0]) * wgt * wgt * eperr(p, d);  // -(W(-g e))^T W (-I)
    }
    T lo = -T(BIK_INF_F), hi = T(BIK_INF_F);
    if (!a.skip_box) { const int qa = dofqadr[d]; box_dof<T, BD>(P, d, qa >= 0 ? qv(qa) : T(0), T(a.dt), &lo, &hi, &bd, &status); }
    if (a.lo_out) { stout<T>(a.lo_out, (long long)b * n + d, a.io64, lo); stout<T>(a.hi_out, (long long)b * n + d, a.io64, hi); }
    if (lo > hi + T(1e-9) * (T(1) + (hi < 0 ? -hi : hi))) status |= 8;   // inconsistent limits (e.g. a configuration far outside its range with a velocity limit): the reference's QP has no solution (solve_ik.py:103)
    if (u >= 0) {
      w.Hp[tri(u) + u] += hd;
      w.c[u] += cd; w.lo[u] = lo; w.hi[u] = hi;
    } else {
      T v = -cd / hd;
      v = v < lo ? lo : (v > hi ? hi : v);
      w.xfull[d] = v;
      if (a.Hout) { a.Hout[((long long)b * n + d) * n + d] = double(hd); a.cout[(long long)b * n + d] = double(cd); }
    }
  }
  k2_sync<W>();
  return status;
}

// ---- packed Cholesky of the free block, right-hand side fused as row nf -------------------------
// On entry Lp holds the lower triangle of the nf x nf block (compact indices) and, as row nf, the
// right-hand side y.  On exit row i (< nf) holds L[i][0..i-1] (the diagonal is kept as its inverse in
// dinv) and row nf holds L^-1 y: the forward substitution is just one more row of the same recurrence.
// Lane i % W owns row i; one warp barrier per column; no division or square root on the critical
// path (rsqrt once per column, by the lane that owns the next diagonal, from a running sum of squares).
template <typename T, int W, int SLOTS>
BIK_NOINLINE int k2_factor(T* __restrict__ Lp, T* __restrict__ dinv, int nf, int lane) {
  BIK_IN_SHARED(Lp); BIK_IN_SHARED(dinv);
  int bad = 0;
  T ss[SLOTS];
#pragma unroll
  for (int s = 0; s < SLOTS; ++s) ss[s] = T(0);
  if (lane == 0 && nf > 0) {
    T d = Lp[0];
    if (!(d > T(0))) { bad = 1; d = T(1e-30); }
    dinv[0] = bik_rsqrt<T>(d);
  }
  k2_sync<W>();
#pragma unroll 1
  for (int j = 0; j < nf; ++j) {
    const T* Lj = Lp + tri(j);
    const T inv = dinv[j];
#pragma unroll
    for (int s = 0; s < SLOTS; ++s) {
      const int i = lane + s * W;
      if (i > j && i <= nf) {
        T* Li = Lp + tri(i);
        T a0 = T(0), a1 = T(0);
        int k = 0;
#pragma unroll 2
        for (; k + 1 < j; k += 2) { a0 += Li[k] * Lj[k]; a1 += Li[k + 1] * Lj[k + 1]; }
        if (k < j) a0 += Li[k] * Lj[k];
        T l = (Li[j] - (a0 + a1)) * inv;
        Li[j] = l;
        ss[s] += l * l;
        if (i == j + 1 && i < nf) {
          T d = Li[i] - ss[s];
          if (!(d > T(0))) { bad = 1; d = T(1e-30); }
          dinv[i] = bik_rsqrt<T>(d);
        }
      }
    }
    k2_sync<W>();
  }
  return bad;
}
// Back substitution x = L^-T y with y in row nf of Lp; each lane keeps its entries in registers and
// the pivot value travels by shuffle.  Writes x_k into out[k] (compact indices).
template <typename T, int W, int SLOTS>
BIK_NOINLINE void k2_backsub(const T* __restrict__ Lp, const T* __restrict__ dinv, int nf, T* out, int lane) {
  BIK_IN_SHARED(Lp); BIK_IN_SHARED(dinv); BIK_IN_SHARED(out);
  T y[SLOTS];
  const T* rhs = Lp + tri(nf);
#pragma unroll
  for (int s = 0; s < SLOTS; ++s) { int i = lane + s * W; y[s] = (i < nf) ? rhs[i] : T(0); }
  for (int k = nf - 1; k >= 0; --k) {
    const int ks = k / W, kl = k - ks * W;
    T cand = y[0];
#pragma unroll
    for (int s = 1; s < SLOTS; ++s) if (ks == s) cand = y[s];
    T xk = warp_bcast<T, W>(cand, kl) * dinv[k];
    if (lane == kl) out[k] = xk;
    const T* Lk = Lp + tri(k);
#pragma unroll
    for (int s = 0; s < SLOTS; ++s) { int i = lane + s * W; if (i < k) y[s] -= Lk[i] * xk; }
  }
  k2_sync<W>();
}
// y <- L^-1 y for a separate vector (general-row path only)
template <typename T, int W>
BIK_NOINLINE void k2_forward(const T* Lp, const T* dinv, T* y, int nf, int lane) {
  BIK_IN_SHARED(Lp); BIK_IN_SHARED(dinv); BIK_IN_SHARED(y);
  for (int k = 0; k < nf; ++k) {
    if (k % W == lane) y[k] = y[k] * dinv[k];
    k2_sync<W>();
    T yk = y[k];
    for (int i = lane; i < nf; i += W) if (i > k) y[i] -= Lp[tri(i) + k] * yk;
  }
  k2_sync<W>();
}

// element j of collision row r of instance b
template <typename T> BIK_HD T k2_grow(const K2Args& a, long long base, int r, int n, int j) { return ldin<T>(a.Gc, base + (long long)r * n + j, a.gc64); }

// Active general rows R (collision): KKT  [H_FF G_RF^T; G_RF 0][x_F; lam] = [y; h_R - G_RA x_A] through the
// factor:  Y_r = L^-1 G_rF^T,  S = Y Y^T,  lam = S^-1 (Y (L^-1 y) - rhs),  rhs row <- L^-1 y - Y^T lam.
// Cold for box-only problems: kept out of line so it does not occupy the instruction cache.
template <typename T, int W>
BIK_NOINLINE int k2_general_rows(const K2Ws<T> w, const K2Args& a, long long gbase, T* rhs, int n, int nf, int ng, int mg, int lane) {
  // local copies: the assumption has to sit on the very pointer values the loops use
  T* const Y = w.Y; T* const S = w.S; T* const lam = w.lam; T* const rg = w.rg; const T* const hg = w.hg; const T* const x = w.x;
  const int* const st = w.st; const int* const idx = w.idx; const int* const gidx = w.gidx; const int* const frow = w.frow;
  BIK_IN_SHARED(frow);
  BIK_IN_SHARED(Y); BIK_IN_SHARED(S); BIK_IN_SHARED(lam); BIK_IN_SHARED(rg); BIK_IN_SHARED(hg); BIK_IN_SHARED(x);
  BIK_IN_SHARED(st); BIK_IN_SHARED(idx); BIK_IN_SHARED(gidx); BIK_IN_SHARED(rhs);
  int bad = 0;
  for (int r = 0; r < ng; ++r) {
    T* Yr = Y + r * n;
    for (int i = lane; i < nf; i += W) Yr[i] = k2_grow<T>(a, gbase, frow[gidx[r]], n, idx[i]);
    if (nf < n) {   // some dofs sit on their bounds: move their part of the row to the right-hand side
      if (lane == 0) { T sv = hg[gidx[r]]; for (int j = 0; j < n; ++j) if (st[j]) sv -= k2_grow<T>(a, gbase, frow[gidx[r]], n, j) * x[j]; rg[r] = sv; }
    } else if (lane == 0) rg[r] = hg[gidx[r]];
    k2_sync<W>();
    k2_forward<T, W>(w.Lp, w.dinv, Yr, nf, lane);
  }
  // S = Y Y^T and the right-hand side Y (L^-1 y) - rhs: one (r, q) entry per lane
  for (int p = lane; p < ng * (ng + 1) / 2 + ng; p += W) {
    int r = 0, q2 = p;
    if (p < ng * (ng + 1) / 2) { while (q2 > r) { q2 -= r + 1; ++r; } } else { r = p - ng * (ng + 1) / 2; q2 = -1; }
    const T* Yr = Y + r * n;
    const T* Yq = q2 >= 0 ? Y + q2 * n : rhs;
    T v = T(0);
    for (int i = 0; i < nf; ++i) v += Yr[i] * Yq[i];
    if (q2 >= 0) { S[r * mg + q2] = v; S[q2 * mg + r] = v; } else lam[r] = v - rg[r];
  }
  k2_sync<W>();
  if (lane == 0) {  // tiny dense solve, serial
    for (int j = 0; j < ng; ++j) {  // Cholesky of S in place + solve
      // Rows between the same two bodies span at most 6 directions, so a working set can hold dependent rows (typically all
      // with h = 0: pairs at the minimum distance).  A relative shift of the diagonal turns the multipliers of such a family
      // into the minimum-norm split of their common multiplier: the signs stay meaningful and the method proceeds instead of
      // cycling (ALOHA with 1 104 pairs, 2 048 sampled instances: 89 flagged without the shift, 0 with it).
      const T sjj = S[j * mg + j] * (T(1) + T(1e-12));
      T d = sjj; for (int k = 0; k < j; ++k) d -= S[j * mg + k] * S[j * mg + k];
      if (!(d > T(1e-14) * sjj)) bad = 1;   // the active rows are (numerically) dependent beyond what the shift absorbs
      d = bik_sqrt<T>(d > T(0) ? d : T(1e-30)); S[j * mg + j] = d;
      for (int i = j + 1; i < ng; ++i) { T v = S[i * mg + j]; for (int k = 0; k < j; ++k) v -= S[i * mg + k] * S[j * mg + k]; S[i * mg + j] = v / d; }
    }
    for (int i = 0; i < ng; ++i) { T v = lam[i]; for (int k = 0; k < i; ++k) v -= S[i * mg + k] * lam[k]; lam[i] = v / S[i * mg + i]; }
    for (int i = ng - 1; i >= 0; --i) { T v = lam[i]; for (int k = i + 1; k < ng; ++k) v -= S[k * mg + i] * lam[k]; lam[i] = v / S[i * mg + i]; }
  }
  k2_sync<W>();
  for (int i = lane; i < nf; i += W) { T v = rhs[i]; for (int r = 0; r < ng; ++r) v -= Y[r * n + i] * lam[r]; rhs[i] = v; }
  k2_sync<W>();
  return warp_max_i<W>(bad);
}

template <typename T> struct K2Tol { static BIK_HD T x() { return T(1e-12); } static BIK_HD T g() { return T(1e-9); } };   // fp64 solve tolerances

// Minimiser of the QP on the working set (w.st: 0 free / 1 at lower / 2 at upper; w.gst: active general rows) into w.x,
// multipliers of the active general rows into w.lam.  Returns status bits (4: factorisation broke down, 2: more than
// k2_max_gen rows active, 32 (internal): the active general rows are linearly dependent, the multipliers are not
// trustworthy); *ng_out = number of active general rows (their indices in w.gidx).
// *fkey remembers which free set the factor in w.Lp belongs to (bit 63 = valid, problems with at most 63 coupled dofs): when only
// the general rows of the working set changed -- always, for a problem without box limits -- the factor is reused and only the
// right-hand side is forward-substituted.
template <typename T, int W, int SLOTS>
BIK_HD int k2_solve_working_set(const PHeader& h, const K2Args& a, long long gbase, K2Ws<T>& w, int lane, int* ng_out, unsigned long long* fkey) {
  const int n = h.nu, np = w.nrows, mg = k2_max_gen(h);   // np: rows in the window
  int status = 0;
  // compact free list / active general rows (every lane writes the same values)
  int nf = 0, ng = 0;
  unsigned long long key = n <= 63 ? 1ull << 63 : 0ull;
#if defined(__CUDA_ARCH__)
  {   // one ballot per W dofs: lane i tests dof base + i, the free ones are numbered by the bits below them
    unsigned lane32;
    asm("mov.u32 %0, %%laneid;" : "=r"(lane32));
    const unsigned gm = k2_gmask<W>(), gshift = lane32 & ~(unsigned)(W - 1);
    for (int base = 0; base < n; base += W) {
      const int i = base + lane;
      const bool fr = i < n && w.st[i] == 0;
      const unsigned bits = __ballot_sync(gm, fr) >> gshift;   // bit k: dof base + k is free
      if (fr) w.idx[nf + __popc(bits & ((1u << lane) - 1u))] = i;
      nf += __popc(bits);
      if (base < 63) key |= ((unsigned long long)bits << base) & 0x7fffffffffffffffull;
    }
  }
#else
  for (int i = 0; i < n; ++i) if (w.st[i] == 0) { w.idx[nf] = i; ++nf; if (i < 63) key |= 1ull << i; }
#endif
  const bool reuse = (key >> 63) != 0ull && key == *fkey;   // bit 63: the mask covers every coupled dof (n <= 63)
  for (int r = 0; r < np; ++r) if (w.gst[r]) { if (ng < mg) { w.gidx[ng] = r; ++ng; } else status |= 2; }
  k2_sync<W>();
  // x on the bounds, rhs of the reduced system, copy of H_FF
  for (int i = lane; i < n; i += W) w.x[i] = w.st[i] == 1 ? w.lo[i] : (w.st[i] == 2 ? w.hi[i] : T(0));
  k2_sync<W>();
  T* rhs = w.Lp + tri(nf);
  for (int i = lane; i < nf; i += W) {
    int ii = w.idx[i];
    const T* Hrow = w.Hp + tri(ii);
    T r = -w.c[ii];
    if (nf < n) {   // some dofs sit on their bounds: their columns move to the right-hand side
      for (int j = 0; j < ii; ++j) if (w.st[j]) r -= Hrow[j] * w.x[j];
      for (int j = ii + 1; j < n; ++j) if (w.st[j]) r -= w.Hp[tri(j) + ii] * w.x[j];
    }
    rhs[i] = r;
    if (!reuse) {
      T* Li = w.Lp + tri(i);
      for (int j = 0; j <= i; ++j) Li[j] = Hrow[w.idx[j]];
    }
  }
  k2_sync<W>();
  if (reuse) k2_forward<T, W>(w.Lp, w.dinv, rhs, nf, lane);
  else if (k2_factor<T, W, SLOTS>(w.Lp, w.dinv, nf, lane)) status |= 4;
  *fkey = key;
  status = warp_max_i<W>(status & 4) | (status & 2);
  if (ng > 0 && k2_general_rows<T, W>(w, a, gbase, rhs, n, nf, ng, mg, lane)) status |= 32;   // internal: active rows dependent
  // x_F = L^-T (.), overwriting the rhs row in place
  k2_backsub<T, W, SLOTS>(w.Lp, w.dinv, nf, rhs, lane);
  for (int i = lane; i < nf; i += W) w.x[w.idx[i]] = rhs[i];
  k2_sync<W>();
  *ng_out = ng;
  return status;
}
// gradient of the Lagrangian on dof i at w.x:  c_i + (H x)_i + sum_r G_ri lam_r
template <typename T>
BIK_HD T k2_grad(const K2Args& a, long long gbase, const K2Ws<T>& w, int n, int ng, int i) {
  T gi = w.c[i];
  const T* Hrow = w.Hp + tri(i);
  for (int j = 0; j <= i; ++j) gi += Hrow[j] * w.x[j];
  for (int j = i + 1; j < n; ++j) gi += w.Hp[tri(j) + i] * w.x[j];
  for (int r = 0; r < ng; ++r) gi += k2_grow<T>(a, gbase, w.frow[w.gidx[r]], n, i) * w.lam[r];
  return gi;
}

// Returns status bits.  On exit w.x holds dq (coupled dofs).
template <typename T, int W, int SLOTS>
BIK_HD int k2_solve(const PView& P, const K2Args& a, int b, K2Ws<T>& w, int lane, int* iters_out) {
  const PHeader& h = P.h();
  const int n = h.nu, npair = h.npairs;   // coupled dofs only (n == nv whenever there are general rows)
  const int MAXIT = 60 + 2 * (n + k2_max_gen(h)), PATIENCE = 2;   // bounds + the general rows that may be active at once
  const T tolx = K2Tol<T>::x(), tolg = K2Tol<T>::g();
  const long long gbase = (long long)b * npair * n;
  for (int i = lane; i < n; i += W) {
    int s0 = a.warm ? (a.warm[(long long)b * n + i] & 3) : 0;   // warm start: last step's active set (bit 2 is the small-group path's marker)
    if ((s0 == 1 && !(w.lo[i] > T(-1e30))) || (s0 == 2 && !(w.hi[i] < T(1e30)))) s0 = 0;
    w.st[i] = s0;
  }
  // gather the finite rows (pairs inside the detection distance) into the window, in pair order
  int np = 0, overflow = 0;
  {
    const int cap = k2_row_cap(h);
    for (int r0 = 0; r0 < npair; r0 += W) {
      const int r = r0 + lane;
      T hv = T(BIK_INF_F);
      if (r < npair) hv = ldin<T>(a.hc, (long long)b * npair + r, a.gc64);
      const bool fin = r < npair && hv < T(1e30);
#if defined(__CUDA_ARCH__)
      unsigned lane32;
      asm("mov.u32 %0, %%laneid;" : "=r"(lane32));
      const unsigned bits = __ballot_sync(k2_gmask<W>(), fin);
      const int pos = np + __popc(bits & ((1u << lane32) - 1u)), cnt = __popc(bits);
#else
      const int pos = np, cnt = fin ? 1 : 0;
#endif
      if (fin && pos < cap) { w.frow[pos] = r; w.hg[pos] = hv; w.gst[pos] = 0; }
      np += cnt;
    }
    if (np > cap) { overflow = 1; np = cap; }
    w.nrows = np;
  }
  k2_sync<W>();
  int status = overflow ? 2 : 0, best = n + np + 1, patience = PATIENCE, it = 0, ng = 0;
  unsigned long long fkey = 0ull;
  bool done = n == 0;
  // One loop, one call site of the working-set solve (the kernel is instruction-cache bound):
  //   mode 0  block principal pivoting;  mode 1  set up the primal method from clip(0);  mode 2  primal active-set method.
  int mode = 0;
  while (!done && it < MAXIT) {
    if (mode == 1) {
      k2_sync<W>();
      for (int i = lane; i < n; i += W) {   // clip(0, lo, hi); a bound that holds the iterate is in the working set
        T v = T(0);
        int s0 = 0;
        if (w.lo[i] > v) { v = w.lo[i]; s0 = 1; }
        if (w.hi[i] < v) { v = w.hi[i]; s0 = 2; }
        w.xf[i] = v; w.st[i] = s0;
      }
      k2_sync<W>();
      int infeas = 0;
      for (int r = lane; r < np; r += W) {
        w.gst[r] = 0;
        T hr = w.hg[r];
        if (hr < T(1e30)) {
          T sv = -hr;
          for (int j = 0; j < n; ++j) sv += k2_grow<T>(a, gbase, w.frow[r], n, j) * w.xf[j];
          if (sv > tolx * (T(1) + (hr < 0 ? -hr : hr))) infeas = 1;
        }
      }
      if (warp_max_i<W>(infeas)) status |= 8;   // no feasible starting point: limits inconsistent with the collision rows
      k2_sync<W>();
      mode = 2;
      if (status & 8) break;
    }
    const int ws = k2_solve_working_set<T, W, SLOTS>(h, a, gbase, w, lane, &ng, &fkey);
    status |= ws & ~32;
    ++it;
    if (ws & 2) break;   // more rows active than the working set holds: the answer is flagged, further iterations cannot repair it
    if (mode == 0) {
      if (ws & 32) { mode = 1; continue; }   // block flips activated dependent rows (the primal method never does)
      // gradient on the active bounds, feasibility of free variables and of general rows.
      // Proposed new states go to w.idx (free after the scatter in the solve) and w.gnew.
      int ninf = 0;
      for (int i = lane; i < n; i += W) {
        int cur = w.st[i], ns = cur;
        if (cur == 0) {
          T xi = w.x[i];
          if (xi < w.lo[i] - tolx * (T(1) + (w.lo[i] < 0 ? -w.lo[i] : w.lo[i]))) ns = 1;
          else if (xi > w.hi[i] + tolx * (T(1) + (w.hi[i] < 0 ? -w.hi[i] : w.hi[i]))) ns = 2;
        } else {
          T gi = k2_grad<T>(a, gbase, w, n, ng, i);
          if (cur == 1 && gi < -tolg) ns = 0;
          else if (cur == 2 && gi > tolg) ns = 0;
        }
        w.idx[i] = ns;
        if (ns != cur) ++ninf;
      }
      for (int r = lane; r < np; r += W) {
        int cur = w.gst[r], ns = cur;
        T hr = w.hg[r];
        if (!(hr < T(1e30))) ns = 0;  // inactive row: h = +inf (collision_avoidance_limit.py:192-199)
        else if (cur == 0) {
          T sv = -hr;
          for (int j = 0; j < n; ++j) sv += k2_grow<T>(a, gbase, w.frow[r], n, j) * w.x[j];
          if (sv > tolx * (T(1) + (hr < 0 ? -hr : hr))) ns = 1;
        } else {
          int k = 0;
          while (k < ng && w.gidx[k] != r) ++k;
          if (k < ng && w.lam[k] < -tolg) ns = 0;
        }
        w.gnew[r] = ns;
        if (ns != cur) ++ninf;
      }
      ninf = warp_sum_i<W>(ninf);
      if (ninf == 0) { done = true; break; }
      if (ninf < best) { best = ninf; patience = PATIENCE; }
      else if (patience > 0) --patience;
      else { mode = 1; continue; }
      k2_sync<W>();
      for (int i = lane; i < n; i += W) w.st[i] = w.idx[i];
      for (int r = lane; r < np; r += W) w.gst[r] = w.gnew[r];
      k2_sync<W>();
      continue;
    }
    // mode 2 -- ratio test: how far can xf move towards x before a bound of a free dof or an inactive general row stops it
    T alpha = T(2);
    int blk = 0x7fffffff;
    for (int i = lane; i < n; i += W) {
      if (w.st[i] != 0) continue;
      const T xi = w.x[i], xo = w.xf[i], lo = w.lo[i], hi = w.hi[i];
      const bool below = xi < lo - tolx * (T(1) + (lo < 0 ? -lo : lo));
      const bool above = !below && xi > hi + tolx * (T(1) + (hi < 0 ? -hi : hi));
      if (below || above) {
        const T d = xi - xo;
        T al = d != T(0) ? ((below ? lo : hi) - xo) / d : T(0);
        al = al < T(0) ? T(0) : al;
        if (al < alpha) { alpha = al; blk = i; }
      }
    }
    for (int r = lane; r < np; r += W) {
      const T hr = w.hg[r];
      if (w.gst[r] || !(hr < T(1e30))) continue;
      T gx = T(0), gf = T(0);
      for (int j = 0; j < n; ++j) { const T gj = k2_grow<T>(a, gbase, w.frow[r], n, j); gx += gj * w.x[j]; gf += gj * w.xf[j]; }
      if (gx > hr + tolx * (T(1) + (hr < 0 ? -hr : hr))) {
        const T d = gx - gf;
        T al = d > T(0) ? (hr - gf) / d : T(0);
        al = al < T(0) ? T(0) : al;
        if (al < alpha) { alpha = al; blk = n + r; }
      }
    }
    const T amin = warp_min_t<W, T>(alpha);
    blk = warp_min_i<W>(alpha == amin ? blk : 0x7fffffff);   // ties: smallest index
    k2_sync<W>();   // every lane has read xf (the shuffles above already gather the lanes; this orders the memory accesses too)
    if (amin < T(1.5)) {   // blocked: partial step, the blocking constraint joins the working set
      const T al = amin > T(1) ? T(1) : amin;
      for (int i = lane; i < n; i += W) if (w.st[i] == 0) w.xf[i] += al * (w.x[i] - w.xf[i]);
      k2_sync<W>();
      if (blk < n) {
        if (lane == 0) { const bool lower = w.x[blk] < w.lo[blk]; w.st[blk] = lower ? 1 : 2; w.xf[blk] = lower ? w.lo[blk] : w.hi[blk]; }
      } else if (lane == 0) w.gst[blk - n] = 1;
      k2_sync<W>();
      continue;
    }
    // feasible subspace minimiser: it becomes the iterate; let go of the constraint with the most negative multiplier
    for (int i = lane; i < n; i += W) w.xf[i] = w.x[i];
    T worst = -tolg;
    int rel = 0x7fffffff;
    for (int i = lane; i < n; i += W) {
      const int cur = w.st[i];
      if (cur == 0) continue;
      T gi = k2_grad<T>(a, gbase, w, n, ng, i);
      if (cur == 2) gi = -gi;   // now: gi < 0 means the bound wants to let go
      if (gi < worst) { worst = gi; rel = i; }
    }
    for (int k = lane; k < ng; k += W) if (w.lam[k] < worst) { worst = w.lam[k]; rel = n + w.gidx[k]; }
    const T wmin = warp_min_t<W, T>(worst);
    rel = warp_min_i<W>(worst == wmin ? rel : 0x7fffffff);
    if (rel == 0x7fffffff) { done = true; break; }
    k2_sync<W>();
    if (lane == 0) { if (rel < n) w.st[rel] = 0; else w.gst[rel - n] = 0; }
    k2_sync<W>();
  }
  if (!done) status |= 2;
  if (a.warm) for (int i = lane; i < n; i += W) a.warm[(long long)b * n + i] = (signed char)w.st[i];
  if (iters_out) *iters_out = it;
  return status;
}

// One instance per warp: assemble, optionally dump (H, c) / (lo, hi), solve, write dq, optionally integrate q.
template <typename T, int W, int SLOTS, bool PW = false, bool BD = false>
BIK_HD void k2_warp(const PView& P, const K2Args& a, int b, void* wsm, int lane) {
  const PHeader& h = P.h();
  const int n = h.nv, nu = h.nu, nq = h.nq;
  const int32_t* umap = P.i(h.off_umap);
  if (a.skip && a.skip[b]) return;
  K2Ws<T> w = k2_carve<T>(h, wsm);
  int st = k2_assemble<T, W, PW, BD>(P, a, b, w, lane);
  if (a.skip_objective) return;
  if (a.Hout) {
    for (int k = lane; k < n * n; k += W) {
      int i = k / n, j = k - i * n, ui = umap[i], uj = umap[j];
      if (ui >= 0 && uj >= 0) a.Hout[(long long)b * n * n + k] = double(Hsym(w.Hp, ui, uj));
      else if (i != j) a.Hout[(long long)b * n * n + k] = 0.0;
    }
    for (int d = lane; d < n; d += W) if (umap[d] >= 0) a.cout[(long long)b * n + d] = double(w.c[umap[d]]);
  }
  if (!a.dq) return;
  int iters = 0;
  if (nu > 0) st |= k2_solve<T, W, SLOTS>(P, a, b, w, lane, &iters);
  for (int d = lane; d < n; d += W) {
    T v = umap[d] >= 0 ? w.x[umap[d]] : w.xfull[d];
    if (!(v == v)) st |= 4;
    w.xfull[d] = v;
    stout<T>(a.dq, (long long)b * n + d, a.io64, v);
  }
  const int bw = st & 32;   // BIK_STATUS_BAD_WEIGHT of a posture weight this lane read (PW only)
  st = warp_max_i<W>(st & 2) | warp_max_i<W>(st & 4) | warp_max_i<W>(st & 8);
  if constexpr (PW) st |= warp_max_i<W>(bw);
  if (lane == 0) {
    if (a.status) a.status[b] |= st;
    if (a.iters) a.iters[b] = iters;
  }
  k2_sync<W>();
  if (a.integrate) {   // q <- q (+) dq, node by node (mj_integratePos); fp32 callers: the sum is rounded once
    for (int nn = lane; nn < h.nnode; nn += W) {
      const NodeRec& r = P.node(nn);
      const int nqn = r.type == JNT_FREE ? 7 : (r.type == JNT_BALL ? 4 : 1);
      T qn[7];
      for (int k = 0; k < nqn; ++k) qn[k] = ldin<T>(a.q, (long long)b * nq + r.qadr + k, a.io64);
      integrate_node<T>(r, qn - r.qadr, w.xfull);
      for (int k = 0; k < nqn; ++k) stout<T>(const_cast<void*>(a.q), (long long)b * nq + r.qadr + k, a.io64, qn[k]);
    }
    k2_sync<W>();
  }
}

}  // namespace bik
