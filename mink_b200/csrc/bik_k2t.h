// bik_k2t.h -- K2, small-group path: the same QP as bik_k2.h (same objective, same box, same tolerances, same optimum),
// laid out for coupled blocks of up to 64 dofs (32-bit active-set masks up to 32, 64-bit ones beyond).
//
// Why: with a whole warp per instance the 18-dof coupled block of the G1 configuration keeps half the
// lanes idle and spends most instructions on run-time index arithmetic, shuffles and barriers
// (14 k warp-instructions per instance, ~45 k cycles per pivoting iteration).  Here G adjacent lanes
// (4 or 8) share one problem, so a warp carries NS = 32/G problems; the solve is in fp64, and its loops are compact
// run-time loops over shared memory so that a whole pivoting iteration stays resident in the instruction cache:
//
//   * per-instance vectors and packed triangles live in shared memory, word w of slot s at [w*NS + s]
//     (the G lanes of a group broadcast-read one address; the NS groups read one 8*NS-byte segment);
//   * instance data from K1 (the packed task blocks -- or, for bik_solve, dense J / e / e_posture -- and q) is staged a task
//     at a time through an instance-major tile with odd row stride: coalesced global reads by the whole warp,
//     conflict-free private reads;
//   * dofs without any finite bound (the free joint) are eliminated once; everything below runs on the Schur
//     complement of that leading block (k2t_schur), and the leading part of dq is recovered at the end;
//   * the active set is guessed by projected Gauss-Seidel sweeps (k2t_pgs_guess), inside a rollout from the
//     previous step's dq; a primal active-set method then starts from that feasible point: every iteration
//     refactors the pivoted block with clamped dofs turned into identity rows/columns (masked loads), so every
//     group executes the same instruction stream whatever its active set is and groups never diverge; a group
//     that has converged idles until its warp is done;
//   * the factorisation is left-looking by blocks of G rows: lane l owns row i0+l, finished rows are
//     broadcast-read from shared memory, the right-hand side rides along as the last row (forward
//     substitution for free), diagonals are kept as reciprocal square roots, entries masked out by the
//     active set are known to be zero and skipped; one warp barrier per row;
//   * back substitution in column form (k2t_backsub): one barrier per row, no shuffles; multipliers are only
//     evaluated on clamped dofs.
//
// Reference semantics: mink/solve_ik.py:13-65,101 (build_ik + qpsolvers), mink/tasks/task.py:105-138.
// Device: G in {4, 8}, NS = 32 / G.  Host emulation (tests/host_emu): G = NS = 1.
#pragma once
#include "bik_k2.h"

#if defined(__CUDA_ARCH__)
#define BIK_WARP_ANY(x) __any_sync(0xffffffffu, (x))
#else
#define BIK_WARP_ANY(x) (x)
#endif

namespace bik {

BIK_HD uint32_t bik_float_bits(float f) {
#if defined(__CUDA_ARCH__)
  return (uint32_t)__float_as_int(f);
#else
  uint32_t u; memcpy(&u, &f, 4); return u;
#endif
}
BIK_HD int bik_popc(uint32_t v) {
#if defined(__CUDA_ARCH__)
  return __popc(v);
#else
  return __builtin_popcount(v);
#endif
}
BIK_HD int bik_popc(uint64_t v) { return bik_popc((uint32_t)v) + bik_popc((uint32_t)(v >> 32)); }

enum { K2T_NMAX = 32, K2T_NMAX_WIDE = 64 };   // 32-bit active-set masks by default, 64-bit in the wide instantiation

// ---- group reductions over G adjacent lanes (every lane of the warp must call them) --------------------
template <int G> BIK_HD int grp_or(int v) {
#if defined(__CUDA_ARCH__)
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) v |= __shfl_xor_sync(0xffffffffu, v, o);
#endif
  return v;
}
template <int G> BIK_HD uint32_t grp_or_m(uint32_t v) { return (uint32_t)grp_or<G>((int)v); }
template <int G> BIK_HD uint64_t grp_or_m(uint64_t v) {
  return (uint64_t)(uint32_t)grp_or<G>((int)(uint32_t)v) | ((uint64_t)(uint32_t)grp_or<G>((int)(uint32_t)(v >> 32)) << 32);
}
template <int G> BIK_HD int grp_add(int v) {
#if defined(__CUDA_ARCH__)
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
#endif
  return v;
}
template <int G> BIK_HD int grp_max(int v) {
#if defined(__CUDA_ARCH__)
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) { int t = __shfl_xor_sync(0xffffffffu, v, o); v = t > v ? t : v; }
#endif
  return v;
}
template <typename T, int G> BIK_HD T grp_sum(T v) {
#if defined(__CUDA_ARCH__)
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
#endif
  return v;
}

// ---- per-warp scratch ------------------------------------------------------------------------------
// T words per slot:   Hp tri(nu) | U (factor incl. rhs row; aliased by the staging tiles) | c nu | vs nu | xf nu (feasible iterate)
// float words / slot: lo nu | hi nu
BIK_HD int k2t_task_tile_words(const PView& P) {  // widest task tile, in T words per instance (odd)
  const PHeader& h = P.h();
  int m = 1;
  #pragma unroll 1
  for (int f = 0; f < h.F; ++f) { int ne = 6 * P.frame(f).ncols + 6; m = ne > m ? ne : m; }
  if (h.C > 0) { int ne = 3 * h.com_ncols + 3; m = ne > m ? ne : m; }
  return m | 1;
}
BIK_HD int k2t_union_words(const PView& P) {
  const PHeader& h = P.h();
  int u = tri(h.nu + 1);
  int t = k2t_task_tile_words(P);
  u = t > u ? t : u;
  int fw = (h.nq + h.P * h.nv) | 1;   // q (+ dense posture errors) of one instance, as T
  return fw > u ? fw : u;
}
BIK_HD int k2t_slot_T_words(const PView& P) { return tri(P.h().nu) + k2t_union_words(P) + 3 * P.h().nu; }
BIK_HD int k2t_slot_bytes(const PView& P, int ts) { return k2t_slot_T_words(P) * ts + 2 * P.h().nu * 4; }
BIK_HD int k2t_warp_bytes(const PView& P, int ts, int NS) { return (NS * k2t_slot_bytes(P, ts) + 15) & ~15; }   // ts: sizeof(T)

// ---- problem tables built by bik_problem_create (bik_build.h) ------------------------------------------------------------
BIK_HD const K2Header& k2t_h(const PView& P) { return *reinterpret_cast<const K2Header*>(P.base + P.h().words64); }
BIK_HD const K2TaskRec& k2t_task(const PView& P, int t) { return reinterpret_cast<const K2TaskRec*>(P.base + k2t_h(P).tasks)[t]; }
BIK_HD const K2DofRec* k2t_dofs(const PView& P) { return reinterpret_cast<const K2DofRec*>(P.base + k2t_h(P).dofs); }
BIK_HD const K2PostRec* k2t_post(const PView& P) { return reinterpret_cast<const K2PostRec*>(P.base + k2t_h(P).post); }

// ---- staging (warp-cooperative, W lanes, NS instances) -------------------------------------------------
// One task's weighted block, column-major like K1's packed record:
//   tile[i][ia*nr + r] = cost_r J[row0+r][col_ia],   tile[i][nr*nc + r] = cost_r (-gain e[row0+r]).
// wk: the weights of the task's nr*nc + nr elements (K2Header::w).
// Source: the packed hand-off (one contiguous run per instance: coalesced without any index arithmetic) or, for bik_solve,
// the dense rows (gather through the task's column list).  PK: the packed hand-off is known to be there.
template <typename T, int W, int NS, bool PK = false>
BIK_HD void k2t_stage_task(T* tile, int S, int lane, int cnt, long long b0, const K2Args& a, int pk64, int dense64, int K, int nv, int pks,
                           const int32_t* cols, const K2TaskRec& tk, const double* wk) {
  const int nj = tk.nr * tk.nc, ne = nj + tk.nr;
  for (int k = lane; k < ne; k += W) {
    const T cr = T(wk[k]);
    if (PK || a.pk) {
      const long long o = b0 * pks + tk.pk_off + k;
#pragma unroll
      for (int i = 0; i < NS; ++i) tile[i * S + k] = i < cnt ? cr * ldin<T>(a.pk, o + (long long)i * pks, pk64) : T(0);
    } else {
      const int ia = k / tk.nr, r = k - ia * tk.nr;
      const bool isj = k < nj;
      const void* src = isj ? a.J : a.e;
      const long long o = isj ? b0 * K * nv + (tk.row0 + r) * nv + (cols[ia] & 0xffff) : b0 * K + tk.row0 + r, stride = isj ? (long long)K * nv : K;
#pragma unroll
      for (int i = 0; i < NS; ++i) tile[i * S + k] = i < cnt ? cr * ldin<T>(src, o + i * stride, dense64) : T(0);
    }
  }
}
template <typename T, int W, int NS>
BIK_HD void k2t_stage_q(T* tile, int S, int lane, int cnt, const void* src, int is64, long long b0, int n) {
  for (int k = lane; k < n; k += W) {
#pragma unroll
    for (int i = 0; i < NS; ++i) tile[i * S + k] = i < cnt ? ldin<T>(src, (b0 + i) * n + k, is64) : T(0);
  }
}
template <typename T, int W, int NS>
BIK_HD void k2t_stage_rows(T* tile, int S, int off, int lane, int cnt, const void* src, int is64, long long o, long long stride, int n) {
  for (int k = lane; k < n; k += W) {
#pragma unroll
    for (int i = 0; i < NS; ++i) tile[i * S + off + k] = i < cnt ? ldin<T>(src, o + i * stride + k, is64) : T(0);
  }
}

// ---- assembly: (W J)^T (W J) and -(W(-g e))^T W J of one task --------------------------------------------------
// Whole columns are dealt to the G lanes, heaviest first in serpentine order (column ia pairs with ia + 1 columns, so lane
// l takes the (l)-th, (2G-1-l)-th, (2G+l)-th ... heaviest).  A lane keeps its column's NR weighted entries in registers and
// walks the columns ib <= ia: NR loads + NR FMAs per entry of H instead of 2 NR loads and a pair-index decode.  Where each entry
// lands comes from the task's tables (K2TaskRec): ucol[ia] = ua, and pairs[tri(ia) + ib] = its packed-triangle offset.
template <typename T, int G, int NS, int NR>
BIK_HD void k2t_task_accumulate_nr(const T* tr, int nc, const int16_t* pairs, const int16_t* ucol, T* Hp, T* c, int l) {
  const T* wev = tr + NR * nc;
  for (int rnd = 0;; ++rnd) {
    const int jj = (rnd & 1) ? (rnd + 1) * G - 1 - l : rnd * G + l;
    if (jj >= nc) break;
    const int ia = nc - 1 - jj;
    T col[NR];
    T cs = T(0);
#pragma unroll
    for (int r = 0; r < NR; ++r) { col[r] = tr[ia * NR + r]; cs += wev[r] * col[r]; }
    c[ucol[ia] * NS] -= cs;
    const int16_t* pr = pairs + tri(ia);
    #pragma unroll 1
    for (int ib = 0; ib <= ia; ++ib) {
      const T* cb = tr + ib * NR;
      T s = T(0);
#pragma unroll
      for (int r = 0; r < NR; ++r) s += col[r] * cb[r];
      Hp[pr[ib] * NS] += s;
    }
  }
}
// The CoM task (at most one per problem) is assembled out of line: its unrolled copy would otherwise sit in the kernel
// beside the frame tasks' one.
template <typename T, int G, int NS>
BIK_NOINLINE void k2t_task_accumulate_com(const T* tr, int nc, const int16_t* pairs, const int16_t* ucol, T* Hp, T* c, int l) {
  BIK_IN_SHARED(tr); BIK_IN_SHARED(Hp); BIK_IN_SHARED(c);
  k2t_task_accumulate_nr<T, G, NS, 3>(tr, nc, pairs, ucol, Hp, c, l);
}
template <typename T, int G, int NS>
BIK_HD void k2t_task_accumulate(const PView& P, const T* tr, const K2TaskRec& tk, T* Hp, T* c, T* mu, int l) {
  const int nr = tk.nr, nc = tk.nc;
  const T* wev = tr + nr * nc;
  if (tk.lm != 0.f) { T s = T(0); for (int r = 0; r < nr; ++r) s += wev[r] * wev[r]; *mu += T(tk.lm) * s; }
  const int16_t* pairs = reinterpret_cast<const int16_t*>(P.base + tk.pairs);
  const int16_t* ucol = reinterpret_cast<const int16_t*>(P.base + tk.ucol);
  if (nr == 6) k2t_task_accumulate_nr<T, G, NS, 6>(tr, nc, pairs, ucol, Hp, c, l);
  else k2t_task_accumulate_com<T, G, NS>(tr, nc, pairs, ucol, Hp, c, l);
}

// ---- solver pieces: compact run-time loops (the whole pivoting iteration must stay resident in the
// instruction cache -- the fully unrolled variants of these routines were instruction-fetch bound).  Every loop here and in
// the assembly carries `#pragma unroll 1`: unrolled by the compiler they made the step's kernel 17.6 k SASS instructions on
// sm_90a, and even the factor's and the assembly's dot loops alone cost 6 % of K2's time in the G1 step on an H100 --------
// Dot product of row i of the symmetric packed matrix with a vector (both slot-strided in shared memory).
template <typename T, int NS>
BIK_HD T k2t_row_dot(const T* __restrict__ Hp, const T* __restrict__ v, int i, int nu, int k0 = 0) {   // sum over m in [k0, nu), i >= k0
  const T* row = Hp + (tri(i) + k0) * NS;
  const T* pv = v + k0 * NS;
  T a0 = T(0), a1 = T(0);
  int k = i + 1 - k0;
  #pragma unroll 1
  for (; k >= 2; k -= 2) { a0 += row[0] * pv[0]; a1 += row[NS] * pv[NS]; row += 2 * NS; pv += 2 * NS; }
  if (k) { a0 += row[0] * pv[0]; pv += NS; }
  const T* col = Hp + (tri(i + 1) + i) * NS;   // entries (m, i), m > i, sit at tri(m) + i
  #pragma unroll 1
  for (int m = i + 1; m < nu; ++m) { a1 += col[0] * pv[0]; col += (m + 1) * NS; pv += NS; }
  return a0 + a1;
}
// Masked factorisation of the coupled block, left-looking by blocks of G rows (lane l owns row i0 + l); rows
// 0..nu-1 are matrix rows, row nu is the right-hand side (already stored in Lp's row nu).  Active dofs (bit set in
// `act`) become identity rows/columns.  On exit Lp row i holds L[i][0..i-1] and 1/L[i][i], row nu holds L^-1 rhs.
// The column window [kb, ke) selects which part of the factor is produced:
//   (0, nu)   the whole factor;
//   (0, nf)   the columns of the nf leading dofs for EVERY row (rows >= nf keep only L[i][0..nf-1]): the one-off
//             elimination of the dofs that have no finite bound (see k2t_warp_tile);
//   (nf, nu)  the factor of the trailing block, whose source (in Hp / the right-hand-side row) must then be the Schur
//             complement of the leading block; columns < nf of Lp are left alone.
// Every lane of the warp must call it (it contains warp barriers).
template <typename T, int G, int NS, typename M>
BIK_NOINLINE int k2t_factor(const T* __restrict__ Hp, T* __restrict__ Lp, int nu, M act, int l, int kb, int ke) {
  int bad = 0;
  T* const rhsrow = Lp + tri(nu) * NS;
  // Row blocks are aligned to the END of the system (rows kb..nu): the last rows are the expensive ones (cost ~ i^2),
  // so the partial block, if any, is the first one and every lane has a row in the last block.
  const int first = (nu + 1 - kb) % G;
  for (int i0 = kb + (first ? first - G : 0); i0 <= nu; i0 += G) {
    const int i = i0 + l;
    const bool has = i >= kb && i <= nu, rhs = i == nu;
    const bool ai = has && !rhs && ((act >> i) & M(1));
    const M msk = rhs ? M(0) : (ai ? ~M(0) : act);
    const int ir = has ? i : kb;
    const T* src = rhs ? rhsrow : Hp + tri(ir) * NS;
    T* dst = Lp + tri(ir) * NS;
    T ss = T(0);
    // one entry of my row: L[i][k] = (A[i][k] - sum_{kb <= m < k} L[i][m] L[k][m]) / L[k][k]; a masked entry is exactly zero
    auto step = [&](int k) {
      T s = T(0);
      if (!((msk >> k) & M(1))) {
        const T* pk = Lp + (tri(k) + kb) * NS;   // row k (finished), walked together with my row
        const T* pi = dst + kb * NS;
        T a0 = T(0), a1 = T(0);
        int m = k - kb;
        #pragma unroll 1
        for (; m >= 2; m -= 2) { a0 += pi[0] * pk[0]; a1 += pi[NS] * pk[NS]; pi += 2 * NS; pk += 2 * NS; }
        if (m) { a0 += pi[0] * pk[0]; pk += NS; }
        s = (src[k * NS] - (a0 + a1)) * pk[0];   // pk now points at 1 / L[k][k]
      }
      dst[k * NS] = s;
      ss += s * s;
    };
    // columns kb .. min(i0 + G, ke) - 1 in order: those above the block are complete; inside the diagonal block the owner of
    // row k closes it first (one barrier), then the rows below use it.  One call site of step(): the kernel carries a single
    // copy of the dot loop.
    const int kend = (i0 + G) < ke ? (i0 + G) : ke;
    for (int k = kb; k < kend; ++k) {
      if (k >= i0) {
        if (has && !rhs && l == k - i0) {
          T d = (ai ? T(1) : src[k * NS]) - ss;
          if (!(d > T(0))) { bad = 1; d = T(1e-30); }
          dst[k * NS] = bik_rsqrt<T>(d);
        }
        if (G > 1) BIK_SYNCWARP();
      }
      if (has && k < i) step(k);
    }
  }
  return bad;
}
// x = L^-T y (y = row nu of Lp, consumed), column form: x_k = y_k / L_kk is computed by every lane from two broadcast reads,
// then the G lanes subtract L[k][m] x_k from the y_m (mlo <= m < k) they own -- row k of the packed factor is contiguous.
// One warp barrier per k, no shuffles, half the instructions of the dot-product form with its butterfly per k.
// Produces x_k for k = khi-1 .. klo.  Every lane of the warp must call it.
template <typename T, int G, int NS>
BIK_HD void k2t_backsub(T* __restrict__ Lp, int nu, int l, T* __restrict__ xs, int khi, int klo, int mlo) {
  T* y = Lp + tri(nu) * NS;
  for (int k = khi - 1; k >= klo; --k) {
    const T* row = Lp + tri(k) * NS;
    const T xk = y[k * NS] * row[k * NS];
    #pragma unroll 1
    for (int m = mlo + l; m < k; m += G) y[m * NS] -= row[m * NS] * xk;
    if (l == 0) xs[k * NS] = xk;
    if (G > 1) BIK_SYNCWARP();   // y_{k-1} is final
  }
}
// y_m -= sum_{k in [klo, khi)} L[k][m] x_k for the m < mhi a lane owns: what the trailing dofs contribute to the leading
// part of the right-hand side (each lane only touches its own m: no barrier inside).
template <typename T, int G, int NS>
BIK_HD void k2t_backsub_cross(T* __restrict__ Lp, int nu, int l, const T* __restrict__ xs, int khi, int klo, int mhi) {
  T* y = Lp + tri(nu) * NS;
  for (int m = l; m < mhi; m += G) {
    T a = y[m * NS];
    #pragma unroll 1
    for (int k = klo; k < khi; ++k) a -= Lp[(tri(k) + m) * NS] * xs[k * NS];
    y[m * NS] = a;
  }
}
// Active-set guess by projected Gauss-Seidel on  min 1/2 x^T S x + c^T x,  lo <= x <= hi  over the dofs [k0, nu):
//   x_i <- clip(-(c_i + sum_{m != i} S_im x_m) / S_ii, lo_i, hi_i),  i = k0 .. nu-1,  `sweeps` times from x = 0.
// Every lane of a group computes x_i and records which bound it sits on; the G lanes split the update of the residual
// (two warp barriers per row).  The guess only has to be
// close: the primal active-set method below starts from it and still ends at the exact optimum.  After the free-joint
// dofs have been eliminated the remaining block is strongly diagonally dominant per limb, and three sweeps cut the
// pivoting iterations of the G1 workload from 3.6 (4.5 for the slowest of the 4 problems in a warp) to 1.1 (1.4).
// dinv and res (nu words each, slot-strided, entries [k0, nu) used) are scratch: 1 / S_ii and the residual c + S x.  At most `sweeps` sweeps; they stop as soon as a sweep leaves the set of
// clamped dofs of every group in the warp unchanged.  Every lane of the warp must call it.
template <typename T, int G, int NS, typename M>
BIK_HD void k2t_pgs_guess(const T* __restrict__ Hp, const T* __restrict__ c, const float* __restrict__ lo, const float* __restrict__ hi,
                          T* __restrict__ xs, T* __restrict__ dinv, T* __restrict__ res, int nu, int k0, int l, int sweeps, bool from_xs,
                          M* lom_out, M* upm_out) {
  // Residual form: res = c + S x is kept up to date, so row i only needs res_i and x_i (broadcast reads, every lane
  // computes the new x_i), after which each lane adds S_mi (x_i' - x_i) to the residuals of the dofs m it owns.
  // from_xs (warp-uniform): xs already holds a feasible starting point (the previous step's dq, clipped), else start from 0
  if (!from_xs) { for (int k = k0 + l; k < nu; k += G) xs[k * NS] = T(0); }
  for (int k = k0 + l; k < nu; k += G) {
    res[k * NS] = c[k * NS] + (from_xs ? k2t_row_dot<T, NS>(Hp, xs, k, nu, k0) : T(0));
    dinv[k * NS] = T(1) / Hp[(tri(k) + k) * NS];
  }
  BIK_SYNCWARP();
  M lom = M(0), upm = M(0);
  for (int s = 0; s < sweeps; ++s) {
    const M plo = lom, pup = upm;
    lom = M(0); upm = M(0);
    for (int i = k0; i < nu; ++i) {
      const T xo = xs[i * NS];
      T xi = xo - res[i * NS] * dinv[i * NS];
      const T bl = T(lo[i * NS]), bu = T(hi[i * NS]);
      if (xi <= bl) { xi = bl; lom |= M(1) << i; }
      else if (xi >= bu) { xi = bu; upm |= M(1) << i; }
      const T dx = xi - xo;
      if (G > 1) BIK_SYNCWARP();   // every lane has read res_i and x_i
      #pragma unroll 1
      for (int m = k0 + l; m < nu; m += G) {
        const int hi_ = m > i ? m : i, lo_ = m > i ? i : m;
        res[m * NS] += Hp[(tri(hi_) + lo_) * NS] * dx;
      }
      if (l == 0) xs[i * NS] = xi;
      if (G > 1) BIK_SYNCWARP();   // res_{i+1} is up to date for the next row
    }
    if (!BIK_WARP_ANY(lom != plo || upm != pup)) break;   // the guess of every group in the warp has settled (first sweep: nothing on a bound)
  }
  *lom_out = lom; *upm_out = upm;
}

// Schur complement of the nf leading dofs, in place: after k2t_factor(.., 0, nf) every row i >= nf of Lp holds
// L[i][0..nf-1] and the right-hand-side row holds y = L_bb^-1 (-c_b).  Then, for i, j >= nf,
//   S[i][j] = H[i][j] - sum_{m<nf} L[i][m] L[j][m],   c~[i] = c[i] + sum_{m<nf} L[i][m] y[m]
// is the QP that remains after minimising over the leading dofs exactly (they have no bounds).
template <typename T, int G, int NS>
BIK_HD void k2t_schur(T* __restrict__ Hp, const T* __restrict__ Lp, T* __restrict__ c, int nu, int nf, int l) {
  const T* y = Lp + tri(nu) * NS;
  for (int i = nf; i < nu; ++i) {
    const T* pi = Lp + tri(i) * NS;
    for (int j = nf + l; j <= i + 1; j += G) {       // j == i + 1 stands for the linear term
      const T* pj = j <= i ? Lp + tri(j) * NS : y;
      T a0 = T(0);
      #pragma unroll 1
      for (int m = 0; m < nf; ++m) a0 += pi[m * NS] * pj[m * NS];
      if (j <= i) Hp[(tri(i) + j) * NS] -= a0;
      else c[i * NS] += a0;
    }
  }
}

// ---- work that runs once per tile, or for few problems: out of line, so that it does not take instruction-cache room
// from the solver loops.  Same arithmetic as in line.
// Levenberg-Marquardt terms of the posture tasks: mu + sum_p lm_p |W_p e_p|^2 (eprow: the staged posture errors).  The sum
// over d stays serial, in dof order: split over the lanes of a group it would be reassociated and change the result's bits.
template <typename T>
BIK_NOINLINE T k2t_posture_lm(PView P, const T* eprow, T mu) {
  BIK_IN_SHARED(eprow);
  const PHeader& h = P.h();
  const int nv = h.nv;
  const K2PostRec* post = k2t_post(P);
  #pragma unroll 1
  for (int p = 0; p < h.P; ++p) {
    const float lm = P.f(h.off_posture)[p * (2 + nv) + 1];
    if (lm != 0.f) {
      T s = T(0);
      #pragma unroll 1
      for (int d = 0; d < nv; ++d) { T v = T(post[p * nv + d].wg) * eprow[p * nv + d]; s += v * v; }
      mu += T(lm) * s;
    }
  }
  return mu;
}
// The same with per-instance posture weights (K2PwArgs): the tabled w gain of (p, d) is scaled by the instance's weight
// before it enters the product.  pw: the instance's [P][nv] weights (element type by pw64), or null for a slot without an
// instance (its result is not used).  Weights are clamped as k2_pw does; the status bit is left to the diagonal loop, which
// reads every weight of the instance too.
template <typename T>
BIK_NOINLINE T k2t_posture_lm_pw(PView P, const T* eprow, T mu, const void* pw, int pw64) {
  BIK_IN_SHARED(eprow);
  const PHeader& h = P.h();
  const int nv = h.nv;
  const K2PostRec* post = k2t_post(P);
  int st = 0;
  #pragma unroll 1
  for (int p = 0; p < h.P; ++p) {
    const float lm = P.f(h.off_posture)[p * (2 + nv) + 1];
    if (lm != 0.f) {
      T s = T(0);
      #pragma unroll 1
      for (int d = 0; d < nv; ++d) {
        const T om = pw ? k2_pw<T>(pw, p * nv + d, pw64, &st) : T(1);
        T v = (T(post[p * nv + d].wg) * om) * eprow[p * nv + d];
        s += v * v;
      }
      mu += T(lm) * s;
    }
  }
  return mu;
}
// Start moving `bytes` bytes at p into L2 (the G lanes of a group take a 32-byte sector each in turn); a no-op on the host.
// The posture weights of a tile's instances are fetched this way when the tile starts: the diagonal loop reads them one
// dependent load per dof, on the tile's serial chain, long after the task assembly has hidden the trip to memory.
template <int G>
BIK_HD void k2t_prefetch_l2(const void* p, int bytes, int l) {
#if defined(__CUDA_ARCH__)
  const uintptr_t a = reinterpret_cast<uintptr_t>(p), a0 = a & ~uintptr_t(31);
  #pragma unroll 1
  for (uintptr_t o = a0 + 32u * l; o < a + bytes; o += 32u * G) asm volatile("prefetch.global.L2 [%0];" ::"l"(o));
#else
  (void)p; (void)bytes; (void)l;
#endif
}
// box_dof (bik_k1.h) from the dof's record: the same bounds, combined in the same order, narrowed as there (BD: dof d of the
// instance's bounds `bd`)
template <typename T, bool BD = false>
BIK_HD void k2t_box_dof(const K2DofRec& r, int ncfg, int has_vel, T qi, T dt, T* lo, T* hi, const BoundsRow* bd = nullptr, int d = 0,
                        int* st = nullptr) {
  T l = -T(BIK_INF_F), u = T(BIK_INF_F);
  if (r.qa >= 0) {
    #pragma unroll 1
    for (int c = 0; c < ncfg; ++c) {
      T up, dn;
      if constexpr (BD) {
        T lc = T(r.cfg[c][1]), uc = T(r.cfg[c][2]);
        bd_narrow_cfg<T>(*bd, d, &lc, &uc, st);
        up = T(r.cfg[c][0]) * (uc - qi); dn = T(r.cfg[c][0]) * (qi - lc);
      } else {
        up = T(r.cfg[c][0]) * (T(r.cfg[c][2]) - qi); dn = T(r.cfg[c][0]) * (qi - T(r.cfg[c][1]));
      }
      u = bik_min(u, up); l = bik_max(l, -dn);
    }
  }
  if (has_vel) {
    T vm;
    if constexpr (BD) vm = dt * bd_narrow_vmax<T>(*bd, d, T(r.vmax), st);
    else vm = dt * T(r.vmax);
    u = bik_min(u, vm); l = bik_max(l, -vm);
  }
  *lo = l; *hi = u;
}
// q <- q (+) dq of one free or ball joint (quaternion update)
template <typename T>
BIK_NOINLINE void k2t_integrate_quat_node(const NodeRec& r, T* q, const T* dq) { integrate_node(r, q, dq); }
// Active set left for the next step's warm start: 0 free, 1 lower, 2 upper, +4 = a.dq holds this step's result
template <typename M>
BIK_NOINLINE void k2t_store_warm(signed char* wm, int nu, M lom, M upm) {
  #pragma unroll 1
  for (int i = 0; i < nu; ++i) wm[i] = (signed char)((((lom >> i) & M(1)) ? 1 : (((upm >> i) & M(1)) ? 2 : 0)) | 4);
}

// ---- one tile of NS instances per warp ----------------------------------------------------------------
// F32IO (compile time): every caller buffer and the hand-off hold fp32 -- the batched fast path: the fp64 load / store /
// integrate code is not even compiled in (it tripled the kernel's SASS and its instruction-fetch stalls).  Otherwise the
// element types follow the run-time flags of K2Args.
// STEP (compile time, with F32IO): the form bik_step / bik_step_host / bik_converge launch -- packed task rows (a.pk set,
// a.ep null).  Only the packed staging is compiled in: no dense-row staging, no staging of dense posture errors.
// PW (compile time): per-instance posture weights (K2PwArgs, which `a` then is; the ..._weighted_ex entry points): the tabled coefficients of
// posture task p on dof d are scaled by the instance's weight (w^2 and (gain w) w by its square) before they enter the same
// sums in the same order, so a weight of 1 gives the bits of the unweighted instantiation.
// BD (compile time, with PW): per-instance bounds (K2BdArgs, which `a` then is) narrow each dof's box where it is formed
// (k2t_box_dof); the posture weights may be null.  The decoupled dofs' clamp and the active-set iterations read the same box.
template <typename T, int G, int NS, typename M = uint32_t, bool F32IO = false, bool STEP = false, bool PW = false, bool BD = false>
BIK_HD void k2t_warp_tile(const PView& P, const K2Args& a, long long b0, void* wsm, int lane, int St = 0, int uw = 0) {
  static_assert(!STEP || F32IO, "the step instantiation reads fp32 buffers");
  if (St == 0) { St = k2t_task_tile_words(P); uw = k2t_union_words(P); }   // callers that loop over tiles pass them in
  const int io64 = F32IO ? 0 : a.io64, pk64 = F32IO ? 0 : a.pk64, dense64 = F32IO ? 0 : a.dense64;
  constexpr int W = G * NS;
  const PHeader& h = P.h();
  const int nv = h.nv, nu = h.nu, K = h.K, nq = h.nq, NP = h.P;
  const int32_t* cols = P.i(h.off_cols);
  const int32_t* ucols = P.i(h.off_ucols);
  const int cnt = (a.B - b0) < NS ? (int)(a.B - b0) : NS;
  const int slot = lane / G, l = lane - slot * G;
  const long long b = b0 + slot;
  const bool live = slot < cnt && !(a.skip && a.skip[b]);
  if (a.skip && !BIK_WARP_ANY(live)) return;   // bik_converge: every instance of this tile has converged
  // PW: this instance's posture weights (null for a slot without a live instance: its results are not stored)
  const void* pw = nullptr;
  if constexpr (PW) {
    if (live && NP > 0 && (!BD || static_cast<const K2PwArgs&>(a).pw)) {
      pw = k2_pw_row(a, h, b, io64);
      k2t_prefetch_l2<G>(pw, NP * nv * (io64 ? 8 : 4), l);
    }
  }
  // BD: this instance's bound rows (null rows for a slot without a live instance), fetched into L2 like the posture weights
  BoundsRow bd{};
  if constexpr (BD) {
    if (live) {
      bd = k2_bd_row(a, nv, b, io64);
      for (const void* r : {bd.lo, bd.up, bd.vm}) if (r) k2t_prefetch_l2<G>(r, nv * (io64 ? 8 : 4), l);
    }
  }
  T* const Tb = reinterpret_cast<T*>(wsm);
  T* const Hp = Tb + slot;
  T* const U = Tb + (size_t)tri(nu) * NS;   // warp-wide base of the union region
  T* const Lp = U + slot;
  T* const c = Tb + (size_t)(tri(nu) + uw) * NS + slot;
  T* const vs = c + (size_t)nu * NS;
  T* const xf = vs + (size_t)nu * NS;
  float* const Fb = reinterpret_cast<float*>(Tb + (size_t)(tri(nu) + uw + 3 * nu) * NS);
  float* const lo = Fb + slot;
  float* const hi = Fb + (size_t)nu * NS + slot;

  // ---- assembly ----
  #pragma unroll 1
  for (int k = l; k < tri(nu); k += G) Hp[k * NS] = T(0);
  #pragma unroll 1
  for (int k = l; k < nu; k += G) c[k * NS] = T(0);
  T mu = T(a.damping);
  for (int t = 0; t < h.F + h.C; ++t) {
    const K2TaskRec& tk = k2t_task(P, t);
    BIK_SYNCWARP();
    k2t_stage_task<T, W, NS, STEP>(U, St, lane, cnt, b0, a, pk64, dense64, K, nv, h.pk_stride, cols + tk.coff, tk, P.d(k2t_h(P).w) + tk.pk_off);
    BIK_SYNCWARP();
    k2t_task_accumulate<T, G, NS>(P, U + (size_t)slot * St, tk, Hp, c, &mu, l);
  }
  // q and posture errors: stage, then diagonal / linear term / box; decoupled dofs are finished on the spot
  BIK_SYNCWARP();
  const int Sq = (nq + NP * nv) | 1;
  k2t_stage_q<T, W, NS>(U, Sq, lane, cnt, a.q, io64, b0, nq);
  if (!STEP && NP > 0 && a.ep) k2t_stage_rows<T, W, NS>(U, Sq, nq, lane, cnt, a.ep, dense64, b0 * NP * nv, (long long)NP * nv, NP * nv);
  BIK_SYNCWARP();
  if (NP > 0 && (STEP || !a.ep)) {   // inside bik_step K1 hands no posture error over: e = q* (-) q from the staged q (posture_task.py:107-118)
    const int per = NP * nv;
    const uint32_t mper = ((1u << 20) + per - 1) / per, mnv = ((1u << 20) + nv - 1) / nv;   // k / per, r / nv by multiplication (exact below 2^20 / divisor)
    for (int k = lane; k < NS * per; k += W) {
      const int i = (int)(((uint32_t)k * mper) >> 20), r = k - i * per, p = (int)(((uint32_t)r * mnv) >> 20), d = r - p * nv;
      const T* qq = U + (size_t)i * Sq;
      const long long t0 = ((long long)(a.pbatched ? (b0 + (i < cnt ? i : 0)) : 0) * NP + p) * nq;
      U[(size_t)i * Sq + nq + r] = posture_err_dof<T>(P, d, [&](int j) { return ldin<T>(a.ptgt, t0 + j, io64); }, [&](int j) { return qq[j]; });
    }
    BIK_SYNCWARP();
  }
  int st = 0;
  {
    const T* qrow = U + (size_t)slot * Sq;
    const T* eprow = qrow + nq;
    if constexpr (PW) { if (NP > 0) mu = k2t_posture_lm_pw<T>(P, eprow, mu, pw, io64); }
    else { if (NP > 0) mu = k2t_posture_lm<T>(P, eprow, mu); }
    const K2DofRec* dofs = k2t_dofs(P);
    const K2PostRec* post = k2t_post(P);
    for (int d = l; d < nv; d += G) {
      const K2DofRec& dr = dofs[d];
      const int u = dr.u;
      // hd += w^2 and cd -= ((gain w) w) e per posture task, in task order, as one FMA each: w^2 is exact in double, so
      // adding the tabled w^2 rounds exactly as fma(w, w, hd) did, and (gain w) w is the product the kernel rounded before
      T hd = mu, cd = T(0);
      #pragma unroll 1
      for (int p = 0; p < NP; ++p) {
        const K2PostRec& pr = post[p * nv + d];
        if constexpr (PW) {
          const T om = pw ? k2_pw<T>(pw, p * nv + d, io64, &st) : T(1), om2 = om * om;
          hd += T(pr.w2) * om2;
          cd -= (T(pr.gw2) * om2) * eprow[p * nv + d];
        } else {
          hd += T(pr.w2);
          cd -= T(pr.gw2) * eprow[p * nv + d];
        }
      }
      T bl, bu;
      k2t_box_dof<T, BD>(dr, h.ncfg, h.has_vel, dr.qa >= 0 ? qrow[dr.qa] : T(0), T(a.dt), &bl, &bu, &bd, d, &st);
      if (bl > bu + T(1e-9) * (T(1) + (bu < 0 ? -bu : bu))) st |= 8;   // inconsistent limits: the reference's QP has no solution (solve_ik.py:103)
      if (u >= 0) { Hp[(tri(u) + u) * NS] += hd; c[u * NS] += cd; lo[u * NS] = float(bl); hi[u * NS] = float(bu); }
      else {
        T v = -cd / hd;
        v = v < bl ? bl : (v > bu ? bu : v);
        if (!(v == v)) st |= 4;
        if (live) stout<T>(a.dq, b * nv + d, io64, v);
      }
    }
  }
  BIK_SYNCWARP();   // the tile is dead; the union region becomes each slot's factor

  // ---- dofs without any finite bound are minimised over once (SURVEY 8a: the free joint has no limits) ----
  // The image lists them first (nf = h.nfree leading coupled dofs).  Their columns of the factor do not depend on the
  // active set, so they are produced once; the pivoting iterations then run on the Schur complement (nu - nf dofs:
  // 12 instead of 18 for the G1 configuration), and the leading part of x is recovered by continuing the last back
  // substitution.  With nf == 0 this block does nothing; with nf == nu (no bounded dof at all) it is the whole solve.
  const int nf = h.nfree;
  T* const rhsrow = Lp + tri(nu) * NS;
  if (nf > 0) {
    for (int k = l; k < nf; k += G) rhsrow[k * NS] = -c[k * NS];
    BIK_SYNCWARP();
    if (k2t_factor<T, G, NS, M>(Hp, Lp, nu, M(0), l, 0, nf)) st |= 4;
    BIK_SYNCWARP();
    k2t_schur<T, G, NS>(Hp, Lp, c, nu, nf, l);
    BIK_SYNCWARP();
  }

  // ---- active-set guess, then the primal active-set method ----
  const int MAXIT = 400;   // the primal active-set method needs ~20 at most
  const T tolx = K2Tol<T>::x(), tolg = K2Tol<T>::g();
  constexpr int IB = sizeof(M) == 8 ? 6 : 5;                       // index bits in the packed (value, index) keys
  constexpr uint32_t KEYV = 0x7fffffffu & ~((1u << IB) - 1u), KEYI = (1u << IB) - 1u;
  M lom = M(0), upm = M(0);
  const bool guess = nf < nu;   // with nf == nu there is no bound to guess and the loop below does not run
  if (guess) {
    // Starting point of the guess: zero, or -- inside a rollout, from its second step on -- the previous step's dq (still
    // in a.dq; the warm-state bytes carry a marker once this kernel has written it), clipped to this step's box.
    const bool have_prev = a.warm != nullptr;   // warp-uniform
    if (have_prev) {
      const bool valid = live && (a.warm[b * nu] & 4);
      for (int k = nf + l; k < nu; k += G) {
        T v = valid ? ldin<T>(a.dq, b * nv + ucols[k], io64) : T(0);
        if (!(v == v)) v = T(0);
        const T bl = T(lo[k * NS]), bu = T(hi[k * NS]);
        vs[k * NS] = v < bl ? bl : (v > bu ? bu : v);
      }
      BIK_SYNCWARP();
    }
    k2t_pgs_guess<T, G, NS, M>(Hp, c, lo, hi, vs, rhsrow, Lp + tri(nu - 1) * NS, nu, nf, l, h.k2_sweeps, have_prev, &lom, &upm);   // scratch: free strips of the factor
    for (int k = nf + l; k < nu; k += G) xf[k * NS] = vs[k * NS];   // the Gauss-Seidel iterate is feasible: it is where the active-set method starts
    BIK_SYNCWARP();
  }
  bool done = nf == nu;    // no bounded dof at all: the elimination above was the whole solve (one factorisation)
  int it = done ? 1 : 0;
  for (;;) {
    if (!BIK_WARP_ANY(!done && it < MAXIT)) break;
    const bool run = !done && it < MAXIT;   // a finished group keeps executing (idempotently) until its warp is done
    const M act = lom | upm;
    // x on the bounds
    for (int k = nf + l; k < nu; k += G) vs[k * NS] = ((lom >> k) & M(1)) ? T(lo[k * NS]) : (((upm >> k) & M(1)) ? T(hi[k * NS]) : T(0));
    BIK_SYNCWARP();
    // right-hand side of the masked system: bound value on clamped dofs, -(c + H_FA x_A) on free ones
    for (int k = nf + l; k < nu; k += G) {
      T rv;
      if ((act >> k) & M(1)) rv = vs[k * NS];
      else { rv = -c[k * NS]; if (act) rv -= k2t_row_dot<T, NS>(Hp, vs, k, nu, nf); }
      rhsrow[k * NS] = rv;
    }
    BIK_SYNCWARP();
    if (k2t_factor<T, G, NS, M>(Hp, Lp, nu, act, l, nf, nu)) st |= 4;
    BIK_SYNCWARP();
    k2t_backsub<T, G, NS>(Lp, nu, l, vs, nu, nf, nf);
    BIK_SYNCWARP();
    // gradient on the clamped dofs, feasibility of the free ones
    M vlo = M(0), vup = M(0), rel = M(0);   // free dofs that violate a bound / clamped dofs whose multiplier has the wrong sign
    int worst = 0;                            // (float bits of the largest wrong-signed multiplier, low 5 bits = its index)
    int blocking = 0x7fffffff;                // (float bits of the smallest step length to a violated bound, low 5 bits = its index)
    for (int k = nf + l; k < nu; k += G) {
      const M bit = M(1) << k;
      if (!(act & bit)) {
        const T xi = vs[k * NS], bl = T(lo[k * NS]), bu = T(hi[k * NS]);
        const bool below = xi < bl - tolx * (T(1) + (bl < 0 ? -bl : bl));
        const bool above = !below && xi > bu + tolx * (T(1) + (bu < 0 ? -bu : bu));
        if (below) vlo |= bit;
        if (above) vup |= bit;
        if (below || above) {   // how far the feasible iterate can move towards x before this bound stops it
          const T xo = xf[k * NS], d = xi - xo;
          T al = d != T(0) ? ((below ? bl : bu) - xo) / d : T(0);
          al = al < T(0) ? T(0) : (al > T(1) ? T(1) : al);
          const int key = (int)((bik_float_bits(float(al)) & KEYV) | (uint32_t)k);
          blocking = key < blocking ? key : blocking;
        }
      } else {
        T gi = c[k * NS] + k2t_row_dot<T, NS>(Hp, vs, k, nu, nf);
        if (upm & bit) gi = -gi;              // now: gi < 0 means the bound wants to let go
        if (gi < -tolg) {
          rel |= bit;
          const int key = (int)((bik_float_bits(float(-gi)) & KEYV) | (uint32_t)k);
          worst = key > worst ? key : worst;
        }
      }
    }
    vlo = grp_or_m<G>(vlo); vup = grp_or_m<G>(vup); rel = grp_or_m<G>(rel);
    worst = grp_max<G>(worst);
    T alpha = T(0), bound = T(0);
    int kb = 0;
    blocking = -grp_max<G>(-blocking);
    if (vlo | vup) {   // exact step length to the blocking bound (the key only ranked the candidates in fp32)
      kb = blocking & (int)KEYI;
      const T xo = xf[kb * NS], d = vs[kb * NS] - xo;
      bound = ((vlo >> kb) & M(1)) ? T(lo[kb * NS]) : T(hi[kb * NS]);
      alpha = d != T(0) ? (bound - xo) / d : T(0);
      alpha = alpha < T(0) ? T(0) : (alpha > T(1) ? T(1) : alpha);
    }
    BIK_SYNCWARP();   // every lane has read x (and the feasible iterate) before anything below or the next iteration overwrites them
    if (run) {
      ++it;
      // Primal active-set step from the feasible iterate xf (started at the Gauss-Seidel guess): block flips cycle on a few
      // instances per thousand once a rollout is under way, and flipping every violated dof at once gives up monotone
      // descent.  Here the objective decreases at every step, so the method terminates: move towards the subspace minimiser
      // x until the first bound stops the move and clamp that dof; at a feasible subspace minimiser let go of the bound with
      // the worst multiplier, or stop if there is none.
      // (a population count, not a test of the mask: with the test, the 64-bit-mask step instantiation is laid out
      // differently and g1_full's step was 0.5 % slower on one H100 80GB HBM3, SXM, 400 W power limit)
      if (bik_popc(vlo | vup | rel) == 0) done = true;
      else if (vlo | vup) {
        for (int k = nf + l; k < nu; k += G) {
          if (k == kb) xf[k * NS] = bound;
          else if (!((act >> k) & M(1))) xf[k * NS] += alpha * (vs[k * NS] - xf[k * NS]);
        }
        const M bit = M(1) << kb;
        if (vlo & bit) lom |= bit; else upm |= bit;
      } else {
        for (int k = nf + l; k < nu; k += G) xf[k * NS] = vs[k * NS];
        const M bit = M(1) << (worst & (int)KEYI);
        lom &= ~bit; upm &= ~bit;
      }
    }
  }
  if (nf > 0) {   // x_b = L_bb^-T (y_b - L_t^T x_t): the back substitution simply continues into the leading rows
    k2t_backsub_cross<T, G, NS>(Lp, nu, l, vs, nu, nf, nf);
    BIK_SYNCWARP();
    k2t_backsub<T, G, NS>(Lp, nu, l, vs, nf, 0, 0);
    BIK_SYNCWARP();
  }
  if (!done) st |= 2;
  // ---- outputs: coupled dofs from vs (the last solve), status, warm-start state ----
  for (int k = l; k < nu; k += G) {
    const T v = vs[k * NS];
    if (!(v == v)) st |= 4;
    if (live) stout<T>(a.dq, b * nv + ucols[k], io64, v);
  }
  st = grp_or<G>(st);
  if (live && l == 0) {
    if (a.status) a.status[b] |= st;
    if (a.iters) a.iters[b] = it;
    if (a.warm) k2t_store_warm<M>(a.warm + b * nu, nu, lom, upm);
  }
  BIK_SYNCWARP();
  // ---- q <- q (+) dq (Configuration.integrate_inplace, configuration.py:228-236): the lanes of a group take the nodes in turn ----
  if (a.integrate) {
    // scalar joints (hinge / slide): the whole warp sweeps the tile's dofs flat -- coalesced, independent loads; free and ball
    // joints (quaternion update) are left to one lane per joint
    const int32_t* dofqadr = P.i(h.off_dofqadr);
    const uint32_t mnv = ((1u << 20) + nv - 1) / nv;
    auto sweep = [&](auto* qg, const auto* dg) {
      #pragma unroll 1
      for (int k = lane; k < cnt * nv; k += W) {
        const int i = (int)(((uint32_t)k * mnv) >> 20), d = k - i * nv, qa = dofqadr[d];
        if (qa >= 0 && !(a.skip && a.skip[b0 + i])) qg[(b0 + i) * nq + qa] += dg[(b0 + i) * nv + d];
      }
      if (live) { const K2Header& kh = k2t_h(P); for (int k = l; k < kh.nquat; k += G) k2t_integrate_quat_node(P.node(P.i(kh.quat)[k]), qg + b * nq, dg + b * nv); }
    };
    if (F32IO || !io64) sweep(reinterpret_cast<float*>(const_cast<void*>(a.q)), reinterpret_cast<const float*>(a.dq));   // fp32 buffers: fp32 arithmetic, as bik_integrate
    else sweep(reinterpret_cast<double*>(const_cast<void*>(a.q)), reinterpret_cast<const double*>(a.dq));
  }
  BIK_SYNCWARP();
}

}  // namespace bik
