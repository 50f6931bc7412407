// bik_k1.cu -- K1 kernels: FK + task errors / Jacobians + collision rows + check_limits (k1_kernel), and the FK / body-frame
// Jacobian kernel behind the Configuration API (fk_kernel).  Both are persistent (grid = SMs x resident CTAs, CTAs loop over
// warp tiles) and begin by staging the problem image into shared memory with one bulk async copy.
#include "bik_dev.cuh"

using namespace bik;

#ifndef BIK_K1_MINBLOCKS
#define BIK_K1_MINBLOCKS 4   // CTAs of 4 warps per SM the register allocation must allow (fp32): 4 -> 128 registers, no spills, 16 warps/SM.
                             // H100 (700 W), G1 at 65 536: K1 of the step 0.090 ms, dense API form 0.213 ms; 5 -> 96 registers with
                             // 44-64 B of spill stores: 0.094 / 0.286 ms
#endif
template <typename T, int G, bool PK, bool TR>
__global__ void __launch_bounds__(128, sizeof(T) == 4 ? BIK_K1_MINBLOCKS : 2) k1_kernel(const uint32_t* __restrict__ gimage, int words, int use_tma, K1Args a) {
  extern __shared__ __align__(16) uint32_t smem[];
  __shared__ __align__(8) uint64_t bar;
  __shared__ __align__(8) uint64_t pbar[4];   // one input-pipeline barrier per warp
  stage_image(smem, gimage, words, &bar, use_tma);
  PView P{smem};
  const PHeader& h = P.h();
  constexpr int IPW = 32 / G;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  T* wsm = reinterpret_cast<T*>(smem + words) + (size_t)warp * k1_warp_words(h, IPW);
  const int ntiles = (a.B + IPW - 1) / IPW, stride = gridDim.x * nwarps;
  int tile = blockIdx.x * nwarps + warp;
  // Input pipeline: tile t computes its Jacobian columns while the q rows and targets of tile t + stride arrive by bulk async
  // copy (BIK_USE_TMA=0 turns it off together with the staged image: plain loads at the top of every tile).
  K1Pipe pipe{&pbar[warp], 0u, -1};
  K1Pipe* pp = use_tma ? &pipe : nullptr;
  if (pp) {
    if (lane == 0) {
      mbar_init(pipe.bar, 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
    if (tile < ntiles && k1_tile_bulk_ok<T, TR>(h, a, tile * IPW, IPW)) {
      T* qtile = wsm + k1_qtile_offset(h, IPW);
      if (lane == 0) k1_pipe_arm<T, TR>(h, a, tile * IPW, IPW, &pipe, qtile, qtile + ((IPW * h.nq + 3) & ~3));
      pipe.armed = tile * IPW;
    }
  }
  for (; tile < ntiles; tile += stride) {
    const int next = tile + stride < ntiles ? (tile + stride) * IPW : -1;
    k1_warp_tile<T, G, 32, PK, TR>(P, a, tile * IPW, wsm, lane, pp, next);
  }
}

// The same with per-instance collision pairs and distances (K1CArgs): the ..._coll entry points.  Packed hand-off only.
// (a kernel of its own rather than a template argument of k1_kernel, so that every k1_kernel instantiation keeps its code)
template <typename T, int G, bool TR>
__global__ void __launch_bounds__(128, sizeof(T) == 4 ? BIK_K1_MINBLOCKS : 2) k1c_kernel(const uint32_t* __restrict__ gimage, int words, int use_tma, K1CArgs a) {
  constexpr bool PK = true;
  extern __shared__ __align__(16) uint32_t smem[];
  __shared__ __align__(8) uint64_t bar;
  __shared__ __align__(8) uint64_t pbar[4];   // one input-pipeline barrier per warp
  stage_image(smem, gimage, words, &bar, use_tma);
  PView P{smem};
  const PHeader& h = P.h();
  constexpr int IPW = 32 / G;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  T* wsm = reinterpret_cast<T*>(smem + words) + (size_t)warp * k1_warp_words(h, IPW);
  const int ntiles = (a.B + IPW - 1) / IPW, stride = gridDim.x * nwarps;
  int tile = blockIdx.x * nwarps + warp;
  // Input pipeline: tile t computes its Jacobian columns while the q rows and targets of tile t + stride arrive by bulk async
  // copy (BIK_USE_TMA=0 turns it off together with the staged image: plain loads at the top of every tile).
  K1Pipe pipe{&pbar[warp], 0u, -1};
  K1Pipe* pp = use_tma ? &pipe : nullptr;
  if (pp) {
    if (lane == 0) {
      mbar_init(pipe.bar, 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
    if (tile < ntiles && k1_tile_bulk_ok<T, TR>(h, a, tile * IPW, IPW)) {
      T* qtile = wsm + k1_qtile_offset(h, IPW);
      if (lane == 0) k1_pipe_arm<T, TR>(h, a, tile * IPW, IPW, &pipe, qtile, qtile + ((IPW * h.nq + 3) & ~3));
      pipe.armed = tile * IPW;
    }
  }
  for (; tile < ntiles; tile += stride) {
    const int next = tile + stride < ntiles ? (tile + stride) * IPW : -1;
    k1_warp_tile<T, G, 32, PK, TR, true>(P, a, tile * IPW, wsm, lane, pp, next);
  }
}

// Track mode with held targets (K1HArgs): the bik_track_hold entry points, with (CO) or without per-instance collision
// arguments.  A kernel of its own for the same reason.
template <typename T, int G, bool CO>
__global__ void __launch_bounds__(128, sizeof(T) == 4 ? BIK_K1_MINBLOCKS : 2) k1h_kernel(const uint32_t* __restrict__ gimage, int words, int use_tma, K1HArgs a) {
  constexpr bool PK = true;
  extern __shared__ __align__(16) uint32_t smem[];
  __shared__ __align__(8) uint64_t bar;
  __shared__ __align__(8) uint64_t pbar[4];   // one input-pipeline barrier per warp
  stage_image(smem, gimage, words, &bar, use_tma);
  PView P{smem};
  const PHeader& h = P.h();
  constexpr int IPW = 32 / G;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  T* wsm = reinterpret_cast<T*>(smem + words) + (size_t)warp * k1_warp_words(h, IPW);
  const int ntiles = (a.B + IPW - 1) / IPW, stride = gridDim.x * nwarps;
  int tile = blockIdx.x * nwarps + warp;
  // Input pipeline: tile t computes its Jacobian columns while the q rows and targets of tile t + stride arrive by bulk async
  // copy (BIK_USE_TMA=0 turns it off together with the staged image: plain loads at the top of every tile).
  K1Pipe pipe{&pbar[warp], 0u, -1};
  K1Pipe* pp = use_tma ? &pipe : nullptr;
  if (pp) {
    if (lane == 0) {
      mbar_init(pipe.bar, 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
    if (tile < ntiles && k1_tile_bulk_ok<T, true>(h, a, tile * IPW, IPW)) {
      T* qtile = wsm + k1_qtile_offset(h, IPW);
      if (lane == 0) k1_pipe_arm<T, true>(h, a, tile * IPW, IPW, &pipe, qtile, qtile + ((IPW * h.nq + 3) & ~3));
      pipe.armed = tile * IPW;
    }
  }
  for (; tile < ntiles; tile += stride) {
    const int next = tile + stride < ntiles ? (tile + stride) * IPW : -1;
    k1_warp_tile<T, G, 32, PK, true, CO, true>(P, a, tile * IPW, wsm, lane, pp, next);
  }
}

// Per-instance frame placement (K1PArgs): the ..._placed entry points, step and converge (TR = false) or track (TR), with held
// targets in track (HO); the collision arguments may be null.  A kernel of its own for the same reason.
template <typename T, int G, bool TR, bool HO>
__global__ void __launch_bounds__(128, sizeof(T) == 4 ? BIK_K1_MINBLOCKS : 2) k1p_kernel(const uint32_t* __restrict__ gimage, int words, int use_tma, K1PArgs a) {
  static_assert(!HO || TR, "held targets are a track-mode feature");
  constexpr bool PK = true;
  extern __shared__ __align__(16) uint32_t smem[];
  __shared__ __align__(8) uint64_t bar;
  __shared__ __align__(8) uint64_t pbar[4];   // one input-pipeline barrier per warp
  stage_image(smem, gimage, words, &bar, use_tma);
  PView P{smem};
  const PHeader& h = P.h();
  constexpr int IPW = 32 / G;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  T* wsm = reinterpret_cast<T*>(smem + words) + (size_t)warp * k1_warp_words(h, IPW);
  const int ntiles = (a.B + IPW - 1) / IPW, stride = gridDim.x * nwarps;
  int tile = blockIdx.x * nwarps + warp;
  // Input pipeline: tile t computes its Jacobian columns while the q rows and targets of tile t + stride arrive by bulk async
  // copy (BIK_USE_TMA=0 turns it off together with the staged image: plain loads at the top of every tile).
  K1Pipe pipe{&pbar[warp], 0u, -1};
  K1Pipe* pp = use_tma ? &pipe : nullptr;
  if (pp) {
    if (lane == 0) {
      mbar_init(pipe.bar, 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
    if (tile < ntiles && k1_tile_bulk_ok<T, TR>(h, a, tile * IPW, IPW)) {
      T* qtile = wsm + k1_qtile_offset(h, IPW);
      if (lane == 0) k1_pipe_arm<T, TR>(h, a, tile * IPW, IPW, &pipe, qtile, qtile + ((IPW * h.nq + 3) & ~3));
      pipe.armed = tile * IPW;
    }
  }
  for (; tile < ntiles; tile += stride) {
    const int next = tile + stride < ntiles ? (tile + stride) * IPW : -1;
    k1_warp_tile<T, G, 32, PK, TR, true, HO, true>(P, a, tile * IPW, wsm, lane, pp, next);
  }
}

template <typename T, int G>
__global__ void __launch_bounds__(128) fk_kernel(const uint32_t* __restrict__ gimage, int words, int use_tma, FkArgs a) {
  extern __shared__ __align__(16) uint32_t smem[];
  __shared__ __align__(8) uint64_t bar;
  stage_image(smem, gimage, words, &bar, use_tma);
  PView P{smem};
  constexpr int IPW = 32 / G;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  T* wsm = reinterpret_cast<T*>(smem + words) + (size_t)warp * fk_warp_words(P.h(), IPW);
  const int ntiles = (a.B + IPW - 1) / IPW;
  for (int tile = blockIdx.x * nwarps + warp; tile < ntiles; tile += gridDim.x * nwarps) fk_warp_tile<T, G, 32>(P, a, tile * IPW, wsm, lane);
}

// Launch K1 kernel `kern` (a k1_kernel, k1c_kernel, k1h_kernel or k1p_kernel instantiation of scalar type T and G lanes per instance).
template <typename T, int G, typename A>
static int launch_k1_kernel(const bik_problem* p, void (*kern)(const uint32_t*, int, int, A), const A& a, cudaStream_t st) {
  const PHeader& h = p->h;
  constexpr int IPW = 32 / G;
  const int words = sizeof(T) == 8 ? h.words64 : h.words32;   // the fp64 side tables only travel with the fp64 instantiation
  int NW = 4;  // warps per CTA: as many as fit next to the image in shared memory
  auto need = [&](int nw) { return (size_t)words * 4 + (size_t)nw * k1_warp_words(h, IPW) * sizeof(T); };
  while (NW > 1 && (int)need(NW) > p->model->max_smem) NW >>= 1;
  size_t smem = need(NW);
  int grid = 1;
  long long tiles = ((long long)a.B + IPW - 1) / IPW;
  int rc = bik_launch_geometry((const void*)kern, p->model, smem, 32 * NW, (tiles + NW - 1) / NW, &grid);
  if (rc) return rc;
  kern<<<grid, 32 * NW, smem, st>>>(p->d_image, words, p->model->use_tma, a);
  CUDA_OK(cudaGetLastError());
  return BIK_OK;
}
template <typename T, int G>
static int launch_k1(const bik_problem* p, const K1Args& a, cudaStream_t st) {
  if (!a.pk) return launch_k1_kernel<T, G>(p, k1_kernel<T, G, false, false>, a, st);
  return launch_k1_kernel<T, G>(p, a.cursor ? k1_kernel<T, G, true, true> : k1_kernel<T, G, true, false>, a, st);
}
template <typename T, int G>
static int launch_k1(const bik_problem* p, const K1CArgs& a, cudaStream_t st) {
  return launch_k1_kernel<T, G>(p, a.cursor ? k1c_kernel<T, G, true> : k1c_kernel<T, G, false>, a, st);
}
template <typename T, int G>
static int launch_k1(const bik_problem* p, const K1HArgs& a, cudaStream_t st) {
  const bool co = a.enabled || a.dmin || a.ddet;
  return launch_k1_kernel<T, G>(p, co ? k1h_kernel<T, G, true> : k1h_kernel<T, G, false>, a, st);
}
template <typename T, int G>
static int launch_k1(const bik_problem* p, const K1PArgs& a, cudaStream_t st) {
  if (!a.cursor) return launch_k1_kernel<T, G>(p, k1p_kernel<T, G, false, false>, a, st);
  return launch_k1_kernel<T, G>(p, a.hold ? k1p_kernel<T, G, true, true> : k1p_kernel<T, G, true, false>, a, st);
}
template <typename T, typename A>
static int dispatch_k1(const bik_problem* p, const A& a, cudaStream_t st) {
  switch (p->h.G) {
    case 1: return launch_k1<T, 1>(p, a, st);
    case 2: return launch_k1<T, 2>(p, a, st);
    case 4: return launch_k1<T, 4>(p, a, st);
    case 8: return launch_k1<T, 8>(p, a, st);
    case 16: return launch_k1<T, 16>(p, a, st);
    default: return launch_k1<T, 32>(p, a, st);
  }
}
int bik_launch_k1(const bik_problem* p, const K1Args& a, bool use_double, cudaStream_t st) {
  if (!use_double && a.in64) return bik_fail(BIK_ERR_INVALID, "fp64 inputs need the fp64 instantiation of K1");
  return use_double ? dispatch_k1<double>(p, a, st) : dispatch_k1<float>(p, a, st);
}
int bik_launch_k1(const bik_problem* p, const K1CArgs& a, bool use_double, cudaStream_t st) {
  if (!use_double && a.in64) return bik_fail(BIK_ERR_INVALID, "fp64 inputs need the fp64 instantiation of K1");
  if (!a.pk) return bik_fail(BIK_ERR_INVALID, "per-instance collision pairs need the packed hand-off");
  return use_double ? dispatch_k1<double>(p, a, st) : dispatch_k1<float>(p, a, st);
}
int bik_launch_k1(const bik_problem* p, const K1HArgs& a, bool use_double, cudaStream_t st) {
  if (!use_double && a.in64) return bik_fail(BIK_ERR_INVALID, "fp64 inputs need the fp64 instantiation of K1");
  if (!a.pk || !a.cursor || !a.held) return bik_fail(BIK_ERR_INVALID, "held targets need track mode's packed hand-off and a held buffer");
  return use_double ? dispatch_k1<double>(p, a, st) : dispatch_k1<float>(p, a, st);
}
int bik_launch_k1(const bik_problem* p, const K1PArgs& a, bool use_double, cudaStream_t st) {
  if (!use_double && a.in64) return bik_fail(BIK_ERR_INVALID, "fp64 inputs need the fp64 instantiation of K1");
  if (!a.pk || !a.placement) return bik_fail(BIK_ERR_INVALID, "frame placement needs the packed hand-off and a placement buffer");
  if (a.hold && (!a.cursor || !a.held)) return bik_fail(BIK_ERR_INVALID, "held targets need track mode and a held buffer");
  return use_double ? dispatch_k1<double>(p, a, st) : dispatch_k1<float>(p, a, st);
}

template <typename T, int G>
static int launch_fk(const bik_model* m, const FkArgs& a, cudaStream_t st) {
  const PHeader& h = m->h;
  constexpr int IPW = 32 / G, THREADS = 128, NW = THREADS / 32;
  const int words = sizeof(T) == 8 ? h.words64 : h.words32;
  size_t smem = (size_t)words * 4 + (size_t)NW * fk_warp_words(h, IPW) * sizeof(T);
  int grid = 1;
  long long tiles = ((long long)a.B + IPW - 1) / IPW;
  int rc = bik_launch_geometry((const void*)fk_kernel<T, G>, m, smem, THREADS, (tiles + NW - 1) / NW, &grid);
  if (rc) return rc;
  fk_kernel<T, G><<<grid, THREADS, smem, st>>>(m->d_image, words, m->use_tma, a);
  CUDA_OK(cudaGetLastError());
  return BIK_OK;
}
template <typename T>
static int dispatch_fk(const bik_model* m, const FkArgs& a, cudaStream_t st) {
  switch (m->h.G) {
    case 1: return launch_fk<T, 1>(m, a, st);
    case 2: return launch_fk<T, 2>(m, a, st);
    case 4: return launch_fk<T, 4>(m, a, st);
    case 8: return launch_fk<T, 8>(m, a, st);
    case 16: return launch_fk<T, 16>(m, a, st);
    default: return launch_fk<T, 32>(m, a, st);
  }
}
int bik_launch_fk(const bik_model* m, const FkArgs& a, cudaStream_t st) { return a.io64 ? dispatch_fk<double>(m, a, st) : dispatch_fk<float>(m, a, st); }
