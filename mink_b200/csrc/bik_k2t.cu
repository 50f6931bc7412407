// bik_k2t.cu -- small-group K2 path (bik_k2t.h): G lanes per problem, 32/G problems per warp; tables are read straight from
// the (L1-resident) global image so that all of shared memory goes to the per-problem triangles; warps are independent.
// Tiles are handed out by an atomic counter (sched[0]) when the launcher has one for this stream: the pivoting count
// differs between instances (G1: 91 % need one iteration, 1 in 10 000 needs six or more), and with a static round-robin
// the warp that meets a slow instance also keeps its whole share of ordinary tiles, which set the kernel time.  The last
// CTA to leave (sched[1] counts them) rewinds the counter for the next launch on the stream.
//
// The kernel is bound by instruction issue and fetch, so its code size is part of its speed.  bik_step, bik_step_host and
// bik_converge launch a STEP instantiation (fp32 buffers, packed rows) that leaves out the dense-row staging, keeps one-off
// work out of line and does not unroll the solver loops: 9 216 SASS instructions on sm_90a for G = 8 instead of 17 592, and
// K2 in the G1 step 0.60 ms instead of 0.78 ms on one H100 80GB HBM3 (SXM, 700 W power limit).
// tests/test_k2_code_size_cpu.py keeps it that size.
#include "bik_dev.cuh"

using namespace bik;

constexpr int K2T_MAXT = 256;   // threads per CTA at most; two CTAs per SM

// The body of both kernels: tiles from the counter, or round-robin.
template <typename T, int G, typename M, bool F32IO, bool STEP, bool PW, bool BD = false>
__device__ __forceinline__ void k2t_tiles(const uint32_t* __restrict__ gimage, int warp_bytes, const K2Args& a, unsigned int* sched) {
  extern __shared__ __align__(16) uint32_t smem[];
  constexpr int NS = 32 / G;
  if (a.gate && *a.gate == 0) return;   // (uniform over the grid: the tile counter is left untouched)
  PView P{gimage};
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  char* wsm = reinterpret_cast<char*>(smem) + (size_t)warp * warp_bytes;
  const long long ntiles = ((long long)a.B + NS - 1) / NS;
  const int St = k2t_task_tile_words(P), uw = k2t_union_words(P);
  if (sched) {
    for (;;) {
      unsigned int t = 0;
      if (lane == 0) t = atomicAdd(&sched[0], 1u);
      t = __shfl_sync(0xffffffffu, t, 0);
      if ((long long)t >= ntiles) break;
      k2t_warp_tile<T, G, NS, M, F32IO, STEP, PW, BD>(P, a, (long long)t * NS, wsm, lane, St, uw);
    }
    __syncthreads();
    if (threadIdx.x == 0 && atomicInc(&sched[1], gridDim.x - 1) == gridDim.x - 1) { __threadfence(); sched[0] = 0u; }
    return;
  }
  for (long long tile = (long long)blockIdx.x * nwarps + warp; tile < ntiles; tile += (long long)gridDim.x * nwarps)
    k2t_warp_tile<T, G, NS, M, F32IO, STEP, PW, BD>(P, a, tile * NS, wsm, lane, St, uw);
}
// Launched as k2t_kernel<double, G, K2T_MAXT, ...> only; T and MAXT stay in the template, and so in the kernel's symbol.
template <typename T, int G, int MAXT, typename M, bool F32IO, bool STEP>
__global__ void __launch_bounds__(MAXT, 512 / MAXT) k2t_kernel(const uint32_t* __restrict__ gimage, int warp_bytes, K2Args a, unsigned int* sched) {
  k2t_tiles<T, G, M, F32IO, STEP, false>(gimage, warp_bytes, a, sched);
}
// The same with per-instance posture weights (K2PwArgs): the ..._weighted_ex entry points with a posture-weights buffer.
template <typename T, int G, int MAXT, typename M, bool F32IO, bool STEP>
__global__ void __launch_bounds__(MAXT, 512 / MAXT) k2t_pw_kernel(const uint32_t* __restrict__ gimage, int warp_bytes, K2PwArgs a, unsigned int* sched) {
  k2t_tiles<T, G, M, F32IO, STEP, true>(gimage, warp_bytes, a, sched);
}
// The same with per-instance bounds and posture weights, which may be null (K2BdArgs): the ..._bounded entry points with bounds.
template <typename T, int G, int MAXT, typename M, bool F32IO, bool STEP>
__global__ void __launch_bounds__(MAXT, 512 / MAXT) k2t_bd_kernel(const uint32_t* __restrict__ gimage, int warp_bytes, K2BdArgs a, unsigned int* sched) {
  k2t_tiles<T, G, M, F32IO, STEP, true, true>(gimage, warp_bytes, a, sched);
}

// warps per CTA: as many as shared memory holds, at most K2T_MAXT / 32
static int k2t_warps(const bik_problem* p, size_t wb) {
  int NW = K2T_MAXT / 32;
  while (NW > 1 && NW * wb > (size_t)p->model->max_smem) --NW;
  return NW;
}
// A: K2Args (k2t_kernel), K2PwArgs (k2t_pw_kernel) or K2BdArgs (k2t_bd_kernel)
template <int G, typename M, bool F32IO, bool STEP, typename A>
static int launch_k2t_io(const bik_problem* p, const A& a, unsigned int* sched, cudaStream_t st) {
  constexpr int NS = 32 / G;
  constexpr bool PW = std::is_same<A, K2PwArgs>::value, BD = std::is_same<A, K2BdArgs>::value;
  PView P{p->image.data()};
  const size_t wb = (size_t)k2t_warp_bytes(P, sizeof(double), NS);
  const int NW = k2t_warps(p, wb);
  const size_t smem = NW * wb;
  int grid = 1;
  long long tiles = ((long long)a.B + NS - 1) / NS;
  const void* kern;
  if constexpr (BD) kern = (const void*)k2t_bd_kernel<double, G, K2T_MAXT, M, F32IO, STEP>;
  else if constexpr (PW) kern = (const void*)k2t_pw_kernel<double, G, K2T_MAXT, M, F32IO, STEP>;
  else kern = (const void*)k2t_kernel<double, G, K2T_MAXT, M, F32IO, STEP>;
  int rc = bik_launch_geometry(kern, p->model, smem, 32 * NW, (tiles + NW - 1) / NW, &grid);
  if (rc) return rc;
  if constexpr (BD) k2t_bd_kernel<double, G, K2T_MAXT, M, F32IO, STEP><<<grid, 32 * NW, smem, st>>>(p->d_image, (int)wb, a, sched);
  else if constexpr (PW) k2t_pw_kernel<double, G, K2T_MAXT, M, F32IO, STEP><<<grid, 32 * NW, smem, st>>>(p->d_image, (int)wb, a, sched);
  else k2t_kernel<double, G, K2T_MAXT, M, F32IO, STEP><<<grid, 32 * NW, smem, st>>>(p->d_image, (int)wb, a, sched);
  CUDA_OK(cudaGetLastError());
  return BIK_OK;
}
// posture weights or bounds (A: K2PwArgs or K2BdArgs): only the packed forms that bik_step / bik_converge / bik_track launch are
// instantiated
template <int G, typename M, typename A>
static int launch_k2t_packed(const bik_problem* p, const A& a, unsigned int* sched, cudaStream_t st) {
  if (!a.pk || a.dense64) return bik_fail(BIK_ERR_UNSUPPORTED, "posture weights and bounds need the packed task rows of bik_step / bik_converge / bik_track");
  if (a.io64 || a.pk64) return launch_k2t_io<G, M, false, false>(p, a, sched, st);
  return launch_k2t_io<G, M, true, true>(p, a, sched, st);
}
template <int G, typename M>
static int launch_k2t(const bik_problem* p, const K2PwArgs& a, unsigned int* sched, cudaStream_t st) { return launch_k2t_packed<G, M>(p, a, sched, st); }
template <int G, typename M>
static int launch_k2t(const bik_problem* p, const K2BdArgs& a, unsigned int* sched, cudaStream_t st) { return launch_k2t_packed<G, M>(p, a, sched, st); }
template <int G, typename M>
static int launch_k2t(const bik_problem* p, const K2Args& a, unsigned int* sched, cudaStream_t st) {
  if (a.io64 || a.pk64 || a.dense64) return launch_k2t_io<G, M, false, false>(p, a, sched, st);
  // fp32 buffers everywhere; packed rows from K1 are the step's form
  return a.pk ? launch_k2t_io<G, M, true, true>(p, a, sched, st) : launch_k2t_io<G, M, true, false>(p, a, sched, st);
}
static int group_of(const bik_problem* p) { return (p->h.nu > K2T_NMAX || p->k2_group == 8) ? 8 : 4; }

bool bik_k2_group_applies(const bik_problem* p) {
  const PHeader& h = p->h;
  if (p->k2_general || h.npairs != 0 || h.nu < 1 || h.nu > K2T_NMAX_WIDE) return false;
  PView P{p->image.data()};
  return k2t_warp_bytes(P, sizeof(double), 32 / group_of(p)) <= p->model->max_smem;
}
long long bik_k2_group_wave(const bik_problem* p) {
  if (!bik_k2_group_applies(p)) return 0;
  PView P{p->image.data()};
  const int NS = 32 / group_of(p);
  const size_t wb = (size_t)k2t_warp_bytes(P, sizeof(double), NS);
  const int NW = k2t_warps(p, wb);
  int per_sm = (int)((size_t)p->model->max_smem / (NW * wb + 1024));   // estimate; only used to size chunks
  if (per_sm < 1) per_sm = 1;
  return (long long)p->model->nsm * per_sm * NW * NS;
}
template <typename A>
static int launch_k2t_group(const bik_problem* p, const A& a, unsigned int* sched, cudaStream_t st) {
  if (p->h.nu > K2T_NMAX) return launch_k2t<8, uint64_t>(p, a, sched, st);   // wide: 64-bit active-set masks
  return group_of(p) == 8 ? launch_k2t<8, uint32_t>(p, a, sched, st) : launch_k2t<4, uint32_t>(p, a, sched, st);
}
int bik_launch_k2_group(const bik_problem* p, const K2Args& a, unsigned int* sched, cudaStream_t st) { return launch_k2t_group(p, a, sched, st); }
int bik_launch_k2_group(const bik_problem* p, const K2PwArgs& a, unsigned int* sched, cudaStream_t st) { return launch_k2t_group(p, a, sched, st); }
int bik_launch_k2_group(const bik_problem* p, const K2BdArgs& a, unsigned int* sched, cudaStream_t st) { return launch_k2t_group(p, a, sched, st); }
const char* bik_k2_describe(const bik_problem* p, char* buf, size_t cap) {
  if (bik_k2_group_applies(p)) snprintf(buf, cap, "small-group G=%d%s", group_of(p), p->h.nu > K2T_NMAX ? " (64-bit masks)" : "");
  else {
    int lanes, slots;
    bik_k2_general_shape(p, &lanes, &slots);
    if (lanes < 32) snprintf(buf, cap, "general %d-lanes-per-problem", lanes);
    else if (slots == 1) snprintf(buf, cap, "general warp-per-problem");
    else snprintf(buf, cap, "general warp-per-problem, %d slots per lane", slots);
  }
  return buf;
}
