// bik_k2.cu -- general K2 path: one warp per problem (collision rows, or more than 64 coupled dofs); bik_k2.h.
#include "bik_dev.cuh"

using namespace bik;

// W lanes per problem (32 / W problems per warp): 8 or 16 when the augmented factor (coupled dofs + right-hand side) has at most
// that many rows -- a 6-dof arm with collision rows leaves 26 of 32 lanes idle with a warp per problem.
template <int W, int SLOTS, bool PW, bool BD = false>
__device__ __forceinline__ void k2_problems(const uint32_t* __restrict__ gimage, int words, int use_tma, const K2Args& a) {
  extern __shared__ __align__(16) uint32_t smem[];
  __shared__ __align__(8) uint64_t bar;
  if (a.gate && *a.gate == 0) return;
  stage_image(smem, gimage, words, &bar, use_tma);
  PView P{smem};
  constexpr int PPW = 32 / W;
  const int warp = threadIdx.x >> 5, lane32 = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  const int grp = lane32 / W, lane = lane32 % W;
  char* wsm = reinterpret_cast<char*>(smem + words) + (size_t)(warp * PPW + grp) * k2_warp_bytes(P.h(), sizeof(double));
  for (long long b = (long long)(blockIdx.x * nwarps + warp) * PPW + grp; b < a.B; b += (long long)gridDim.x * nwarps * PPW)
    k2_warp<double, W, SLOTS, PW, BD>(P, a, (int)b, wsm, lane);
}
template <int W, int SLOTS>
__global__ void __launch_bounds__(256) k2_kernel(const uint32_t* __restrict__ gimage, int words, int use_tma, K2Args a) {
  k2_problems<W, SLOTS, false>(gimage, words, use_tma, a);
}
// The same with per-instance posture weights (K2PwArgs): the ..._weighted_ex entry points with a posture-weights buffer.
template <int W, int SLOTS>
__global__ void __launch_bounds__(256) k2_pw_kernel(const uint32_t* __restrict__ gimage, int words, int use_tma, K2PwArgs a) {
  k2_problems<W, SLOTS, true>(gimage, words, use_tma, a);
}
// The same with per-instance bounds and posture weights, which may be null (K2BdArgs): the ..._bounded entry points with bounds.
template <int W, int SLOTS>
__global__ void __launch_bounds__(256) k2_bd_kernel(const uint32_t* __restrict__ gimage, int words, int use_tma, K2BdArgs a) {
  k2_problems<W, SLOTS, true, true>(gimage, words, use_tma, a);
}

// A: K2Args (k2_kernel), K2PwArgs (k2_pw_kernel) or K2BdArgs (k2_bd_kernel)
template <int W, int SLOTS, typename A>
static int launch_k2(const bik_problem* p, const A& a, cudaStream_t st) {
  constexpr bool PW = std::is_same<A, K2PwArgs>::value, BD = std::is_same<A, K2BdArgs>::value;
  const PHeader& h = p->h;
  constexpr int PPW = 32 / W;
  int NW = p->k2_warps;
  auto need = [&](int nw) { return (size_t)h.words32 * 4 + (size_t)nw * PPW * k2_warp_bytes(h, sizeof(double)); };
  while (NW > 1 && (int)need(NW) > p->model->max_smem) NW >>= 1;
  size_t smem = need(NW);
  int grid = 1;
  const long long per_cta = (long long)NW * PPW;
  const void* kern = BD ? (const void*)k2_bd_kernel<W, SLOTS> : PW ? (const void*)k2_pw_kernel<W, SLOTS> : (const void*)k2_kernel<W, SLOTS>;
  int rc = bik_launch_geometry(kern, p->model, smem, 32 * NW, ((long long)a.B + per_cta - 1) / per_cta, &grid);
  if (rc) return rc;
  if constexpr (BD) k2_bd_kernel<W, SLOTS><<<grid, 32 * NW, smem, st>>>(p->d_image, h.words32, p->model->use_tma, a);
  else if constexpr (PW) k2_pw_kernel<W, SLOTS><<<grid, 32 * NW, smem, st>>>(p->d_image, h.words32, p->model->use_tma, a);
  else k2_kernel<W, SLOTS><<<grid, 32 * NW, smem, st>>>(p->d_image, h.words32, p->model->use_tma, a);
  CUDA_OK(cudaGetLastError());
  return BIK_OK;
}
void bik_k2_general_shape(const bik_problem* p, int* lanes, int* slots) {
  const int rows = p->h.nu + 1;           // rows of the augmented factor (coupled dofs + rhs): lanes x SLOTS must cover them
  *lanes = rows <= 8 ? 8 : (rows <= 16 ? 16 : 32);
  *slots = (rows + *lanes - 1) / *lanes;
}
template <typename A>
static int launch_k2_shape(const bik_problem* p, const A& a, cudaStream_t st) {
  int lanes, slots;
  bik_k2_general_shape(p, &lanes, &slots);
  if (lanes == 8) return launch_k2<8, 1>(p, a, st);
  if (lanes == 16) return launch_k2<16, 1>(p, a, st);
  if (slots <= 1) return launch_k2<32, 1>(p, a, st);
  if (slots == 2) return launch_k2<32, 2>(p, a, st);
  return launch_k2<32, 3>(p, a, st);
}
int bik_launch_k2_general(const bik_problem* p, const K2Args& a, cudaStream_t st) { return launch_k2_shape(p, a, st); }
int bik_launch_k2_general(const bik_problem* p, const K2PwArgs& a, cudaStream_t st) { return launch_k2_shape(p, a, st); }
int bik_launch_k2_general(const bik_problem* p, const K2BdArgs& a, cudaStream_t st) { return launch_k2_shape(p, a, st); }
