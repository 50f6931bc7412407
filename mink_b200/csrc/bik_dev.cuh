// bik_dev.cuh -- what the translation units of libbik share: PTX helpers (mbarrier + 1-D bulk async copy), the handle
// structs behind the C ABI and the launcher entry points each .cu exports to bik_api.cu.
//
//   bik_k1.cu   k1_kernel<T,G> (FK + task rows + collision rows + check_limits), fk_kernel<T,G> (Configuration API)
//   bik_k2.cu   k2_kernel<W,SLOTS>  (general QP path, fp64: W = 8 / 16 / 32 lanes per problem)
//   bik_k2t.cu  k2t_kernel<double,G,256,M,..>  (small-group QP path, fp64: G lanes per problem, 32- or 64-bit active-set masks)
//   bik_api.cu  C ABI (include/bik.h), workspace, bik_step / bik_converge / bik_step_host, small tiled kernels
//
// There is no CPU fallback in this library: without a CUDA device every entry point fails.
#pragma once
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>

#include <mutex>
#include <string>
#include <vector>

#include "bik_build.h"
#include "bik_ptx.cuh"
#include "bik_k2t.h"
#include "bik_loop.h"

namespace bik {

// Stage the first `words` words of the problem image into shared memory: one elected thread issues a single bulk copy and
// everybody waits on the mbarrier (bounded spin; traps instead of hanging the GPU).
__device__ __forceinline__ void stage_image(uint32_t* smem_image, const uint32_t* gimage, int words, uint64_t* bar, int use_tma) {
  if (use_tma) {
    if (threadIdx.x == 0) {
      mbar_init(bar, 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      mbar_expect_tx(bar, (uint32_t)words * 4u);
      bulk_g2s(smem_image, gimage, (uint32_t)words * 4u, bar);
    }
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, 0)) {
      if (++spins > (1u << 24)) __trap();
    }
  } else {
    const uint4* src = reinterpret_cast<const uint4*>(gimage);
    uint4* dst = reinterpret_cast<uint4*>(smem_image);
    for (int k = threadIdx.x; k < words / 4; k += blockDim.x) dst[k] = src[k];
    __syncthreads();
  }
}

}  // namespace bik

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
int bik_fail(int code, const std::string& msg);   // records the message for bik_last_error(), returns code
#define CUDA_OK(expr)                                                                                       \
  do {                                                                                                      \
    cudaError_t _e = (expr);                                                                                \
    if (_e != cudaSuccess) return bik_fail(BIK_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e)); \
  } while (0)

struct bik_model {
  int device = 0, nsm = 0, max_smem = 0;
  int G = 4, use_tma = 1;
  bik::HostModel hm;
  std::vector<uint32_t> image;  // model-only image (no tasks)
  uint32_t* d_image = nullptr;
};

enum { BIK_SCHED_SLOTS = 8 };
struct bik_problem {
  const bik_model* model = nullptr;
  int device = 0;  // copy: the model may be destroyed first
  std::vector<uint32_t> image;
  uint32_t* d_image = nullptr;
  bik::PHeader h;
  int k2_general = 0;     // BIK_K2_PATH=dense: every problem takes the general warp-per-problem path
  int k2_group = 8;       // lanes per problem on the small-group path (BIK_K2_GROUP = 4 | 8)
  int k2_warps = 8;       // warps per CTA of the general K2 kernel (BIK_K2_WARPS)
  int k2_dynamic = 1;     // BIK_K2_DYNAMIC=0: static tile assignment in the small-group K2
  int k1_prec = 0;        // BIK_K1_PRECISION: 0 auto (by conditioning estimate), 1 f32, 2 f64
  bik::K1Conditioning k1cond;   // what the automatic choice of K1's precision rests on
  // K1 -> K2 hand-off (one caller at a time per problem)
  std::mutex mu;
  size_t ws_B = 0;
  int ws_elem = 0;        // element size the hand-off buffers were sized for (4 or 8)
  void *pk = nullptr, *Gc = nullptr, *hc = nullptr;
  signed char* warm = nullptr;          // [B][nu] active-set guess carried between the steps of one bik_step call
  // the hand-off buffers, tile counters and the warm start belong to the problem, not to a stream: a call on another stream
  // than the previous one first waits for that call's kernels (event recorded at the end of every call that uses them)
  cudaEvent_t ws_event = nullptr;
  cudaStream_t ws_stream = nullptr;
  int ws_pending = 0;
  unsigned int* d_sched = nullptr;      // BIK_SCHED_SLOTS x 32 words: {next tile, finished CTAs} per launching stream (own 128-byte line each)
  cudaStream_t sched_stream[BIK_SCHED_SLOTS];
  int n_sched = 0;
  // bik_step_host staging
  size_t host_B = 0;
  float *hq = nullptr, *hft = nullptr, *hpt = nullptr, *hct = nullptr, *hdq = nullptr;
  int32_t* hst = nullptr;
  size_t host_pt_elems = 0;
  cudaStream_t hs[4] = {nullptr, nullptr, nullptr, nullptr};   // upload, compute A, compute B, download
  std::vector<cudaEvent_t> hev;
  // bik_converge state
  size_t conv_B = 0;
  int conv_elem = 0;           // bytes per conv_dq element: 4, or 8 once an fp64 call (bik_converge64 / bik_track64) needed it
  int32_t* conv_done = nullptr;
  void* conv_dq = nullptr;     // [conv_B][nv] K2's dq of the previous pass (its warm start)
  int* conv_count = nullptr;   // device: { steps taken so far, unconverged instances }
  int* conv_host = nullptr;    // pinned mirror
  // bik_track state (the same loop, per-instance frame cursor)
  int32_t* conv_cursor = nullptr;   // [B] frame each instance is on
  int32_t* conv_step = nullptr;     // [B] steps taken in that frame, -1 = no frames left
  int32_t* conv_status = nullptr;   // [B] status of the frame in progress
};

// resident CTAs per SM for (kernel, dynamic smem, threads): attribute + occupancy queries run once per combination
int bik_launch_geometry(const void* kern, const bik_model* m, size_t smem, int threads, long long work_ctas, int* grid);

// launchers (each returns BIK_OK or records an error)
int bik_launch_k1(const bik_problem* p, const bik::K1Args& a, bool use_double, cudaStream_t st);
int bik_launch_fk(const bik_model* m, const bik::FkArgs& a, cudaStream_t st);
int bik_launch_k2_general(const bik_problem* p, const bik::K2Args& a, cudaStream_t st);
int bik_launch_k2_group(const bik_problem* p, const bik::K2Args& a, unsigned int* sched, cudaStream_t st);
bool bik_k2_group_applies(const bik_problem* p);                  // box-only, at most 64 coupled dofs, fits in shared memory
long long bik_k2_group_wave(const bik_problem* p);                // instances one resident wave of the small-group K2 covers
const char* bik_k2_describe(const bik_problem* p, char* buf, size_t cap);
