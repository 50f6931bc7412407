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
  bik::PHeader h;               // the image's header
};

// One device allocation: move-only, freed with its owner (whose destroy function selects the device).
struct DevBuf {
  void* ptr = nullptr;
  size_t bytes = 0;
  DevBuf() = default;
  DevBuf(DevBuf&& o) noexcept : ptr(o.ptr), bytes(o.bytes) { o.ptr = nullptr; o.bytes = 0; }
  ~DevBuf() { cudaFree(ptr); }
  // Grow-only, contents not kept.  A larger request moves the allocation: work enqueued earlier on some stream may still
  // use the old one, so the device is idle first, and *moves is counted up before the old one is freed.
  cudaError_t reserve(size_t n, unsigned* moves) {
    if (n <= bytes) return cudaSuccess;
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) return e;
    ++*moves;
    cudaFree(ptr);
    ptr = nullptr; bytes = 0;
    e = cudaMalloc(&ptr, n);
    if (e == cudaSuccess) bytes = n;
    return e;
  }
  template <typename T> T* as() const { return static_cast<T*>(ptr); }
};

// K1 -> K2 hand-off (bik_loop.h: handoff_sizes), 4- or 8-byte elements by K1's precision.  It belongs to the problem, not to
// a stream, as the tile counters do: a call on another stream than the previous one first waits for that call's kernels
// (event recorded at the end of every call that uses them).
struct Handoff {
  DevBuf pk, Gc, hc;
  DevBuf warm;                 // [B][nu] active-set guess carried between the steps of one bik_step call
  cudaEvent_t event = nullptr;
  cudaStream_t stream = nullptr;
  int pending = 0;
  int reserve(const bik::PHeader& h, size_t B, int elem, unsigned* moves);
  ~Handoff() { if (event) cudaEventDestroy(event); }
};

// The cached CUDA graph of bik_converge / bik_track and the call it was built for.  The key is compared as bytes: it is
// zero-filled before its members are assigned.
struct ConvKey {
  bik::ConvCall c;             // `in` cleared: the struct it points to is the caller's, its contents are in `in`
  bik_inputs in;               // q cleared (the loop takes q from the call)
  unsigned moves;              // bik_problem::moves when the graph captured the hand-off and loop-state addresses
};
struct ConvGraph {
  ConvKey key;
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t exec = nullptr;
  cudaStream_t cap = nullptr;
  void drop() {
    if (exec) cudaGraphExecDestroy(exec);
    if (graph) cudaGraphDestroy(graph);
    if (cap) cudaStreamDestroy(cap);
    exec = nullptr; graph = nullptr; cap = nullptr;
  }
};

// bik_converge / bik_track loop state (bik_loop.h: ConvBufs)
struct LoopState {
  DevBuf done;                 // [B]
  DevBuf dq;                   // [B][nv] K2's dq of the previous pass (its warm start), 4- or 8-byte elements by the caller's precision
  DevBuf cursor, step, status; // [B] each: bik_track's frame cursor, steps taken in that frame, status of the frame in progress
  DevBuf count;                // device: { steps taken so far, unconverged instances, go }
  DevBuf ptcur;                // [B][P][nq] bik_track's posture targets of each instance's current frame (bik_loop.h: uses_ptcur)
  DevBuf held;                 // [B][7F + 3C] bik_track_hold's held frame and CoM targets (calls with a hold mask only)
  int* host = nullptr;         // pinned mirror of count
  ConvGraph graph;
  // elem: bytes of the caller's elements; ptcur: the call keeps posture targets in ptcur; hold: the call has a hold mask
  int reserve(const bik::PHeader& h, size_t B, int elem, bool ptcur, bool hold, unsigned* moves);
  ~LoopState() { graph.drop(); if (host) cudaFreeHost(host); }
};

// bik_step_host staging (fp32)
struct HostStaging {
  DevBuf q, ft, pt, ct, dq, st;
  cudaStream_t hs[4] = {nullptr, nullptr, nullptr, nullptr};   // upload, compute A, compute B, download
  std::vector<cudaEvent_t> hev;
  int reserve(const bik::PHeader& h, size_t B, size_t pt_elems);
  ~HostStaging() {
    for (cudaStream_t s : hs) if (s) cudaStreamDestroy(s);
    for (cudaEvent_t e : hev) cudaEventDestroy(e);
  }
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
  std::mutex mu;          // one caller at a time per problem
  Handoff hand;
  LoopState loop;
  unsigned moves = 0;     // times a buffer of `hand` or `loop` has moved: a graph built before the last move is stale
  HostStaging stage;
  unsigned int* d_sched = nullptr;      // BIK_SCHED_SLOTS x 32 words: {next tile, finished CTAs} per launching stream (own 128-byte line each)
  cudaStream_t sched_stream[BIK_SCHED_SLOTS];
  int n_sched = 0;
};

// resident CTAs per SM for (kernel, dynamic smem, threads): attribute + occupancy queries run once per combination
int bik_launch_geometry(const void* kern, const bik_model* m, size_t smem, int threads, long long work_ctas, int* grid);

// launchers (each returns BIK_OK or records an error)
int bik_launch_k1(const bik_problem* p, const bik::K1Args& a, bool use_double, cudaStream_t st);
int bik_launch_k1(const bik_problem* p, const bik::K1CArgs& a, bool use_double, cudaStream_t st);   // per-instance collision pairs (k1c_kernel)
int bik_launch_k1(const bik_problem* p, const bik::K1HArgs& a, bool use_double, cudaStream_t st);   // held targets (k1h_kernel)
int bik_launch_k1(const bik_problem* p, const bik::K1PArgs& a, bool use_double, cudaStream_t st);   // frame placement (k1p_kernel)
int bik_launch_fk(const bik_model* m, const bik::FkArgs& a, cudaStream_t st);
int bik_launch_k2_general(const bik_problem* p, const bik::K2Args& a, cudaStream_t st);
int bik_launch_k2_general(const bik_problem* p, const bik::K2PwArgs& a, cudaStream_t st);   // posture-weighted instantiations
int bik_launch_k2_general(const bik_problem* p, const bik::K2BdArgs& a, cudaStream_t st);   // bounded instantiations
void bik_k2_general_shape(const bik_problem* p, int* lanes, int* slots);   // the (W, SLOTS) bik_launch_k2_general picks
int bik_launch_k2_group(const bik_problem* p, const bik::K2Args& a, unsigned int* sched, cudaStream_t st);
int bik_launch_k2_group(const bik_problem* p, const bik::K2PwArgs& a, unsigned int* sched, cudaStream_t st);   // posture-weighted
int bik_launch_k2_group(const bik_problem* p, const bik::K2BdArgs& a, unsigned int* sched, cudaStream_t st);   // bounded
bool bik_k2_group_applies(const bik_problem* p);                  // box-only, at most 64 coupled dofs, fits in shared memory
long long bik_k2_group_wave(const bik_problem* p);                // instances one resident wave of the small-group K2 covers
const char* bik_k2_describe(const bik_problem* p, char* buf, size_t cap);
