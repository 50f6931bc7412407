// bik_api.cu -- the C ABI of libbik (include/bik.h): handles, workspace, bik_step / bik_converge / bik_step_host, and the
// small tiled kernels (stand-alone integrate / check_limits).  The hot kernels live in bik_k1.cu / bik_k2.cu / bik_k2t.cu.
//
// There is no CPU fallback in this library: without a CUDA device every entry point fails.
#include "bik_dev.cuh"

using namespace bik;

// ------------------------------------------------------------------------------------------------
// small kernels
// ------------------------------------------------------------------------------------------------
// A CTA of 128 threads moves the q (and dq) rows of its 64 instances through a shared-memory tile with odd row stride
// (flat, contiguous global traffic), then one thread per instance integrates / checks its row in the tile.
enum { TILE_INST = 64, TILE_THREADS = 128 };
template <typename T>
__device__ __forceinline__ void tile_rows_in(T* tile, int S, const T* __restrict__ g, int n, int len) {
  const int total = n * len;
#pragma unroll 4
  for (int k = threadIdx.x; k < total; k += TILE_THREADS) { int i = k / len; tile[i * S + (k - i * len)] = g[k]; }
}
template <typename T>
__global__ void __launch_bounds__(TILE_THREADS) integrate_tiled_kernel(const uint32_t* __restrict__ gimage, int B, T* q, const T* __restrict__ dq) {
  extern __shared__ __align__(16) unsigned char tile_raw[];
  T* tile = reinterpret_cast<T*>(tile_raw);
  PView P{gimage};
  const int nq = P.h().nq, nv = P.h().nv, Sq = nq | 1, Sd = nv | 1;
  const long long b0 = (long long)blockIdx.x * TILE_INST;
  const int n = (B - b0) < TILE_INST ? (int)(B - b0) : TILE_INST;
  T* tq = tile; T* td = tile + TILE_INST * Sq;
  tile_rows_in<T>(tq, Sq, q + b0 * nq, n, nq);
  tile_rows_in<T>(td, Sd, dq + b0 * nv, n, nv);
  __syncthreads();
  if ((int)threadIdx.x < n) integrate_instance<T>(P, tq + threadIdx.x * Sq, td + threadIdx.x * Sd);
  __syncthreads();
  T* gq = q + b0 * nq;
  const int total = n * nq;
#pragma unroll 4
  for (int k = threadIdx.x; k < total; k += TILE_THREADS) { int i = k / nq; gq[k] = tq[i * Sq + (k - i * nq)]; }
}
template <typename T>
__global__ void __launch_bounds__(TILE_THREADS) check_limits_tiled_kernel(const uint32_t* __restrict__ gimage, int B, const T* __restrict__ q, float tol, int32_t* status) {
  extern __shared__ __align__(16) unsigned char tile_raw[];
  T* tile = reinterpret_cast<T*>(tile_raw);
  PView P{gimage};
  const int nq = P.h().nq, Sq = nq | 1;
  const long long b0 = (long long)blockIdx.x * TILE_INST;
  const int n = (B - b0) < TILE_INST ? (int)(B - b0) : TILE_INST;
  tile_rows_in<T>(tile, Sq, q + b0 * nq, n, nq);
  __syncthreads();
  if ((int)threadIdx.x < n) status[b0 + threadIdx.x] = check_limits_instance<T>(P, tile + threadIdx.x * Sq, tol);
}
template <typename T>
__global__ void integrate_kernel(const uint32_t* __restrict__ gimage, int B, T* q, const T* dq) {
  PView P{gimage};
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B) integrate_instance<T>(P, q + (size_t)b * P.h().nq, dq + (size_t)b * P.h().nv);
}
template <typename T>
__global__ void check_limits_kernel(const uint32_t* __restrict__ gimage, int B, const T* q, float tol, int32_t* status) {
  PView P{gimage};
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B) status[b] = check_limits_instance<T>(P, q + (size_t)b * P.h().nq, tol);
}
// bik_converge / bik_track bookkeeping (bik_loop.h): the per-instance reset before the loop, the one-thread tick and
// condition around K1 of every pass (the condition also sets the WHILE node's), and the per-instance finish of converge.
__global__ void conv_reset_kernel(int B, bool track, int T, const int32_t* __restrict__ lengths, ConvBufs s) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B) conv_reset(track, T, lengths, s, b);
}
__global__ void conv_tick_kernel(bool track, int* count) { conv_tick(track, count); }
__global__ void conv_cond_kernel(bool track, int max_iters, int* count, cudaGraphConditionalHandle handle, int use_handle) {
  const int go = conv_cond(track, max_iters, count);
  if (use_handle) cudaGraphSetConditional(handle, go ? 1u : 0u);
}
__global__ void conv_finish_kernel(int B, int max_iters, const int32_t* __restrict__ done, int32_t* iters, int32_t* status) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B) conv_finish(max_iters, done, iters, status, b);
}

// CUDA-core FMA peak, measured: 16 independent dependent-chains of fused multiply-adds per thread, enough CTAs to fill every SM.
// This is the denominator of K2's roofline (bench.py): the QP solve runs on the FMA pipes, not on tensor cores.
template <typename T>
__global__ void __launch_bounds__(256) fma_peak_kernel(int iters, T seed, T* sink) {
  T a[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) a[k] = seed + T(k + threadIdx.x) * T(1e-3);
  const T m = T(0.999), c = T(1e-3);
  for (int i = 0; i < iters; ++i) {
#pragma unroll
    for (int k = 0; k < 16; ++k) a[k] = a[k] * m + c;
  }
  T s = T(0);
#pragma unroll
  for (int k = 0; k < 16; ++k) s += a[k];
  if (s == T(-1)) sink[0] = s;   // never true: keeps the chains alive
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static thread_local std::string g_err;
int bik_fail(int code, const std::string& msg) { g_err = msg; return code; }

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    cudaGetDevice(&prev);
    if (prev != dev) cudaSetDevice(dev); else prev = -1;
    (void)cudaGetLastError();  // drop stale errors of earlier, unrelated calls on this thread
  }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

static int env_int(const char* name, int dflt) { const char* v = getenv(name); return v ? atoi(v) : dflt; }

// (kernel, smem, threads) -> resident CTAs per SM; the attribute/occupancy queries run once per combination.
struct GeomKey { const void* kern; size_t smem; int threads; int device; };
static std::mutex g_geom_mu;
static std::vector<std::pair<GeomKey, int>> g_geom;

int bik_launch_geometry(const void* kern, const bik_model* m, size_t smem, int threads, long long work_ctas, int* grid) {
  if ((int)smem > m->max_smem) return bik_fail(BIK_ERR_UNSUPPORTED, "problem does not fit in shared memory (" + std::to_string(smem) + " B)");
  int per_sm = 0;
  {
    std::lock_guard<std::mutex> lock(g_geom_mu);
    for (auto& e : g_geom)
      if (e.first.kern == kern && e.first.smem == smem && e.first.threads == threads && e.first.device == m->device) per_sm = e.second;
  }
  if (per_sm == 0) {
    // the opt-in limit is per kernel and must never shrink below what an earlier, cached combination needs
    size_t prev_max = 0;
    {
      std::lock_guard<std::mutex> lock(g_geom_mu);
      for (auto& e : g_geom) if (e.first.kern == kern && e.first.device == m->device && e.first.smem > prev_max) prev_max = e.first.smem;
    }
    if (smem > prev_max) CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, threads, smem));
    if (per_sm < 1) return bik_fail(BIK_ERR_UNSUPPORTED, "kernel cannot be resident");
    std::lock_guard<std::mutex> lock(g_geom_mu);
    g_geom.push_back({GeomKey{kern, smem, threads, m->device}, per_sm});
  }
  long long g = (long long)m->nsm * per_sm;  // persistent: one wave, CTAs loop over tiles
  if (work_ctas < g) g = work_ctas;
  *grid = (int)(g < 1 ? 1 : g);
  return BIK_OK;
}

// bik_integrate[64] / bik_check_limits[64]: tiled (coalesced) when the tile fits the default 48 KB of dynamic shared memory
template <typename T>
static int integrate_common(const bik_model* m, int B, T* q, const T* dq, void* stream) {
  if (!m || !q || !dq || B < 0) return bik_fail(BIK_ERR_INVALID, "null argument");
  if (B == 0) return BIK_OK;
  DeviceGuard g(m->device);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t smem = (size_t)TILE_INST * ((m->h.nq | 1) + (m->h.nv | 1)) * sizeof(T);
  if (smem <= 48 * 1024) integrate_tiled_kernel<T><<<(B + TILE_INST - 1) / TILE_INST, TILE_THREADS, smem, st>>>(m->d_image, B, q, dq);
  else integrate_kernel<T><<<(B + 127) / 128, 128, 0, st>>>(m->d_image, B, q, dq);
  CUDA_OK(cudaGetLastError());
  return BIK_OK;
}
template <typename T>
static int check_limits_common(const bik_model* m, int B, const T* q, float tol, int32_t* status, void* stream) {
  if (!m || !q || !status || B < 0) return bik_fail(BIK_ERR_INVALID, "null argument");
  if (B == 0) return BIK_OK;
  DeviceGuard g(m->device);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t smem = (size_t)TILE_INST * (m->h.nq | 1) * sizeof(T);
  if (smem <= 48 * 1024) check_limits_tiled_kernel<T><<<(B + TILE_INST - 1) / TILE_INST, TILE_THREADS, smem, st>>>(m->d_image, B, q, tol, status);
  else check_limits_kernel<T><<<(B + 127) / 128, 128, 0, st>>>(m->d_image, B, q, tol, status);
  CUDA_OK(cudaGetLastError());
  return BIK_OK;
}

static int valid_group(int G) { return G == 1 || G == 2 || G == 4 || G == 8 || G == 16 || G == 32; }

extern "C" int bik_version(void) { return BIK_VERSION; }
extern "C" const char* bik_last_error(void) { return g_err.c_str(); }

extern "C" int bik_model_create(const void* blob, size_t nbytes, int device, bik_model** out) {
  if (!blob || !out) return bik_fail(BIK_ERR_INVALID, "null argument");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return bik_fail(BIK_ERR_CUDA, "no CUDA device: libbik has no CPU path");
  if (device < 0 || device >= ndev) return bik_fail(BIK_ERR_INVALID, "bad device index");
  bik_model* m = new bik_model;
  std::string err;
  if (!parse_model_blob(blob, nbytes, &m->hm, &err)) { delete m; return bik_fail(BIK_ERR_INVALID, err); }
  m->device = device;
  m->G = env_int("BIK_K1_GROUP", 0);  // 0: chosen per problem from the visited tree (bik_build.h)
  if (m->G != 0 && !valid_group(m->G)) { delete m; return bik_fail(BIK_ERR_INVALID, "BIK_K1_GROUP must be 1,2,4,8,16 or 32"); }
  m->use_tma = env_int("BIK_USE_TMA", 1);
  if (!build_image(m->hm, nullptr, 0, nullptr, 0, m->G, &m->image, &err)) { delete m; return bik_fail(BIK_ERR_UNSUPPORTED, err); }
  memcpy(&m->h, m->image.data(), sizeof(PHeader));
  DeviceGuard g(device);
  cudaDeviceProp prop;
  CUDA_OK(cudaGetDeviceProperties(&prop, device));
  m->nsm = prop.multiProcessorCount;
  m->max_smem = (int)prop.sharedMemPerBlockOptin;
  CUDA_OK(cudaMalloc(&m->d_image, m->image.size() * 4));
  CUDA_OK(cudaMemcpy(m->d_image, m->image.data(), m->image.size() * 4, cudaMemcpyHostToDevice));
  *out = m;
  return BIK_OK;
}
extern "C" void bik_model_destroy(bik_model* m) {
  if (!m) return;
  DeviceGuard g(m->device);
  cudaFree(m->d_image);
  delete m;
}

extern "C" int bik_problem_create(const bik_model* model, const bik_task_desc* tasks, int ntasks, const bik_limit_desc* limits, int nlimits,
                                  bik_problem** out) {
  if (!model || !out || ntasks < 0 || nlimits < 0 || (ntasks && !tasks) || (nlimits && !limits)) return bik_fail(BIK_ERR_INVALID, "null argument");
  bik_problem* p = new bik_problem;
  p->model = model;
  p->device = model->device;
  std::string err;
  if (!build_image(model->hm, tasks, ntasks, limits, nlimits, model->G, &p->image, &err)) { delete p; return bik_fail(BIK_ERR_UNSUPPORTED, err); }
  {  // launch-independent solver knob kept in the image header so that every K2 entry point sees it
    PHeader* hh = reinterpret_cast<PHeader*>(p->image.data());
    hh->k2_sweeps = std::max(1, std::min(16, env_int("BIK_K2_SWEEPS", hh->k2_sweeps)));
  }
  memcpy(&p->h, p->image.data(), sizeof(PHeader));
  const char* path = getenv("BIK_K2_PATH");
  p->k2_general = path && (std::string(path) == "dense" || std::string(path) == "general");
  p->k2_group = env_int("BIK_K2_GROUP", p->h.nu > 8 ? 8 : 4) == 8 ? 8 : 4;
  p->k2_warps = env_int("BIK_K2_WARPS", 8);
  p->k2_dynamic = env_int("BIK_K2_DYNAMIC", 1) != 0;
  if (p->k2_warps != 1 && p->k2_warps != 2 && p->k2_warps != 4 && p->k2_warps != 8) p->k2_warps = 8;
  const char* k1p = getenv("BIK_K1_PRECISION");
  p->k1_prec = k1p ? (std::string(k1p) == "f64" ? 2 : (std::string(k1p) == "f32" ? 1 : 0)) : 0;
  p->k1cond = k1_conditioning(model->hm, p->image, tasks, ntasks);
  DeviceGuard g(model->device);
  CUDA_OK(cudaMalloc(&p->d_image, p->image.size() * 4));
  CUDA_OK(cudaMemcpy(p->d_image, p->image.data(), p->image.size() * 4, cudaMemcpyHostToDevice));
  *out = p;
  return BIK_OK;
}
extern "C" void bik_problem_destroy(bik_problem* p) {
  if (!p) return;
  DeviceGuard g(p->device);
  cudaFree(p->d_sched); cudaFree(p->d_image);
  delete p;   // the buffer groups free themselves
}
extern "C" int bik_problem_dims(const bik_problem* p, bik_dims* out) {
  if (!p || !out) return bik_fail(BIK_ERR_INVALID, "null argument");
  out->nq = p->h.nq; out->nv = p->h.nv; out->nnode = p->h.nnode; out->nframe = p->h.F; out->nposture = p->h.P; out->ncom = p->h.C;
  out->nrows = p->h.K; out->npairs = p->h.npairs;
  return BIK_OK;
}
// hand-off element size: 8 when K1 runs in fp64 for this (problem, damping, caller precision, posture weights or not)
static bool k1_double(const bik_problem* p, double damping, bool io64, bool posture_weighted = false) {
  if (io64 || p->k1_prec == 2) return true;
  if (p->k1_prec == 1) return false;
  return k1_auto_double(p->h, p->k1cond, damping, posture_weighted);
}
extern "C" size_t bik_workspace_bytes(const bik_problem* p, int B) {
  if (!p || B <= 0) return 0;
  const PHeader& h = p->h;
  return (size_t)B * 8 * ((size_t)h.pk_stride + (size_t)h.npairs * (h.nv + 1)) + (size_t)B * (h.nu + 4);
}

// One (next tile, finished CTAs) pair per stream that launches the small-group K2 of this problem: launches on one stream
// are ordered, launches on different streams must not share a counter.  More than BIK_SCHED_SLOTS streams, or
// BIK_K2_DYNAMIC=0: static round-robin.  Caller holds p->mu.
static unsigned int* tile_counter(bik_problem* p, cudaStream_t st) {
  if (!p->k2_dynamic) return nullptr;
  if (!p->d_sched) {
    if (cudaMalloc(&p->d_sched, BIK_SCHED_SLOTS * 32 * sizeof(unsigned int)) != cudaSuccess) { cudaGetLastError(); p->k2_dynamic = 0; return nullptr; }
    cudaMemset(p->d_sched, 0, BIK_SCHED_SLOTS * 32 * sizeof(unsigned int));
  }
  for (int i = 0; i < p->n_sched; ++i) if (p->sched_stream[i] == st) return p->d_sched + 32 * i;
  if (p->n_sched == BIK_SCHED_SLOTS) return nullptr;
  p->sched_stream[p->n_sched] = st;
  return p->d_sched + 32 * p->n_sched++;
}
// K2 dispatch.  Caller holds p->mu when a.dq is set (the small-group path owns a per-stream tile counter).  A: K2Args, or
// K2PwArgs for the posture-weighted instantiations.
template <typename A>
static int dispatch_k2(bik_problem* p, const A& a, cudaStream_t st) {
  const bool solving = a.dq && !a.Hout && !a.lo_out;
  if (solving && bik_k2_group_applies(p)) return bik_launch_k2_group(p, a, tile_counter(p, st), st);
  return bik_launch_k2_general(p, a, st);
}

static int fk_common(const bik_model* model, int B, const void* q, const bik_frame* frames, int nframes, void* poses, void* com, void* J, int io64, void* stream) {
  if (!model || B < 0 || !q || nframes < 0 || (nframes && !frames)) return bik_fail(BIK_ERR_INVALID, "null argument");
  if (B == 0) return BIK_OK;
  DeviceGuard g(model->device);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // frames travel by value in the kernel arguments (the Configuration API asks for one or two)
  if (nframes > 16) return bik_fail(BIK_ERR_UNSUPPORTED, "at most 16 frames per bik_fk / bik_frame_jacobian call");
  FkArgs a;
  memset(&a, 0, sizeof a);
  a.B = B; a.nframes = nframes; a.q = q; a.poses = poses; a.com = com; a.J = J; a.io64 = io64;
  for (int f = 0; f < nframes; ++f) {
    if (frames[f].node >= model->hm.nnode) return bik_fail(BIK_ERR_INVALID, "frame node out of range");
    a.frames[f].node = frames[f].node;
    put_frame64(frames[f], a.frames[f].lpos, a.frames[f].lquat);
  }
  return bik_launch_fk(model, a, st);
}
extern "C" int bik_fk(const bik_model* model, int B, const float* q, const bik_frame* frames, int nframes, float* poses, float* com, void* stream) {
  return fk_common(model, B, q, frames, nframes, poses, com, nullptr, 0, stream);
}
extern "C" int bik_frame_jacobian(const bik_model* model, int B, const float* q, const bik_frame* frames, int nframes, float* J, void* stream) {
  return fk_common(model, B, q, frames, nframes, nullptr, nullptr, J, 0, stream);
}
extern "C" int bik_fk64(const bik_model* model, int B, const double* q, const bik_frame* frames, int nframes, double* poses, double* com, void* stream) {
  return fk_common(model, B, q, frames, nframes, poses, com, nullptr, 1, stream);
}
extern "C" int bik_frame_jacobian64(const bik_model* model, int B, const double* q, const bik_frame* frames, int nframes, double* J, void* stream) {
  return fk_common(model, B, q, frames, nframes, nullptr, nullptr, J, 1, stream);
}

// track: a bik_track entry point, the only ones that take a posture target sequence
// bounds: the ..._bounded entry points' bounds (as from bounds_of), or null; coll: the ..._coll entry points' collision
// arguments (as from coll_of), or null; placement: the ..._placed entry points' frame placements, or null
static int check_inputs(const bik_problem* p, const bik_inputs* in, bool need_q, int f64, bool track = false, const void* posture_weights = nullptr,
                        const bik_bounds* bounds = nullptr, const bik_collision* coll = nullptr, const void* placement = nullptr) {
  if (!p || !in) return bik_fail(BIK_ERR_INVALID, "null argument");
  const PHeader& h = p->h;
  if (coll && h.npairs == 0) return bik_fail(BIK_ERR_INVALID, "coll given for a problem without a CollisionAvoidanceLimit");
  if (placement && h.F == 0) return bik_fail(BIK_ERR_INVALID, "placement given for a problem without a FrameTask or RelativeFrameTask");
  if (posture_weights && h.P == 0) return bik_fail(BIK_ERR_INVALID, "posture_weights given for a problem without a PostureTask or DampingTask");
  if (bounds && (bounds->lower || bounds->upper) && h.ncfg == 0)
    return bik_fail(BIK_ERR_INVALID, "bounds.lower / bounds.upper given for a problem without a ConfigurationLimit");
  if (bounds && bounds->vmax && !h.has_vel) return bik_fail(BIK_ERR_INVALID, "bounds.vmax given for a problem without a VelocityLimit");
  if (!track && posture_seq(in))
    return bik_fail(BIK_ERR_INVALID, "posture_batched = " + std::to_string(in->posture_batched) +
                                         " (a posture target sequence) is accepted by bik_track, bik_track64 and bik_track_weighted[64] only");
  if ((in->f64 != 0) != (f64 != 0)) return bik_fail(BIK_ERR_INVALID, f64 ? "bik_inputs.f64 must be 1 for the fp64 entry points" : "bik_inputs.f64 must be 0 for the fp32 entry points");
  if (need_q && !in->q) return bik_fail(BIK_ERR_INVALID, "inputs.q is null");
  if (h.F > 0 && !in->frame_targets) return bik_fail(BIK_ERR_INVALID, "No target set for FrameTask");
  if (h.P > 0 && !in->posture_targets) return bik_fail(BIK_ERR_INVALID, "No target set for PostureTask");
  if (h.C > 0 && !in->com_targets) return bik_fail(BIK_ERR_INVALID, "No target set for ComTask");
  return BIK_OK;
}

static int fk_jac_common(const bik_problem* p, int B, const bik_inputs* in, double dt, void* J, void* e, void* e_posture, void* G_coll, void* h_coll, int f64, void* stream) {
  if (B == 0 && p) return BIK_OK;
  int rc = check_inputs(p, in, true, f64);
  if (rc) return rc;
  const PHeader& h = p->h;
  if (B < 0 || (h.K > 0 && (!J || !e)) || (h.P > 0 && !e_posture) || (h.npairs > 0 && (!G_coll || !h_coll))) return bik_fail(BIK_ERR_INVALID, "null output");
  DeviceGuard g(p->model->device);
  K1Args a;
  memset(&a, 0, sizeof a);
  a.B = B; a.q = in->q; a.ftgt = in->frame_targets; a.ptgt = in->posture_targets; a.ctgt = in->com_targets; a.in64 = f64; a.pbatched = in->posture_batched;
  a.dt = dt; a.J = J; a.e = e; a.ep = e_posture; a.Gc = G_coll; a.hc = h_coll;
  return bik_launch_k1(p, a, f64 != 0, static_cast<cudaStream_t>(stream));
}
extern "C" int bik_fk_jac(const bik_problem* p, int B, const bik_inputs* in, float dt, float* J, float* e, float* e_posture, float* G_coll,
                          float* h_coll, void* stream) {
  return fk_jac_common(p, B, in, dt, J, e, e_posture, G_coll, h_coll, 0, stream);
}
extern "C" int bik_fk_jac64(const bik_problem* p, int B, const bik_inputs* in, double dt, double* J, double* e, double* e_posture, double* G_coll,
                            double* h_coll, void* stream) {
  return fk_jac_common(p, B, in, dt, J, e, e_posture, G_coll, h_coll, 1, stream);
}

static int objective_common(const bik_problem* cp, int B, const void* J, const void* e, const void* e_posture, double damping, double* H, double* c, int f64, void* stream) {
  if (!cp || !H || !c || B < 0) return bik_fail(BIK_ERR_INVALID, "null argument");
  if (B == 0) return BIK_OK;
  bik_problem* p = const_cast<bik_problem*>(cp);
  DeviceGuard g(p->model->device);
  K2Args a;
  memset(&a, 0, sizeof a);
  a.B = B; a.J = J; a.e = e; a.ep = e_posture; a.dense64 = f64; a.dt = 1.0; a.damping = damping; a.Hout = H; a.cout = c;
  a.skip_box = 1;
  return dispatch_k2(p, a, static_cast<cudaStream_t>(stream));
}
extern "C" int bik_qp_objective(const bik_problem* p, int B, const float* J, const float* e, const float* e_posture, double damping, double* H,
                                double* c, void* stream) {
  return objective_common(p, B, J, e, e_posture, damping, H, c, 0, stream);
}
extern "C" int bik_qp_objective64(const bik_problem* p, int B, const double* J, const double* e, const double* e_posture, double damping, double* H,
                                  double* c, void* stream) {
  return objective_common(p, B, J, e, e_posture, damping, H, c, 1, stream);
}

static int box_common(const bik_problem* cp, int B, const void* q, double dt, void* lo, void* hi, int f64, void* stream) {
  if (!cp || !q || !lo || !hi || B < 0) return bik_fail(BIK_ERR_INVALID, "null argument");
  if (B == 0) return BIK_OK;
  bik_problem* p = const_cast<bik_problem*>(cp);
  DeviceGuard g(p->model->device);
  K2Args a;
  memset(&a, 0, sizeof a);
  a.B = B; a.q = q; a.io64 = f64; a.dt = dt; a.lo_out = lo; a.hi_out = hi; a.skip_objective = 1;
  return dispatch_k2(p, a, static_cast<cudaStream_t>(stream));
}
extern "C" int bik_limits_box(const bik_problem* p, int B, const float* q, float dt, float* lo, float* hi, void* stream) {
  return box_common(p, B, q, dt, lo, hi, 0, stream);
}
extern "C" int bik_limits_box64(const bik_problem* p, int B, const double* q, double dt, double* lo, double* hi, void* stream) {
  return box_common(p, B, q, dt, lo, hi, 1, stream);
}

// Cross-stream ordering of the per-problem hand-off (callers hold p->mu).
static int ws_acquire(bik_problem* p, cudaStream_t st) {
  if (p->hand.pending && p->hand.stream != st) CUDA_OK(cudaStreamWaitEvent(st, p->hand.event, 0));
  return BIK_OK;
}
static int ws_release(bik_problem* p, cudaStream_t st, int rc) {
  if (rc) return rc;
  if (!p->hand.event) CUDA_OK(cudaEventCreateWithFlags(&p->hand.event, cudaEventDisableTiming));
  CUDA_OK(cudaEventRecord(p->hand.event, st));
  p->hand.stream = st; p->hand.pending = 1;
  return BIK_OK;
}

static int solve_common(const bik_problem* cp, int B, const void* q, const void* J, const void* e, const void* e_posture, const void* G_coll,
                        const void* h_coll, double dt, double damping, void* dq, int32_t* status, int32_t* iters, int f64, void* stream) {
  if (!cp || !q || !dq || B < 0) return bik_fail(BIK_ERR_INVALID, "null argument");
  const PHeader& h = cp->h;
  if ((h.K > 0 && (!J || !e)) || (h.P > 0 && !e_posture) || (h.npairs > 0 && (!G_coll || !h_coll))) return bik_fail(BIK_ERR_INVALID, "null input");
  if (B == 0) return BIK_OK;
  bik_problem* p = const_cast<bik_problem*>(cp);
  DeviceGuard g(p->model->device);
  K2Args a;
  memset(&a, 0, sizeof a);
  a.B = B; a.q = q; a.io64 = f64; a.J = J; a.e = e; a.ep = e_posture; a.dense64 = f64; a.Gc = G_coll; a.hc = h_coll; a.gc64 = f64;
  a.dt = dt; a.damping = damping; a.dq = dq; a.status = status; a.iters = iters;
  if (status) CUDA_OK(cudaMemsetAsync(status, 0, sizeof(int32_t) * (size_t)B, static_cast<cudaStream_t>(stream)));
  std::lock_guard<std::mutex> lock(p->mu);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int rc = ws_acquire(p, st);   // the tile counters live in the problem
  if (rc) return rc;
  return ws_release(p, st, dispatch_k2(p, a, st));
}
extern "C" int bik_solve_ex(const bik_problem* p, int B, const float* q, const float* J, const float* e, const float* e_posture, const float* G_coll,
                            const float* h_coll, float dt, double damping, float* dq, int32_t* status, int32_t* iters, void* stream) {
  return solve_common(p, B, q, J, e, e_posture, G_coll, h_coll, dt, damping, dq, status, iters, 0, stream);
}
extern "C" int bik_solve(const bik_problem* p, int B, const float* q, const float* J, const float* e, const float* e_posture, const float* G_coll,
                         const float* h_coll, float dt, double damping, float* dq, int32_t* status, void* stream) {
  return solve_common(p, B, q, J, e, e_posture, G_coll, h_coll, dt, damping, dq, status, nullptr, 0, stream);
}
extern "C" int bik_solve64(const bik_problem* p, int B, const double* q, const double* J, const double* e, const double* e_posture, const double* G_coll,
                           const double* h_coll, double dt, double damping, double* dq, int32_t* status, int32_t* iters, void* stream) {
  return solve_common(p, B, q, J, e, e_posture, G_coll, h_coll, dt, damping, dq, status, iters, 1, stream);
}

extern "C" int bik_integrate(const bik_model* m, int B, float* q, const float* dq, void* stream) { return integrate_common(m, B, q, dq, stream); }
extern "C" int bik_integrate64(const bik_model* m, int B, double* q, const double* dq, void* stream) { return integrate_common(m, B, q, dq, stream); }
extern "C" int bik_check_limits(const bik_model* m, int B, const float* q, float tol, int32_t* status, void* stream) {
  return check_limits_common(m, B, q, tol, status, stream);
}
extern "C" int bik_check_limits64(const bik_model* m, int B, const double* q, double tol, int32_t* status, void* stream) {
  return check_limits_common(m, B, q, (float)tol, status, stream);
}

// The buffer groups of a problem (bik_dev.cuh).  Callers hold p->mu.
int Handoff::reserve(const PHeader& h, size_t B, int elem, unsigned* moves) {
  const HandoffSizes n = handoff_sizes(h);
  CUDA_OK(pk.reserve(elem * B * n.pk, moves));
  CUDA_OK(Gc.reserve(elem * B * n.Gc, moves));
  CUDA_OK(hc.reserve(elem * B * n.hc, moves));
  CUDA_OK(warm.reserve(B * n.warm, moves));
  return BIK_OK;
}
int LoopState::reserve(const PHeader& h, size_t B, int elem, bool ptc, bool hold, unsigned* moves) {
  for (DevBuf* b : {&done, &cursor, &step, &status}) CUDA_OK(b->reserve(sizeof(int32_t) * B, moves));
  CUDA_OK(dq.reserve(elem * B * h.nv, moves));
  CUDA_OK(count.reserve(4 * sizeof(int), moves));
  if (ptc) CUDA_OK(ptcur.reserve(elem * B * (size_t)(h.P > 0 ? h.P : 1) * h.nq, moves));
  if (hold) CUDA_OK(held.reserve(elem * B * (size_t)(k1_tgt_words(h) > 0 ? k1_tgt_words(h) : 1), moves));
  if (!host) CUDA_OK(cudaMallocHost(&host, 4 * sizeof(int)));
  return BIK_OK;
}
int HostStaging::reserve(const PHeader& h, size_t B, size_t pt_elems) {
  unsigned moves = 0;   // nothing keeps these addresses between calls
  CUDA_OK(q.reserve(4 * B * h.nq, &moves));
  CUDA_OK(ft.reserve(4 * B * (h.F > 0 ? h.F : 1) * 7, &moves));
  CUDA_OK(pt.reserve(4 * (pt_elems > 0 ? pt_elems : 1), &moves));
  CUDA_OK(ct.reserve(4 * B * (h.C > 0 ? h.C : 1) * 3, &moves));
  CUDA_OK(dq.reserve(4 * B * h.nv, &moves));
  CUDA_OK(st.reserve(4 * B, &moves));
  return BIK_OK;
}

// One or more solve_ik steps on device buffers: per step K1 (check_limits + FK + packed task rows + collision rows) and
// K2 (QP + integrate).  Caller holds p->mu and has reserved the hand-off for `k1d ? 8 : 4`-byte elements.
// bounds: per-instance bounds (the bounded K2), or null.  coll: per-instance collision pairs and distances (k1c_kernel), or null.
// placement: per-instance frame placements (k1p_kernel, with coll's members or null ones), or null.
static int step_core(bik_problem* p, int B, size_t ws_off, void* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                     const bik_bounds* bounds, const bik_collision* coll, const void* placement, double dt, double damping, int nsteps, int integrate, void* dq,
                     int32_t* status, int io64, bool k1d, cudaStream_t st) {
  // hand-off rows [ws_off, ws_off + B): chunks of one batch may be in flight on different streams (bik_step_host)
  const HandoffSizes n = handoff_sizes(p->h);
  const size_t es = k1d ? 8 : 4;
  char* const pk = p->hand.pk.as<char>() + ws_off * n.pk * es;
  char* const Gc = p->hand.Gc.as<char>() + ws_off * n.Gc * es;
  char* const hc = p->hand.hc.as<char>() + ws_off * n.hc * es;
  signed char* const warmb = p->hand.warm.as<signed char>() + ws_off * n.warm;
  const bool warm = nsteps > 1;   // rollouts: carry the active set (and the previous dq) from step to step
  const int phase = env_int("BIK_STEP_PHASE", 0);   // measurement aid: 1 = only K1, 2 = only K2 (on the rows the last K1 left)
  if (warm) CUDA_OK(cudaMemsetAsync(warmb, 0, (size_t)B * n.warm, st));
  for (int s = 0; s < nsteps; ++s) {
    K1Args a1;
    memset(&a1, 0, sizeof a1);
    a1.B = B; a1.q = q; a1.ftgt = in->frame_targets; a1.ptgt = in->posture_targets; a1.ctgt = in->com_targets; a1.in64 = io64; a1.pbatched = in->posture_batched;
    a1.dt = dt; a1.pk = pk; a1.Gc = Gc; a1.hc = hc; a1.weights = weights;
    a1.status = status; a1.accumulate = s > 0; a1.tol = 1e-6f;   // Configuration.check_limits(safety_break=False) of solve_ik.py:99
    int rc = BIK_OK;
    if (phase != 2 && placement) {
      K1PArgs pa;
      memset(&pa, 0, sizeof pa);
      static_cast<K1Args&>(pa) = a1;
      if (coll) { pa.enabled = coll->enabled; pa.dmin = coll->minimum_distance; pa.ddet = coll->detection_distance; }
      pa.placement = placement;
      rc = bik_launch_k1(p, pa, k1d, st);
    } else if (phase != 2 && coll) {
      K1CArgs ca;
      memset(&ca, 0, sizeof ca);
      static_cast<K1Args&>(ca) = a1;
      ca.enabled = coll->enabled; ca.dmin = coll->minimum_distance; ca.ddet = coll->detection_distance;
      rc = bik_launch_k1(p, ca, k1d, st);
    } else if (phase != 2) {
      rc = bik_launch_k1(p, a1, k1d, st);
    }
    if (rc) return rc;
    if (phase == 1) continue;
    K2Args a2;
    memset(&a2, 0, sizeof a2);
    a2.B = B; a2.q = q; a2.io64 = io64; a2.pk = pk; a2.pk64 = k1d; a2.ptgt = in->posture_targets; a2.pbatched = in->posture_batched;
    a2.Gc = Gc; a2.hc = hc; a2.gc64 = k1d; a2.dt = dt; a2.damping = damping; a2.dq = dq; a2.integrate = integrate; a2.status = status;
    a2.warm = warm ? warmb : nullptr;
    if (bounds) {
      K2BdArgs ba;
      memset(&ba, 0, sizeof ba);
      static_cast<K2Args&>(ba) = a2;
      ba.pw = posture_weights; ba.lower = bounds->lower; ba.upper = bounds->upper; ba.vmax = bounds->vmax;
      rc = dispatch_k2(p, ba, st);
    } else if (posture_weights) {
      K2PwArgs pa;
      memset(&pa, 0, sizeof pa);
      static_cast<K2Args&>(pa) = a2;
      pa.pw = posture_weights;
      rc = dispatch_k2(p, pa, st);
    } else {
      rc = dispatch_k2(p, a2, st);
    }
    if (rc) return rc;
  }
  return BIK_OK;
}

// The bounds of a ..._bounded call, or null when it narrows nothing (no struct, or three null members): such a call runs what
// the ..._weighted_ex call runs.
static const bik_bounds* bounds_of(const bik_bounds* bounds) { return bounds && has_bounds(*bounds) ? bounds : nullptr; }
// The collision arguments of a ..._coll call, or null when they change nothing (no struct, or three null members): such a
// call runs what the ..._bounded call runs.
static const bik_collision* coll_of(const bik_collision* coll) { return coll && has_coll(*coll) ? coll : nullptr; }

// placement: the ..._placed entry points' frame placements, or null (what the ..._coll entry points run).
static int step_common(const bik_problem* cp, int B, void* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                       const bik_bounds* bounds, const bik_collision* coll, double dt, double damping, int nsteps, int integrate, void* dq, int32_t* status, int f64,
                       void* stream, const void* placement = nullptr) {
  if (B == 0 && cp) return BIK_OK;
  bounds = bounds_of(bounds);
  coll = coll_of(coll);
  int rc = check_inputs(cp, in, false, f64, false, posture_weights, bounds, coll, placement);
  if (rc) return rc;
  if (!q || !dq || B < 0 || nsteps < 1) return bik_fail(BIK_ERR_INVALID, "bad argument");
  bik_problem* p = const_cast<bik_problem*>(cp);
  std::lock_guard<std::mutex> lock(p->mu);
  DeviceGuard g(p->model->device);
  const bool k1d = k1_double(p, damping, f64 != 0, posture_weights != nullptr);
  rc = p->hand.reserve(p->h, B, k1d ? 8 : 4, &p->moves);
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  rc = ws_acquire(p, st);
  if (rc) return rc;
  // (status needs no clearing: K1's fused check_limits assigns it on the first step, everything later ORs into it)
  return ws_release(p, st, step_core(p, B, 0, q, in, weights, posture_weights, bounds, coll, placement, dt, damping, nsteps, integrate, dq, status, f64, k1d, st));
}
extern "C" int bik_step(const bik_problem* p, int B, float* q, const bik_inputs* in, float dt, double damping, int nsteps, int integrate, float* dq,
                        int32_t* status, void* stream) {
  return step_common(p, B, q, in, nullptr, nullptr, nullptr, nullptr, dt, damping, nsteps, integrate, dq, status, 0, stream);
}
extern "C" int bik_step64(const bik_problem* p, int B, double* q, const bik_inputs* in, double dt, double damping, int nsteps, int integrate, double* dq,
                          int32_t* status, void* stream) {
  return step_common(p, B, q, in, nullptr, nullptr, nullptr, nullptr, dt, damping, nsteps, integrate, dq, status, 1, stream);
}
extern "C" int bik_step_weighted(const bik_problem* p, int B, float* q, const bik_inputs* in, const void* weights, float dt, double damping, int nsteps,
                                 int integrate, float* dq, int32_t* status, void* stream) {
  return step_common(p, B, q, in, weights, nullptr, nullptr, nullptr, dt, damping, nsteps, integrate, dq, status, 0, stream);
}
extern "C" int bik_step_weighted64(const bik_problem* p, int B, double* q, const bik_inputs* in, const void* weights, double dt, double damping,
                                   int nsteps, int integrate, double* dq, int32_t* status, void* stream) {
  return step_common(p, B, q, in, weights, nullptr, nullptr, nullptr, dt, damping, nsteps, integrate, dq, status, 1, stream);
}
extern "C" int bik_step_weighted_ex(const bik_problem* p, int B, float* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                                    float dt, double damping, int nsteps, int integrate, float* dq, int32_t* status, void* stream) {
  return step_common(p, B, q, in, weights, posture_weights, nullptr, nullptr, dt, damping, nsteps, integrate, dq, status, 0, stream);
}
extern "C" int bik_step_weighted_ex64(const bik_problem* p, int B, double* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                                      double dt, double damping, int nsteps, int integrate, double* dq, int32_t* status, void* stream) {
  return step_common(p, B, q, in, weights, posture_weights, nullptr, nullptr, dt, damping, nsteps, integrate, dq, status, 1, stream);
}
extern "C" int bik_step_bounded(const bik_problem* p, int B, float* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                                const bik_bounds* bounds, float dt, double damping, int nsteps, int integrate, float* dq, int32_t* status,
                                void* stream) {
  return step_common(p, B, q, in, weights, posture_weights, bounds, nullptr, dt, damping, nsteps, integrate, dq, status, 0, stream);
}
extern "C" int bik_step_bounded64(const bik_problem* p, int B, double* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                                  const bik_bounds* bounds, double dt, double damping, int nsteps, int integrate, double* dq, int32_t* status,
                                  void* stream) {
  return step_common(p, B, q, in, weights, posture_weights, bounds, nullptr, dt, damping, nsteps, integrate, dq, status, 1, stream);
}
extern "C" int bik_step_coll(const bik_problem* p, int B, float* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                             const bik_bounds* bounds, const bik_collision* coll, float dt, double damping, int nsteps, int integrate, float* dq,
                             int32_t* status, void* stream) {
  return step_common(p, B, q, in, weights, posture_weights, bounds, coll, dt, damping, nsteps, integrate, dq, status, 0, stream);
}
extern "C" int bik_step_coll64(const bik_problem* p, int B, double* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                               const bik_bounds* bounds, const bik_collision* coll, double dt, double damping, int nsteps, int integrate, double* dq,
                               int32_t* status, void* stream) {
  return step_common(p, B, q, in, weights, posture_weights, bounds, coll, dt, damping, nsteps, integrate, dq, status, 1, stream);
}
extern "C" int bik_step_placed(const bik_problem* p, int B, float* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                               const bik_bounds* bounds, const bik_collision* coll, const void* placement, float dt, double damping, int nsteps,
                               int integrate, float* dq, int32_t* status, void* stream) {
  return step_common(p, B, q, in, weights, posture_weights, bounds, coll, dt, damping, nsteps, integrate, dq, status, 0, stream, placement);
}
extern "C" int bik_step_placed64(const bik_problem* p, int B, double* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                                 const bik_bounds* bounds, const bik_collision* coll, const void* placement, double dt, double damping, int nsteps,
                                 int integrate, double* dq, int32_t* status, void* stream) {
  return step_common(p, B, q, in, weights, posture_weights, bounds, coll, dt, damping, nsteps, integrate, dq, status, 1, stream, placement);
}

extern "C" int bik_problem_describe(const bik_problem* p, double damping, char* buf, size_t cap) {
  if (!p) return bik_fail(BIK_ERR_INVALID, "null argument");
  const PHeader& h = p->h;
  char k2[96];
  bik_k2_describe(p, k2, sizeof k2);
  const bool grp = bik_k2_group_applies(p);
  std::string d = "k1: " + std::to_string(h.G) + " lanes/instance, " + std::to_string(h.nneeded) + "/" + std::to_string(h.nnode) + " nodes visited, " +
                  (k1_double(p, damping, false) ? "f64" : "f32") + " for fp32 callers; nv=" + std::to_string(h.nv) + " coupled=" + std::to_string(h.nu) +
                  " (unbounded, eliminated once: " + std::to_string(grp ? h.nfree : 0) + ") rows=" + std::to_string(h.K) + " pairs=" + std::to_string(h.npairs) +
                  " packed=" + std::to_string(h.pk_stride) + "; k2: " + k2 + " f64";
  if (buf && cap) { size_t n = d.size() < cap - 1 ? d.size() : cap - 1; memcpy(buf, d.c_str(), n); buf[n] = 0; }
  return (int)d.size();
}

// solve_ik + integrate until every frame task of an instance is within (pos_threshold, ori_threshold) or max_iters steps were
// taken -- the inner loop of the reference's examples (examples/quadruped_spot.py:89-104, examples/arm_aloha.py:146-169), per
// instance.  One pass = a one-thread tick, K1 (which also tests the thresholds on the errors it has just computed: instances
// that pass are marked done and keep their q), a one-thread condition, K2 (skips the done instances, integrates the others).
// The loop itself runs ON THE DEVICE: the passes are the body of a CUDA-graph WHILE node whose condition the condition kernel
// sets (cudaGraphSetConditional), so the host enqueues one graph launch and never polls.  The graph is kept and reused as long
// as the call's arguments and the problem's buffers do not change (the usual control loop).  BIK_CONVERGE_GRAPH=0, or any failure to build the graph,
// falls back to a host loop that reads the device counter back every `check_every` steps.
// bik_track (below) runs the same passes with K1 in track mode; `track` selects the mode everywhere in this driver.
// The pass's arguments (ConvCall), its buffers and its bookkeeping rules are defined in bik_loop.h.
static ConvBufs conv_bufs(const bik_problem* p) {
  const Handoff& w = p->hand;
  const LoopState& l = p->loop;
  return ConvBufs{w.pk.ptr, w.Gc.ptr, w.hc.ptr, l.dq.ptr, w.warm.as<signed char>(), l.done.as<int32_t>(), l.cursor.as<int32_t>(), l.step.as<int32_t>(),
                  l.status.as<int32_t>(), l.count.as<int>(), l.ptcur.ptr, l.held.ptr};
}
// `status` is the call's status buffer, or null (the warm-up pass before a graph capture)
static int converge_pass(bik_problem* p, const ConvCall& c, int32_t* status, cudaGraphConditionalHandle handle, int use_handle, cudaStream_t st) {
  const ConvBufs s = conv_bufs(p);
  conv_tick_kernel<<<1, 1, 0, st>>>(c.track, s.count);
  int rc = c.placement ? bik_launch_k1(p, conv_k1p_args(c, s, status), c.k1d, st)
           : c.hold ? bik_launch_k1(p, conv_k1h_args(c, s, status), c.k1d, st)
           : (has_coll(c.coll) ? bik_launch_k1(p, conv_k1c_args(c, s, status), c.k1d, st) : bik_launch_k1(p, conv_k1_args(c, s, status), c.k1d, st));
  if (rc) return rc;
  conv_cond_kernel<<<1, 1, 0, st>>>(c.track, c.max_iters, s.count, handle, use_handle);
  if (has_bounds(c.bounds)) rc = dispatch_k2(p, conv_k2_bd_args(c, s, status), st);
  else rc = c.posture_weights ? dispatch_k2(p, conv_k2_pw_args(c, s, status), st) : dispatch_k2(p, conv_k2_args(c, s, status), st);
  if (rc) return rc;
  CUDA_OK(cudaGetLastError());
  return BIK_OK;
}

// The graph of the call: the one the problem keeps if it was built for these arguments and these buffers, else a new one
// that replaces it.  *exec stays null when the graph cannot be built (the caller then runs the host-polled loop).
static int conv_graph_for(bik_problem* p, const ConvCall& c, cudaStream_t st, cudaGraphExec_t* exec) {
  ConvKey key;
  memset(&key, 0, sizeof key);
  key.c = c; key.c.in = nullptr;   // (every ConvCall is zero-filled before it is assigned)
  key.in = *c.in; key.in.q = nullptr;
  key.moves = p->moves;
  ConvGraph& g = p->loop.graph;
  if (g.exec && memcmp(&g.key, &key, sizeof key) == 0) { *exec = g.exec; return BIK_OK; }
  g.drop();
  // warm the launch-geometry cache and the tile counter outside the capture (those paths allocate / query attributes):
  // one K1 + a K2 that skips every instance (track mode: every instance is marked as having no frames left).  The warm-up
  // rewrites the loop state on its own stream, so an earlier call that may still be running on `st` finishes first.
  CUDA_OK(cudaStreamSynchronize(st));
  const ConvBufs s = conv_bufs(p);
  bool built = false;
  do {
    if (cudaStreamCreateWithFlags(&g.cap, cudaStreamNonBlocking) != cudaSuccess) break;
    cudaMemsetAsync(s.done, 1, sizeof(int32_t) * (size_t)c.B, g.cap);
    if (c.track) cudaMemsetAsync(s.step, 0xff, sizeof(int32_t) * (size_t)c.B, g.cap);
    cudaMemsetAsync(s.count, 0, 4 * sizeof(int), g.cap);
    cudaGraphConditionalHandle none{};
    if (converge_pass(p, c, nullptr, none, 0, g.cap) != BIK_OK) break;
    if (cudaStreamSynchronize(g.cap) != cudaSuccess) break;
    if (cudaGraphCreate(&g.graph, 0) != cudaSuccess) break;
    cudaGraphConditionalHandle handle;
    if (cudaGraphConditionalHandleCreate(&handle, g.graph, 1, cudaGraphCondAssignDefault) != cudaSuccess) break;
    cudaGraphNodeParams cp2 = {cudaGraphNodeTypeConditional};
    cp2.conditional.handle = handle; cp2.conditional.type = cudaGraphCondTypeWhile; cp2.conditional.size = 1;
    cudaGraphNode_t node;
    if (cudaGraphAddNode(&node, g.graph, nullptr, 0, &cp2) != cudaSuccess) break;
    cudaGraph_t body = cp2.conditional.phGraph_out[0];
    if (cudaStreamBeginCaptureToGraph(g.cap, body, nullptr, nullptr, 0, cudaStreamCaptureModeRelaxed) != cudaSuccess) break;
    const int prc = converge_pass(p, c, c.status, handle, 1, g.cap);
    if (cudaStreamEndCapture(g.cap, nullptr) != cudaSuccess || prc != BIK_OK) break;
    if (cudaGraphInstantiate(&g.exec, g.graph, 0) != cudaSuccess) break;
    built = true;
  } while (false);
  if (built) g.key = key;
  else { (void)cudaGetLastError(); g.drop(); }
  *exec = g.exec;
  return BIK_OK;
}

// The passes from the host.  converge: polled after step `it` every check_every steps; track: polled every check_every passes.
static int conv_host_loop(bik_problem* p, const ConvCall& c, int check_every, cudaStream_t st) {
  const long long cap = conv_pass_cap(c);
  bool all_done = false;
  cudaGraphConditionalHandle none{};
  for (long long it = 0; it < cap && !all_done; ++it) {
    int rc = converge_pass(p, c, c.status, none, 0, st);
    if (rc) return rc;
    const bool poll = c.track ? ((it + 1) % check_every == 0 || it + 1 == cap) : (it > 0 && (it == c.max_iters || it % check_every == 0));
    if (poll) {
      CUDA_OK(cudaMemcpyAsync(p->loop.host, p->loop.count.ptr, 4 * sizeof(int), cudaMemcpyDeviceToHost, st));
      CUDA_OK(cudaStreamSynchronize(st));
      all_done = p->loop.host[1] == 0;
    }
  }
  return BIK_OK;
}

// The loop of bik_converge / bik_track.  Caller has validated the arguments.
static int converge_run(bik_problem* p, const ConvCall& c, int check_every, int32_t* passes, cudaStream_t st) {
  std::lock_guard<std::mutex> lock(p->mu);
  DeviceGuard g(p->model->device);
  int rc = p->hand.reserve(p->h, c.B, c.k1d ? 8 : 4, &p->moves);
  if (rc) return rc;
  rc = p->loop.reserve(p->h, c.B, c.io64 ? 8 : 4, uses_ptcur(c), c.hold != nullptr, &p->moves);   // K2 writes dq in the caller's precision and reads it back as the next pass's warm start
  if (rc) return rc;
  rc = ws_acquire(p, st);
  if (rc) return rc;
  cudaGraphExec_t exec = nullptr;
  if (env_int("BIK_CONVERGE_GRAPH", 1) != 0) rc = conv_graph_for(p, c, st, &exec);
  if (rc) return rc;
  const ConvBufs s = conv_bufs(p);
  const int blocks = (c.B + 127) / 128;
  conv_reset_kernel<<<blocks, 128, 0, st>>>(c.B, c.track, c.T, c.lengths, s);
  CUDA_OK(cudaGetLastError());
  CUDA_OK(cudaMemsetAsync(s.warm, 0, (size_t)c.B * handoff_sizes(p->h).warm, st));
  if (exec) CUDA_OK(cudaGraphLaunch(exec, st));
  else rc = conv_host_loop(p, c, check_every, st);
  if (rc) return rc;
  if (c.track) {
    if (passes) CUDA_OK(cudaMemcpyAsync(passes, s.count, sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  } else {
    conv_finish_kernel<<<blocks, 128, 0, st>>>(c.B, c.max_iters, s.done, c.iters, c.status);
    CUDA_OK(cudaGetLastError());
  }
  return ws_release(p, st, BIK_OK);
}

// placement: the ..._placed entry points' frame placements, or null.
static int converge_common(const bik_problem* cp, int B, void* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                           const bik_bounds* bounds, const bik_collision* coll, double dt, double damping, int max_iters, double pos_threshold, double ori_threshold,
                           int check_every, int32_t* iters, int32_t* status, int io64, void* stream, const void* placement = nullptr) {
  if (B == 0 && cp) return BIK_OK;
  bounds = bounds_of(bounds);
  coll = coll_of(coll);
  int rc = check_inputs(cp, in, false, io64, false, posture_weights, bounds, coll, placement);
  if (rc) return rc;
  if (!q || !iters || B < 0 || max_iters < 1) return bik_fail(BIK_ERR_INVALID, "bad argument");
  if (check_every < 1) check_every = 1;
  bik_problem* p = const_cast<bik_problem*>(cp);
  ConvCall c;
  memset(&c, 0, sizeof c);
  c.B = B; c.T = 1; c.max_iters = max_iters; c.dt = dt; c.pos = pos_threshold; c.ori = ori_threshold; c.damping = damping; c.q = q; c.in = in;
  c.iters = iters; c.status = status; c.track = false; c.k1d = k1_double(p, damping, io64 != 0, posture_weights != nullptr); c.io64 = io64 != 0;
  c.weights = weights; c.posture_weights = posture_weights;
  if (bounds) c.bounds = *bounds;
  if (coll) c.coll = *coll;
  c.placement = placement;
  return converge_run(p, c, check_every, nullptr, static_cast<cudaStream_t>(stream));
}
extern "C" int bik_converge(const bik_problem* cp, int B, float* q, const bik_inputs* in, float dt, double damping, int max_iters, float pos_threshold,
                            float ori_threshold, int check_every, int32_t* iters, int32_t* status, void* stream) {
  return converge_common(cp, B, q, in, nullptr, nullptr, nullptr, nullptr, dt, damping, max_iters, pos_threshold, ori_threshold, check_every, iters, status, 0, stream);
}
extern "C" int bik_converge64(const bik_problem* cp, int B, double* q, const bik_inputs* in, double dt, double damping, int max_iters,
                              double pos_threshold, double ori_threshold, int check_every, int32_t* iters, int32_t* status, void* stream) {
  return converge_common(cp, B, q, in, nullptr, nullptr, nullptr, nullptr, dt, damping, max_iters, pos_threshold, ori_threshold, check_every, iters, status, 1, stream);
}
extern "C" int bik_converge_weighted(const bik_problem* cp, int B, float* q, const bik_inputs* in, const void* weights, float dt, double damping,
                                     int max_iters, float pos_threshold, float ori_threshold, int check_every, int32_t* iters, int32_t* status,
                                     void* stream) {
  return converge_common(cp, B, q, in, weights, nullptr, nullptr, nullptr, dt, damping, max_iters, pos_threshold, ori_threshold, check_every, iters, status, 0, stream);
}
extern "C" int bik_converge_weighted64(const bik_problem* cp, int B, double* q, const bik_inputs* in, const void* weights, double dt, double damping,
                                       int max_iters, double pos_threshold, double ori_threshold, int check_every, int32_t* iters, int32_t* status,
                                       void* stream) {
  return converge_common(cp, B, q, in, weights, nullptr, nullptr, nullptr, dt, damping, max_iters, pos_threshold, ori_threshold, check_every, iters, status, 1, stream);
}
extern "C" int bik_converge_weighted_ex(const bik_problem* cp, int B, float* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                                        float dt, double damping, int max_iters, float pos_threshold, float ori_threshold, int check_every,
                                        int32_t* iters, int32_t* status, void* stream) {
  return converge_common(cp, B, q, in, weights, posture_weights, nullptr, nullptr, dt, damping, max_iters, pos_threshold, ori_threshold, check_every, iters, status, 0,
                         stream);
}
extern "C" int bik_converge_weighted_ex64(const bik_problem* cp, int B, double* q, const bik_inputs* in, const void* weights,
                                          const void* posture_weights, double dt, double damping, int max_iters, double pos_threshold,
                                          double ori_threshold, int check_every, int32_t* iters, int32_t* status, void* stream) {
  return converge_common(cp, B, q, in, weights, posture_weights, nullptr, nullptr, dt, damping, max_iters, pos_threshold, ori_threshold, check_every, iters, status, 1,
                         stream);
}
extern "C" int bik_converge_bounded(const bik_problem* cp, int B, float* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                                    const bik_bounds* bounds, float dt, double damping, int max_iters, float pos_threshold, float ori_threshold,
                                    int check_every, int32_t* iters, int32_t* status, void* stream) {
  return converge_common(cp, B, q, in, weights, posture_weights, bounds, nullptr, dt, damping, max_iters, pos_threshold, ori_threshold, check_every, iters, status, 0,
                         stream);
}
extern "C" int bik_converge_bounded64(const bik_problem* cp, int B, double* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                                      const bik_bounds* bounds, double dt, double damping, int max_iters, double pos_threshold, double ori_threshold,
                                      int check_every, int32_t* iters, int32_t* status, void* stream) {
  return converge_common(cp, B, q, in, weights, posture_weights, bounds, nullptr, dt, damping, max_iters, pos_threshold, ori_threshold, check_every, iters, status, 1,
                         stream);
}
extern "C" int bik_converge_coll(const bik_problem* cp, int B, float* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                                 const bik_bounds* bounds, const bik_collision* coll, float dt, double damping, int max_iters, float pos_threshold,
                                 float ori_threshold, int check_every, int32_t* iters, int32_t* status, void* stream) {
  return converge_common(cp, B, q, in, weights, posture_weights, bounds, coll, dt, damping, max_iters, pos_threshold, ori_threshold, check_every, iters, status, 0,
                         stream);
}
extern "C" int bik_converge_coll64(const bik_problem* cp, int B, double* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                                   const bik_bounds* bounds, const bik_collision* coll, double dt, double damping, int max_iters, double pos_threshold,
                                   double ori_threshold, int check_every, int32_t* iters, int32_t* status, void* stream) {
  return converge_common(cp, B, q, in, weights, posture_weights, bounds, coll, dt, damping, max_iters, pos_threshold, ori_threshold, check_every, iters, status, 1,
                         stream);
}
extern "C" int bik_converge_placed(const bik_problem* cp, int B, float* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                                   const bik_bounds* bounds, const bik_collision* coll, const void* placement, float dt, double damping, int max_iters,
                                   float pos_threshold, float ori_threshold, int check_every, int32_t* iters, int32_t* status, void* stream) {
  return converge_common(cp, B, q, in, weights, posture_weights, bounds, coll, dt, damping, max_iters, pos_threshold, ori_threshold, check_every, iters, status, 0,
                         stream, placement);
}
extern "C" int bik_converge_placed64(const bik_problem* cp, int B, double* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                                     const bik_bounds* bounds, const bik_collision* coll, const void* placement, double dt, double damping, int max_iters,
                                     double pos_threshold, double ori_threshold, int check_every, int32_t* iters, int32_t* status, void* stream) {
  return converge_common(cp, B, q, in, weights, posture_weights, bounds, coll, dt, damping, max_iters, pos_threshold, ori_threshold, check_every, iters, status, 1,
                         stream, placement);
}

// The examples' outer loop: for each frame of a target sequence, the bik_converge loop, every instance on its own cursor.
// One pass works like a bik_converge pass; K1's test, when it ends an instance's frame, records that frame's results and
// moves the instance to its next frame (K1Args, track mode).  The loop ends when no instance has frames left.
// hold: the bik_track_hold entry points' hold mask, or null.  placement: the bik_track_placed entry points' frame placements, or
// null.
static int track_common(const bik_problem* cp, int B, int T, void* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                        const bik_bounds* bounds, const bik_collision* coll, const int32_t* lengths, double dt, double damping, int max_iters, double pos_threshold,
                        double ori_threshold, int check_every, void* q_traj, int32_t* iters, int32_t* status, int32_t* passes, int io64, void* stream,
                        const uint8_t* hold = nullptr, const void* placement = nullptr) {
  if (B == 0 && cp) return BIK_OK;
  bounds = bounds_of(bounds);
  coll = coll_of(coll);
  int rc = check_inputs(cp, in, false, io64, true, posture_weights, bounds, coll, placement);
  if (rc) return rc;
  if (!q || !q_traj || !iters || B < 0 || max_iters < 1) return bik_fail(BIK_ERR_INVALID, "bad argument");
  if (T < 1) return bik_fail(BIK_ERR_INVALID, "T must be at least 1");
  if (check_every < 1) check_every = 1;
  bik_problem* p = const_cast<bik_problem*>(cp);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (lengths) {   // a length beyond T would read another instance's targets: check them before anything is enqueued
    DeviceGuard g(p->model->device);
    std::vector<int32_t> hl((size_t)B);
    CUDA_OK(cudaMemcpyAsync(hl.data(), lengths, sizeof(int32_t) * (size_t)B, cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaStreamSynchronize(st));
    for (int b = 0; b < B; ++b)
      if (hl[b] < 0 || hl[b] > T) return bik_fail(BIK_ERR_INVALID, "lengths[" + std::to_string(b) + "] = " + std::to_string(hl[b]) + " is outside 0..T");
  }
  ConvCall c;
  memset(&c, 0, sizeof c);
  c.B = B; c.T = T; c.max_iters = max_iters; c.dt = dt; c.pos = pos_threshold; c.ori = ori_threshold; c.damping = damping; c.q = q; c.in = in;
  c.lengths = lengths; c.q_traj = q_traj; c.iters = iters; c.status = status; c.track = true;
  c.k1d = k1_double(p, damping, io64 != 0, posture_weights != nullptr); c.io64 = io64 != 0; c.weights = weights; c.posture_weights = posture_weights;
  if (bounds) c.bounds = *bounds;
  if (coll) c.coll = *coll;
  c.hold = hold;
  c.placement = placement;
  return converge_run(p, c, check_every, passes, st);
}
extern "C" int bik_track(const bik_problem* cp, int B, int T, float* q, const bik_inputs* in, const int32_t* lengths, float dt, double damping,
                         int max_iters, float pos_threshold, float ori_threshold, int check_every, float* q_traj, int32_t* iters, int32_t* status,
                         int32_t* passes, void* stream) {
  return track_common(cp, B, T, q, in, nullptr, nullptr, nullptr, nullptr, lengths, dt, damping, max_iters, pos_threshold, ori_threshold, check_every, q_traj, iters, status, passes, 0,
                      stream);
}
extern "C" int bik_track_weighted(const bik_problem* cp, int B, int T, float* q, const bik_inputs* in, const void* weights, const int32_t* lengths,
                                  float dt, double damping, int max_iters, float pos_threshold, float ori_threshold, int check_every, float* q_traj,
                                  int32_t* iters, int32_t* status, int32_t* passes, void* stream) {
  return track_common(cp, B, T, q, in, weights, nullptr, nullptr, nullptr, lengths, dt, damping, max_iters, pos_threshold, ori_threshold, check_every, q_traj, iters, status, passes,
                      0, stream);
}
extern "C" int bik_track_weighted64(const bik_problem* cp, int B, int T, double* q, const bik_inputs* in, const void* weights, const int32_t* lengths,
                                    double dt, double damping, int max_iters, double pos_threshold, double ori_threshold, int check_every,
                                    double* q_traj, int32_t* iters, int32_t* status, int32_t* passes, void* stream) {
  return track_common(cp, B, T, q, in, weights, nullptr, nullptr, nullptr, lengths, dt, damping, max_iters, pos_threshold, ori_threshold, check_every, q_traj, iters, status, passes,
                      1, stream);
}
extern "C" int bik_track_weighted_ex(const bik_problem* cp, int B, int T, float* q, const bik_inputs* in, const void* weights,
                                     const void* posture_weights, const int32_t* lengths, float dt, double damping, int max_iters, float pos_threshold,
                                     float ori_threshold, int check_every, float* q_traj, int32_t* iters, int32_t* status, int32_t* passes,
                                     void* stream) {
  return track_common(cp, B, T, q, in, weights, posture_weights, nullptr, nullptr, lengths, dt, damping, max_iters, pos_threshold, ori_threshold, check_every, q_traj,
                      iters, status, passes, 0, stream);
}
extern "C" int bik_track_weighted_ex64(const bik_problem* cp, int B, int T, double* q, const bik_inputs* in, const void* weights,
                                       const void* posture_weights, const int32_t* lengths, double dt, double damping, int max_iters,
                                       double pos_threshold, double ori_threshold, int check_every, double* q_traj, int32_t* iters, int32_t* status,
                                       int32_t* passes, void* stream) {
  return track_common(cp, B, T, q, in, weights, posture_weights, nullptr, nullptr, lengths, dt, damping, max_iters, pos_threshold, ori_threshold, check_every, q_traj,
                      iters, status, passes, 1, stream);
}
extern "C" int bik_track_bounded(const bik_problem* cp, int B, int T, float* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                                 const bik_bounds* bounds, const int32_t* lengths, float dt, double damping, int max_iters, float pos_threshold,
                                 float ori_threshold, int check_every, float* q_traj, int32_t* iters, int32_t* status, int32_t* passes, void* stream) {
  return track_common(cp, B, T, q, in, weights, posture_weights, bounds, nullptr, lengths, dt, damping, max_iters, pos_threshold, ori_threshold, check_every, q_traj,
                      iters, status, passes, 0, stream);
}
extern "C" int bik_track_bounded64(const bik_problem* cp, int B, int T, double* q, const bik_inputs* in, const void* weights,
                                   const void* posture_weights, const bik_bounds* bounds, const int32_t* lengths, double dt, double damping,
                                   int max_iters, double pos_threshold, double ori_threshold, int check_every, double* q_traj, int32_t* iters,
                                   int32_t* status, int32_t* passes, void* stream) {
  return track_common(cp, B, T, q, in, weights, posture_weights, bounds, nullptr, lengths, dt, damping, max_iters, pos_threshold, ori_threshold, check_every, q_traj,
                      iters, status, passes, 1, stream);
}
extern "C" int bik_track_coll(const bik_problem* cp, int B, int T, float* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                              const bik_bounds* bounds, const bik_collision* coll, const int32_t* lengths, float dt, double damping, int max_iters,
                              float pos_threshold, float ori_threshold, int check_every, float* q_traj, int32_t* iters, int32_t* status, int32_t* passes,
                              void* stream) {
  return track_common(cp, B, T, q, in, weights, posture_weights, bounds, coll, lengths, dt, damping, max_iters, pos_threshold, ori_threshold, check_every, q_traj,
                      iters, status, passes, 0, stream);
}
extern "C" int bik_track_coll64(const bik_problem* cp, int B, int T, double* q, const bik_inputs* in, const void* weights,
                                const void* posture_weights, const bik_bounds* bounds, const bik_collision* coll, const int32_t* lengths, double dt,
                                double damping, int max_iters, double pos_threshold, double ori_threshold, int check_every, double* q_traj,
                                int32_t* iters, int32_t* status, int32_t* passes, void* stream) {
  return track_common(cp, B, T, q, in, weights, posture_weights, bounds, coll, lengths, dt, damping, max_iters, pos_threshold, ori_threshold, check_every, q_traj,
                      iters, status, passes, 1, stream);
}
extern "C" int bik_track_hold(const bik_problem* cp, int B, int T, float* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                              const bik_bounds* bounds, const bik_collision* coll, const uint8_t* hold, const int32_t* lengths, float dt, double damping,
                              int max_iters, float pos_threshold, float ori_threshold, int check_every, float* q_traj, int32_t* iters, int32_t* status,
                              int32_t* passes, void* stream) {
  return track_common(cp, B, T, q, in, weights, posture_weights, bounds, coll, lengths, dt, damping, max_iters, pos_threshold, ori_threshold, check_every, q_traj,
                      iters, status, passes, 0, stream, hold);
}
extern "C" int bik_track_hold64(const bik_problem* cp, int B, int T, double* q, const bik_inputs* in, const void* weights,
                                const void* posture_weights, const bik_bounds* bounds, const bik_collision* coll, const uint8_t* hold,
                                const int32_t* lengths, double dt, double damping, int max_iters, double pos_threshold, double ori_threshold,
                                int check_every, double* q_traj, int32_t* iters, int32_t* status, int32_t* passes, void* stream) {
  return track_common(cp, B, T, q, in, weights, posture_weights, bounds, coll, lengths, dt, damping, max_iters, pos_threshold, ori_threshold, check_every, q_traj,
                      iters, status, passes, 1, stream, hold);
}
extern "C" int bik_track_placed(const bik_problem* cp, int B, int T, float* q, const bik_inputs* in, const void* weights, const void* posture_weights,
                                const bik_bounds* bounds, const bik_collision* coll, const uint8_t* hold, const void* placement, const int32_t* lengths,
                                float dt, double damping, int max_iters, float pos_threshold, float ori_threshold, int check_every, float* q_traj,
                                int32_t* iters, int32_t* status, int32_t* passes, void* stream) {
  return track_common(cp, B, T, q, in, weights, posture_weights, bounds, coll, lengths, dt, damping, max_iters, pos_threshold, ori_threshold, check_every, q_traj,
                      iters, status, passes, 0, stream, hold, placement);
}
extern "C" int bik_track_placed64(const bik_problem* cp, int B, int T, double* q, const bik_inputs* in, const void* weights,
                                  const void* posture_weights, const bik_bounds* bounds, const bik_collision* coll, const uint8_t* hold,
                                  const void* placement, const int32_t* lengths, double dt, double damping, int max_iters, double pos_threshold,
                                  double ori_threshold, int check_every, double* q_traj, int32_t* iters, int32_t* status, int32_t* passes, void* stream) {
  return track_common(cp, B, T, q, in, weights, posture_weights, bounds, coll, lengths, dt, damping, max_iters, pos_threshold, ori_threshold, check_every, q_traj,
                      iters, status, passes, 1, stream, hold, placement);
}
extern "C" int bik_track64(const bik_problem* cp, int B, int T, double* q, const bik_inputs* in, const int32_t* lengths, double dt, double damping,
                           int max_iters, double pos_threshold, double ori_threshold, int check_every, double* q_traj, int32_t* iters,
                           int32_t* status, int32_t* passes, void* stream) {
  return track_common(cp, B, T, q, in, nullptr, nullptr, nullptr, nullptr, lengths, dt, damping, max_iters, pos_threshold, ori_threshold, check_every, q_traj, iters, status, passes, 1,
                      stream);
}

// Host-buffer variant: device staging lives in the problem (separate allocations).  The batch is cut into chunks that flow
// through an upload stream, two compute streams taken in turn and a download stream, chained by events, so that the copies of
// neighbouring chunks overlap the kernels (PCIe is full duplex: chunk i+1 goes up while chunk i computes and chunk i-1 comes
// down) and the kernels of chunk i+1 fill the SMs that chunk i's K2 frees while its last tiles finish.  Default plan: whole K2 waves per chunk
// (see below), 1:3:4:4:3:1 where the wave size is unknown; BIK_HOST_CHUNKS=n forces n equal chunks.
extern "C" int bik_step_host(const bik_problem* cp, int B, float* q_host, const bik_inputs* in, float dt, double damping, int nsteps, int integrate,
                             float* dq_host, int32_t* status_host, size_t* h2d_bytes, size_t* d2h_bytes) {
  int rc = check_inputs(cp, in, false, 0);
  if (rc) return rc;
  if (!q_host || !dq_host || B < 0) return bik_fail(BIK_ERR_INVALID, "bad argument");
  if (B == 0) return BIK_OK;
  bik_problem* p = const_cast<bik_problem*>(cp);
  const PHeader& h = p->h;
  DeviceGuard g(p->model->device);
  size_t nq = h.nq, nv = h.nv, b = (size_t)B;
  size_t pt_elems = (in->posture_batched ? b : 1) * (size_t)h.P * nq;
  std::lock_guard<std::mutex> lock(p->mu);
  if (p->hand.pending) { CUDA_OK(cudaEventSynchronize(p->hand.event)); p->hand.pending = 0; }   // this call runs on the problem's own streams
  HostStaging& hb = p->stage;
  rc = hb.reserve(h, b, pt_elems);
  if (rc) return rc;
  if (!hb.hs[0]) for (int i = 0; i < 4; ++i) CUDA_OK(cudaStreamCreateWithFlags(&hb.hs[i], cudaStreamNonBlocking));
  float *const hq = hb.q.as<float>(), *const hft = hb.ft.as<float>(), *const hpt = hb.pt.as<float>(), *const hct = hb.ct.as<float>(),
        *const hdq = hb.dq.as<float>();
  int32_t* const hst = hb.st.as<int32_t>();
  // chunk plan
  std::vector<size_t> cuts;
  const int forced = env_int("BIK_HOST_CHUNKS", 0);
  const long long wave = bik_k2_group_wave(p);   // instances one resident wave of the small-group K2 covers (0: other path)
  if (forced > 0 || b < 8192) {
    const int NC = forced > 0 ? forced : 1;
    const size_t chunk = (b + NC - 1) / NC;
    for (size_t o = 0; o < b; o += chunk) cuts.push_back(std::min(chunk, b - o));
  } else if (wave > 0 && b > (size_t)(2 * wave)) {
    // K2's time is quantised in waves (a tile takes as long however few there are), so chunks are whole waves: one wave first
    // (the pipeline fills after the shortest possible upload), two-wave chunks in the middle, the fractional wave last (the
    // shortest possible download drains it).
    const size_t w = (size_t)wave, rem = b % w;
    size_t left = b - w - rem;
    cuts.push_back(w);
    while (left > 0) { const size_t n = std::min(left, 2 * w); cuts.push_back(n); left -= n; }
    if (rem) cuts.push_back(rem);
    else if (cuts.size() > 2 && cuts.back() == 2 * w) { cuts.back() = w; cuts.push_back(w); }
  } else {
    const int w[6] = {1, 3, 4, 4, 3, 1};
    size_t used = 0;
    for (int i = 0; i < 6; ++i) {
      size_t n = i == 5 ? b - used : ((b * w[i] / 16 + 63) & ~(size_t)63);
      n = std::min(n, b - used);
      if (n) cuts.push_back(n);
      used += n;
    }
  }
  while (hb.hev.size() < 2 * cuts.size() + 1) { cudaEvent_t e; CUDA_OK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming)); hb.hev.push_back(e); }
  const bool k1d = k1_double(p, damping, false);
  rc = p->hand.reserve(h, b, k1d ? 8 : 4, &p->moves);   // chunks keep disjoint hand-off rows: two of them compute at the same time
  if (rc) return rc;
  cudaStream_t s_up = hb.hs[0], s_dn = hb.hs[3];
  size_t up = 0, down = 0;
  // BIK_HOST_TRACE=1: timed events around every stage of every chunk, printed after the call (measurement aid)
  const bool trace = env_int("BIK_HOST_TRACE", 0) != 0;
  std::vector<cudaEvent_t> tev;
  auto mark = [&](cudaStream_t st) { if (trace) { cudaEvent_t e; cudaEventCreate(&e); cudaEventRecord(e, st); tev.push_back(e); } };
  mark(s_up);
  if (h.P) { CUDA_OK(cudaMemcpyAsync(hpt, in->posture_targets, 4 * pt_elems, cudaMemcpyHostToDevice, s_up)); up += 4 * pt_elems; }
  // every upload is enqueued first: the copy engine then streams the chunks back to back, whatever the host spends on
  // enqueuing kernels and downloads afterwards
  size_t o = 0;
  for (size_t ci = 0; ci < cuts.size(); ++ci) {
    const size_t n = cuts[ci];
    CUDA_OK(cudaMemcpyAsync(hq + o * nq, q_host + o * nq, 4 * n * nq, cudaMemcpyHostToDevice, s_up)); up += 4 * n * nq;
    if (h.F) { CUDA_OK(cudaMemcpyAsync(hft + o * h.F * 7, static_cast<const float*>(in->frame_targets) + o * h.F * 7, 4 * n * h.F * 7, cudaMemcpyHostToDevice, s_up)); up += 4 * n * h.F * 7; }
    if (h.C) { CUDA_OK(cudaMemcpyAsync(hct + o * h.C * 3, static_cast<const float*>(in->com_targets) + o * h.C * 3, 4 * n * h.C * 3, cudaMemcpyHostToDevice, s_up)); up += 4 * n * h.C * 3; }
    CUDA_OK(cudaEventRecord(hb.hev[2 * ci], s_up));
    mark(s_up);
    o += n;
  }
  o = 0;
  for (size_t ci = 0; ci < cuts.size(); ++ci) {
    const size_t n = cuts[ci];
    cudaStream_t s_cmp = hb.hs[1 + (ci & 1)];   // two compute streams in turn: the tail of one chunk's K2 (CTAs waiting for their
    CUDA_OK(cudaStreamWaitEvent(s_cmp, hb.hev[2 * ci], 0));   // slowest tile) is filled by the next chunk's kernels
    mark(s_cmp);
    bik_inputs din = *in;
    din.q = hq + o * nq; din.frame_targets = hft + o * h.F * 7; din.com_targets = hct + o * h.C * 3;
    din.posture_targets = in->posture_batched ? hpt + o * (size_t)h.P * nq : hpt;
    rc = step_core(p, (int)n, o, hq + o * nq, &din, nullptr, nullptr, nullptr, nullptr, nullptr, dt, damping, nsteps, integrate, hdq + o * nv, status_host ? hst + o : nullptr, 0, k1d, s_cmp);
    if (rc) return rc;
    CUDA_OK(cudaEventRecord(hb.hev[2 * ci + 1], s_cmp));
    mark(s_cmp);
    CUDA_OK(cudaStreamWaitEvent(s_dn, hb.hev[2 * ci + 1], 0));
    mark(s_dn);
    CUDA_OK(cudaMemcpyAsync(dq_host + o * nv, hdq + o * nv, 4 * n * nv, cudaMemcpyDeviceToHost, s_dn)); down += 4 * n * nv;
    if (integrate) { CUDA_OK(cudaMemcpyAsync(q_host + o * nq, hq + o * nq, 4 * n * nq, cudaMemcpyDeviceToHost, s_dn)); down += 4 * n * nq; }
    if (status_host) { CUDA_OK(cudaMemcpyAsync(status_host + o, hst + o, 4 * n, cudaMemcpyDeviceToHost, s_dn)); down += 4 * n; }
    mark(s_dn);
    o += n;
  }
  CUDA_OK(cudaStreamSynchronize(s_dn));
  CUDA_OK(cudaStreamSynchronize(hb.hs[1]));
  CUDA_OK(cudaStreamSynchronize(hb.hs[2]));
  CUDA_OK(cudaStreamSynchronize(s_up));
  if (trace) {   // uploads done (one per chunk), then per chunk: compute start, end, download start, end  (ms since the call's first event)
    std::string line = "bik_step_host trace (ms): up";
    const size_t nc = cuts.size();
    for (size_t k = 1; k < tev.size(); ++k) {
      float ms = 0; cudaEventElapsedTime(&ms, tev[0], tev[k]);
      char buf[32]; snprintf(buf, sizeof buf, "%s%.3f", (k > nc && (k - 1 - nc) % 4 == 0) ? " | " : " ", ms); line += buf;
    }
    fprintf(stderr, "%s\n", line.c_str());
    for (cudaEvent_t e : tev) cudaEventDestroy(e);
  }
  if (h2d_bytes) *h2d_bytes = up;
  if (d2h_bytes) *d2h_bytes = down;
  return BIK_OK;
}

// Measured FMA throughput of the CUDA cores (2 flops per FMA), best of `repeats` launches timed with CUDA events.
extern "C" int bik_measure_fma_peak(int device, int use_double, int repeats, double* tflops) {
  if (!tflops) return bik_fail(BIK_ERR_INVALID, "null argument");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) return bik_fail(BIK_ERR_CUDA, "no such CUDA device");
  DeviceGuard g(device);
  cudaDeviceProp prop;
  CUDA_OK(cudaGetDeviceProperties(&prop, device));
  const int iters = use_double ? 4096 : 8192, grid = prop.multiProcessorCount * 8, threads = 256;
  void* sink = nullptr;
  CUDA_OK(cudaMalloc(&sink, 8));
  cudaEvent_t e0, e1;
  CUDA_OK(cudaEventCreate(&e0)); CUDA_OK(cudaEventCreate(&e1));
  double best = 0;
  for (int r = 0; r < (repeats > 0 ? repeats : 5) + 1; ++r) {
    CUDA_OK(cudaEventRecord(e0));
    if (use_double) fma_peak_kernel<double><<<grid, threads>>>(iters, 1.0, static_cast<double*>(sink));
    else fma_peak_kernel<float><<<grid, threads>>>(iters, 1.0f, static_cast<float*>(sink));
    CUDA_OK(cudaEventRecord(e1));
    CUDA_OK(cudaEventSynchronize(e1));
    float ms = 0;
    CUDA_OK(cudaEventElapsedTime(&ms, e0, e1));
    const double tf = 2.0 * 16.0 * iters * (double)grid * threads / (ms * 1e-3) / 1e12;
    if (r > 0 && tf > best) best = tf;   // first launch is the warm-up
  }
  cudaEventDestroy(e0); cudaEventDestroy(e1); cudaFree(sink);
  *tflops = best;
  return BIK_OK;
}
