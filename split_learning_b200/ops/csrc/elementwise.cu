// Memory-bound kernels of the VGG-family stages (SURVEY §2.7 G4, G5, G7-G10, G12-G14):
// BatchNorm(train)+ReLU+MaxPool forward/backward on NHWC bf16, the first-layer direct conv
// (Cin <= 4), Linear finalisation (bias/ReLU/dropout), fused CE forward+backward, fused
// flat optimisers (SGD-momentum, AdamW), the FedAvg weighted n-ary reduction over (peer)
// pointers, and the mailbox flag primitives.  All vectorised to 16-byte accesses.
#include "sm90.cuh"

#include <climits>
#include <map>
#include <mutex>
#include <utility>
#include <vector>

namespace slb {

// ============================================================================ per-stream reduction scratch (sm90.cuh Det)
// A stream gets its scratch when this library creates it (slb_stream_create) or first uses it outside a CUDA-graph capture:
// its own allocation, counters zeroed by a memset ordered before its first reduction.  Inside a capture (torch records
// graphs on a side stream) nothing may be allocated or memset, so a stream first seen there takes a pre-zeroed slot from
// the device's reserve, filled at the first use outside a capture.  Slots go back (or are freed) when the stream is destroyed.
constexpr long long DET_PART_FLOATS = 1ll << 20;  // 4 MB of partial rows per stream
constexpr size_t DET_CTR_BYTES = static_cast<size_t>(DET_COUNTERS) * sizeof(uint32_t);
constexpr int DET_RESERVE = 32;
struct DetSlot {
  Det d;
  bool owned;           // own allocation (freed with the stream) or a reserve slot (returned)
};
static std::mutex g_det_mu;
static std::map<std::pair<int, cudaStream_t>, DetSlot> g_det_slots;
static std::map<int, std::vector<Det>> g_det_reserve;
static std::map<int, bool> g_det_reserve_filled;

// caller holds g_det_mu; st is not capturing
static bool det_fill_reserve(int dev, cudaStream_t st) {
  if (g_det_reserve_filled[dev]) return true;
  float* part = nullptr;
  uint32_t* ctr = nullptr;
  if (cudaMalloc(reinterpret_cast<void**>(&part), DET_RESERVE * DET_PART_FLOATS * sizeof(float)) != cudaSuccess) return false;
  if (cudaMalloc(reinterpret_cast<void**>(&ctr), DET_RESERVE * DET_CTR_BYTES) != cudaSuccess ||
      cudaMemsetAsync(ctr, 0, DET_RESERVE * DET_CTR_BYTES, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess) {
    cudaFree(part);
    return false;
  }
  for (int i = DET_RESERVE - 1; i >= 0; --i)
    g_det_reserve[dev].push_back({part + i * DET_PART_FLOATS, ctr + static_cast<long long>(i) * DET_COUNTERS, DET_PART_FLOATS});
  g_det_reserve_filled[dev] = true;
  return true;
}

Det slb_det(cudaStream_t st) {
  const Det none = {nullptr, nullptr, 0};
  int dev = 0;
  cudaGetDevice(&dev);
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(st, &cs) != cudaSuccess) return none;
  std::lock_guard<std::mutex> lock(g_det_mu);
  auto it = g_det_slots.find({dev, st});
  if (it != g_det_slots.end()) return it->second.d;
  if (cs != cudaStreamCaptureStatusNone) {
    std::vector<Det>& res = g_det_reserve[dev];
    if (res.empty()) return none;
    const Det d = res.back();
    res.pop_back();
    g_det_slots[{dev, st}] = {d, false};
    return d;
  }
  if (!det_fill_reserve(dev, st)) return none;
  float* part = nullptr;
  uint32_t* ctr = nullptr;
  if (cudaMalloc(reinterpret_cast<void**>(&part), DET_PART_FLOATS * sizeof(float)) != cudaSuccess) return none;
  if (cudaMalloc(reinterpret_cast<void**>(&ctr), DET_CTR_BYTES) != cudaSuccess ||
      cudaMemsetAsync(ctr, 0, DET_CTR_BYTES, st) != cudaSuccess) {
    cudaFree(part);
    return none;
  }
  const Det d = {part, ctr, DET_PART_FLOATS};
  g_det_slots[{dev, st}] = {d, true};
  return d;
}

void slb_det_release(cudaStream_t st) {
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> lock(g_det_mu);
  auto it = g_det_slots.find({dev, st});
  if (it == g_det_slots.end()) return;
  cudaStreamSynchronize(st);
  if (it->second.owned) {
    cudaFree(it->second.d.part);
    cudaFree(it->second.d.ctr);
  } else {
    g_det_reserve[dev].push_back(it->second.d);      // counters are zero at rest
  }
  g_det_slots.erase(it);
}

struct alignas(16) bf16x8 { __nv_bfloat162 v[4]; };

__device__ __forceinline__ void unpack8(const bf16x8& p, float (&f)[8]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __bfloat1622float2(p.v[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ bf16x8 pack8(const float (&f)[8]) {
  bf16x8 p;
#pragma unroll
  for (int i = 0; i < 4; ++i) p.v[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return p;
}

// 8 consecutive channels of one pixel, activation-typed (bf16: one 16-byte access, fp32: two)
__device__ __forceinline__ void load8(const __nv_bfloat16* p, float (&f)[8]) { unpack8(*reinterpret_cast<const bf16x8*>(p), f); }
__device__ __forceinline__ void load8(const float* p, float (&f)[8]) {
  const float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}
__device__ __forceinline__ void store8(__nv_bfloat16* p, const float (&f)[8]) { *reinterpret_cast<bf16x8*>(p) = pack8(f); }
__device__ __forceinline__ void store8(float* p, const float (&f)[8]) {
  reinterpret_cast<float4*>(p)[0] = make_float4(f[0], f[1], f[2], f[3]);
  reinterpret_cast<float4*>(p)[1] = make_float4(f[4], f[5], f[6], f[7]);
}
__device__ __forceinline__ float to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float to_f32(float v) { return v; }
template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16(v); }
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }

// "last block done" publication of a mailbox flag: every block fences its (possibly peer) stores,
// the last one to arrive releases the flag system-wide and re-arms the ticket counter.
// The flag value is a per-slot sequence number kept in device memory (`seq`), so the same
// captured CUDA graph publishes 1, 2, 3, ... on successive replays.
__device__ __forceinline__ void publish_flag(uint32_t* ticket, uint32_t* flag, uint32_t* seq, uint32_t* hint) {
  if (flag == nullptr) return;
  __syncthreads();
  if (threadIdx.x == 0 && threadIdx.y == 0) {
    __threadfence_system();
    const uint32_t t = atomicAdd(ticket, 1u);
    if (t == gridDim.x * gridDim.y - 1) {
      *ticket = 0;
      const uint32_t value = *seq + 1;
      *seq = value;
      __threadfence_system();
      st_release_sys(flag, value);
      if (hint != nullptr) st_release_sys(hint, value);
    }
  }
}

// ============================================================================ zero / flags
__global__ void zero_kernel(float4* p, long long n4) {
  pdl_trigger();
  pdl_wait();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x)
    p[i] = make_float4(0.f, 0.f, 0.f, 0.f);
}

// First kernel of a stage program that consumes a mailbox slot: zero the scratch region AND acquire the slot flag (block 0,
// thread 0 spins with ld.acquire.sys while the other blocks zero) — the stand-alone one-thread wait launch disappears
// from every F / B / L program.  No pdl_trigger(), like wait_flag_kernel: dependents must not occupy SM slots while we spin.
__global__ void zero_wait_kernel(float4* p, long long n4, const uint32_t* flag, uint32_t* expect_ctr, unsigned long long max_spins,
                                 int* status) {
  pdl_wait();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x)
    p[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const uint32_t expected = *expect_ctr + 1;
    unsigned long long spins = 0;
    while (ld_acquire_sys(flag) < expected) {
      __nanosleep(64);
      if (++spins > max_spins) {
        if (status) *status = 1;
        return;
      }
    }
    *expect_ctr = expected;
  }
}

// Spin until *flag >= expected (acquire, system scope).  `expect_ctr` (nullable): device counter; the
// kernel waits for *expect_ctr + 1 and stores it back (graph-replay friendly).  `status` (nullable)
// receives 1 on timeout so a dead producer turns into an error instead of a hung GPU.
__global__ void wait_flag_kernel(const uint32_t* flag, uint32_t expected, uint32_t* expect_ctr, unsigned long long max_spins,
                                 int* status) {
  // no pdl_trigger(): dependents must not become resident (and hog SM slots) while this kernel spins on a flag that
  // another stream of the same GPU has yet to publish
  pdl_wait();
  if (expect_ctr) expected = *expect_ctr + 1;
  unsigned long long spins = 0;
  while (ld_acquire_sys(flag) < expected) {
    __nanosleep(64);
    if (++spins > max_spins) {
      if (status) *status = 1;
      return;
    }
  }
  if (expect_ctr) *expect_ctr = expected;
}
__global__ void set_flag_kernel(uint32_t* flag, uint32_t value, uint32_t* seq, uint32_t* hint) {
  pdl_trigger();
  pdl_wait();
  if (seq) { value = *seq + 1; *seq = value; }
  __threadfence_system();
  st_release_sys(flag, value);
  if (hint) st_release_sys(hint, value);
}
__global__ void counter_inc_kernel(uint32_t* c) {
  pdl_trigger();
  pdl_wait(); *c += 1; }

// ============================================================================ BN + ReLU + MaxPool forward
template <typename T>
struct BnFwdParams {
  const T* y;               // [P][C] conv output (pre-BN)
  const float* sum;         // [C]
  const float* sumsq;       // [C]
  const float* gamma;
  const float* beta;
  float* running_mean;
  float* running_var;
  long long* num_batches_tracked;
  float* save_mean;         // [C]
  float* save_invstd;       // [C]
  T* out;                   // [P or P/4][C]   (may be a peer pointer: cut-edge mailbox slot)
  int P, C, H, W;
  int relu, pool;
  float momentum, eps;
  int update_running;
  int identity;             // 1: no normalisation (orphan ReLU/MaxPool at the head of a stage)
  uint32_t* ticket;
  uint32_t* flag;
  uint32_t* seq;
  uint32_t* hint;
};

// INFER: BatchNorm in inference mode (module.eval()): scale / shift from running_mean / running_var, no batch statistics
// and no writes to the running statistics, num_batches_tracked or save_*.
// ODD: MaxPool2 over a map with odd H or W (nn.MaxPool2d(2) floor semantics: the last row / column is dropped, the
// output is floor(H/2) x floor(W/2)).  A separate instantiation, so the even-size kernels keep their code.
template <typename T, bool INFER = false, bool ODD = false>
__global__ void __launch_bounds__(256) bn_relu_pool_fwd_kernel(const BnFwdParams<T> p) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ float s_aff[];     // scale[C], shift[C]
  float* s_scale = s_aff;
  float* s_shift = s_aff + p.C;
  const float invP = 1.f / static_cast<float>(p.P);
  for (int c = threadIdx.x; c < p.C; c += blockDim.x) {
    if constexpr (INFER) {
      const float invstd = rsqrtf(p.running_var[c] + p.eps);
      const float g = p.gamma[c];
      s_scale[c] = g * invstd;
      s_shift[c] = p.beta[c] - p.running_mean[c] * g * invstd;
      continue;
    }
    if (p.identity) { s_scale[c] = 1.f; s_shift[c] = 0.f; continue; }
    const float mean = p.sum[c] * invP;
    const float var = fmaxf(p.sumsq[c] * invP - mean * mean, 0.f);
    const float invstd = rsqrtf(var + p.eps);
    const float g = p.gamma[c];
    s_scale[c] = g * invstd;
    s_shift[c] = p.beta[c] - mean * g * invstd;
    if (blockIdx.x == 0) {
      p.save_mean[c] = mean;
      p.save_invstd[c] = invstd;
      if (p.update_running) {
        const float unbiased = p.P > 1 ? var * static_cast<float>(p.P) / static_cast<float>(p.P - 1) : var;
        p.running_mean[c] = (1.f - p.momentum) * p.running_mean[c] + p.momentum * mean;
        p.running_var[c] = (1.f - p.momentum) * p.running_var[c] + p.momentum * unbiased;
      }
    }
  }
  if (!INFER && blockIdx.x == 0 && threadIdx.x == 0 && p.update_running && !p.identity && p.num_batches_tracked)
    *p.num_batches_tracked += 1;
  __syncthreads();

  const int cg = p.C >> 3;                                  // 8-channel groups
  const int OW = p.pool ? p.W >> 1 : p.W, OH = p.pool ? p.H >> 1 : p.H;
  const long long outP = ODD ? static_cast<long long>(p.P / (p.H * p.W)) * OH * OW
                              : (p.pool ? static_cast<long long>(p.P) >> 2 : p.P);
  const long long total = outP * cg;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int g = static_cast<int>(i % cg);
    const long long op = i / cg;
    float sc[8], sh[8], r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { sc[j] = s_scale[g * 8 + j]; sh[j] = s_shift[g * 8 + j]; }
    if (!p.pool) {
      float f[8];
      load8(p.y + op * p.C + g * 8, f);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float z = fmaf(f[j], sc[j], sh[j]);
        r[j] = p.relu ? fmaxf(z, 0.f) : z;
      }
    } else {
      const int ow = static_cast<int>(op % OW);
      const long long t = op / OW;
      const int oh = static_cast<int>(t % OH);
      const long long b = t / OH;
      const long long base = ((b * p.H + 2 * oh) * p.W + 2 * ow);
#pragma unroll
      for (int j = 0; j < 8; ++j) r[j] = -INFINITY;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const long long ip = base + (q >> 1) * p.W + (q & 1);
        float f[8];
        load8(p.y + ip * p.C + g * 8, f);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float z = fmaf(f[j], sc[j], sh[j]);
          if (p.relu) z = fmaxf(z, 0.f);
          r[j] = fmaxf(r[j], z);
        }
      }
    }
    store8(p.out + op * p.C + g * 8, r);
  }
  publish_flag(p.ticket, p.flag, p.seq, p.hint);
}

// ============================================================================ BN + ReLU + MaxPool backward
template <typename T>
struct BnBwdParams {
  const T* dout;               // [P or P/4][C] gradient w.r.t. the (pooled) activation  (may be a mailbox slot)
  const T* y;                  // [P][C] saved conv output
  const float* gamma;
  const float* beta;
  const float* save_mean;
  const float* save_invstd;
  float* dgamma;               // [C] (zeroed by caller; accumulated)
  float* dbeta;                // [C]
  T* dy;                       // [P][C] gradient w.r.t. conv output
  int P, C, H, W;
  int relu, pool;
  int identity;
  Det det;                     // reproducible dgamma / dbeta reduction
};

// dz for the 1 (no pool) or 4 (pool) input pixels of output position `op`, 8 channels.
template <bool POOL, typename T>
__device__ __forceinline__ void bn_dz(const BnBwdParams<T>& p, long long op, int g, const float (&sc)[8], const float (&sh)[8],
                                      float (&yv)[POOL ? 4 : 1][8], float (&dz)[POOL ? 4 : 1][8], long long (&ip)[POOL ? 4 : 1]) {
  float d[8];
  load8(p.dout + op * p.C + g * 8, d);
  if constexpr (!POOL) {
    ip[0] = op;
    load8(p.y + op * p.C + g * 8, yv[0]);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float z = fmaf(yv[0][j], sc[j], sh[j]);
      dz[0][j] = (p.relu && z <= 0.f) ? 0.f : d[j];
    }
  } else {
    const int OW = p.W >> 1, OH = p.H >> 1;
    const int ow = static_cast<int>(op % OW);
    const long long t = op / OW;
    const int oh = static_cast<int>(t % OH);
    const long long b = t / OH;
    const long long base = ((b * p.H + 2 * oh) * p.W + 2 * ow);
    float best[8];
    int arg[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { best[j] = -INFINITY; arg[j] = 0; }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      ip[q] = base + (q >> 1) * p.W + (q & 1);
      load8(p.y + ip[q] * p.C + g * 8, yv[q]);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float z = fmaf(yv[q][j], sc[j], sh[j]);
        if (p.relu) z = fmaxf(z, 0.f);
        if (z > best[j]) { best[j] = z; arg[j] = q; }   // first maximum wins, like torch
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int j = 0; j < 8; ++j) dz[q][j] = (arg[j] == q && !(p.relu && best[j] <= 0.f)) ? d[j] : 0.f;
  }
}

// Odd H or W with MaxPool2 (the ODD kernels): position `op` walks the ceil(H/2) x ceil(W/2) grid, so that every pre-pool
// pixel belongs to exactly one position.  A window on the dropped last row or column has no pooled output: its dz is zero,
// but its dy is not (the BatchNorm-backward mean terms), so the apply passes still write it.  ip[q] = -1: no pixel.
template <typename T>
__device__ __forceinline__ void bn_dz_odd(const BnBwdParams<T>& p, long long op, int g, const float (&sc)[8], const float (&sh)[8],
                                          float (&yv)[4][8], float (&dz)[4][8], long long (&ip)[4]) {
  const int OW = p.W >> 1, OH = p.H >> 1, CW = (p.W + 1) >> 1, CH = (p.H + 1) >> 1;
  const int ow = static_cast<int>(op % CW);
  const long long t = op / CW;
  const int oh = static_cast<int>(t % CH);
  const long long b = t / CH;
  const bool pooled = ow < OW && oh < OH;
  float d[8];
  if (pooled) {
    load8(p.dout + ((b * OH + oh) * OW + ow) * p.C + g * 8, d);
  } else {
#pragma unroll
    for (int j = 0; j < 8; ++j) d[j] = 0.f;
  }
  const long long base = ((b * p.H + 2 * oh) * p.W + 2 * ow);
  float best[8];
  int arg[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { best[j] = -INFINITY; arg[j] = 0; }
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const bool in = 2 * oh + (q >> 1) < p.H && 2 * ow + (q & 1) < p.W;
    ip[q] = in ? base + (q >> 1) * p.W + (q & 1) : -1;
    if (in) {
      load8(p.y + ip[q] * p.C + g * 8, yv[q]);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) yv[q][j] = 0.f;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float z = fmaf(yv[q][j], sc[j], sh[j]);
      if (p.relu) z = fmaxf(z, 0.f);
      if (in && z > best[j]) { best[j] = z; arg[j] = q; }   // first maximum wins, like torch
    }
  }
#pragma unroll
  for (int q = 0; q < 4; ++q)
#pragma unroll
    for (int j = 0; j < 8; ++j) dz[q][j] = (pooled && arg[j] == q && !(p.relu && best[j] <= 0.f)) ? d[j] : 0.f;
}

// positions walked by the backward kernels: pooled windows, or (ODD) the ceil grid of bn_dz_odd
template <bool POOL, bool ODD, typename T>
__device__ __forceinline__ long long bn_bwd_positions(const BnBwdParams<T>& p) {
  if constexpr (ODD) return static_cast<long long>(p.P / (p.H * p.W)) * ((p.H + 1) >> 1) * ((p.W + 1) >> 1);
  else return POOL ? static_cast<long long>(p.P) >> 2 : p.P;
}

// pass 1: dgamma / dbeta.  blockDim = (C/8, 256/(C/8)); grid-stride over output positions.
template <bool POOL, typename T, bool ODD = false>
__global__ void __launch_bounds__(256) bn_bwd_reduce_kernel(const BnBwdParams<T> p) {
  pdl_trigger();
  pdl_wait();
  constexpr int NP = POOL ? 4 : 1;
  const int g = threadIdx.x;
  float sc[8], sh[8], mean[8], istd[8], ag[8], ab[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = g * 8 + j;
    mean[j] = p.save_mean[c];
    istd[j] = p.save_invstd[c];
    sc[j] = p.gamma[c] * istd[j];
    sh[j] = p.beta[c] - mean[j] * sc[j];
    ag[j] = ab[j] = 0.f;
  }
  const long long outP = bn_bwd_positions<POOL, ODD>(p);
  for (long long op = blockIdx.x * (long long)blockDim.y + threadIdx.y; op < outP; op += (long long)gridDim.x * blockDim.y) {
    float yv[NP][8], dz[NP][8];
    long long ip[NP];
    if constexpr (ODD) bn_dz_odd<T>(p, op, g, sc, sh, yv, dz, ip);
    else bn_dz<POOL, T>(p, op, g, sc, sh, yv, dz, ip);
#pragma unroll
    for (int q = 0; q < NP; ++q)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        ab[j] += dz[q][j];
        ag[j] += dz[q][j] * (yv[q][j] - mean[j]) * istd[j];
      }
  }
  extern __shared__ float s_red[];            // [2][C]
  for (int i = threadIdx.y * blockDim.x + threadIdx.x; i < 2 * p.C; i += blockDim.x * blockDim.y) s_red[i] = 0.f;
  __syncthreads();
  for (int r = 0; r < static_cast<int>(blockDim.y); ++r) {     // rows in order: a reproducible sum
    if (threadIdx.y == r) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        s_red[g * 8 + j] += ag[j];
        s_red[p.C + g * 8 + j] += ab[j];
      }
    }
    __syncthreads();
  }
  det_commit<-1>(p.det, 0, blockIdx.x, gridDim.x, s_red, 2 * p.C, p.dgamma, p.C, p.dbeta,
                 threadIdx.y * blockDim.x + threadIdx.x, blockDim.x * blockDim.y);
}

// pass 2: dy = gamma*invstd*(dz - dbeta/P - xhat*dgamma/P)
template <bool POOL, typename T, bool ODD = false>
__global__ void __launch_bounds__(256) bn_bwd_apply_kernel(const BnBwdParams<T> p) {
  pdl_trigger();
  pdl_wait();
  constexpr int NP = POOL ? 4 : 1;
  const int g = threadIdx.x;
  const float invP = 1.f / static_cast<float>(p.P);
  float sc[8], sh[8], mean[8], istd[8], k1[8], k2[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = g * 8 + j;
    if (p.identity) { mean[j] = 0.f; istd[j] = 1.f; sc[j] = 1.f; sh[j] = 0.f; k1[j] = 0.f; k2[j] = 0.f; continue; }
    mean[j] = p.save_mean[c];
    istd[j] = p.save_invstd[c];
    sc[j] = p.gamma[c] * istd[j];
    sh[j] = p.beta[c] - mean[j] * sc[j];
    k1[j] = p.dbeta[c] * invP;
    k2[j] = p.dgamma[c] * invP;
  }
  const long long outP = bn_bwd_positions<POOL, ODD>(p);
  for (long long op = blockIdx.x * (long long)blockDim.y + threadIdx.y; op < outP; op += (long long)gridDim.x * blockDim.y) {
    float yv[NP][8], dz[NP][8];
    long long ip[NP];
    if constexpr (ODD) bn_dz_odd<T>(p, op, g, sc, sh, yv, dz, ip);
    else bn_dz<POOL, T>(p, op, g, sc, sh, yv, dz, ip);
#pragma unroll
    for (int q = 0; q < NP; ++q) {
      if constexpr (ODD) { if (ip[q] < 0) continue; }
      float r[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float xhat = (yv[q][j] - mean[j]) * istd[j];
        r[j] = sc[j] * (dz[q][j] - k1[j] - xhat * k2[j]);
      }
      store8(p.dy + ip[q] * p.C + g * 8, r);
    }
  }
}

// Single-launch BatchNorm backward for small feature maps (P <= 4096 pixels: the 8x8 / 4x4 / 2x2 layers of VGG at
// microbatch 32).  BatchNorm statistics are per channel, so a block that owns 8 channels and walks *all* pixels needs no
// cross-block reduction at all: pass 1 (dgamma, dbeta) -> block reduction -> pass 2 (dy), one launch instead of the
// reduce + apply pair (whose second kernel re-reads what the first just read, after a kernel boundary).  The re-read of
// pass 2 hits L1/L2.  Threads read 32-byte sectors (8 fp32 channels) — full sector efficiency.
template <bool POOL, typename T, bool ODD = false>
__global__ void __launch_bounds__(256) bn_bwd_chan_kernel(const BnBwdParams<T> p) {
  pdl_trigger();
  pdl_wait();
  constexpr int NP = POOL ? 4 : 1;
  const int g = blockIdx.x;                         // channel group of 8
  float sc[8], sh[8], mean[8], istd[8], ag[8], ab[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = g * 8 + j;
    mean[j] = p.save_mean[c];
    istd[j] = p.save_invstd[c];
    sc[j] = p.gamma[c] * istd[j];
    sh[j] = p.beta[c] - mean[j] * sc[j];
    ag[j] = ab[j] = 0.f;
  }
  const int outP = ODD ? static_cast<int>(bn_bwd_positions<POOL, ODD>(p)) : (POOL ? p.P >> 2 : p.P);
  for (int op = threadIdx.x; op < outP; op += blockDim.x) {
    float yv[NP][8], dz[NP][8];
    long long ip[NP];
    if constexpr (ODD) bn_dz_odd<T>(p, op, g, sc, sh, yv, dz, ip);
    else bn_dz<POOL, T>(p, op, g, sc, sh, yv, dz, ip);
#pragma unroll
    for (int q = 0; q < NP; ++q)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        ab[j] += dz[q][j];
        ag[j] += dz[q][j] * (yv[q][j] - mean[j]) * istd[j];
      }
  }
  __shared__ float s_part[8][16];                   // [warp][dgamma 8 | dbeta 8]
  __shared__ float s_tot[16];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      ag[j] += __shfl_xor_sync(0xffffffffu, ag[j], o);
      ab[j] += __shfl_xor_sync(0xffffffffu, ab[j], o);
    }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
#pragma unroll
    for (int j = 0; j < 8; ++j) { s_part[warp][j] = ag[j]; s_part[warp][8 + j] = ab[j]; }
  }
  __syncthreads();
  if (threadIdx.x < 16) {
    float t = 0.f;
    for (int w = 0; w < (blockDim.x >> 5); ++w) t += s_part[w][threadIdx.x];
    s_tot[threadIdx.x] = t;
    float* dst = threadIdx.x < 8 ? p.dgamma + g * 8 + threadIdx.x : p.dbeta + g * 8 + (threadIdx.x - 8);
    *dst += t;                                      // this block is the only writer of its channels (buffers pre-zeroed / accumulated)
  }
  __syncthreads();
  const float invP = 1.f / static_cast<float>(p.P);
  float k1[8], k2[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { k2[j] = s_tot[j] * invP; k1[j] = s_tot[8 + j] * invP; }
  for (int op = threadIdx.x; op < outP; op += blockDim.x) {
    float yv[NP][8], dz[NP][8];
    long long ip[NP];
    if constexpr (ODD) bn_dz_odd<T>(p, op, g, sc, sh, yv, dz, ip);
    else bn_dz<POOL, T>(p, op, g, sc, sh, yv, dz, ip);
#pragma unroll
    for (int q = 0; q < NP; ++q) {
      if constexpr (ODD) { if (ip[q] < 0) continue; }
      float r[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float xhat = (yv[q][j] - mean[j]) * istd[j];
        r[j] = sc[j] * (dz[q][j] - k1[j] - xhat * k2[j]);
      }
      store8(p.dy + ip[q] * p.C + g * 8, r);
    }
  }
}

// Single-launch BatchNorm backward: reduce (dgamma, dbeta) -> software grid barrier -> apply.  Every block of the grid
// is co-resident (<= 296 blocks of 256 threads, a few KB of smem: 8 fit per SM), so the barrier cannot dead-lock; kernels
// of other streams that may share the SMs always terminate on their own.  grid_bar: [0] arrivals (monotonic),
// [1] generation, [2] finish ticket — owned by one call site, zero-initialised.
template <bool POOL, typename T>
__global__ void __launch_bounds__(256, 2) bn_bwd_fused_kernel(const BnBwdParams<T> p, uint32_t* grid_bar) {
  pdl_trigger();
  pdl_wait();
  constexpr int NP = POOL ? 4 : 1;
  const int g = threadIdx.x;
  const bool leader = threadIdx.x == 0 && threadIdx.y == 0;
  const uint32_t G = gridDim.x;
  uint32_t gen = 0;
  if (leader) gen = ld_acquire_gpu(grid_bar + 1);
  float sc[8], sh[8], mean[8], istd[8], ag[8], ab[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = g * 8 + j;
    mean[j] = p.save_mean[c];
    istd[j] = p.save_invstd[c];
    sc[j] = p.gamma[c] * istd[j];
    sh[j] = p.beta[c] - mean[j] * sc[j];
    ag[j] = ab[j] = 0.f;
  }
  const long long outP = POOL ? static_cast<long long>(p.P) >> 2 : p.P;
  for (long long op = blockIdx.x * (long long)blockDim.y + threadIdx.y; op < outP; op += (long long)gridDim.x * blockDim.y) {
    float yv[NP][8], dz[NP][8];
    long long ip[NP];
    bn_dz<POOL, T>(p, op, g, sc, sh, yv, dz, ip);
#pragma unroll
    for (int q = 0; q < NP; ++q)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        ab[j] += dz[q][j];
        ag[j] += dz[q][j] * (yv[q][j] - mean[j]) * istd[j];
      }
  }
  extern __shared__ float s_red[];            // [2][C]
  for (int i = threadIdx.y * blockDim.x + threadIdx.x; i < 2 * p.C; i += blockDim.x * blockDim.y) s_red[i] = 0.f;
  __syncthreads();
  for (int r = 0; r < static_cast<int>(blockDim.y); ++r) {     // rows in order: a reproducible sum
    if (threadIdx.y == r) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        s_red[g * 8 + j] += ag[j];
        s_red[p.C + g * 8 + j] += ab[j];
      }
    }
    __syncthreads();
  }
  det_commit<-1>(p.det, 0, blockIdx.x, gridDim.x, s_red, 2 * p.C, p.dgamma, p.C, p.dbeta,
                 threadIdx.y * blockDim.x + threadIdx.x, blockDim.x * blockDim.y);
  // ---- grid barrier ----
  __syncthreads();
  if (leader) {
    __threadfence();
    atomicAdd(grid_bar, 1u);
    const uint32_t target = (gen + 1u) * G;
    uint32_t spins = 0;
    while (static_cast<int32_t>(ld_acquire_gpu(grid_bar) - target) < 0) {
      __nanosleep(32);
      if (++spins > (1u << 26)) { printf("slb: bn_bwd grid barrier timeout\n"); __trap(); }
    }
  }
  __syncthreads();
  // ---- apply ----
  const float invP = 1.f / static_cast<float>(p.P);
  float k1[8], k2[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    k1[j] = __ldcg(p.dbeta + g * 8 + j) * invP;
    k2[j] = __ldcg(p.dgamma + g * 8 + j) * invP;
  }
  for (long long op = blockIdx.x * (long long)blockDim.y + threadIdx.y; op < outP; op += (long long)gridDim.x * blockDim.y) {
    float yv[NP][8], dz[NP][8];
    long long ip[NP];
    bn_dz<POOL, T>(p, op, g, sc, sh, yv, dz, ip);
#pragma unroll
    for (int q = 0; q < NP; ++q) {
      float r[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float xhat = (yv[q][j] - mean[j]) * istd[j];
        r[j] = sc[j] * (dz[q][j] - k1[j] - xhat * k2[j]);
      }
      store8(p.dy + ip[q] * p.C + g * 8, r);
    }
  }
  __syncthreads();
  if (leader) {
    const uint32_t tk = atomicAdd(grid_bar + 2, 1u);
    if (tk == G - 1u) {
      grid_bar[2] = 0;
      __threadfence();
      atomicExch(grid_bar + 1, gen + 1u);
    }
  }
}

// Column sums / sums of squares of an activation-typed [P][C] matrix (BN statistics fallback, bias gradients).
template <typename T>
__global__ void __launch_bounds__(256) col_stats_kernel(const T* y, float* sum, float* sumsq, long long P, int C, const Det det) {
  pdl_trigger();
  pdl_wait();
  const int g = threadIdx.x;
  float a[8], b[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) a[j] = b[j] = 0.f;
  for (long long r = blockIdx.x * (long long)blockDim.y + threadIdx.y; r < P; r += (long long)gridDim.x * blockDim.y) {
    float f[8];
    load8(y + r * C + g * 8, f);
#pragma unroll
    for (int j = 0; j < 8; ++j) { a[j] += f[j]; b[j] += f[j] * f[j]; }
  }
  extern __shared__ float s_red[];
  for (int i = threadIdx.y * blockDim.x + threadIdx.x; i < 2 * C; i += blockDim.x * blockDim.y) s_red[i] = 0.f;
  __syncthreads();
  for (int r = 0; r < static_cast<int>(blockDim.y); ++r) {     // rows in order: a reproducible sum
    if (threadIdx.y == r) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        s_red[g * 8 + j] += a[j];
        s_red[C + g * 8 + j] += b[j];
      }
    }
    __syncthreads();
  }
  det_commit<-1>(det, 0, blockIdx.x, gridDim.x, s_red, sumsq ? 2 * C : C, sum, C, sumsq, threadIdx.y * blockDim.x + threadIdx.x,
                 blockDim.x * blockDim.y);
}

// Split-K epilogue of the wgmma conv: y = bf16(acc + bias) and the BN statistics of the rounded values
// (acc: fp32 [P][C] partial-sum buffer filled with red.add by the K-slices).  bias/y/sum may be null.
template <typename T>
__global__ void __launch_bounds__(256) conv_finalize_kernel(const float* acc, const float* bias, T* y, float* sum,
                                                           float* sumsq, long long P, int C, const Det det) {
  pdl_trigger();
  pdl_wait();
  const int g = threadIdx.x;
  float a[8], b[8], bs[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { a[j] = b[j] = 0.f; bs[j] = bias ? bias[g * 8 + j] : 0.f; }
  for (long long r = blockIdx.x * (long long)blockDim.y + threadIdx.y; r < P; r += (long long)gridDim.x * blockDim.y) {
    const float4 v0 = *reinterpret_cast<const float4*>(acc + r * C + g * 8);
    const float4 v1 = *reinterpret_cast<const float4*>(acc + r * C + g * 8 + 4);
    float f[8] = {v0.x + bs[0], v0.y + bs[1], v0.z + bs[2], v0.w + bs[3], v1.x + bs[4], v1.y + bs[5], v1.z + bs[6], v1.w + bs[7]};
    store8(y + r * C + g * 8, f);
    if (sum) {
      float q[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) q[j] = to_f32(from_f32<T>(f[j]));      // statistics of the stored values
#pragma unroll
      for (int j = 0; j < 8; ++j) { a[j] += q[j]; b[j] += q[j] * q[j]; }
    }
  }
  if (sum == nullptr) return;
  extern __shared__ float s_red[];
  for (int i = threadIdx.y * blockDim.x + threadIdx.x; i < 2 * C; i += blockDim.x * blockDim.y) s_red[i] = 0.f;
  __syncthreads();
  for (int r = 0; r < static_cast<int>(blockDim.y); ++r) {     // rows in order: a reproducible sum
    if (threadIdx.y == r) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        s_red[g * 8 + j] += a[j];
        s_red[C + g * 8 + j] += b[j];
      }
    }
    __syncthreads();
  }
  det_commit<-1>(det, 0, blockIdx.x, gridDim.x, s_red, 2 * C, sum, C, sumsq, threadIdx.y * blockDim.x + threadIdx.x,
                 blockDim.x * blockDim.y);
}

// ============================================================================ first-layer direct conv (Cin <= 4)
// x: fp32 NCHW [B][Cin][H][W]; w: fp32 [Cout][3][3][Cin]; y: bf16 NHWC [B][H][W][Cout] (pre-BN) + BN statistics.
// One thread = one output pixel, all COUT channels in registers; weights are warp-broadcast smem reads; the BN
// statistics are reduced across the 32 pixels of a warp with the register butterfly, then smem, then one red per CTA.
__device__ __forceinline__ float warp_col_reduce32e(float (&v)[32]) {
  const uint32_t lane = threadIdx.x & 31;
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) {
    const bool upper = (lane & off) != 0;
#pragma unroll
    for (int i = 0; i < off; ++i) {
      const float send = upper ? v[i] : v[i + off];
      const float keep = upper ? v[i + off] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
    }
  }
  return v[0];
}

template <int CIN, int COUT, typename T>
__global__ void __launch_bounds__(128) conv3x3_small_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                               const float* __restrict__ bias, T* y,
                                                               float* sum, float* sumsq, int B, int H, int W, const Det det) {
  pdl_trigger();
  pdl_wait();
  constexpr int KK = 9 * CIN;
  __shared__ float s_w[COUT * KK];
  __shared__ float s_b[COUT];
  __shared__ float s_st[2 * COUT];
  for (int i = threadIdx.x; i < COUT * KK; i += blockDim.x) s_w[i] = w[i];
  for (int i = threadIdx.x; i < COUT; i += blockDim.x) { s_b[i] = bias ? bias[i] : 0.f; s_st[i] = 0.f; s_st[COUT + i] = 0.f; }
  __syncthreads();
  const long long P = (long long)B * H * W;
  const long long pix = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const bool ok = pix < P;
  float patch[KK];
  if (ok) {
    const int ww = static_cast<int>(pix % W);
    const int hh = static_cast<int>((pix / W) % H);
    const long long b = pix / ((long long)W * H);
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const int ih = hh + t / 3 - 1, iw = ww + t % 3 - 1;
      const bool in = ih >= 0 && ih < H && iw >= 0 && iw < W;
#pragma unroll
      for (int c = 0; c < CIN; ++c) patch[t * CIN + c] = in ? __ldg(x + ((b * CIN + c) * H + ih) * W + iw) : 0.f;
    }
  } else {
#pragma unroll
    for (int k = 0; k < KK; ++k) patch[k] = 0.f;
  }
#pragma unroll 1
  for (int c0 = 0; c0 < COUT; c0 += 32) {
    float acc[32];
#pragma unroll
    for (int o = 0; o < 32; ++o) {
      const float* wr = s_w + (c0 + o) * KK;
      float a = s_b[c0 + o];
#pragma unroll
      for (int k = 0; k < KK; ++k) a = fmaf(patch[k], wr[k], a);
      acc[o] = a;
    }
    if (ok) store_row32(y + pix * COUT + c0, acc);
    if (sum) {
      float s1[32], s2[32];
#pragma unroll
      for (int o = 0; o < 32; ++o) {
        const float r = ok ? stored_value(acc[o], static_cast<const T*>(nullptr)) : 0.f;
        s1[o] = r;
        s2[o] = r * r;
      }
      const float c1 = warp_col_reduce32e(s1);
      const float c2 = warp_col_reduce32e(s2);
      for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w) {   // warps in order: a reproducible sum
        if ((threadIdx.x >> 5) == w) {
          s_st[c0 + (threadIdx.x & 31)] += c1;
          s_st[COUT + c0 + (threadIdx.x & 31)] += c2;
        }
        __syncthreads();
      }
    }
  }
  if (sum) det_commit<-1>(det, 0, blockIdx.x, gridDim.x, s_st, 2 * COUT, sum, COUT, sumsq, threadIdx.x, blockDim.x);
}

// dw[Cout][9*CIN] += sum_pix dy[pix][Cout] * patch[pix][9*CIN]  (first conv of the network: CIN = 3 or 1, Cout <= 64).
// A [Cout x KK] x [pix] GEMM with K = all pixels.  Per 128-pixel chunk the block stages the im2col patch [128][KP] and dy
// [128][Cout] in shared memory; thread (slice, cg, kg) owns a 4 (channels) x KG (taps) register tile and walks the pixels
// of its slice: one LDS.128 of dy + KG scalar patch loads feed 4*KG FMAs (the previous one-output-per-thread version
// issued two shared loads per FMA and ran at the LDS limit: 140 us for conv1 of VGG16 at batch 32).  Partial tiles of
// the pixel slices are combined with shared-memory atomics, then one global red per output and block.
template <int CIN, typename T>
__global__ void __launch_bounds__(256) conv3x3_small_wgrad_kernel(const float* __restrict__ x, const T* __restrict__ dy,
                                                                 float* dw, int B, int H, int W, int Cout, const Det det) {
  pdl_trigger();
  pdl_wait();
  constexpr int KK = 9 * CIN;
  constexpr int KG = (KK + 3) / 4;                // taps per thread (4 tap groups)
  constexpr int KP = 4 * KG;                      // padded patch row
  extern __shared__ float s_buf[];                // patch[128][KP] | dy[128][Cout] | out[Cout][KP]
  float* s_patch = s_buf;
  float* s_dy = s_buf + 128 * KP;
  float* s_out = s_dy + 128 * Cout;
  const int P = B * H * W;
  const int HW = H * W;
  const int n_cg = Cout / 4;                      // channel groups of 4
  const int lanes = n_cg * 4;                     // threads that cover every output once
  const int slices = 256 / lanes;                 // pixel slices processed in parallel (Cout = 64 -> 4)
  const int slice = threadIdx.x / lanes, within = threadIdx.x % lanes;
  const int cg = within >> 2, kg = within & 3;
  const bool active = slice < slices;
  float acc[4][KG];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int j = 0; j < KG; ++j) acc[a][j] = 0.f;
  for (int i = threadIdx.x; i < Cout * KP; i += blockDim.x) s_out[i] = 0.f;
  for (int pix0 = blockIdx.x * 128; pix0 < P; pix0 += gridDim.x * 128) {
    __syncthreads();
    for (int i = threadIdx.x; i < 128 * KP; i += blockDim.x) {
      const int lp = i / KP, k = i - lp * KP;
      const int pix = pix0 + lp;
      float v = 0.f;
      if (pix < P && k < KK) {
        const int t = k / CIN, c = k - t * CIN;
        const int b = pix / HW, r = pix - b * HW;
        const int hh = r / W, ww = r - hh * W;
        const int ih = hh + t / 3 - 1, iw = ww + t % 3 - 1;
        if (ih >= 0 && ih < H && iw >= 0 && iw < W) v = x[((b * CIN + c) * H + ih) * W + iw];
      }
      s_patch[i] = v;
    }
    for (int i = threadIdx.x; i < 128 * Cout; i += blockDim.x) {
      const int pix = pix0 + i / Cout;
      s_dy[i] = pix < P ? to_f32(dy[(long long)pix * Cout + (i % Cout)]) : 0.f;
    }
    __syncthreads();
    if (active) {
      for (int lp = slice; lp < 128; lp += slices) {
        const float4 d = *reinterpret_cast<const float4*>(s_dy + lp * Cout + cg * 4);
        const float* pr = s_patch + lp * KP + kg * KG;
#pragma unroll
        for (int j = 0; j < KG; ++j) {
          const float pv = pr[j];
          acc[0][j] = fmaf(d.x, pv, acc[0][j]);
          acc[1][j] = fmaf(d.y, pv, acc[1][j]);
          acc[2][j] = fmaf(d.z, pv, acc[2][j]);
          acc[3][j] = fmaf(d.w, pv, acc[3][j]);
        }
      }
    }
  }
  for (int sl = 0; sl < slices; ++sl) {                           // pixel slices in order: a reproducible sum
    if (active && slice == sl) {
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int j = 0; j < KG; ++j) s_out[(cg * 4 + a) * KP + kg * KG + j] += acc[a][j];
    }
    __syncthreads();
  }
  for (int i = threadIdx.x; i < Cout * KK; i += blockDim.x) s_patch[i] = s_out[(i / KK) * KP + i % KK];   // drop the padding
  __syncthreads();
  det_commit<-1>(det, 0, blockIdx.x, gridDim.x, s_patch, Cout * KK, dw, Cout * KK, nullptr, threadIdx.x, blockDim.x);
}

// ============================================================================ Linear finalisation
__device__ __forceinline__ uint32_t hash_u32(uint32_t a, uint32_t b, uint32_t c) {
  uint32_t h = a * 0x9E3779B1u ^ (b + 0x7F4A7C15u) * 0x85EBCA77u ^ (c + 0x165667B1u) * 0xC2B2AE3Du;
  h ^= h >> 16; h *= 0x7FEB352Du; h ^= h >> 15; h *= 0x846CA68Bu; h ^= h >> 16;
  return h;
}
// Value i of a sliced fp32 Linear result (linear_fwd_f32 / linear_dgrad_f32): +0 plus the `parts` slice partials
// p[i + z * stride] in slice order, each added with add.rn.ftz — the arithmetic of red.global.add.f32 into a zeroed buffer
// in slice order, so the sum is the same every run without the slices waiting for one another.  parts == 0: p[i] is final.
__device__ __forceinline__ float slice_sum(const float* p, long long stride, int parts, long long i) {
  if (parts == 0) return p[i];
  float s = 0.f;
#pragma unroll 8
  for (int z = 0; z < parts; ++z) {
    const float v = p[i + z * stride];
    asm("add.rn.ftz.f32 %0, %0, %1;" : "+f"(s) : "f"(v));
  }
  return s;
}

// out[b][n] = dropout(relu(acc[b][n] + bias[n]))  -> activation type (ld = ldo) ; also keeps fp32 logits when out_f32 != null
// acc: `parts` slice partials [parts][B][N] (slice_sum)
template <typename T>
__global__ void linear_finalize_kernel(const float* acc, int parts, const float* bias, T* out, float* out_f32, uint8_t* mask,
                                       int B, int N, int ldo, int relu, float drop_p, uint32_t seed, const uint32_t* step_ptr) {
  pdl_trigger();
  pdl_wait();
  const uint32_t step = step_ptr ? *step_ptr : 0u;
  const long long total = (long long)B * N;
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  const uint32_t thresh = static_cast<uint32_t>(drop_p * 4294967296.0);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int n = static_cast<int>(i % N), b = static_cast<int>(i / N);
    float v = slice_sum(acc, total, parts, i) + (bias ? bias[n] : 0.f);
    if (relu) v = fmaxf(v, 0.f);
    if (drop_p > 0.f) {
      const bool keep = hash_u32(seed, step, static_cast<uint32_t>(i)) >= thresh;
      mask[i] = keep ? 1 : 0;
      v = keep ? v * keep_scale : 0.f;
    }
    if (out) out[(long long)b * ldo + n] = from_f32<T>(v);
    if (out_f32) out_f32[i] = v;
  }
}
// dz[b][n] = dy[b][n] * dropmask * (relu ? y>0 : 1)  (bf16, ld = ldz) ; db[n] = sum_b dz[b][n] (bf16-rounded values)
// blockDim = (32 columns, 8 row groups): rows are split over threadIdx.y, the bias gradient is combined in smem
template <typename T>
__global__ void __launch_bounds__(256) linear_bwd_prep_kernel(const float* dacc, int parts, const T* yout, const uint8_t* mask,
                                                             T* dz, float* dbias, int B, int N, int ldy, int ldz,
                                                             int relu, float drop_p) {
  pdl_trigger();
  pdl_wait();
  __shared__ float s_part[8][33];
  const int n = blockIdx.x * 32 + threadIdx.x;
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  float s = 0.f;
  if (n < N) {
    for (int b = threadIdx.y; b < B; b += 8) {
      float g = slice_sum(dacc, (long long)B * N, parts, (long long)b * N + n);
      if (drop_p > 0.f) g = mask[(long long)b * N + n] ? g * keep_scale : 0.f;
      if (relu && !(to_f32(yout[(long long)b * ldy + n]) > 0.f)) g = 0.f;
      const T r = from_f32<T>(g);
      dz[(long long)b * ldz + n] = r;
      s += to_f32(r);
    }
  }
  s_part[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && n < N && dbias) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += s_part[k][threadIdx.x];
    dbias[n] = t;
  }
}
// dropout on a dense activation (VGG layer 46) and its backward
template <typename T>
__global__ void dropout_fwd_kernel(const T* x, T* y, uint8_t* mask, long long n, float p, uint32_t seed,
                                   const uint32_t* step_ptr) {
  pdl_trigger();
  pdl_wait();
  const uint32_t step = step_ptr ? *step_ptr : 0u;
  const float ks = 1.f / (1.f - p);
  const uint32_t thresh = static_cast<uint32_t>(p * 4294967296.0);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const bool keep = hash_u32(seed, step, static_cast<uint32_t>(i)) >= thresh;
    mask[i] = keep ? 1 : 0;
    y[i] = from_f32<T>(keep ? to_f32(x[i]) * ks : 0.f);
  }
}
template <typename T>
__global__ void dropout_bwd_kernel(const float* dacc, int parts, const uint8_t* mask, T* dx, long long n, float p) {
  pdl_trigger();
  pdl_wait();
  const float ks = 1.f / (1.f - p);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    dx[i] = from_f32<T>((mask == nullptr || mask[i]) ? slice_sum(dacc, n, parts, i) * (mask ? ks : 1.f) : 0.f);
}


// ============================================================================ fp32 Linear on the CUDA cores (parity mode)
// The reference runs nn.Linear as a plain fp32 cuBLAS GEMM (PyTorch keeps TF32 off for matmuls, SURVEY §2.7 note), so
// the parity mode computes the classifier with IEEE fp32 FMAs.  At microbatch 32 these layers are weight-streaming ops
// (16 FLOP per weight byte): the kernels below read every weight exactly once with 16-byte coalesced loads and keep the
// whole batch tile in registers / shared memory.

// Two batch rows per accumulator pair: f32x2 packs (row 2bp, row 2bp + 1); ffma2 is two IEEE round-to-nearest fp32 FMAs
// (sm_90 has no packed fp32 FMA instruction, so it is two FFMAs).
// Ampere-style asynchronous copies (LDGSTS): the weight stream of the fp32 Linear kernels is staged through a ring of
// shared-memory stages so that several steps of HBM traffic are in flight per SM without holding registers (ncu on the
// register-prefetch version: 22 % of the stall samples on the first use of the prefetched weights, DRAM at 13 % of peak).
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

typedef unsigned long long f32x2;
__device__ __forceinline__ f32x2 pack2(float lo, float hi) {
  f32x2 r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
  return r;
}
__device__ __forceinline__ void unpack2(f32x2 v, float& lo, float& hi) { asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v)); }
__device__ __forceinline__ f32x2 ffma2(f32x2 a, f32x2 b, f32x2 c) {
  float a0, a1, b0, b1, c0, c1;
  unpack2(a, a0, a1);
  unpack2(b, b0, b1);
  unpack2(c, c0, c1);
  return pack2(fmaf(a0, b0, c0), fmaf(a1, b1, c1));
}

// part[s][b][n] = sum_{k in slice s} x[b][k] * w[n][k]          grid (ceil(N/32), ceil(K/kc), ceil(B/32)), 256 threads
// warp = (feature group of 8) x (batch half of 16); lanes stride K in float4 steps; partial sums are reduced across the
// warp with the register butterfly and stored as slice s's partial (the consumer adds the slices in order: slice_sum).
__global__ void __launch_bounds__(256) linear_fwd_f32_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                            float* part, int B, int N, int K, int ldx, int ldw, int kc) {
  pdl_trigger();
  pdl_wait();
  constexpr int ST = 4;                                          // weight stages in flight (16 KB each)
  // x of the current step, transposed for the packed FMAs: [j = k % 4][lane = k / 4][b], lane stride padded to 36 floats
  // (16-byte loads of 4 consecutive batch rows by the 32 lanes of a warp hit 8 distinct bank groups per phase)
  __shared__ __align__(16) float s_x[4 * 32 * 36];
  extern __shared__ __align__(16) float s_w[];                   // [ST][32 features][128 k]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int fg = warp >> 1, bh = warp & 1;
  const int n0 = blockIdx.x * 32 + fg * 8;
  const int k_begin = blockIdx.y * kc, k_end = min(K, k_begin + kc);
  const int b0 = blockIdx.z * 32;
  f32x2 ac2[8][8];                                               // [feature][batch pair of this warp's half]
#pragma unroll
  for (int f = 0; f < 8; ++f)
#pragma unroll
    for (int bp = 0; bp < 8; ++bp) ac2[f][bp] = 0ull;
  const int steps = (k_end - k_begin + 127) / 128;
  float4 xr[4];
  auto fetch_x = [&](int step) {
    const int kb = k_begin + step * 128;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int e = threadIdx.x + i * 256, b = e >> 5, c = (e & 31) * 4;
      xr[i] = (b0 + b < B && kb + c < k_end) ? __ldg(reinterpret_cast<const float4*>(x + (long long)(b0 + b) * ldx + kb + c))
                                             : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto issue_w = [&](int step) {                                 // 32 rows x 128 k = 1024 float4: four per thread
    if (step < steps) {
      const int kb = k_begin + step * 128;
      float* dst = s_w + (step % ST) * 32 * 128;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int e = threadIdx.x + i * 256, r = e >> 5, c = (e & 31) * 4;
        const int n = blockIdx.x * 32 + r;
        if (n < N && kb + c < k_end) cp_async16(dst + r * 128 + c, w + (long long)n * ldw + kb + c);
        else *reinterpret_cast<float4*>(dst + r * 128 + c) = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    cp_async_commit();                                           // one group per step, also when empty: uniform counting
  };
#pragma unroll
  for (int s0 = 0; s0 < ST - 1; ++s0) issue_w(s0);
  if (steps > 0) fetch_x(0);
  for (int step = 0; step < steps; ++step) {
    cp_async_wait<ST - 2>();                                     // this thread's copies of stage `step` have landed
    __syncthreads();                                             // ... everybody's have; previous step's readers are done
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int e = threadIdx.x + i * 256, b = e >> 5, c4 = e & 31;
      s_x[(0 * 32 + c4) * 36 + b] = xr[i].x;
      s_x[(1 * 32 + c4) * 36 + b] = xr[i].y;
      s_x[(2 * 32 + c4) * 36 + b] = xr[i].z;
      s_x[(3 * 32 + c4) * 36 + b] = xr[i].w;
    }
    issue_w(step + ST - 1);                                      // refills the stage that was read during step - 1
    float4 wc[8];
    const float* ws = s_w + ((step % ST) * 32 + fg * 8) * 128 + 4 * lane;
#pragma unroll
    for (int f = 0; f < 8; ++f) wc[f] = *reinterpret_cast<const float4*>(ws + f * 128);
    __syncthreads();
    if (step + 1 < steps) fetch_x(step + 1);                     // x is L2-resident: one step of register prefetch suffices
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      f32x2 xp[8];
      const float* row = s_x + (j * 32 + lane) * 36 + bh * 16;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const ulonglong2 v = *reinterpret_cast<const ulonglong2*>(row + q * 4);
        xp[2 * q] = v.x;
        xp[2 * q + 1] = v.y;
      }
#pragma unroll
      for (int f = 0; f < 8; ++f) {
        const float wv = j == 0 ? wc[f].x : (j == 1 ? wc[f].y : (j == 2 ? wc[f].z : wc[f].w));
        const f32x2 wp = pack2(wv, wv);
#pragma unroll
        for (int bp = 0; bp < 8; ++bp) ac2[f][bp] = ffma2(wp, xp[bp], ac2[f][bp]);
      }
    }
  }
  cp_async_wait<0>();
  float a[4][32];
#pragma unroll
  for (int f = 0; f < 8; ++f)
#pragma unroll
    for (int bp = 0; bp < 8; ++bp) unpack2(ac2[f][bp], a[f >> 1][(f & 1) * 16 + 2 * bp], a[f >> 1][(f & 1) * 16 + 2 * bp + 1]);
  float v[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) v[q] = warp_col_reduce32e(a[q]);  // lane j: sum over lanes of a[q][j]
  float* ps = part + (long long)blockIdx.y * B * N;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int f = 2 * q + (lane >> 4), b = b0 + bh * 16 + (lane & 15);
    if (n0 + f < N && b < B) ps[(long long)b * N + n0 + f] = v[q];
  }
}

// part[s][b][k] = sum_{n in slice s} dz[b][n] * w[n][k]         grid (ceil(K/(4*T)), ceil(N/nc), ceil(B/32)), T threads
// a thread owns 4 consecutive k for the whole batch tile (128 accumulators); the dz slice sits in shared memory as
// [n][32 b] and is read with warp-broadcast 16-byte loads; weights stream through with coalesced float4 loads.
// The consumer adds the slices in order (slice_sum).
__global__ void __launch_bounds__(128) linear_dgrad_f32_kernel(const float* __restrict__ dz, const float* __restrict__ w, float* part,
                                                              int B, int N, int K, int lddz, int ldw, int nc) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ __align__(16) float s_dz[];                  // [nc][32]
  const int n_begin = blockIdx.y * nc, n_cnt = min(nc, N - n_begin);
  const int b0 = blockIdx.z * 32;
  const int k0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  for (int i = threadIdx.x; i < nc * 32; i += blockDim.x) {
    const int nn = i >> 5, b = i & 31;
    s_dz[i] = (nn < n_cnt && b0 + b < B) ? dz[(long long)(b0 + b) * lddz + n_begin + nn] : 0.f;
  }
  __syncthreads();
  if (k0 >= K) return;
  f32x2 acc[16][4];                                              // [batch pair][k]: (row 2bp, row 2bp+1)
#pragma unroll
  for (int bp = 0; bp < 16; ++bp) { acc[bp][0] = acc[bp][1] = acc[bp][2] = acc[bp][3] = 0ull; }
  // weights: every thread streams its own 16-byte column segment of the rows n through a private ring in shared memory
  // (DST stages of 4 rows): DST * 64 bytes in flight per thread instead of one 4-row register group
  constexpr int DST = 6;
  float* s_ring = s_dz + nc * 32;                                // [DST][4 rows][blockDim.x] float4
  const float* wp = w + (long long)n_begin * ldw + k0;
  const int groups = (n_cnt + 3) / 4;
  auto issue = [&](int g) {
    if (g < groups) {
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        float* dst = s_ring + (((g % DST) * 4 + u) * blockDim.x + threadIdx.x) * 4;
        if (g * 4 + u < n_cnt) cp_async16(dst, wp + (long long)(g * 4 + u) * ldw);
        else *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    cp_async_commit();
  };
#pragma unroll
  for (int g = 0; g < DST - 1; ++g) issue(g);
  for (int g = 0; g < groups; ++g) {
    cp_async_wait<DST - 2>();                                    // my own copies of group g have landed (nobody else reads them)
    float4 wv[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) wv[u] = *reinterpret_cast<const float4*>(s_ring + (((g % DST) * 4 + u) * blockDim.x + threadIdx.x) * 4);
    issue(g + DST - 1);                                          // the slot of group g - 1: its values are in registers / consumed
    const int nn = g * 4;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const f32x2 w0 = pack2(wv[u].x, wv[u].x), w1 = pack2(wv[u].y, wv[u].y), w2 = pack2(wv[u].z, wv[u].z), w3 = pack2(wv[u].w, wv[u].w);
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const ulonglong2 d = *reinterpret_cast<const ulonglong2*>(s_dz + (nn + u) * 32 + q * 4);   // rows 4q..4q+3 (warp broadcast)
        acc[2 * q][0] = ffma2(d.x, w0, acc[2 * q][0]); acc[2 * q][1] = ffma2(d.x, w1, acc[2 * q][1]);
        acc[2 * q][2] = ffma2(d.x, w2, acc[2 * q][2]); acc[2 * q][3] = ffma2(d.x, w3, acc[2 * q][3]);
        acc[2 * q + 1][0] = ffma2(d.y, w0, acc[2 * q + 1][0]); acc[2 * q + 1][1] = ffma2(d.y, w1, acc[2 * q + 1][1]);
        acc[2 * q + 1][2] = ffma2(d.y, w2, acc[2 * q + 1][2]); acc[2 * q + 1][3] = ffma2(d.y, w3, acc[2 * q + 1][3]);
      }
    }
  }
  cp_async_wait<0>();
  float a[32][4];
#pragma unroll
  for (int bp = 0; bp < 16; ++bp)
#pragma unroll
    for (int k = 0; k < 4; ++k) unpack2(acc[bp][k], a[2 * bp][k], a[2 * bp + 1][k]);
  float* ps = part + (long long)blockIdx.y * B * K;
#pragma unroll
  for (int b = 0; b < 32; ++b)
    if (b0 + b < B)
      *reinterpret_cast<float4*>(ps + (long long)(b0 + b) * K + k0) = make_float4(a[b][0], a[b][1], a[b][2], a[b][3]);
}

// g[n][k] = sum_b dz[b][n] * x[b][k]  (K = batch: the weight gradient is written exactly once, so the optimizer step
// rides on it).  A thread owns 4 consecutive k, keeps x[32 b][4 k] in registers and walks `nr` rows n.
//   mode 0: G[n][k]  = g          mode 1: G[n][k] += g        (plain gradient, e.g. for clip-grad-norm / batch > 32)
//   mode 2: m = mu*m + g ; p -= lr*m   — fused SGD-momentum (torch.optim.SGD semantics); G is not touched at all,
//           which removes the gradient write + the optimizer's gradient read/zero from the 134 MB classifier update.
// The bias rows of the block (gradient produced by linear_bwd_prep) are updated by the blockIdx.x == 0 column in mode 2.
__global__ void __launch_bounds__(128) linear_wgrad_f32_kernel(const float* __restrict__ dz, const float* __restrict__ x, float* G,
                                                              float* P, float* M, float* bias_p, float* bias_m, float* bias_g,
                                                              int B, int b0, int N, int K, int lddz, int ldx, int ld, int nr,
                                                              int mode, float lr, float mu) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ __align__(16) float s_dz[];                  // [nr][32]
  const int n_begin = blockIdx.y * nr, n_cnt = min(nr, N - n_begin);
  const int k0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  for (int i = threadIdx.x; i < nr * 32; i += blockDim.x) {
    const int nn = i >> 5, b = i & 31;
    s_dz[i] = (nn < n_cnt && b0 + b < B) ? dz[(long long)(b0 + b) * lddz + n_begin + nn] : 0.f;
  }
  if (mode == 2 && blockIdx.x == 0 && bias_p != nullptr && threadIdx.x < n_cnt) {
    const int n = n_begin + threadIdx.x;
    const float mb = __fadd_rn(__fmul_rn(mu, bias_m[n]), bias_g[n]);
    bias_m[n] = mb;
    bias_p[n] = __fmaf_rn(-lr, mb, bias_p[n]);
    bias_g[n] = 0.f;
  }
  __syncthreads();
  if (k0 >= K) return;
  f32x2 xp[16][4];                                               // [batch pair][k] = (x[2bp][k], x[2bp+1][k])
#pragma unroll
  for (int bp = 0; bp < 16; ++bp) {
    const float4 e = (b0 + 2 * bp < B) ? __ldg(reinterpret_cast<const float4*>(x + (long long)(b0 + 2 * bp) * ldx + k0)) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 o = (b0 + 2 * bp + 1 < B) ? __ldg(reinterpret_cast<const float4*>(x + (long long)(b0 + 2 * bp + 1) * ldx + k0)) : make_float4(0.f, 0.f, 0.f, 0.f);
    xp[bp][0] = pack2(e.x, o.x); xp[bp][1] = pack2(e.y, o.y); xp[bp][2] = pack2(e.z, o.z); xp[bp][3] = pack2(e.w, o.w);
  }
  const long long base = (long long)n_begin * ld + k0;
  float4 pc = make_float4(0.f, 0.f, 0.f, 0.f), mc = pc;
  if (mode == 2 && n_cnt > 0) { pc = *reinterpret_cast<const float4*>(P + base); mc = *reinterpret_cast<const float4*>(M + base); }
  if (mode == 1 && n_cnt > 0) pc = *reinterpret_cast<const float4*>(G + base);
  for (int nn = 0; nn < n_cnt; ++nn) {
    const long long off = base + (long long)nn * ld;
    float4 pn = pc, mn = mc;
    if (nn + 1 < n_cnt) {                                         // next row's optimizer state is in flight during the FMAs
      if (mode == 2) { pn = *reinterpret_cast<const float4*>(P + off + ld); mn = *reinterpret_cast<const float4*>(M + off + ld); }
      if (mode == 1) pn = *reinterpret_cast<const float4*>(G + off + ld);
    }
    f32x2 g2[4] = {0ull, 0ull, 0ull, 0ull};                        // (sum over even rows, sum over odd rows) per k
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const ulonglong2 d = *reinterpret_cast<const ulonglong2*>(s_dz + nn * 32 + q * 4);      // (d[4q], d[4q+1]), (d[4q+2], d[4q+3])
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        g2[k] = ffma2(d.x, xp[2 * q][k], g2[k]);
        g2[k] = ffma2(d.y, xp[2 * q + 1][k], g2[k]);
      }
    }
    float4 g;
    {
      float lo, hi;
      unpack2(g2[0], lo, hi); g.x = __fadd_rn(lo, hi);
      unpack2(g2[1], lo, hi); g.y = __fadd_rn(lo, hi);
      unpack2(g2[2], lo, hi); g.z = __fadd_rn(lo, hi);
      unpack2(g2[3], lo, hi); g.w = __fadd_rn(lo, hi);
    }
    if (mode == 2) {
      mc.x = __fadd_rn(__fmul_rn(mu, mc.x), g.x); mc.y = __fadd_rn(__fmul_rn(mu, mc.y), g.y);      // same rounding
      mc.z = __fadd_rn(__fmul_rn(mu, mc.z), g.z); mc.w = __fadd_rn(__fmul_rn(mu, mc.w), g.w);      // sequence as
      pc.x = __fmaf_rn(-lr, mc.x, pc.x); pc.y = __fmaf_rn(-lr, mc.y, pc.y);                        // sgd_momentum_kernel
      pc.z = __fmaf_rn(-lr, mc.z, pc.z); pc.w = __fmaf_rn(-lr, mc.w, pc.w);
      *reinterpret_cast<float4*>(M + off) = mc;
      *reinterpret_cast<float4*>(P + off) = pc;
    } else if (mode == 1) {
      *reinterpret_cast<float4*>(G + off) = make_float4(pc.x + g.x, pc.y + g.y, pc.z + g.z, pc.w + g.w);
    } else {
      *reinterpret_cast<float4*>(G + off) = g;
    }
    pc = pn; mc = mn;
  }
}

// sum of squares of a flat fp32 buffer (gradient norm for clip-grad-norm), accumulated into *out (zeroed by the caller)
__global__ void __launch_bounds__(256) sumsq_kernel(const float4* g, long long n4, float* out) {
  pdl_trigger();
  pdl_wait();
  float s = 0.f;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = g[i];
    s += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  __shared__ float part[8];
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += part[k];
    atomicAdd(out, t);
  }
}
// g *= min(1, max_norm / (sqrt(*sumsq) + 1e-6))   (torch.nn.utils.clip_grad_norm_)
__global__ void __launch_bounds__(256) clip_scale_kernel(float4* g, long long n4, const float* sumsq, float max_norm) {
  pdl_trigger();
  pdl_wait();
  const float c = fminf(1.f, max_norm / (sqrtf(*sumsq) + 1e-6f));
  if (c >= 1.f) return;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 v = g[i];
    v.x *= c; v.y *= c; v.z *= c; v.w *= c;
    g[i] = v;
  }
}

// ============================================================================ cross-entropy forward + backward
// one warp per sample: loss_sum += -log softmax[label] / B; dlogits = (softmax - onehot) / B  (fp32, ld = ldd)
__global__ void ce_fwd_bwd_kernel(const float* logits, const long long* labels, float* dlogits, float* loss_sum,
                                  int* nan_flag, int B, int C, int ldd, const Det det) {
  pdl_trigger();
  pdl_wait();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  __shared__ float s_loss[32];
  float loss_v = 0.f;
  if (warp < B) {
  const float* row = logits + (long long)warp * C;
  float mx = -INFINITY;
  for (int c = lane; c < C; c += 32) mx = fmaxf(mx, row[c]);
  for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float se = 0.f;
  for (int c = lane; c < C; c += 32) se += __expf(row[c] - mx);
  for (int o = 16; o; o >>= 1) se += __shfl_xor_sync(0xffffffffu, se, o);
  const int lab = static_cast<int>(labels[warp]);
  const float lse = mx + __logf(se);
  const float invB = 1.f / static_cast<float>(B);
  for (int c = lane; c < ldd; c += 32) {
    float g = 0.f;
    if (c < C) g = (__expf(row[c] - lse) - (c == lab ? 1.f : 0.f)) * invB;
    dlogits[(long long)warp * ldd + c] = g;
  }
  if (lane == 0) {
    const float loss = lse - row[lab];
    loss_v = loss * invB;
    if (loss != loss) *nan_flag = 1;
  }
  }
  if (lane == 0) s_loss[threadIdx.x >> 5] = loss_v;
  __syncthreads();
  if (threadIdx.x == 0) {                 // rows in order (blocks behind a turn counter): the same loss every run
    uint32_t* turn = det.ctr + DET_TURN_BASE;
    if (gridDim.x > 1) turn_wait(turn, blockIdx.x);
    float sum = *loss_sum;
    for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w) sum += s_loss[w];
    *loss_sum = sum;
    if (gridDim.x > 1) turn_pass(turn, blockIdx.x, gridDim.x);
  }
}

// ============================================================================ evaluation loss / accuracy
// (value, index) of a row maximum with torch.argmax's rules: a NaN beats every number, and among equal values (or NaNs)
// the smaller index wins.  idx == INT_MAX marks "no element yet".
__device__ __forceinline__ bool argmax_better(float v, int i, float best, int bi) {
  if (bi == INT_MAX) return true;
  const bool vn = v != v, bn = best != best;
  if (vn || bn) return vn && (!bn || i < bi);
  return v > best || (v == best && i < bi);
}

// One block of 8 warps, warp w takes rows w, w + 8, ...: per row the max-subtracted log-sum-exp (fp64) and the argmax.
// The batch-mean loss is added to loss_total (fp64), the correct predictions to correct and B to count.  Every sum runs
// in a fixed order, so the totals are the same bits every run.  Nothing that changes per batch is a launch argument.
__global__ void __launch_bounds__(256) eval_metrics_kernel(const float* logits, const long long* labels, int B, int C,
                                                           double* loss_total, long long* correct, long long* count) {
  pdl_trigger();
  pdl_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  __shared__ double s_loss[32];
  __shared__ long long s_hit[32];
  double wl = 0.0;
  long long wh = 0;
  for (int r = warp; r < B; r += nw) {
    const float* row = logits + (long long)r * C;
    float best = 0.f;
    int bi = INT_MAX;
    for (int c = lane; c < C; c += 32) {
      const float v = row[c];
      if (argmax_better(v, c, best, bi)) { best = v; bi = c; }
    }
    for (int o = 16; o; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (oi != INT_MAX && argmax_better(ov, oi, best, bi)) { best = ov; bi = oi; }
    }
    const double mx = static_cast<double>(best);
    double se = 0.0;
    for (int c = lane; c < C; c += 32) se += exp(static_cast<double>(row[c]) - mx);
    for (int o = 16; o; o >>= 1) se += __shfl_xor_sync(0xffffffffu, se, o);
    if (lane == 0) {
      const long long lab = labels[r];
      wl += mx + log(se) - static_cast<double>(row[lab]);
      wh += (bi == lab) ? 1 : 0;
    }
  }
  if (lane == 0) { s_loss[warp] = wl; s_hit[warp] = wh; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    long long h = 0;
    for (int w = 0; w < nw; ++w) { s += s_loss[w]; h += s_hit[w]; }
    *loss_total += s / static_cast<double>(B);
    *correct += h;
    *count += B;
  }
}

// ============================================================================ optimisers (flat)
// v = mu*v + g ; p -= lr*v ; g = 0 ; optional bf16 shadow copy of p  (torch.optim.SGD, no dampening/nesterov/wd)
__global__ void sgd_momentum_kernel(float4* p, float4* g, float4* m, uint2* p_bf16, long long n4, float lr, float mu, int first_step) {
  pdl_trigger();
  pdl_wait();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 gi = g[i];
    float4 mi = m[i], pi = p[i];
    // Rounding sequence of torch.optim.SGD (foreach): buf.mul_(mu) [rounded], buf.add_(g) [rounded], p.add_(buf, alpha=-lr)
    // [one fused multiply-add] -> the update is bitwise identical to the reference optimizer.
    if (first_step) { mi = gi; }            // torch initialises the buffer with the first gradient
    else {
      mi.x = __fadd_rn(__fmul_rn(mu, mi.x), gi.x); mi.y = __fadd_rn(__fmul_rn(mu, mi.y), gi.y);
      mi.z = __fadd_rn(__fmul_rn(mu, mi.z), gi.z); mi.w = __fadd_rn(__fmul_rn(mu, mi.w), gi.w);
    }
    pi.x = __fmaf_rn(-lr, mi.x, pi.x); pi.y = __fmaf_rn(-lr, mi.y, pi.y);
    pi.z = __fmaf_rn(-lr, mi.z, pi.z); pi.w = __fmaf_rn(-lr, mi.w, pi.w);
    m[i] = mi;
    p[i] = pi;
    g[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (p_bf16) p_bf16[i] = make_uint2(pack_bf16x2(pi.x, pi.y), pack_bf16x2(pi.z, pi.w));
  }
}
__global__ void adamw_kernel(float4* p, float4* g, float4* m, float4* v, uint2* p_bf16, long long n4, float lr, float b1, float b2,
                             float eps, float wd, float bc1, float bc2, const uint32_t* step_ptr) {
  pdl_trigger();
  pdl_wait();
  if (step_ptr != nullptr) {          // step count lives on the device: a captured graph stays valid across replays
    const float t = static_cast<float>(*step_ptr);
    bc1 = 1.f - powf(b1, t);
    bc2 = 1.f - powf(b2, t);
  }
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 gi = g[i];
    float4 mi = m[i], vi = v[i], pi = p[i];
    float* pp = reinterpret_cast<float*>(&pi);
    float* mm = reinterpret_cast<float*>(&mi);
    float* vv = reinterpret_cast<float*>(&vi);
    const float* gg = reinterpret_cast<const float*>(&gi);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      pp[k] *= (1.f - lr * wd);
      mm[k] = b1 * mm[k] + (1.f - b1) * gg[k];
      vv[k] = b2 * vv[k] + (1.f - b2) * gg[k] * gg[k];
      pp[k] -= lr * (mm[k] / bc1) / (sqrtf(vv[k] / bc2) + eps);
    }
    m[i] = mi; v[i] = vi; p[i] = pi;
    g[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (p_bf16) p_bf16[i] = make_uint2(pack_bf16x2(pi.x, pi.y), pack_bf16x2(pi.z, pi.w));
  }
}
__global__ void cast_f32_bf16_kernel(const float4* x, uint2* y, long long n4) {
  pdl_trigger();
  pdl_wait();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = x[i];
    y[i] = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
  }
}

// ============================================================================ GPU-resident image loader
// One training microbatch straight from a uint8 dataset that lives in HBM (reference recipe,
// src/dataset/dataloader.py:61-84: RandomCrop(32, padding 4) + RandomHorizontalFlip + ToTensor + Normalize):
//   out[b][c][y][x] = (img[idx[b]][y + dy[b]][x' + dx[b]][c] / 255 - mean[c]) / std[c],  x' = flip[b] ? W-1-x : x,
// zero outside the image (the padding is applied to the raw image, i.e. it normalises to -mean/std).
// data: [N][H][W][C] uint8 (torchvision's layout), out: [B][C][H][W] fp32 (the stage input).
__global__ void __launch_bounds__(256)
image_batch_kernel(const uint8_t* __restrict__ data, const long long* __restrict__ idx, const int* __restrict__ dx,
                   const int* __restrict__ dy, const int* __restrict__ flip, float* __restrict__ out, int B, int C, int H,
                   int W, float m0, float m1, float m2, float s0, float s1, float s2) {
  pdl_trigger();
  pdl_wait();
  const long long total = static_cast<long long>(B) * C * H * W;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(i % W);
    const int y = static_cast<int>((i / W) % H);
    const int c = static_cast<int>((i / (static_cast<long long>(W) * H)) % C);
    const int b = static_cast<int>(i / (static_cast<long long>(W) * H * C));
    const int sx = (flip[b] ? W - 1 - x : x) + dx[b], sy = y + dy[b];
    float v = 0.f;
    if (sx >= 0 && sx < W && sy >= 0 && sy < H)
      v = static_cast<float>(data[((idx[b] * H + sy) * W + sx) * C + c]) * (1.f / 255.f);
    const float mean = c == 0 ? m0 : (c == 1 ? m1 : m2), sd = c == 0 ? s0 : (c == 1 ? s1 : s2);
    out[i] = (v - mean) / sd;
  }
}

// ============================================================================ FedAvg n-ary weighted reduction
// out[i] = sum_r coef[r] * nan_to_num(src[r][i]) ; src pointers may be peer (NVLink) addresses.  (SURVEY G12)
struct FedAvgParams {
  const float* src[16];
  float coef[16];
  int nsrc;
};
__global__ void __launch_bounds__(512) fedavg_kernel(float4* out, uint2* out_bf16, const FedAvgParams p, long long n4) {
  pdl_trigger();
  pdl_wait();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
    for (int r = 0; r < p.nsrc; ++r) {
      const float4 v = __ldcg(reinterpret_cast<const float4*>(p.src[r]) + i);
      const float c = p.coef[r];
      acc.x += c * (v.x == v.x ? v.x : 0.f);
      acc.y += c * (v.y == v.y ? v.y : 0.f);
      acc.z += c * (v.z == v.z ? v.z : 0.f);
      acc.w += c * (v.w == v.w ? v.w : 0.f);
    }
    out[i] = acc;
    if (out_bf16) out_bf16[i] = make_uint2(pack_bf16x2(acc.x, acc.y), pack_bf16x2(acc.z, acc.w));
  }
}

static inline int grid_for(long long work, int block, int max_blocks = 132 * 8) {
  long long g = (work + block - 1) / block;
  if (g < 1) g = 1;
  if (g > max_blocks) g = max_blocks;
  return static_cast<int>(g);
}
static inline int last_err() {
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : -static_cast<int>(e) - 2000;
}

}  // namespace slb
using namespace slb;

extern "C" {

int slb_preload_elementwise() {
  using bf = __nv_bfloat16;
  cudaFuncAttributes a;
  int bad = 0;
  bad += slb_det(nullptr).part != nullptr ? 0 : 1;                // reduction scratch, before any graph capture
#define SLB_PRELOAD(k) bad += (cudaFuncGetAttributes(&a, k) != cudaSuccess)
#define SLB_PRELOAD_T(T) \
  { auto k = bn_relu_pool_fwd_kernel<T>; SLB_PRELOAD(k); } { auto k = bn_relu_pool_fwd_kernel<T, true>; SLB_PRELOAD(k); } \
  { auto k = bn_bwd_reduce_kernel<true, T>; SLB_PRELOAD(k); } { auto k = bn_bwd_reduce_kernel<false, T>; SLB_PRELOAD(k); } \
  { auto k = bn_bwd_apply_kernel<true, T>; SLB_PRELOAD(k); } { auto k = bn_bwd_apply_kernel<false, T>; SLB_PRELOAD(k); } \
  { auto k = bn_bwd_fused_kernel<true, T>; SLB_PRELOAD(k); } { auto k = bn_bwd_fused_kernel<false, T>; SLB_PRELOAD(k); } \
  { auto k = bn_bwd_chan_kernel<true, T>; SLB_PRELOAD(k); } { auto k = bn_bwd_chan_kernel<false, T>; SLB_PRELOAD(k); } \
  { auto k = bn_relu_pool_fwd_kernel<T, false, true>; SLB_PRELOAD(k); } { auto k = bn_bwd_chan_kernel<true, T, true>; SLB_PRELOAD(k); } \
  { auto k = bn_bwd_reduce_kernel<true, T, true>; SLB_PRELOAD(k); } { auto k = bn_bwd_apply_kernel<true, T, true>; SLB_PRELOAD(k); } \
  { auto k = col_stats_kernel<T>; SLB_PRELOAD(k); } { auto k = conv_finalize_kernel<T>; SLB_PRELOAD(k); } \
  { auto k = conv3x3_small_fwd_kernel<3, 64, T>; SLB_PRELOAD(k); } { auto k = conv3x3_small_fwd_kernel<1, 64, T>; SLB_PRELOAD(k); } \
  { auto k = conv3x3_small_fwd_kernel<3, 32, T>; SLB_PRELOAD(k); } { auto k = conv3x3_small_fwd_kernel<1, 32, T>; SLB_PRELOAD(k); } \
  { auto k = conv3x3_small_wgrad_kernel<3, T>; SLB_PRELOAD(k); } { auto k = conv3x3_small_wgrad_kernel<1, T>; SLB_PRELOAD(k); } \
  { auto k = linear_finalize_kernel<T>; SLB_PRELOAD(k); } { auto k = linear_bwd_prep_kernel<T>; SLB_PRELOAD(k); } \
  { auto k = dropout_fwd_kernel<T>; SLB_PRELOAD(k); } { auto k = dropout_bwd_kernel<T>; SLB_PRELOAD(k); }
  SLB_PRELOAD_T(bf)
  SLB_PRELOAD_T(float)
  SLB_PRELOAD(zero_kernel); SLB_PRELOAD(zero_wait_kernel); SLB_PRELOAD(wait_flag_kernel); SLB_PRELOAD(set_flag_kernel); SLB_PRELOAD(counter_inc_kernel);
  SLB_PRELOAD(linear_fwd_f32_kernel); SLB_PRELOAD(linear_dgrad_f32_kernel); SLB_PRELOAD(linear_wgrad_f32_kernel);
  SLB_PRELOAD(sumsq_kernel); SLB_PRELOAD(clip_scale_kernel);
  SLB_PRELOAD(ce_fwd_bwd_kernel); SLB_PRELOAD(eval_metrics_kernel); SLB_PRELOAD(sgd_momentum_kernel); SLB_PRELOAD(adamw_kernel); SLB_PRELOAD(cast_f32_bf16_kernel);
  SLB_PRELOAD(fedavg_kernel); SLB_PRELOAD(image_batch_kernel);
#undef SLB_PRELOAD_T
#undef SLB_PRELOAD
  return bad;
}

int slb_zero(void* p, long long bytes, cudaStream_t st) {
  if (bytes % 16) return -1;
  launch_k(zero_kernel, grid_for(bytes / 16, 256), 256, 0, st, reinterpret_cast<float4*>(p), bytes / 16);
  return last_err();
}
int slb_zero_wait(void* p, long long bytes, const uint32_t* flag, uint32_t* expect_ctr, unsigned long long max_spins, int* status,
                  cudaStream_t st) {
  if (bytes % 16) return -1;
  static bool carve = false;
  if (!carve) {
    cudaFuncSetAttribute(zero_wait_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    carve = true;
  }
  launch_k(zero_wait_kernel, grid_for(bytes / 16, 256, 64), 256, 0, st, reinterpret_cast<float4*>(p), bytes / 16, flag, expect_ctr,
           max_spins, status);
  return last_err();
}
int slb_wait_flag(const uint32_t* flag, uint32_t expected, uint32_t* expect_ctr, unsigned long long max_spins, int* status,
                  cudaStream_t st) {
  static bool carve = false;
  if (!carve) {   // an SM hosting this spinner should already be configured for large-smem CTAs of sibling kernels
    cudaFuncSetAttribute(wait_flag_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    carve = true;
  }
  launch_k(wait_flag_kernel, 1, 1, 0, st, flag, expected, expect_ctr, max_spins, status);
  return last_err();
}
int slb_set_flag(uint32_t* flag, uint32_t value, uint32_t* seq, uint32_t* hint, cudaStream_t st) {
  launch_k(set_flag_kernel, 1, 1, 0, st, flag, value, seq, hint);
  return last_err();
}
int slb_counter_inc(uint32_t* c, cudaStream_t st) {
  launch_k(counter_inc_kernel, 1, 1, 0, st, c);
  return last_err();
}

// dtype everywhere below: 0 = bf16 activations, 1 = fp32 activations (parity mode)
}  // extern "C"
template <typename T>
static int bn_fwd_t(const void* y, const float* sum, const float* sumsq, const float* gamma, const float* beta,
                    float* running_mean, float* running_var, long long* nbt, float* save_mean, float* save_invstd,
                    void* out, int P, int C, int H, int W, int relu, int pool, float momentum, float eps,
                    int update_running, int identity, uint32_t* ticket, uint32_t* flag, uint32_t* seq, uint32_t* hint,
                    cudaStream_t st) {
  BnFwdParams<T> p = {reinterpret_cast<const T*>(y), sum, sumsq, gamma, beta, running_mean, running_var, nbt,
                      save_mean, save_invstd, reinterpret_cast<T*>(out), P, C, H, W, relu, pool, momentum, eps,
                      update_running, identity, ticket, flag, seq, hint};
  if (pool && ((H | W) & 1)) {                    // odd map: floor(H/2) x floor(W/2) windows
    const long long work = (long long)(P / (H * W)) * (H >> 1) * (W >> 1) * (C / 8);
    launch_k(bn_relu_pool_fwd_kernel<T, false, true>, grid_for(work, 256, 132 * 4), 256, 2 * C * sizeof(float), st, p);
    return last_err();
  }
  const long long work = (pool ? (long long)P / 4 : P) * (C / 8);
  launch_k(bn_relu_pool_fwd_kernel<T>, grid_for(work, 256, 132 * 4), 256, 2 * C * sizeof(float), st, p);
  return last_err();
}
extern "C" {
int slb_bn_relu_pool_fwd(const void* y, const float* sum, const float* sumsq, const float* gamma, const float* beta,
                         float* running_mean, float* running_var, long long* nbt, float* save_mean, float* save_invstd,
                         void* out, int P, int C, int H, int W, int relu, int pool, float momentum, float eps,
                         int update_running, int identity, uint32_t* ticket, uint32_t* flag, uint32_t* seq, uint32_t* hint,
                         int dtype, cudaStream_t st) {
  if (C % 8) return -1;
  if (pool && ((H | W) & 1) && (H < 1 || W < 1 || P % (H * W))) return -1;
  if (dtype == 1)
    return bn_fwd_t<float>(y, sum, sumsq, gamma, beta, running_mean, running_var, nbt, save_mean, save_invstd, out, P, C, H, W,
                           relu, pool, momentum, eps, update_running, identity, ticket, flag, seq, hint, st);
  return bn_fwd_t<__nv_bfloat16>(y, sum, sumsq, gamma, beta, running_mean, running_var, nbt, save_mean, save_invstd, out, P, C,
                                 H, W, relu, pool, momentum, eps, update_running, identity, ticket, flag, seq, hint, st);
}

}  // extern "C"
template <typename T>
static int bn_infer_t(const void* y, const float* gamma, const float* beta, const float* running_mean, const float* running_var,
                      void* out, int P, int C, int H, int W, int relu, int pool, float eps, cudaStream_t st) {
  BnFwdParams<T> p = {reinterpret_cast<const T*>(y), nullptr, nullptr, gamma, beta, const_cast<float*>(running_mean),
                      const_cast<float*>(running_var), nullptr, nullptr, nullptr, reinterpret_cast<T*>(out), P, C, H, W, relu,
                      pool, 0.f, eps, 0, 0, nullptr, nullptr, nullptr, nullptr};
  const long long work = (pool ? (long long)P / 4 : P) * (C / 8);
  launch_k(bn_relu_pool_fwd_kernel<T, true>, grid_for(work, 256, 132 * 4), 256, 2 * C * sizeof(float), st, p);
  return last_err();
}
extern "C" {
// BatchNorm (inference mode) + ReLU + MaxPool2 forward: the running statistics are read, never written.
int slb_bn_relu_pool_infer(const void* y, const float* gamma, const float* beta, const float* running_mean,
                           const float* running_var, void* out, int P, int C, int H, int W, int relu, int pool, float eps,
                           int dtype, cudaStream_t st) {
  if (C % 8 || gamma == nullptr || beta == nullptr || running_mean == nullptr || running_var == nullptr) return -1;
  if (pool && ((H | W) & 1)) return -2;          // the eval plan pools even maps only
  if (dtype == 1) return bn_infer_t<float>(y, gamma, beta, running_mean, running_var, out, P, C, H, W, relu, pool, eps, st);
  return bn_infer_t<__nv_bfloat16>(y, gamma, beta, running_mean, running_var, out, P, C, H, W, relu, pool, eps, st);
}

}  // extern "C"
static int bn_bwd_chan_max_p() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("SLB200_BN_BWD_CHAN_MAX_P");
    v = e ? atoi(e) : 4096;
  }
  return v;
}
template <typename T>
static int bn_bwd_t(const void* dout, const void* y, const float* gamma, const float* beta, const float* save_mean,
                    const float* save_invstd, float* dgamma, float* dbeta, void* dy, int P, int C, int H, int W, int relu,
                    int pool, int identity, uint32_t* grid_bar, cudaStream_t st) {
  // identity == 2: dgamma / dbeta already hold the reduction (done by the downstream dgrad epilogue) -> apply pass only
  const bool skip_reduce = identity == 2;
  if (skip_reduce) { identity = 0; grid_bar = nullptr; }
  BnBwdParams<T> p = {reinterpret_cast<const T*>(dout), reinterpret_cast<const T*>(y), gamma, beta,
                      save_mean, save_invstd, dgamma, dbeta, reinterpret_cast<T*>(dy), P, C, H, W, relu, pool, identity,
                      slb_det(st)};
  const int tx = C / 8;
  const int ty = tx >= 256 ? 1 : 256 / tx;
  dim3 block(tx, ty);
  const bool odd = pool && ((H | W) & 1);
  // odd map: positions on the ceil(H/2) x ceil(W/2) grid, so the dropped last row / column also receives its dy
  const long long outP = odd ? (long long)(P / (H * W)) * ((H + 1) >> 1) * ((W + 1) >> 1) : (pool ? (long long)P / 4 : P);
  const int grid = grid_for(outP, ty, 132 * 2);
  if (p.det.part == nullptr || (long long)grid * 2 * C > p.det.cap) return -30;
  if (odd) {                                        // channel-owned or two-pass kernels; the grid-barrier kernel is even-only
    if (grid_bar != nullptr && !identity) return -2;
    if (!identity && !skip_reduce && P <= bn_bwd_chan_max_p()) {
      const int thr = outP >= 256 ? 256 : (outP >= 128 ? 128 : 64);
      launch_k(bn_bwd_chan_kernel<true, T, true>, C / 8, thr, 0, st, p);
      return last_err();
    }
    if (!identity && !skip_reduce) launch_k(bn_bwd_reduce_kernel<true, T, true>, grid, block, 2 * C * sizeof(float), st, p);
    launch_k(bn_bwd_apply_kernel<true, T, true>, grid, block, 0, st, p);
    return last_err();
  }
  if (grid_bar != nullptr && !identity) {          // one launch: reduce -> grid barrier -> apply
    // the software barrier needs every block co-resident: cap the grid at (SMs - 4) x measured occupancy
    static int cap[2] = {0, 0};
    if (cap[pool ? 1 : 0] == 0) {
      int per_sm = 0, dev = 0, sms = 132;
      cudaGetDevice(&dev);
      cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
      if (pool) cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, bn_bwd_fused_kernel<true, T>, 256, 2 * 2048 * sizeof(float));
      else      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, bn_bwd_fused_kernel<false, T>, 256, 2 * 2048 * sizeof(float));
      if (per_sm < 1) per_sm = 1;
      if (per_sm > 2) per_sm = 2;
      cap[pool ? 1 : 0] = (sms > 8 ? sms - 4 : sms) * per_sm;
    }
    const int g2 = grid < cap[pool ? 1 : 0] ? grid : cap[pool ? 1 : 0];
    if (pool) launch_k(bn_bwd_fused_kernel<true, T>, g2, block, 2 * C * sizeof(float), st, p, grid_bar);
    else      launch_k(bn_bwd_fused_kernel<false, T>, g2, block, 2 * C * sizeof(float), st, p, grid_bar);
    return last_err();
  }
  if (!identity && !skip_reduce && P <= bn_bwd_chan_max_p()) {       // small maps: channel-owned blocks, one launch
    const int thr = outP >= 256 ? 256 : (outP >= 128 ? 128 : 64);
    if (pool) launch_k(bn_bwd_chan_kernel<true, T>, C / 8, thr, 0, st, p);
    else      launch_k(bn_bwd_chan_kernel<false, T>, C / 8, thr, 0, st, p);
    return last_err();
  }
  if (pool) {
    if (!identity && !skip_reduce) launch_k(bn_bwd_reduce_kernel<true, T>, grid, block, 2 * C * sizeof(float), st, p);
    launch_k(bn_bwd_apply_kernel<true, T>, grid, block, 0, st, p);
  } else {
    if (!identity && !skip_reduce) launch_k(bn_bwd_reduce_kernel<false, T>, grid, block, 2 * C * sizeof(float), st, p);
    launch_k(bn_bwd_apply_kernel<false, T>, grid, block, 0, st, p);
  }
  return last_err();
}
extern "C" {
int slb_bn_relu_pool_bwd(const void* dout, const void* y, const float* gamma, const float* beta, const float* save_mean,
                         const float* save_invstd, float* dgamma, float* dbeta, void* dy, int P, int C, int H, int W, int relu,
                         int pool, int identity, uint32_t* grid_bar, int dtype, cudaStream_t st) {
  if (C % 8 || C > 2048) return -1;
  if (pool && ((H | W) & 1) && (H < 1 || W < 1 || P % (H * W))) return -1;
  if (dtype == 1)
    return bn_bwd_t<float>(dout, y, gamma, beta, save_mean, save_invstd, dgamma, dbeta, dy, P, C, H, W, relu, pool, identity, grid_bar, st);
  return bn_bwd_t<__nv_bfloat16>(dout, y, gamma, beta, save_mean, save_invstd, dgamma, dbeta, dy, P, C, H, W, relu, pool, identity, grid_bar, st);
}

int slb_conv_finalize(const float* acc, const float* bias, void* y, float* sum, float* sumsq, long long P, int C, int dtype,
                      cudaStream_t st) {
  if (C % 8) return -1;
  const int tx = C / 8, ty = tx >= 256 ? 1 : 256 / tx;
  const Det det = slb_det(st);
  if (det.part == nullptr || (long long)grid_for(P, ty, 132 * 2) * 2 * C > det.cap) return -30;
  if (dtype == 1)
    launch_k(conv_finalize_kernel<float>, grid_for(P, ty, 132 * 2), dim3(tx, ty), 2 * C * sizeof(float), st, acc, bias,
             reinterpret_cast<float*>(y), sum, sumsq, P, C, det);
  else
    launch_k(conv_finalize_kernel<__nv_bfloat16>, grid_for(P, ty, 132 * 2), dim3(tx, ty), 2 * C * sizeof(float), st, acc, bias,
             reinterpret_cast<__nv_bfloat16*>(y), sum, sumsq, P, C, det);
  return last_err();
}
int slb_col_stats(const void* y, float* sum, float* sumsq, long long P, int C, int dtype, cudaStream_t st) {
  if (C % 8) return -1;
  const int tx = C / 8, ty = tx >= 256 ? 1 : 256 / tx;
  const Det det = slb_det(st);
  if (det.part == nullptr || (long long)grid_for(P, ty, 132 * 2) * 2 * C > det.cap) return -30;
  if (dtype == 1)
    launch_k(col_stats_kernel<float>, grid_for(P, ty, 132 * 2), dim3(tx, ty), 2 * C * sizeof(float), st,
             reinterpret_cast<const float*>(y), sum, sumsq, P, C, det);
  else
    launch_k(col_stats_kernel<__nv_bfloat16>, grid_for(P, ty, 132 * 2), dim3(tx, ty), 2 * C * sizeof(float), st,
             reinterpret_cast<const __nv_bfloat16*>(y), sum, sumsq, P, C, det);
  return last_err();
}

}  // extern "C"
template <typename T>
static int small_fwd_t(const float* x, const float* w, const float* bias, void* y, float* sum, float* sumsq, int B, int Cin,
                       int H, int W, int Cout, cudaStream_t st) {
  const long long P = (long long)B * H * W;
  const int grid = static_cast<int>((P + 127) / 128);
  T* yy = reinterpret_cast<T*>(y);
  const Det det = slb_det(st);
  if (det.part == nullptr || (long long)grid * 2 * Cout > det.cap) return -30;
  if (Cin == 3 && Cout == 64) launch_k(conv3x3_small_fwd_kernel<3, 64, T>, grid, 128, 0, st, x, w, bias, yy, sum, sumsq, B, H, W, det);
  else if (Cin == 3 && Cout == 32) launch_k(conv3x3_small_fwd_kernel<3, 32, T>, grid, 128, 0, st, x, w, bias, yy, sum, sumsq, B, H, W, det);
  else if (Cin == 1 && Cout == 64) launch_k(conv3x3_small_fwd_kernel<1, 64, T>, grid, 128, 0, st, x, w, bias, yy, sum, sumsq, B, H, W, det);
  else if (Cin == 1 && Cout == 32) launch_k(conv3x3_small_fwd_kernel<1, 32, T>, grid, 128, 0, st, x, w, bias, yy, sum, sumsq, B, H, W, det);
  else return -2;
  return last_err();
}
extern "C" {
int slb_conv3x3_small_fwd(const float* x, const float* w, const float* bias, void* y, float* sum, float* sumsq, int B, int Cin,
                          int H, int W, int Cout, int dtype, cudaStream_t st) {
  return dtype == 1 ? small_fwd_t<float>(x, w, bias, y, sum, sumsq, B, Cin, H, W, Cout, st)
                    : small_fwd_t<__nv_bfloat16>(x, w, bias, y, sum, sumsq, B, Cin, H, W, Cout, st);
}
}  // extern "C"
template <typename T>
static int small_wgrad_t(const float* x, const void* dy, float* dw, int B, int Cin, int H, int W, int Cout, cudaStream_t st) {
  if (Cout % 4 || Cout > 64 || (long long)B * H * W > (1LL << 30)) return -3;
  const int kp = 4 * ((9 * Cin + 3) / 4);
  const size_t smem = (size_t)(128 * kp + 128 * Cout + Cout * kp) * sizeof(float);
  const long long chunks = ((long long)B * H * W + 127) / 128;
  const int grid = static_cast<int>(chunks < 296 ? chunks : 296);   // 2 CTAs per SM: the staging phase of one hides behind the FMAs of the other
  const T* d = reinterpret_cast<const T*>(dy);
  const Det det = slb_det(st);
  if (det.part == nullptr || (long long)grid * Cout * 9 * Cin > det.cap) return -30;
  if (Cin == 3) {
    static bool done3 = false;
    if (!done3) { cudaFuncSetAttribute(conv3x3_small_wgrad_kernel<3, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024); done3 = true; }
    launch_k(conv3x3_small_wgrad_kernel<3, T>, grid, 256, smem, st, x, d, dw, B, H, W, Cout, det);
  } else if (Cin == 1) {
    static bool done1 = false;
    if (!done1) { cudaFuncSetAttribute(conv3x3_small_wgrad_kernel<1, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024); done1 = true; }
    launch_k(conv3x3_small_wgrad_kernel<1, T>, grid, 256, smem, st, x, d, dw, B, H, W, Cout, det);
  } else return -2;
  return last_err();
}
extern "C" {
int slb_conv3x3_small_wgrad(const float* x, const void* dy, float* dw, int B, int Cin, int H, int W, int Cout, int dtype,
                            cudaStream_t st) {
  return dtype == 1 ? small_wgrad_t<float>(x, dy, dw, B, Cin, H, W, Cout, st)
                    : small_wgrad_t<__nv_bfloat16>(x, dy, dw, B, Cin, H, W, Cout, st);
}

// acc / dacc below: `parts` slice partials [parts][B][N] of linear_fwd_f32 / linear_dgrad_f32, summed in slice order, or
// (parts == 0) one finished [B][N] buffer
int slb_linear_finalize(const float* acc, int parts, const float* bias, void* out, float* out_f32, uint8_t* mask, int B, int N,
                        int ldo, int relu, float drop_p, uint32_t seed, const uint32_t* step_ptr, int dtype, cudaStream_t st) {
  if (parts < 0) return -1;
  if (dtype == 1)
    launch_k(linear_finalize_kernel<float>, grid_for((long long)B * N, 256), 256, 0, st, acc, parts, bias,
             reinterpret_cast<float*>(out), out_f32, mask, B, N, ldo, relu, drop_p, seed, step_ptr);
  else
    launch_k(linear_finalize_kernel<__nv_bfloat16>, grid_for((long long)B * N, 256), 256, 0, st, acc, parts, bias,
             reinterpret_cast<__nv_bfloat16*>(out), out_f32, mask, B, N, ldo, relu, drop_p, seed, step_ptr);
  return last_err();
}
int slb_linear_bwd_prep(const float* dacc, int parts, const void* yout, const uint8_t* mask, void* dz, float* dbias, int B, int N,
                        int ldy, int ldz, int relu, float drop_p, int dtype, cudaStream_t st) {
  if (parts < 0) return -1;
  if (dtype == 1)
    launch_k(linear_bwd_prep_kernel<float>, (N + 31) / 32, dim3(32, 8), 0, st, dacc, parts, reinterpret_cast<const float*>(yout),
             mask, reinterpret_cast<float*>(dz), dbias, B, N, ldy, ldz, relu, drop_p);
  else
    launch_k(linear_bwd_prep_kernel<__nv_bfloat16>, (N + 31) / 32, dim3(32, 8), 0, st, dacc, parts,
             reinterpret_cast<const __nv_bfloat16*>(yout), mask, reinterpret_cast<__nv_bfloat16*>(dz), dbias, B, N, ldy, ldz, relu,
             drop_p);
  return last_err();
}
int slb_dropout_fwd(const void* x, void* y, uint8_t* mask, long long n, float p, uint32_t seed, const uint32_t* step_ptr,
                    int dtype, cudaStream_t st) {
  if (dtype == 1)
    launch_k(dropout_fwd_kernel<float>, grid_for(n, 256), 256, 0, st, reinterpret_cast<const float*>(x), reinterpret_cast<float*>(y),
             mask, n, p, seed, step_ptr);
  else
    launch_k(dropout_fwd_kernel<__nv_bfloat16>, grid_for(n, 256), 256, 0, st, reinterpret_cast<const __nv_bfloat16*>(x),
             reinterpret_cast<__nv_bfloat16*>(y), mask, n, p, seed, step_ptr);
  return last_err();
}
int slb_dropout_bwd(const float* dacc, int parts, const uint8_t* mask, void* dx, long long n, float p, int dtype, cudaStream_t st) {
  if (parts < 0) return -1;
  if (dtype == 1)
    launch_k(dropout_bwd_kernel<float>, grid_for(n, 256), 256, 0, st, dacc, parts, mask, reinterpret_cast<float*>(dx), n, p);
  else
    launch_k(dropout_bwd_kernel<__nv_bfloat16>, grid_for(n, 256), 256, 0, st, dacc, parts, mask,
             reinterpret_cast<__nv_bfloat16*>(dx), n, p);
  return last_err();
}

// ---- fp32 Linear (CUDA cores).  K % 4 == 0 and 16-byte aligned rows required.  Both kernels store one partial per slice
// into part[slices][B][out] (no atomics, no zeroing); `part_cap` is the buffer's size in floats.
// forward, K slices: enough CTAs for >= 2 waves when the layer allows, at least 128 k per slice
static int linear_fwd_kc(int N, int K) {
  const int fgroups = (N + 31) / 32;
  int kc = 1024;
  while (kc > 128 && fgroups * ((K + kc - 1) / kc) < 296) kc >>= 1;
  return kc;
}
static int linear_dgrad_threads(int K) { return K >= 512 ? 128 : 64; }
// input gradient, N slices of nc rows
static int linear_dgrad_nc(int N, int K) {
  const int threads = linear_dgrad_threads(K);
  const int ktiles = (K / 4 + threads - 1) / threads;
  int nc = 256;
  while (nc > 32 && ktiles * ((N + nc - 1) / nc) < 296) nc >>= 1;
  return nc;
}
// number of slice partials the forward (dgrad = 0) or input-gradient (dgrad = 1) kernel writes; N = out, K = in features
int slb_linear_f32_slices(int dgrad, int N, int K) {
  if (N < 1 || K < 1) return -1;
  if (dgrad) { const int nc = linear_dgrad_nc(N, K); return (N + nc - 1) / nc; }
  const int kc = linear_fwd_kc(N, K);
  return (K + kc - 1) / kc;
}
int slb_linear_fwd_f32(const float* x, const float* w, float* part, long long part_cap, int B, int N, int K, int ldx, int ldw,
                       cudaStream_t st) {
  if (K % 4 || ldx % 4 || ldw % 4) return -1;
  const int kc = linear_fwd_kc(N, K);
  dim3 grid((N + 31) / 32, (K + kc - 1) / kc, (B + 31) / 32);
  if ((long long)grid.y * B * N > part_cap) return -3;
  static bool attr = false;
  if (!attr) { cudaFuncSetAttribute(linear_fwd_f32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * 32 * 128 * 4); attr = true; }
  launch_k(linear_fwd_f32_kernel, grid, dim3(256), (size_t)4 * 32 * 128 * sizeof(float), st, x, w, part, B, N, K, ldx, ldw, kc);
  return last_err();
}
int slb_linear_dgrad_f32(const float* dz, const float* w, float* part, long long part_cap, int B, int N, int K, int lddz, int ldw,
                         cudaStream_t st) {
  if (K % 4 || ldw % 4 || (reinterpret_cast<uintptr_t>(part) & 15)) return -1;
  const int threads = linear_dgrad_threads(K);
  const int ktiles = (K / 4 + threads - 1) / threads;
  const int nc = linear_dgrad_nc(N, K);
  dim3 grid(ktiles, (N + nc - 1) / nc, (B + 31) / 32);
  if ((long long)grid.y * B * K > part_cap) return -3;
  const size_t smem = (size_t)nc * 32 * sizeof(float) + (size_t)6 * 4 * threads * 16;      // dz slice + per-thread weight ring
  static bool attr = false;
  if (!attr) { cudaFuncSetAttribute(linear_dgrad_f32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024); attr = true; }
  launch_k(linear_dgrad_f32_kernel, grid, dim3(threads), smem, st, dz, w, part, B, N, K, lddz, ldw, nc);
  return last_err();
}
// mode 0: G = g, 1: G += g, 2: fused SGD-momentum on (P, M) [+ bias rows].  Batches > 32 are looped here (mode 2 needs B <= 32).
int slb_linear_wgrad_f32(const float* dz, const float* x, float* G, float* P, float* M, float* bias_p, float* bias_m,
                         float* bias_g, int B, int N, int K, int lddz, int ldx, int ld, int mode, float lr, float mu,
                         cudaStream_t st) {
  if (K % 4 || ldx % 4 || ld % 4) return -1;
  if (mode == 2 && B > 32) return -2;
  const int threads = K >= 512 ? 128 : 64;
  const int nr = 32;
  dim3 grid((K / 4 + threads - 1) / threads, (N + nr - 1) / nr, 1);
  for (int b0 = 0; b0 < B; b0 += 32) {
    const int m = (mode == 2) ? 2 : ((mode == 1 || b0 > 0) ? 1 : 0);
    launch_k(linear_wgrad_f32_kernel, grid, dim3(threads), (size_t)nr * 32 * sizeof(float), st, dz, x, G, P, M, bias_p, bias_m,
             bias_g, B, b0, N, K, lddz, ldx, ld, nr, m, lr, mu);
  }
  return last_err();
}
int slb_sumsq(const float* g, long long n, float* out, cudaStream_t st) {
  if (n % 4) return -1;
  launch_k(sumsq_kernel, grid_for(n / 4, 256, 132 * 8), 256, 0, st, reinterpret_cast<const float4*>(g), n / 4, out);
  return last_err();
}
int slb_clip_scale(float* g, long long n, const float* sumsq, float max_norm, cudaStream_t st) {
  if (n % 4) return -1;
  launch_k(clip_scale_kernel, grid_for(n / 4, 256, 132 * 8), 256, 0, st, reinterpret_cast<float4*>(g), n / 4, sumsq, max_norm);
  return last_err();
}

int slb_ce_fwd_bwd(const float* logits, const long long* labels, float* dlogits, float* loss_sum, int* nan_flag, int B, int C,
                   int ldd, cudaStream_t st) {
  const Det det = slb_det(st);
  if (det.part == nullptr) return -30;
  launch_k(ce_fwd_bwd_kernel, (B * 32 + 127) / 128, 128, 0, st, logits, labels, dlogits, loss_sum, nan_flag, B, C, ldd, det);
  return last_err();
}
int slb_eval_metrics(const float* logits, const long long* labels, int B, int C, double* loss_total, long long* correct,
                     long long* count, cudaStream_t st) {
  if (B < 1 || C < 1) return -1;
  launch_k(eval_metrics_kernel, 1, 256, 0, st, logits, labels, B, C, loss_total, correct, count);
  return last_err();
}
int slb_sgd_momentum(float* p, float* g, float* m, void* p_bf16, long long n, float lr, float mu, int first_step, cudaStream_t st) {
  if (n % 4) return -1;
  launch_k(sgd_momentum_kernel, grid_for(n / 4, 256, 132 * 16), 256, 0, st, reinterpret_cast<float4*>(p), reinterpret_cast<float4*>(g),
                                                                     reinterpret_cast<float4*>(m), reinterpret_cast<uint2*>(p_bf16),
                                                                     n / 4, lr, mu, first_step);
  return last_err();
}
int slb_adamw(float* p, float* g, float* m, float* v, void* p_bf16, long long n, float lr, float b1, float b2, float eps, float wd,
              float bc1, float bc2, const uint32_t* step_ptr, cudaStream_t st) {
  if (n % 4) return -1;
  launch_k(adamw_kernel, grid_for(n / 4, 256, 132 * 16), 256, 0, st, reinterpret_cast<float4*>(p), reinterpret_cast<float4*>(g),
                                                              reinterpret_cast<float4*>(m), reinterpret_cast<float4*>(v),
                                                              reinterpret_cast<uint2*>(p_bf16), n / 4, lr, b1, b2, eps, wd, bc1, bc2, step_ptr);
  return last_err();
}
int slb_image_batch(const void* data, const long long* idx, const int* dx, const int* dy, const int* flip, float* out, int B,
                    int C, int H, int W, const float* mean3, const float* std3, cudaStream_t st) {
  if (C < 1 || C > 3) return -1;
  const long long total = (long long)B * C * H * W;
  launch_k(image_batch_kernel, grid_for(total, 256, 132 * 8), 256, 0, st, reinterpret_cast<const uint8_t*>(data), idx, dx, dy,
           flip, out, B, C, H, W, mean3[0], mean3[1], mean3[2], std3[0], std3[1], std3[2]);
  return last_err();
}
int slb_cast_f32_bf16(const float* x, void* y, long long n, cudaStream_t st) {
  if (n % 4) return -1;
  launch_k(cast_f32_bf16_kernel, grid_for(n / 4, 256, 132 * 16), 256, 0, st, reinterpret_cast<const float4*>(x), reinterpret_cast<uint2*>(y), n / 4);
  return last_err();
}
// srcs: host array of nsrc device pointers (local or peer-mapped), coefs: host array
int slb_fedavg(float* out, void* out_bf16, const float* const* srcs, const float* coefs, int nsrc, long long n, cudaStream_t st) {
  if (nsrc < 1 || nsrc > 16 || n % 4) return -1;
  FedAvgParams p;
  for (int i = 0; i < 16; ++i) { p.src[i] = i < nsrc ? srcs[i] : nullptr; p.coef[i] = i < nsrc ? coefs[i] : 0.f; }
  p.nsrc = nsrc;
  launch_k(fedavg_kernel, grid_for(n / 4, 512, 132 * 4), 512, 0, st, reinterpret_cast<float4*>(out), reinterpret_cast<uint2*>(out_bf16), p, n / 4);
  return last_err();
}

}  // extern "C"
