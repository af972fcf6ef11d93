// Cut-tail forward kernel (SURVEY §2.7 G1+G4+G5+G13, §7.4 "hard part" #1):
//
//   conv3x3 (wgmma implicit GEMM, the accumulator tile then stays in shared memory)
//     -> per-channel batch statistics from the accumulators (+bias)
//     -> grid-wide barrier (persistent launch, every tile resident in shared memory)
//     -> BatchNorm(train) + ReLU + 2x2 MaxPool applied straight out of shared memory
//     -> bf16 tiles stored into the NEXT stage's mailbox slot (local or NVLink-peer pointer)
//     -> last CTA publishes the slot flag with st.release.sys.
//
// The pre-BN activation never touches HBM on the forward-only pass of a recomputing stage:
// the only global traffic is x, w, 2*C floats of statistics and the (pooled) cut payload that
// crosses the link.  One persistent CTA per SM; CTA c owns tiles c, c+G, ... (at most MAX_TILES:
// the fp32 accumulators of the last tile re-use the pipeline buffers, earlier ones have their own slot).
#include "sm90.cuh"

#include <cooperative_groups.h>

namespace slb {

struct FusedCutParams {
  int M, N, C;              // pixels, Cout, Cin
  int H, W;
  int tiles_m, tiles_n;
  const float* bias;
  const float* gamma;
  const float* beta;
  float* running_mean;
  float* running_var;
  long long* nbt;
  float* save_mean;
  float* save_invstd;
  float* sum;               // [N] zeroed by the caller
  float* sumsq;
  void* y;                  // optional local copy of the pre-BN conv output (needed when not recomputing)
  void* out;                // [M or M/4][N]  — mailbox slot (may be a peer pointer); activation-typed (bf16 / fp32)
  int relu, pool;
  float momentum, eps;
  int update_running;
  uint32_t* grid_bar;       // [0] arrivals (monotonic)  [1] generation  [2] finish ticket
  uint32_t* flag;
  uint32_t* seq;
  uint32_t* hint;
  Det det;                  // reproducible cross-CTA sum of the batch statistics
};

template <int BLOCK_N>
struct FusedSmem {
  static constexpr int A_BYTES = 128 * 128;
  static constexpr int B_BYTES = BLOCK_N * 128;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = (BLOCK_N >= 128) ? 4 : 6;
  static constexpr int TILE_BYTES = STAGES * STAGE_BYTES;
  // after the MMAs the ring holds the pooling stage tile [128][33] and the last tile's fp32 accumulators [128][ACC_LD]
  static constexpr int ACC_OFF = 17 * 1024;
  static constexpr int ACC_LD = BLOCK_N + 4;
  static constexpr int ACC_BYTES = 128 * ACC_LD * 4;
  static constexpr int MAX_TILES = BLOCK_N <= 128 ? 2 : 1;
  static constexpr int TAIL_BYTES = 4096;
  static constexpr int TR_BYTES = 4 * 32 * 33 * 4;   // warp-private transpose tiles of the statistics reduction
  static constexpr int EXTRA_OFF = TILE_BYTES + TAIL_BYTES + TR_BYTES;   // accumulators of the earlier tiles
  static constexpr int TOTAL = EXTRA_OFF + (MAX_TILES - 1) * ACC_BYTES + 1024;
  static constexpr int TOT_OFF = ACC_OFF + ACC_BYTES;   // per-CTA statistics [2][N], N <= MAX_N, behind the last tile
  static constexpr int MAX_N = 512;
  static_assert(TOT_OFF + 2 * MAX_N * 4 <= TILE_BYTES, "statistics must fit in the pipeline buffers");
  static_assert(128 * 33 * 4 <= ACC_OFF, "staging tile must fit in front of the accumulator tile");
  static_assert(ACC_OFF + 128 * ACC_LD * 4 <= TILE_BYTES, "accumulator tile must fit in the pipeline buffers");
};

__device__ __forceinline__ float warp_col_reduce32f(float (&v)[32]) {
  const uint32_t lane = lane_id();
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

template <int BLOCK_N, typename T>
__global__ void __launch_bounds__(288, 1)
conv_bn_act_p2p_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                       const FusedCutParams p) {
  using L = FusedSmem<BLOCK_N>;
  using OT = OperandTraits<T>;
  constexpr int KE = OT::KE;          // K elements (channels) per 128-byte pipeline stage: 64 bf16 / 32 tf32
  pdl_trigger();
  // __align__(1024): the dynamic shared-memory window starts on a swizzle-atom boundary, and — unlike rounding the pointer
  // up by hand through an integer cast — the compiler keeps the shared address space (LDS/STS instead of generic LD/ST)
  extern __shared__ __align__(1024) uint8_t smem[];
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::TILE_BYTES);
  uint64_t* empty_bar = full_bar + L::STAGES;
  float* s_scale = reinterpret_cast<float*>(empty_bar + L::STAGES);   // [BLOCK_N]
  float* s_shift = s_scale + BLOCK_N;                           // [BLOCK_N]
  float* s_bias = s_shift + BLOCK_N;                            // [BLOCK_N] bias of the current tile's columns
  float* s_tr_all = reinterpret_cast<float*>(smem + L::TILE_BYTES + L::TAIL_BYTES);   // 4 x [32][33]
  float* s_stage = reinterpret_cast<float*>(smem);              // [128][33] fp32, reuses the pipeline buffers
  float* s_acc = reinterpret_cast<float*>(smem + L::ACC_OFF);   // [128][ACC_LD] accumulators of this CTA's last tile
  float* s_extra = reinterpret_cast<float*>(smem + L::EXTRA_OFF); // [MAX_TILES - 1][128][ACC_LD] the earlier tiles

  const int warp = threadIdx.x >> 5;
  const int G = gridDim.x;
  const int total_tiles = p.tiles_m * p.tiles_n;
  int my_tiles = 0;
  for (int t = blockIdx.x; t < total_tiles; t += G) ++my_tiles;
  auto tile_acc = [&](int j) { return j == my_tiles - 1 ? s_acc : s_extra + j * (L::ACC_BYTES / 4); };
  const int k_iters = 9 * (p.C / KE);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < L::STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);                 // one arrival per consumer warpgroup
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ============================== TMA producer ==============================
    if (elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      const int kc_per_tap = p.C / KE;
      const int pix_per_img = p.H * p.W;
      for (int j = 0; j < my_tiles; ++j) {
        const int t = blockIdx.x + j * G;
        const int m0 = (t / p.tiles_n) * 128, n0 = (t % p.tiles_n) * BLOCK_N;
        const int b0 = m0 / pix_per_img;
        const int h0 = (m0 - b0 * pix_per_img) / p.W;
        for (int it = 0; it < k_iters; ++it) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * L::STAGE_BYTES;
          mbar_expect_tx(&full_bar[stage], L::STAGE_BYTES);
          const int tap = it / kc_per_tap, kc = it - tap * kc_per_tap;
          tma_load_4d(sa, &tmA, &full_bar[stage], kc * KE, tap % 3 - 1, h0 + tap / 3 - 1, b0);
          tma_load_2d(sa + L::A_BYTES, &tmB, &full_bar[stage], tap * p.C + kc * KE, n0);
          if (++stage == L::STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ============================== two wgmma warpgroups ==============================
    int stage = 0;
    uint32_t phase = 0;
    for (int j = 0; j < my_tiles; ++j) {
      float acc[BLOCK_N / 2];
      wg_mainloop<T, BLOCK_N>(smem, nullptr, L::STAGE_BYTES, L::A_BYTES, L::STAGES, full_bar, empty_bar, k_iters, 0, 0, acc,
                              stage, phase);
      if (j == my_tiles - 1) asm volatile("bar.sync 2, 256;" ::: "memory");   // no MMA reads the ring any more
      wg_store_acc<BLOCK_N>(tile_acc(j) + (threadIdx.x >> 7) * 64 * L::ACC_LD, L::ACC_LD, acc);
    }
    asm volatile("bar.sync 2, 256;" ::: "memory");
  }
  if (warp < 4) {
    // ============================== epilogue ==============================
    const int q = warp;
    const int lrow = q * 32 + lane_id();            // row inside the tile
    const int et = threadIdx.x;
    const uint32_t gen = ld_acquire_gpu(p.grid_bar + 1);
    float* s_tot = reinterpret_cast<float*>(smem + L::TOT_OFF);     // this CTA's column sums, all its tiles
    for (int i = et; i < 2 * p.N; i += 128) s_tot[i] = 0.f;

    // ---- phase 1: statistics (and optional y) from the accumulators ----
    for (int j = 0; j < my_tiles; ++j) {
      const int t = blockIdx.x + j * G;
      const int m0 = (t / p.tiles_n) * 128, n0 = (t % p.tiles_n) * BLOCK_N;
      const int row = m0 + lrow;
      const bool row_ok = row < p.M;
      asm volatile("bar.sync 1, 128;");                 // previous tile's readers are done with s_bias
      for (int i = et; i < BLOCK_N; i += 128) s_bias[i] = __ldg(p.bias + n0 + i);
      asm volatile("bar.sync 1, 128;");
      float* s_tr = s_tr_all + warp * (32 * 33);
#pragma unroll 1
      for (int c = 0; c < BLOCK_N; c += 32) {
        uint32_t v[32];
        acc_ld32(tile_acc(j), L::ACC_LD, lrow, c, v);
        float s1[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) s1[i] = row_ok ? __uint_as_float(v[i]) + s_bias[c + i] : 0.f;
        if (p.y != nullptr && row_ok)
          store_row32(reinterpret_cast<T*>(p.y) + static_cast<long long>(row) * p.N + n0 + c, s1);
        // column sums through the warp-private transpose tile (lane l writes its row, reads column l)
#pragma unroll
        for (int i = 0; i < 32; ++i) s_tr[lane_id() * 33 + i] = s1[i];
        __syncwarp();
        float c1 = 0.f, c2 = 0.f;
#pragma unroll
        for (int r = 0; r < 32; ++r) {
          const float x = s_tr[r * 33 + lane_id()];
          c1 += x;
          c2 = fmaf(x, x, c2);
        }
        __syncwarp();
        for (int w = 0; w < 4; ++w) {                       // warps in order: a reproducible sum
          if (warp == w) { s_tot[n0 + c + lane_id()] += c1; s_tot[p.N + n0 + c + lane_id()] += c2; }
          asm volatile("bar.sync 1, 128;" ::: "memory");
        }
      }
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");
    det_commit<1>(p.det, 0, blockIdx.x, G, s_tot, 2 * p.N, p.sum, p.N, p.sumsq, et, 128);   // CTA order
    // ---- grid barrier: every CTA has contributed its partial sums ----
    asm volatile("bar.sync 1, 128;");
    if (et == 0) {
      __threadfence();
      atomicAdd(p.grid_bar, 1u);
      const uint32_t target = (gen + 1u) * static_cast<uint32_t>(G);
      uint32_t spins = 0;
      while (static_cast<int32_t>(ld_acquire_gpu(p.grid_bar) - target) < 0) {
        __nanosleep(32);
        if (++spins > (1u << 26)) __trap();                         // no printf: see mbar_wait
      }
    }
    asm volatile("bar.sync 1, 128;");

    // ---- phase 2: BN + ReLU (+pool) out of the accumulator tile, store to the mailbox ----
    const float invM = 1.f / static_cast<float>(p.M);
    const int OW = p.W >> 1, OH = p.H >> 1;
    for (int j = 0; j < my_tiles; ++j) {
      const int t = blockIdx.x + j * G;
      const int mt = t / p.tiles_n;
      const int m0 = mt * 128, n0 = (t % p.tiles_n) * BLOCK_N;
      for (int c = et; c < BLOCK_N; c += 128) {
        const int ch = n0 + c;
        s_bias[c] = __ldg(p.bias + ch);
        const float mean = __ldcg(p.sum + ch) * invM;
        const float var = fmaxf(__ldcg(p.sumsq + ch) * invM - mean * mean, 0.f);
        const float invstd = rsqrtf(var + p.eps);
        const float g = p.gamma[ch];
        s_scale[c] = g * invstd;
        s_shift[c] = p.beta[ch] - mean * g * invstd + 0.f;
        if (mt == 0) {
          p.save_mean[ch] = mean;
          p.save_invstd[ch] = invstd;
          if (p.update_running) {
            const float unbiased = p.M > 1 ? var * static_cast<float>(p.M) / static_cast<float>(p.M - 1) : var;
            p.running_mean[ch] = (1.f - p.momentum) * p.running_mean[ch] + p.momentum * mean;
            p.running_var[ch] = (1.f - p.momentum) * p.running_var[ch] + p.momentum * unbiased;
          }
        }
      }
      if (t == 0 && et == 0 && p.update_running && p.nbt) *p.nbt += 1;
      asm volatile("bar.sync 1, 128;");
      const int row = m0 + lrow;
      const bool row_ok = row < p.M;
#pragma unroll 1
      for (int c = 0; c < BLOCK_N; c += 32) {
        uint32_t v[32];
        acc_ld32(tile_acc(j), L::ACC_LD, lrow, c, v);
        float z[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          float x = fmaf(__uint_as_float(v[i]) + s_bias[c + i], s_scale[c + i], s_shift[c + i]);
          if (p.relu) x = fmaxf(x, 0.f);
          z[i] = x;
        }
        if (!p.pool) {
          if (row_ok) store_row32(reinterpret_cast<T*>(p.out) + static_cast<long long>(row) * p.N + n0 + c, z);
        } else {
          // stage the 128 x 32 activated tile, then 128 threads emit 32 pooled pixels x 32 channels
#pragma unroll
          for (int i = 0; i < 32; ++i) s_stage[lrow * 33 + i] = z[i];
          asm volatile("bar.sync 1, 128;");
          const int pp = et >> 2;                   // pooled pixel inside the tile: 0..31
          const int cg = (et & 3) * 8;              // 8-channel group
          // tile = rows_in_tile full-width image rows; pooled pixel pp -> (pooled row pr, pooled col pc)
          const int pr = pp / OW, pc = pp - pr * OW;
          const int r00 = (2 * pr) * p.W + 2 * pc;  // top-left source row inside the tile
          const int src_pix = m0 + r00;
          if (src_pix < p.M) {
            float r[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const float a = s_stage[r00 * 33 + cg + i], b = s_stage[(r00 + 1) * 33 + cg + i];
              const float cc = s_stage[(r00 + p.W) * 33 + cg + i], d = s_stage[(r00 + p.W + 1) * 33 + cg + i];
              r[i] = fmaxf(fmaxf(a, b), fmaxf(cc, d));
            }
            // global pooled pixel index: image b, row oh, col ow
            const int pix_per_img = p.H * p.W;
            const int b = src_pix / pix_per_img;
            const int rem = src_pix - b * pix_per_img;
            const int oh = (rem / p.W) >> 1, ow = (rem % p.W) >> 1;
            const long long opix = (static_cast<long long>(b) * OH + oh) * OW + ow;
            store_row8(reinterpret_cast<T*>(p.out) + opix * p.N + n0 + c + cg, r);
          }
          asm volatile("bar.sync 1, 128;");
        }
      }
      asm volatile("bar.sync 1, 128;");             // s_scale/s_shift reused by the next tile
    }
    // ---- publish: last CTA to finish releases the mailbox flag ----
    asm volatile("bar.sync 1, 128;");
    if (et == 0) {
      __threadfence_system();
      const uint32_t tk = atomicAdd(p.grid_bar + 2, 1u);
      if (tk == static_cast<uint32_t>(G) - 1u) {
        p.grid_bar[2] = 0;
        __threadfence();
        atomicExch(p.grid_bar + 1, gen + 1u);
        if (p.flag != nullptr) {
          const uint32_t value = *p.seq + 1;
          *p.seq = value;
          __threadfence_system();
          st_release_sys(p.flag, value);
          if (p.hint != nullptr) st_release_sys(p.hint, value);
        }
      }
    }
  }
}

typedef CUresult (*PFN_encodeTiled2)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                     const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                     CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled2 get_encode2() {
  // cuTensorMapEncodeTiled is a driver call: it needs a context bound to *this* thread.  Autograd worker threads may
  // reach us before any runtime call has bound the primary context (seen as CUresult 201) -> bind it once per thread.
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) { int d = 0; cudaGetDevice(&d); cudaSetDevice(d); ctx_bound = true; }   // capture-safe, unlike cudaFree(0)
  static PFN_encodeTiled2 fn = nullptr;
  if (!fn) {
    void* q = nullptr;
    cudaDriverEntryPointQueryResult r;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &q, cudaEnableDefault, &r) != cudaSuccess || !q) return nullptr;
    fn = reinterpret_cast<PFN_encodeTiled2>(q);
  }
  return fn;
}
static int encode_typed(CUtensorMap* m, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides,
                        const cuuint32_t* box, int dtype) {
  PFN_encodeTiled2 enc = get_encode2();
  if (!enc) return -1;
  cuuint32_t es[5] = {1, 1, 1, 1, 1};
  CUtensorMapDataType dt = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  if (dtype == 1) {                      // fp32 in memory, rounded to tf32 by the copy engine (see umma_gemm.cu)
    const char* e = getenv("SLB200_TMAP_F32");
    dt = (e && e[0] == '1') ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_TFLOAT32;
  }
  CUresult r = enc(m, dt, rank, const_cast<void*>(base), dims, strides, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -static_cast<int>(r) - 100;
}

template <int BN, typename T>
static int launch_fused(const CUtensorMap& a, const CUtensorMap& b, const FusedCutParams& p, int grid, cudaStream_t st) {
  auto k = conv_bn_act_p2p_kernel<BN, T>;
  static bool attr_done = false;
  if (!attr_done) {
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, FusedSmem<BN>::TOTAL);
    if (e != cudaSuccess) return -static_cast<int>(e) - 1000;
    attr_done = true;
  }
  // Plain (non-cooperative) launch with grid <= #SMs and one CTA per SM (150+ KB of smem each): co-residency of the
  // software grid barrier holds as soon as every SM has drained whatever independent kernel of another stream it was
  // running.  cudaLaunchCooperativeKernel is NOT used: the driver would not start it while any other kernel of the
  // context is resident — e.g. the next stage's flag-wait kernel that only this kernel can release (observed dead-lock).
  k<<<dim3(grid), dim3(288), FusedSmem<BN>::TOTAL, st>>>(a, b, p);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : -static_cast<int>(e) - 2000;
}

}  // namespace slb
using namespace slb;

extern "C" {

int slb_preload_fused() {
  cudaFuncAttributes a;
  int bad = 0;
  bad += cudaFuncGetAttributes(&a, conv_bn_act_p2p_kernel<64, __nv_bfloat16>) != cudaSuccess;
  bad += cudaFuncGetAttributes(&a, conv_bn_act_p2p_kernel<128, __nv_bfloat16>) != cudaSuccess;
  bad += cudaFuncGetAttributes(&a, conv_bn_act_p2p_kernel<256, __nv_bfloat16>) != cudaSuccess;
  bad += cudaFuncGetAttributes(&a, conv_bn_act_p2p_kernel<64, float>) != cudaSuccess;
  bad += cudaFuncGetAttributes(&a, conv_bn_act_p2p_kernel<128, float>) != cudaSuccess;
  bad += cudaFuncGetAttributes(&a, conv_bn_act_p2p_kernel<256, float>) != cudaSuccess;
  return bad;
}

// Fused cut-tail forward.  x [B,H,W,Cin], w [Cout][3][3][Cin], y_opt / out: bf16 (dtype 0) or fp32 (dtype 1, wgmma tf32).
// `out` may be a peer pointer.
// `grid_bar`: 4 zero-initialised uint32 owned by this call site.  sum/sumsq: zeroed by the caller.
int slb_conv_bn_act_p2p(const void* x, const void* w, const float* bias, const float* gamma, const float* beta,
                        float* running_mean, float* running_var, long long* nbt, float* save_mean, float* save_invstd,
                        float* sum, float* sumsq, void* y_opt, void* out, int B, int H, int W, int Cin, int Cout, int relu,
                        int pool, float momentum, float eps, int update_running, uint32_t* grid_bar, uint32_t* flag,
                        uint32_t* seq, uint32_t* hint, int num_sms, int dtype, cudaStream_t st) {
  const int esz = dtype == 1 ? 4 : 2, KE = 128 / esz;
  if (Cin % KE || Cout % 64 || (128 % W)) return -10;
  const int M = B * H * W;
  int tw = W, rows = 128 / W, th, tb;
  if (rows <= H) { th = rows; tb = 1; } else { th = H; tb = rows / H; }
  if (pool && ((th & 1) || (H & 1) || (W & 1))) return -14;
  const int bn = Cout >= 256 ? 256 : Cout;
  FusedCutParams p = {};
  p.M = M; p.N = Cout; p.C = Cin; p.H = H; p.W = W;
  p.tiles_m = (M + 127) / 128; p.tiles_n = Cout / bn;
  const int total = p.tiles_m * p.tiles_n;
  // Leave a few SMs out of the persistent grid: an SM that currently hosts a small flag-wait kernel of another stream
  // cannot switch its shared-memory carve-out to admit a 150 KB CTA until that kernel exits — and that kernel may be
  // waiting for *this* kernel's flag.  With spare SMs every CTA of the software grid barrier can always become resident.
  const int usable = num_sms > 8 ? num_sms - 4 : num_sms;
  int grid = total < usable ? total : usable;
  if ((total + grid - 1) / grid > (bn <= 128 ? 2 : 1)) return -15;   // FusedSmem<bn>::MAX_TILES
  CUtensorMap ta, tbm;
  {
    cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t str[3] = {(cuuint64_t)Cin * esz, (cuuint64_t)W * Cin * esz, (cuuint64_t)H * W * Cin * esz};
    cuuint32_t box[4] = {(cuuint32_t)KE, (cuuint32_t)tw, (cuuint32_t)th, (cuuint32_t)tb};
    int r = encode_typed(&ta, x, 4, dims, str, box, dtype);
    if (r) return r;
  }
  {
    cuuint64_t dims[2] = {(cuuint64_t)9 * Cin, (cuuint64_t)Cout};
    cuuint64_t str[1] = {(cuuint64_t)9 * Cin * esz};
    cuuint32_t box[2] = {(cuuint32_t)KE, (cuuint32_t)bn};
    int r = encode_typed(&tbm, w, 2, dims, str, box, dtype);
    if (r) return r;
  }
  p.bias = bias; p.gamma = gamma; p.beta = beta; p.running_mean = running_mean; p.running_var = running_var; p.nbt = nbt;
  p.save_mean = save_mean; p.save_invstd = save_invstd; p.sum = sum; p.sumsq = sumsq;
  p.y = y_opt; p.out = out;
  p.relu = relu; p.pool = pool; p.momentum = momentum; p.eps = eps; p.update_running = update_running;
  p.grid_bar = grid_bar; p.flag = flag; p.seq = seq; p.hint = hint;
  p.det = slb_det(st);
  if (p.det.part == nullptr || Cout > 512 || (long long)grid * 2 * Cout > p.det.cap) return -30;
  if (dtype == 1) {
    switch (bn) {
      case 64: return launch_fused<64, float>(ta, tbm, p, grid, st);
      case 128: return launch_fused<128, float>(ta, tbm, p, grid, st);
      case 256: return launch_fused<256, float>(ta, tbm, p, grid, st);
      default: return -3;
    }
  }
  switch (bn) {
    case 64: return launch_fused<64, __nv_bfloat16>(ta, tbm, p, grid, st);
    case 128: return launch_fused<128, __nv_bfloat16>(ta, tbm, p, grid, st);
    case 256: return launch_fused<256, __nv_bfloat16>(ta, tbm, p, grid, st);
    default: return -3;
  }
}

}  // extern "C"
