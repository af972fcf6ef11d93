// One warp-specialised wgmma GEMM pipeline, instantiated for every GEMM-shaped op of the
// split-learning stages (SURVEY §2.7 G1-G3, G6):
//
//   MODE_CONV   conv3x3 s1 p1 forward and input-gradient as implicit GEMM.
//               A = NHWC activations, one 4-D TMA box per filter tap (signed coordinates ->
//               zero padding for free), K-major;  B = [Cout][3][3][Cin] weights, K-major
//               (forward) or MN-major view of the same tensor (dgrad, taps mirrored).
//   MODE_WGRAD  conv3x3 weight gradient, K = all pixels, both operands MN-major,
//               split-K over CTAs with fp32 red.add into the [Cout][3][3][Cin] gradient.
//   MODE_GEMM   plain C[M,N] (+)= A * B with any major combination: the three Linear GEMMs
//               (swap-AB so the 4096-wide dimension sits on the MMA M axis).
//
// Roles (288 threads): warps 0..7 = two consumer warpgroups issuing wgmma (rows [0,64) and [64,128)
// of the tile, fp32 accumulators in registers), warp 8 = TMA producer.  BLOCK_M = 128, BLOCK_K = one
// 128-byte swizzle row.  After the mainloop the accumulators go to shared memory and warps 0..3 run the
// epilogue with one output row per thread.
//
// Two operand precisions share the pipeline (template parameter T, sm100.cuh OperandTraits):
//   float          fp32 tensors in HBM and shared memory, wgmma tf32 (the reference's precision: PyTorch
//                  runs cuDNN convolutions on TF32 tensor cores by default, SURVEY §2.7 note), BLOCK_K = 32, fp32 outputs
//   __nv_bfloat16  bf16 operands / outputs, wgmma bf16, BLOCK_K = 64 (opt-in fast mode)
#include "sm90.cuh"

namespace slb {

enum { MODE_CONV = 0, MODE_WGRAD = 1, MODE_GEMM = 2 };
enum { EPI_BF16 = 0 /* activation-typed store (bf16 or fp32) */, EPI_F32_ATOMIC = 1, EPI_F32_ATOMIC_T = 2, EPI_F32_STORE = 3 };

struct GemmParams {
  // generic
  int M, N;             // logical output extent (rows x columns of the accumulator tiles)
  int k_iters;          // total K iterations of 64
  int k_split;          // gridDim.z
  int a_mn, b_mn;       // operand majors (1 = MN-major)
  int epi;              // epilogue kind
  void* out;            // output tensor
  long long ldo;        // output leading dimension (elements)
  const float* bias;    // per-column bias (EPI_BF16) or nullptr
  float* col_sum;       // per-column sum / sum of squares (BN statistics) or nullptr
  float* col_sumsq;
  // row remap for wgrad: row r -> (r % rmod) * rmul1 + (r / rmod) * rmul2   (rmod == 0: r * ldo)
  int rmod;
  long long rmul1, rmul2;
  int m_valid_mod;      // wgrad: rows r with r / rmod >= 9 are padding
  // conv geometry
  int C;                // channels of the A tensor (GEMM-K per tap)
  int tw, th, tb;       // pixel-tile box (W, H, B) ; tw*th*tb == 128 (conv) or 64 (wgrad)
  int H, W;
  int flip;             // 1: dgrad (mirrored taps)
  int b_row_stride;     // conv: columns of B per tap (= Cin of the weight tensor)
  int Cout;             // wgrad: number of output channels (rows per tap)
  // split-K with in-kernel finalisation: the last K-slice of a tile to arrive adds the fp32 partial tiles of all slices
  // (slice z at out + z * M * ldo) and converts them into the result + BN statistics — no separate finalize launch.
  uint32_t* tile_counters;   // [m_tiles * n_tiles], zero at rest (self-resetting)
  void* fin_out;             // activation-typed destination [M][fin_ld]
  long long fin_ld;
  // dgrad epilogue doubling as the BatchNorm-backward reduction of the *upstream* block (whose ReLU output this dX is
  // the gradient of): col_sum += sum_p m*dX (dbeta), col_sumsq += sum_p m*dX*xhat (dgamma), m = ReLU mask recomputed
  // from the saved conv output.  Removes one launch per conv block from the backward critical path.
  const __nv_bfloat16* bnb_y;     // [M][N] saved pre-BN conv output of the upstream block, or nullptr
  const float* bnb_mean;
  const float* bnb_istd;
  const float* bnb_gamma;
  const float* bnb_beta;
  int bnb_relu;
  int bnb_pool;                   // 1: the upstream block ends in MaxPool2 — dX lives on the pooled grid (H x W here),
                                  //    bnb_y on the 2H x 2W grid; the gradient goes to the window's (first) maximum
  // transformer epilogue (EPI_BF16, MODE_GEMM): out = act(acc + bias + residual); aux_out keeps the pre-activation
  // cut-head dgrad: the gradient tiles land in the upstream stage's mailbox (peer pointer); the last CTA of the grid
  // publishes the slot flag itself (st.release.sys) — no separate flag kernel on the backward edge
  uint32_t* pub_ticket;           // zero at rest (self-resetting)
  uint32_t* pub_flag;             // mailbox flag (may be a peer pointer) or nullptr
  uint32_t* pub_seq;              // device sequence counter of the edge
  long long* trace;               // optional [16] cycle stamps of CTA (0,0,0) (tools/trace_gemm.py): where a launch spends its time
  int act;                        // 0 none, 1 ReLU, 2 GELU (erf), 3 tanh
  __nv_bfloat16* aux_out;         // [M][ldo] or nullptr
  const __nv_bfloat16* residual;  // [M][ldo] or nullptr
  Det det;                        // reproducible reductions: BN statistics across m-tiles, split-K turns without tile_counters
};

// May 32 columns at `ptr` be moved as 16-byte vectors?  Conv and wgrad rows always start 16-byte aligned (the host
// requires Nout % 32 == 0), so only MODE_GEMM tests the pointer: its ldo is free (a Linear with 36 or 100 outputs).
template <int MODE>
__device__ __forceinline__ bool vec16_ok(const void* ptr) {
  return MODE != MODE_GEMM || (reinterpret_cast<uintptr_t>(ptr) & 15) == 0;
}

__device__ __forceinline__ float apply_act(float x, int act) {
  if (act == 1) return fmaxf(x, 0.f);
  if (act == 2) return 0.5f * x * (1.f + erff(x * 0.70710678118654752f));
  if (act == 3) return tanhf(x);
  return x;
}

template <int BLOCK_N, typename T>
struct SmemLayout {
  static constexpr int A_BYTES = 128 * 128;      // 16 KB
  static constexpr int B_BYTES = BLOCK_N * 128;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES_FIT = 196 * 1024 / STAGE_BYTES;
  static constexpr int STAGES = STAGES_FIT < 6 ? STAGES_FIT : 6;
  // tf32 MN-major operands are transposed in place one stage ahead of the MMAs (sm90.cuh wg_mainloop)
  static_assert(STAGES >= 3, "the in-place tf32 transpose needs a third stage");
  static constexpr int TILE_BYTES = STAGES * STAGE_BYTES;
  // once the MMAs are done the ring holds the epilogue's transpose tiles [0, 17 KB) and the fp32 accumulator tile
  static constexpr int ACC_OFF = 17 * 1024;
  static constexpr int ACC_LD = BLOCK_N + 4;     // row pitch in floats: 16-byte row reads without bank conflicts
  static constexpr int BAR_BYTES = 4096;
  static constexpr int TOTAL = TILE_BYTES + BAR_BYTES + 1024 /*align slack*/;
  static_assert(ACC_OFF + 128 * ACC_LD * 4 <= TILE_BYTES, "accumulator tile must fit in the pipeline buffers");
};

// Sum of v[c] over the 32 lanes of a warp for every c in 0..31; lane j returns column j.
__device__ __forceinline__ float warp_col_reduce32(float (&v)[32]) {
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

// Column sums of a 32 x 32 block held one row per lane (f[j] = column j of this lane's row), through a warp-private
// [32][33] shared-memory tile: lane l writes its row, then reads column l top to bottom.  Returns sum and sum of squares
// of column `lane` — about a third of the instructions of the register butterfly (measured 0.78 us -> ~0.25 us per chunk).
__device__ __forceinline__ void warp_col_sums_smem(float* tile, const float (&f)[32], float& c1, float& c2) {
  const uint32_t lane = lane_id();
#pragma unroll
  for (int j = 0; j < 32; ++j) tile[lane * 33 + j] = f[j];
  __syncwarp();
  float a = 0.f, b = 0.f;
#pragma unroll
  for (int r = 0; r < 32; ++r) {
    const float x = tile[r * 33 + lane];
    a += x;
    b = fmaf(x, x, b);
  }
  __syncwarp();
  c1 = a;
  c2 = b;
}

// Per-element terms of the two column reductions of an epilogue chunk (row = pixel, 32 consecutive channels):
// BatchNorm forward statistics (x, x^2) or, with bnb_y, the BatchNorm backward sums of the upstream block.
template <bool BNB, typename T>
__device__ __forceinline__ void stat_terms(const GemmParams& p, int row, bool row_ok, int col0, const float (&f)[32],
                                           float (&s1)[32], float (&s2)[32]) {
  if (!BNB || p.bnb_y == nullptr) {
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const float r = row_ok ? stored_value(f[j], static_cast<const T*>(nullptr)) : 0.f;   // statistics of the stored values
      s1[j] = r;
      s2[j] = r * r;
    }
    return;
  }
  if constexpr (BNB) {
  if (!row_ok) {
#pragma unroll
    for (int j = 0; j < 32; ++j) { s1[j] = 0.f; s2[j] = 0.f; }
    return;
  }
  if (!p.bnb_pool) {
    const uint4* y4 = reinterpret_cast<const uint4*>(p.bnb_y + static_cast<long long>(row) * p.N + col0);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint4 u = __ldg(y4 + q);
      const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 yy = __bfloat1622float2(h2[e]);
#pragma unroll
        for (int t = 0; t < 2; ++t) {
          const int j = 8 * q + 2 * e + t, c = col0 + j;
          const float y = t ? yy.y : yy.x;
          const float mean = __ldg(p.bnb_mean + c), istd = __ldg(p.bnb_istd + c);
          const float sc = __ldg(p.bnb_gamma + c) * istd, sh = __ldg(p.bnb_beta + c) - mean * sc;
          const float r = __bfloat162float(__float2bfloat16(f[j]));
          const float dz = (p.bnb_relu && fmaf(y, sc, sh) <= 0.f) ? 0.f : r;          // same test as bn_dz()
          s1[j] = dz;
          s2[j] = dz * (y - mean) * istd;
        }
      }
    }
    return;
  }
  // pooled upstream block: row = (b, oh, ow) on the H x W grid of this dgrad; window = 2x2 pixels of the 2H x 2W grid
  const int ow = row % p.W, t0 = row / p.W, oh = t0 % p.H, bb = t0 / p.H;
  const long long base = (static_cast<long long>(bb) * (2 * p.H) + 2 * oh) * (2 * p.W) + 2 * ow;
  float best[32], ybest[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) { best[j] = -INFINITY; ybest[j] = 0.f; }
#pragma unroll 1
  for (int q = 0; q < 4; ++q) {
    const long long ip = base + (q >> 1) * (2 * p.W) + (q & 1);
    const uint4* y4 = reinterpret_cast<const uint4*>(p.bnb_y + ip * p.N + col0);
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      const uint4 u = __ldg(y4 + v);
      const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 yy = __bfloat1622float2(h2[e]);
#pragma unroll
        for (int t = 0; t < 2; ++t) {
          const int j = 8 * v + 2 * e + t, c = col0 + j;
          const float y = t ? yy.y : yy.x;
          const float istd = __ldg(p.bnb_istd + c), sc = __ldg(p.bnb_gamma + c) * istd;
          float z = fmaf(y, sc, __ldg(p.bnb_beta + c) - __ldg(p.bnb_mean + c) * sc);
          if (p.bnb_relu) z = fmaxf(z, 0.f);
          if (z > best[j]) { best[j] = z; ybest[j] = y; }                            // first maximum wins, like bn_dz()
        }
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int c = col0 + j;
    const float r = __bfloat162float(__float2bfloat16(f[j]));
    const float dz = (p.bnb_relu && best[j] <= 0.f) ? 0.f : r;
    s1[j] = dz;
    s2[j] = dz * (ybest[j] - __ldg(p.bnb_mean + c)) * __ldg(p.bnb_istd + c);
  }
  }  // BNB
}

// Ragged pixel tiles (RAG): a tile is one padded power-of-two box (tb x th x tw pixel slots, tw >= W, th >= min(H, ...))
// at (b0, h0, 0) of the NHWC tensor; slots outside the tensor are TMA out-of-bounds zero fill.  Tile t of a conv has
// b0 = (t / tiles_h) * tb and h0 = (t % tiles_h) * th, tiles_h = ceil(H / th); a wgrad K step is one such box.
__device__ __forceinline__ int rag_tiles_h(const GemmParams& p) { return (p.H + p.th - 1) / p.th; }

// Row r of ragged conv tile `t` is pixel (b0 + r / (tw th), h0 + (r / tw) % th, r % tw); false for padding slots.
__device__ __forceinline__ bool rag_row(const GemmParams& p, int t, int r, long long& off) {
  const int tiles_h = rag_tiles_h(p);
  const int b = (t / tiles_h) * p.tb + r / (p.tw * p.th);
  const int h = (t % tiles_h) * p.th + (r / p.tw) % p.th;
  const int w = r % p.tw;
  off = ((static_cast<long long>(b) * p.H + h) * p.W + w) * p.ldo;
  return b < p.M / (p.H * p.W) && h < p.H && w < p.W;
}

// BNB: instantiate the upstream-BatchNorm-backward epilogue (dgrad only).  A separate instantiation on purpose: with the
// code in the common kernel every conv paid ~1.8 % (205 vs 154 registers; same-box A/B, profiles/README.md).
// RAG: ragged pixel tiles (above) for maps whose width does not divide the tile; also a separate instantiation, so the
// power-of-two kernels keep their code.  The host gives a ragged conv k_split == 1 and no statistics, BNB or publish.
template <int MODE, int BLOCK_N, typename T, bool BNB = false, bool RAG = false>
__global__ void __launch_bounds__(288, 1)
umma_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const GemmParams p) {
  using L = SmemLayout<BLOCK_N, T>;
  using OT = OperandTraits<T>;
  constexpr int KE = OT::KE;                       // K elements per stage == elements per MN-major group (128 bytes)
  constexpr int GROUP_BYTES = KE * 128;            // one MN-major group: KE k-rows of 128 bytes
  static_assert(!BNB || !OT::TF32, "the fused BatchNorm-backward epilogue is a bf16-only option");
  pdl_trigger();                      // the next kernel may start its prologue now
  // __align__(1024): the dynamic shared-memory window starts on a swizzle-atom boundary, and — unlike rounding the pointer
  // up by hand through an integer cast — the compiler keeps the shared address space (LDS/STS instead of generic LD/ST)
  extern __shared__ __align__(1024) uint8_t smem[];
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::TILE_BYTES);
  uint64_t* empty_bar = full_bar + L::STAGES;
  uint32_t* s_flag = reinterpret_cast<uint32_t*>(empty_bar + L::STAGES);
  float* s_stats = reinterpret_cast<float*>(s_flag + 4);      // [2][BLOCK_N] floats (<= 2 KB of the 4 KB tail)
  float* s_acc = reinterpret_cast<float*>(smem + L::ACC_OFF); // [128][ACC_LD] accumulators for the epilogue

  const int warp = threadIdx.x >> 5;
  const int m_tile = blockIdx.x, n_tile = blockIdx.y, z = blockIdx.z;
  const int m0 = m_tile * 128, n0 = n_tile * BLOCK_N;
  long long* const tr = (p.trace != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) ? p.trace : nullptr;
#define SLB_STAMP(i) do { if (tr != nullptr) tr[i] = clock64(); } while (0)
  if (threadIdx.x == 0) SLB_STAMP(0);

  // K range of this CTA (split-K)
  const int per = (p.k_iters + p.k_split - 1) / p.k_split;
  const int k_begin = z * per;
  const int k_end = min(p.k_iters, k_begin + per);
  const int my_iters = max(0, k_end - k_begin);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < L::STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);                 // one arrival per consumer warpgroup
    }
    mbar_fence_init();
    s_flag[1] = 0;
  }
  __syncthreads();
  if (threadIdx.x == 0) SLB_STAMP(1);
  pdl_wait();                         // predecessor grids complete + visible; prologue above overlapped with their tail
  if (threadIdx.x == 0) SLB_STAMP(2);

  if (my_iters > 0) {
    if (warp == 8) {
      // ============================== TMA producer ==============================
      if (elect_one()) {
        int stage = 0;
        uint32_t phase = 0;
        for (int it = k_begin; it < k_end; ++it) {
          if (it == k_begin + L::STAGES) SLB_STAMP(3);        // producer: the first ring of loads is in flight
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * L::STAGE_BYTES;
          uint8_t* sb = sa + L::A_BYTES;
          mbar_expect_tx(&full_bar[stage], L::STAGE_BYTES);
          if constexpr (MODE == MODE_CONV) {
            const int kc_per_tap = p.C / KE;
            const int tap = it / kc_per_tap, kc = it - tap * kc_per_tap;
            int dh = tap / 3 - 1, dw = tap % 3 - 1;
            if (p.flip) { dh = -dh; dw = -dw; }
            int b0, h0;
            if constexpr (RAG) {
              const int tiles_h = rag_tiles_h(p);
              b0 = (m_tile / tiles_h) * p.tb;
              h0 = (m_tile % tiles_h) * p.th;
            } else {
              // pixel tile origin: 128 consecutive NHWC pixels starting at m0
              const int pix_per_img = p.H * p.W;
              b0 = m0 / pix_per_img;
              const int rem = m0 - b0 * pix_per_img;
              h0 = rem / p.W;
            }
            tma_load_4d(sa, &tmA, &full_bar[stage], kc * KE, dw, h0 + dh, b0);
            if (!p.b_mn) {
              tma_load_2d(sb, &tmB, &full_bar[stage], tap * p.b_row_stride + kc * KE, n0);
            } else {
#pragma unroll
              for (int g = 0; g < BLOCK_N / KE; ++g)
                tma_load_2d(sb + g * GROUP_BYTES, &tmB, &full_bar[stage], tap * p.b_row_stride + n0 + g * KE, kc * KE);
            }
          } else if constexpr (MODE == MODE_WGRAD) {
            int b0, h0;
            if constexpr (RAG) {
              // K iteration = one padded box of KE pixel slots; empty slots are zero in both operands
              const int tiles_h = rag_tiles_h(p);
              b0 = (it / tiles_h) * p.tb;
              h0 = (it % tiles_h) * p.th;
            } else {
              // K iteration = KE consecutive pixels starting at it*KE
              const int pix0 = it * KE;
              const int pix_per_img = p.H * p.W;
              b0 = pix0 / pix_per_img;
              const int rem = pix0 - b0 * pix_per_img;
              h0 = rem / p.W;
            }
#pragma unroll
            for (int g = 0; g < 128 / KE; ++g) {
              const int r = m0 + g * KE;
              const int tap = r / p.Cout, c0 = r - tap * p.Cout;
              if (tap < 9) {
                const int dh = tap / 3 - 1, dw = tap % 3 - 1;
                // dW[co][tap][ci] = sum_q dY[q - tap][co] * X[q][ci]
                tma_load_4d(sa + g * GROUP_BYTES, &tmA, &full_bar[stage], c0, -dw, h0 - dh, b0);
              } else {
                // padding group (9 * Cout is not a multiple of 128 when Cout == 64): re-load tap 8, result is discarded
                tma_load_4d(sa + g * GROUP_BYTES, &tmA, &full_bar[stage], c0, 0, h0, b0);
              }
            }
#pragma unroll
            for (int g = 0; g < BLOCK_N / KE; ++g)
              tma_load_4d(sb + g * GROUP_BYTES, &tmB, &full_bar[stage], n0 + g * KE, 0, h0, b0);
          } else {
            if (!p.a_mn) {
              tma_load_2d(sa, &tmA, &full_bar[stage], it * KE, m0);
            } else {
#pragma unroll
              for (int g = 0; g < 128 / KE; ++g)
                tma_load_2d(sa + g * GROUP_BYTES, &tmA, &full_bar[stage], m0 + g * KE, it * KE);
            }
            if (!p.b_mn) {
              tma_load_2d(sb, &tmB, &full_bar[stage], it * KE, n0);
            } else {
#pragma unroll
              for (int g = 0; g < (BLOCK_N + KE - 1) / KE; ++g)
                tma_load_2d(sb + g * GROUP_BYTES, &tmB, &full_bar[stage], n0 + g * KE, it * KE);
            }
          }
          if (++stage == L::STAGES) { stage = 0; phase ^= 1; }
        }
      }
    } else {
      // ========================= two wgmma warpgroups, then the epilogue (warps 0..3) =========================
      const int et = threadIdx.x;                  // 0..127: epilogue thread id
      const bool want_stats = (p.col_sum != nullptr);
      // the bias of this tile's columns is staged in shared memory before the mainloop (32 dependent-latency global
      // loads per 32-column chunk would otherwise sit on the epilogue's critical path)
      float* s_bias = s_stats + 2 * BLOCK_N;
      if (warp < 4) {
        for (int i = et; i < 2 * BLOCK_N; i += 128) s_stats[i] = 0.f;
        for (int i = et; i < BLOCK_N; i += 128) s_bias[i] = (p.bias != nullptr && n0 + i < p.N) ? __ldg(p.bias + n0 + i) : 0.f;
      }
      float acc[BLOCK_N / 2];
      int stage = 0;
      uint32_t phase = 0;
      wg_mainloop<T, BLOCK_N>(smem, L::STAGE_BYTES, L::A_BYTES, L::STAGES, full_bar, empty_bar, my_iters, p.a_mn, p.b_mn,
                              acc, stage, phase);
      if (et == 0) SLB_STAMP(6);                               // accumulator complete
      asm volatile("bar.sync 2, 256;" ::: "memory");           // no MMA reads the ring any more
      wg_store_acc<BLOCK_N>(s_acc + (threadIdx.x >> 7) * 64 * L::ACC_LD, L::ACC_LD, acc);
      asm volatile("bar.sync 2, 256;" ::: "memory");
      if (warp < 4) {
      const int q = warp;                           // rows [32q, 32q + 32) of the tile
      const int row = m0 + q * 32 + lane_id();      // output row of this thread
      // warp-private transpose tile for the statistics, in front of the accumulator tile
      float* s_tr = reinterpret_cast<float*>(smem) + warp * (32 * 33);
      static_assert(L::ACC_OFF >= 4 * 32 * 33 * 4, "transpose tiles must fit in front of the accumulator tile");
      constexpr bool RAG_ROWS = RAG && MODE == MODE_CONV;        // a ragged wgrad keeps its [Cout][3][3][Cin] rows
      long long rag_off = 0;
      const bool row_ok = RAG_ROWS ? rag_row(p, m_tile, q * 32 + lane_id(), rag_off) : row < p.M;
      long long row_off;
      bool row_store = row_ok;
      if (p.rmod > 0) {
        const int hi = row / p.rmod, lo = row - hi * p.rmod;
        row_off = lo * p.rmul1 + hi * p.rmul2;
        row_store = row_ok && hi < p.m_valid_mod;
      } else {
        row_off = RAG_ROWS ? rag_off : static_cast<long long>(row) * p.ldo;
      }
      // split-K with in-kernel finalisation (tile_counters): every K slice stores its partial tile into slice z of `out`
      // ([k_split][M][ldo]); the last slice of the tile to arrive adds the k_split partials in slice order.  Without
      // tile_counters the slices add into `out` in slice order (blockIdx.z) behind a turn counter.  Either way the fp32
      // sums are the same every run.
      const uint32_t tix = blockIdx.x * gridDim.y + blockIdx.y;
      uint32_t* turn = nullptr;
      if ((p.epi == EPI_F32_ATOMIC || p.epi == EPI_F32_ATOMIC_T) && gridDim.z > 1 && p.tile_counters == nullptr) {
        turn = p.det.ctr + DET_TURN_BASE + tix;
        if (et == 0) turn_wait(turn, blockIdx.z);
        asm volatile("bar.sync 1, 128;" ::: "memory");
      }
      const long long slice = static_cast<long long>(p.M) * p.ldo;   // floats per partial tile set
#pragma unroll 1
      for (int c = 0; c < BLOCK_N; c += 32) {
        uint32_t v[32];
        acc_ld32(s_acc, L::ACC_LD, q * 32 + lane_id(), c, v);
        if (et == 0 && c == 0) SLB_STAMP(11);
        const int col0 = n0 + c;
        if (p.epi == EPI_BF16) {
          float f[32];
#pragma unroll
          for (int j = 0; j < 32; ++j) f[j] = __uint_as_float(v[j]) + s_bias[c + j];
          if (et == 0 && c == 0) SLB_STAMP(12);
          if constexpr (MODE == MODE_GEMM && !OT::TF32) {
            if (p.residual != nullptr && row_store) {
              const __nv_bfloat16* rs = p.residual + row_off + col0;
              if (col0 + 32 <= p.N && vec16_ok<MODE>(rs)) {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                  const uint4 u = __ldg(reinterpret_cast<const uint4*>(rs) + j);
                  const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
                  for (int e = 0; e < 4; ++e) {
                    const float2 t = __bfloat1622float2(h2[e]);
                    f[8 * j + 2 * e] += t.x;
                    f[8 * j + 2 * e + 1] += t.y;
                  }
                }
              } else {
                {
_Pragma("unroll") for (int j = 0; j < 32; ++j) if (col0 + j < p.N) f[j] += __bfloat162float(rs[j]); }
              }
            }
            if (p.aux_out != nullptr && row_store) {
              __nv_bfloat16* ao = p.aux_out + row_off + col0;
              if (col0 + 32 <= p.N && vec16_ok<MODE>(ao)) {
                uint4* a4 = reinterpret_cast<uint4*>(ao);
#pragma unroll
                for (int j = 0; j < 4; ++j)
                  a4[j] = make_uint4(pack_bf16x2(f[8 * j], f[8 * j + 1]), pack_bf16x2(f[8 * j + 2], f[8 * j + 3]),
                                     pack_bf16x2(f[8 * j + 4], f[8 * j + 5]), pack_bf16x2(f[8 * j + 6], f[8 * j + 7]));
              } else {
                {
_Pragma("unroll") for (int j = 0; j < 32; ++j) if (col0 + j < p.N) ao[j] = __float2bfloat16(f[j]); }
              }
            }
            if (p.act != 0) {
#pragma unroll
              for (int j = 0; j < 32; ++j) f[j] = apply_act(f[j], p.act);
            }
          }
          if (row_store) {
            T* o = reinterpret_cast<T*>(p.out) + row_off + col0;
            if (col0 + 32 <= p.N && vec16_ok<MODE>(o)) {   // tf32 (T = float) outputs are conv / wgrad only: aligned
              store_row32(o, f);
            } else {
              {
_Pragma("unroll") for (int j = 0; j < 32; ++j) if (col0 + j < p.N) o[j] = static_cast<T>(f[j]); }
            }
          }
          if (et == 0 && c == 0) SLB_STAMP(13);
          if (want_stats) {
            // statistics of the values that were stored (what the consumer normalises; bf16-rounded in bf16 mode)
            float c1, c2;
            if constexpr (BNB) {
              float s1[32], s2[32];
              stat_terms<BNB, T>(p, row, row_ok, col0, f, s1, s2);
              c1 = warp_col_reduce32(s1);
              c2 = warp_col_reduce32(s2);
            } else {
              float s1[32];
#pragma unroll
              for (int j = 0; j < 32; ++j) s1[j] = row_ok ? stored_value(f[j], static_cast<const T*>(nullptr)) : 0.f;
              warp_col_sums_smem(s_tr, s1, c1, c2);
            }
            if (et == 0 && c == 0) SLB_STAMP(14);
            for (int w = 0; w < 4; ++w) {                       // warps in order: a reproducible sum
              if (warp == w) { s_stats[c + lane_id()] += c1; s_stats[BLOCK_N + c + lane_id()] += c2; }
              asm volatile("bar.sync 1, 128;" ::: "memory");
            }
          }
          if (et == 0 && c == 0) SLB_STAMP(15);
        } else if (p.epi == EPI_F32_ATOMIC) {
          if (row_store && p.tile_counters != nullptr) {
            // conv split-K partial (Nout % 32 == 0: whole, 16-byte aligned 32-column chunks)
            float4* o4 = reinterpret_cast<float4*>(reinterpret_cast<float*>(p.out) + blockIdx.z * slice + row_off + col0);
#pragma unroll
            for (int j = 0; j < 8; ++j)
              __stcg(o4 + j, make_float4(__uint_as_float(v[4 * j]), __uint_as_float(v[4 * j + 1]),
                                         __uint_as_float(v[4 * j + 2]), __uint_as_float(v[4 * j + 3])));
          } else if (row_store) {
            float* o = reinterpret_cast<float*>(p.out) + row_off + col0;
            if (col0 + 32 <= p.N && ((reinterpret_cast<uintptr_t>(o) & 15) == 0)) {
#pragma unroll
              for (int j = 0; j < 32; j += 4)   // 16-byte vector reductions: 4x fewer L2 atomic operations
                asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(o + j), "f"(__uint_as_float(v[j])),
                             "f"(__uint_as_float(v[j + 1])), "f"(__uint_as_float(v[j + 2])), "f"(__uint_as_float(v[j + 3]))
                             : "memory");
            } else {
#pragma unroll
              for (int j = 0; j < 32; ++j)
                if (col0 + j < p.N) atomicAdd(o + j, __uint_as_float(v[j]));
            }
          }
        } else if (p.epi == EPI_F32_ATOMIC_T) {
          if (row_ok) {
            float* o = reinterpret_cast<float*>(p.out) + row;
#pragma unroll
            for (int j = 0; j < 32; ++j)
              if (col0 + j < p.N) atomicAdd(o + static_cast<long long>(col0 + j) * p.ldo, __uint_as_float(v[j]));
          }
        } else {  // EPI_F32_STORE (MODE_GEMM with a bias: fp32 logits = acc + bias, slb_gemm_bf16_bias_f32)
          if constexpr (MODE == MODE_GEMM) {
            if (p.bias != nullptr) {
#pragma unroll
              for (int j = 0; j < 32; ++j) v[j] = __float_as_uint(__uint_as_float(v[j]) + s_bias[c + j]);
            }
          }
          if (row_store) {
            float* o = reinterpret_cast<float*>(p.out) + row_off + col0;
            if (col0 + 32 <= p.N && vec16_ok<MODE>(o)) {
              float4* o4 = reinterpret_cast<float4*>(o);
#pragma unroll
              for (int j = 0; j < 8; ++j)
                o4[j] = make_float4(__uint_as_float(v[4 * j]), __uint_as_float(v[4 * j + 1]),
                                    __uint_as_float(v[4 * j + 2]), __uint_as_float(v[4 * j + 3]));
            } else {
              {
_Pragma("unroll") for (int j = 0; j < 32; ++j) if (col0 + j < p.N) o[j] = __uint_as_float(v[j]); }
            }
          }
        }
      }
      if (et == 0) SLB_STAMP(7);                               // accumulators drained / stores or reds issued
      if (turn != nullptr) {
        __threadfence();
        if (et == 0) SLB_STAMP(8);                             // reds globally visible
        asm volatile("bar.sync 1, 128;" ::: "memory");
        if (et == 0) turn_pass(turn, blockIdx.z, gridDim.z);
      }
      if (p.epi == EPI_F32_ATOMIC && p.tile_counters != nullptr) {
        // ---- split-K tail: the last slice of this tile to arrive sums the partials and finalises the tile ----
        __threadfence();                                       // this slice's partial is visible before it arrives
        asm volatile("bar.sync 1, 128;" ::: "memory");
        if (et == 0) {
          const uint32_t t = atomicAdd(p.tile_counters + tix, 1u);
          s_flag[1] = (t == gridDim.z - 1u) ? 1u : 0u;
          if (s_flag[1]) p.tile_counters[tix] = 0;             // zero at rest
        }
        asm volatile("bar.sync 1, 128;" ::: "memory");
        if (s_flag[1]) {
          __threadfence();
#pragma unroll 1
          for (int c = 0; c < BLOCK_N; c += 32) {
            const int col0 = n0 + c;
            float f[32];
#pragma unroll
            for (int j = 0; j < 32; ++j) f[j] = 0.f;
            if (row_ok) {
              // +0 plus the slices in slice order with add.rn.ftz: the arithmetic of red.global.add.f32 into a zeroed buffer.
              // Unrolled by four slices so that 32 independent L2 loads are in flight, not 8 per dependent round trip.
              const float4* a4 = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p.out) + row_off + col0);
#pragma unroll 4
              for (int zz = 0; zz < static_cast<int>(gridDim.z); ++zz) {
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                  const float4 t4 = __ldcg(a4 + zz * (slice / 4) + j);
                  asm("add.rn.ftz.f32 %0, %0, %1;" : "+f"(f[4 * j]) : "f"(t4.x));
                  asm("add.rn.ftz.f32 %0, %0, %1;" : "+f"(f[4 * j + 1]) : "f"(t4.y));
                  asm("add.rn.ftz.f32 %0, %0, %1;" : "+f"(f[4 * j + 2]) : "f"(t4.z));
                  asm("add.rn.ftz.f32 %0, %0, %1;" : "+f"(f[4 * j + 3]) : "f"(t4.w));
                }
              }
            }
#pragma unroll
            for (int j = 0; j < 32; ++j) f[j] += s_bias[c + j];
            // fin_out / fin_ld exist for the conv split-K path only, where fin_ld = Nout % 32 == 0: rows stay aligned
            if (row_ok) store_row32(reinterpret_cast<T*>(p.fin_out) + static_cast<long long>(row) * p.fin_ld + col0, f);
            if (want_stats) {
              float c1, c2;
              if constexpr (BNB) {
                float s1[32], s2[32];
                stat_terms<BNB, T>(p, row, row_ok, col0, f, s1, s2);
                c1 = warp_col_reduce32(s1);
                c2 = warp_col_reduce32(s2);
              } else {
                float s1[32];
#pragma unroll
                for (int j = 0; j < 32; ++j) s1[j] = row_ok ? stored_value(f[j], static_cast<const T*>(nullptr)) : 0.f;
                warp_col_sums_smem(s_tr, s1, c1, c2);
              }
              for (int w = 0; w < 4; ++w) {                     // warps in order: a reproducible sum
                if (warp == w) { s_stats[c + lane_id()] += c1; s_stats[BLOCK_N + c + lane_id()] += c2; }
                asm volatile("bar.sync 1, 128;" ::: "memory");
              }
            }
          }
        }
      }
      if (want_stats && (p.epi == EPI_BF16 || s_flag[1])) {
        // one committing CTA per (m-tile, n-tile): the n-tile's column sums are added in m-tile order
        asm volatile("bar.sync 1, 128;" ::: "memory");
        det_commit<1>(p.det, blockIdx.y, blockIdx.x, gridDim.x, s_stats, 2 * BLOCK_N, p.col_sum + n0, BLOCK_N, p.col_sumsq + n0,
                      et, 128);
      }
      }  // epilogue warps
    }
  }
  if (p.pub_flag != nullptr && warp < 4 && my_iters > 0) {
    // ---- publish: every CTA fences its (peer) stores; the last one to arrive releases the mailbox flag system-wide ----
    asm volatile("bar.sync 1, 128;");
    if (threadIdx.x == 0) {
      __threadfence_system();
      const uint32_t t = atomicAdd(p.pub_ticket, 1u);
      if (t == gridDim.x * gridDim.y * gridDim.z - 1u) {
        *p.pub_ticket = 0;
        const uint32_t value = *p.pub_seq + 1;
        *p.pub_seq = value;
        __threadfence_system();
        st_release_sys(p.pub_flag, value);
      }
    }
  }
  if (threadIdx.x == 0) SLB_STAMP(9);                          // epilogue thread 0 done
  __syncthreads();
  if (threadIdx.x == 0) SLB_STAMP(10);
#undef SLB_STAMP
}

// ----------------------------------------------------------------------------- host side
static long long* g_gemm_trace = nullptr;
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  // cuTensorMapEncodeTiled is a driver call: it needs a context bound to *this* thread.  Autograd worker threads may
  // reach us before any runtime call has bound the primary context (seen as CUresult 201) -> bind it once per thread.
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) { int d = 0; cudaGetDevice(&d); cudaSetDevice(d); ctx_bound = true; }   // capture-safe, unlike cudaFree(0)
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p) return nullptr;
    fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

// Tensor map, SWIZZLE_128B, inner box = 128 bytes.  dims/strides innermost first.  fp32 operands are encoded as
// TFLOAT32 (same 4-byte memory format; the copy engine rounds to tf32 on the way into shared memory, which is what
// cuDNN's TF32 convolutions do to their inputs).  SLB200_TMAP_F32=1 selects plain FLOAT32 (the MMA then truncates).
static int esize(int dtype) { return dtype == 1 ? 4 : 2; }
static CUtensorMapDataType tmap_dtype(int dtype) {
  if (dtype != 1) return CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  static int plain = -1;
  if (plain < 0) { const char* e = getenv("SLB200_TMAP_F32"); plain = (e && e[0] == '1') ? 1 : 0; }
  return plain ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_TFLOAT32;
}
static int make_tmap(CUtensorMap* m, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                     const uint32_t* box, int dtype, int mn_major = 0) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return -1;
  cuuint64_t gdim[5], gstr[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (i > 0) gstr[i - 1] = strides_bytes[i];
  }
  // MN-major fp32 (tf32) operands land unswizzled and are transposed in shared memory (sm90.cuh transpose_tf32_inplace)
  const CUtensorMapSwizzle sw = (dtype == 1 && mn_major) ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B;
  CUresult r = enc(m, tmap_dtype(dtype), rank, const_cast<void*>(base), gdim, gstr, bx, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -static_cast<int>(r) - 100;
}

static int tmap_2d(CUtensorMap* m, const void* base, uint64_t cols, uint64_t rows, uint64_t ld_elems, uint32_t box_cols,
                   uint32_t box_rows, int dtype = 0, int mn_major = 0) {
  const uint64_t e = esize(dtype);
  uint64_t dims[2] = {cols, rows};
  uint64_t str[2] = {e, ld_elems * e};
  uint32_t box[2] = {box_cols, box_rows};
  return make_tmap(m, base, 2, dims, str, box, dtype, mn_major);
}
static int tmap_nhwc(CUtensorMap* m, const void* base, int B, int H, int W, int C, int tb, int th, int tw, int dtype = 0,
                     int mn_major = 0) {
  const uint64_t e = esize(dtype);
  uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)B};
  uint64_t str[4] = {e, (uint64_t)C * e, (uint64_t)W * C * e, (uint64_t)H * W * C * e};
  uint32_t box[4] = {(uint32_t)(128 / e), (uint32_t)tw, (uint32_t)th, (uint32_t)tb};
  return make_tmap(m, base, 4, dims, str, box, dtype, mn_major);
}

template <int MODE, int BN, typename T, bool BNB = false, bool RAG = false>
static int launch(const CUtensorMap& a, const CUtensorMap& b, const GemmParams& p_in, dim3 grid, cudaStream_t st) {
  auto k = umma_gemm_kernel<MODE, BN, T, BNB, RAG>;
  GemmParams p = p_in;
  p.det = slb_det(st);
  if (p.det.part == nullptr) return -30;
  if (p.col_sum != nullptr && (grid.y > DET_TURN_BASE || (long long)grid.x * grid.y * 2 * BN > p.det.cap)) return -31;
  if (grid.z > 1 && p.tile_counters == nullptr && (long long)grid.x * grid.y > DET_COUNTERS - DET_TURN_BASE) return -32;
  static bool attr_done = false;
  if (!attr_done) {
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, SmemLayout<BN, T>::TOTAL);
    if (e != cudaSuccess) return -static_cast<int>(e) - 1000;
    attr_done = true;
  }
  cudaError_t e0 = launch_k(k, grid, dim3(288), SmemLayout<BN, T>::TOTAL, st, a, b, p);
  if (e0 != cudaSuccess) return -static_cast<int>(e0) - 2000;
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : -static_cast<int>(e) - 2000;
}

template <int MODE, bool RAG = false>
static int dispatch_bn(int bn, int dtype, const CUtensorMap& a, const CUtensorMap& b, const GemmParams& p, dim3 grid,
                       cudaStream_t st) {
  using bf = __nv_bfloat16;
  if constexpr (RAG) {                            // ragged pixel tiles: bf16 conv / dgrad / wgrad
    static_assert(MODE != MODE_GEMM, "ragged tiles are a conv geometry");
    if (dtype != 0 || p.bnb_y != nullptr) return -13;
    switch (bn) {
      case 32: if constexpr (MODE == MODE_CONV) return launch<MODE, 32, bf, false, true>(a, b, p, grid, st); else return -3;
      case 64: return launch<MODE, 64, bf, false, true>(a, b, p, grid, st);
      case 128: return launch<MODE, 128, bf, false, true>(a, b, p, grid, st);
      case 256: return launch<MODE, 256, bf, false, true>(a, b, p, grid, st);
      default: return -3;
    }
  }
  if (dtype == 1) {                               // fp32 tensors, wgmma tf32 (conv fwd / dgrad / wgrad only)
    if constexpr (MODE == MODE_GEMM) return -5;
    else {
      if (p.bnb_y != nullptr) return -6;
      switch (bn) {
        case 32: return launch<MODE, 32, float>(a, b, p, grid, st);
        case 64: return launch<MODE, 64, float>(a, b, p, grid, st);
        case 128: return launch<MODE, 128, float>(a, b, p, grid, st);
        case 256: return launch<MODE, 256, float>(a, b, p, grid, st);
        default: return -3;
      }
    }
  }
  if constexpr (MODE == MODE_CONV) {
    if (p.bnb_y != nullptr) {
      switch (bn) {
        case 64: return launch<MODE, 64, bf, true>(a, b, p, grid, st);
        case 128: return launch<MODE, 128, bf, true>(a, b, p, grid, st);
        case 256: return launch<MODE, 256, bf, true>(a, b, p, grid, st);
        default: return -3;
      }
    }
  }
  switch (bn) {
    case 32: return launch<MODE, 32, bf>(a, b, p, grid, st);
    case 64: return launch<MODE, 64, bf>(a, b, p, grid, st);
    case 128: return launch<MODE, 128, bf>(a, b, p, grid, st);
    case 256: return launch<MODE, 256, bf>(a, b, p, grid, st);
    default: return -3;
  }
}

template <int MODE, int BN, typename T, bool BNB = false, bool RAG = false>
static int preload_one() {
  cudaFuncAttributes a;
  return cudaFuncGetAttributes(&a, umma_gemm_kernel<MODE, BN, T, BNB, RAG>) == cudaSuccess ? 0 : 1;
}

static void pixel_box(int H, int W, int pixels, int* tb, int* th, int* tw) {
  *tw = W;
  int rows = pixels / W;           // full-width rows in the tile
  if (rows <= H) { *th = rows; *tb = 1; }
  else { *th = H; *tb = rows / H; }
}

// Does pixel_box tile the map exactly, so that tile t is the `pixels` consecutive NHWC pixels from t * pixels?  Power-of-
// two maps do.  Every other map (W = 28, 14, 7, 3, ...) takes the ragged instantiation with padded_box.
static bool pixel_box_exact(int H, int W, int pixels) {
  if (W > pixels || pixels % W != 0) return false;
  const int rows = pixels / W;
  return rows <= H ? H % rows == 0 : rows % H == 0;
}

// Padded power-of-two box of `pixels` slots for W <= pixels: tw = the smallest power of two >= W, th = min(the smallest
// power of two >= H, pixels / tw), tb = the rest.  Equal to pixel_box for power-of-two H and W.
static void padded_box(int H, int W, int pixels, int* tb, int* th, int* tw) {
  int w = 1, h = 1;
  while (w < W) w <<= 1;
  while (h < H) h <<= 1;
  if (h > pixels / w) h = pixels / w;
  *tw = w; *th = h; *tb = pixels / (w * h);
}

}  // namespace slb

using namespace slb;

extern "C" {

// Force-load every instantiation (CUDA lazy loading would otherwise load a kernel at its first launch, which can
// block behind a running flag-spinning kernel of a sibling stage sharing the GPU).
int slb_preload_gemm() {
  using bf = __nv_bfloat16;
  int bad = 0;
  bad += preload_one<MODE_CONV, 64, bf>() + preload_one<MODE_CONV, 128, bf>() + preload_one<MODE_CONV, 256, bf>() + preload_one<MODE_CONV, 32, bf>();
  bad += preload_one<MODE_WGRAD, 64, bf>() + preload_one<MODE_WGRAD, 128, bf>() + preload_one<MODE_WGRAD, 256, bf>() + preload_one<MODE_WGRAD, 32, bf>();
  bad += preload_one<MODE_GEMM, 32, bf>() + preload_one<MODE_GEMM, 64, bf>() + preload_one<MODE_GEMM, 128, bf>() + preload_one<MODE_GEMM, 256, bf>();
  bad += preload_one<MODE_CONV, 64, bf, true>() + preload_one<MODE_CONV, 128, bf, true>() + preload_one<MODE_CONV, 256, bf, true>();
  bad += preload_one<MODE_CONV, 64, float>() + preload_one<MODE_CONV, 128, float>() + preload_one<MODE_CONV, 256, float>() + preload_one<MODE_CONV, 32, float>();
  bad += preload_one<MODE_WGRAD, 64, float>() + preload_one<MODE_WGRAD, 128, float>() + preload_one<MODE_WGRAD, 256, float>() + preload_one<MODE_WGRAD, 32, float>();
  bad += preload_one<MODE_CONV, 32, bf, false, true>() + preload_one<MODE_CONV, 64, bf, false, true>() + preload_one<MODE_CONV, 128, bf, false, true>() + preload_one<MODE_CONV, 256, bf, false, true>();
  bad += preload_one<MODE_WGRAD, 64, bf, false, true>() + preload_one<MODE_WGRAD, 128, bf, false, true>() + preload_one<MODE_WGRAD, 256, bf, false, true>();
  return bad;
}

// The pixel box of a conv tile (pixels = 128) or wgrad K step (pixels = 64 bf16 / 32 fp32): out = {tb, th, tw, ragged}.
// ragged = 0: pixel_box over consecutive pixels; 1: padded_box; -1: no box (W > pixels).
void slb_conv_pixel_box(int H, int W, int pixels, int padded, int* out) {
  int tb = 0, th = 0, tw = 0, rag = 0;
  if (W < 1 || H < 1 || W > pixels) rag = -1;
  else if (!padded && pixel_box_exact(H, W, pixels)) pixel_box(H, W, pixels, &tb, &th, &tw);
  else { padded_box(H, W, pixels, &tb, &th, &tw); rag = 1; }
  out[0] = tb; out[1] = th; out[2] = tw; out[3] = rag;
}

// y[B,H,W,Cout] (pre-BN) = conv3x3(x[B,H,W,Cin], w[Cout][3][3][Cin]) + bias ; optional per-channel
// sum / sum-of-squares accumulation (caller zeroes them).  flip=1 computes the input gradient:
// x := dY [B,H,W,Cout_w], w as stored, out = dX[B,H,W,Cin_w]  (then Cin here means channels of A = Cout_w).
// dtype: 0 = bf16 tensors (wgmma bf16), 1 = fp32 tensors (wgmma tf32); x, w and y share it.
// block_n in {64,128,256} (0 = auto); k_split > 1 with tile_counters: every K slice stores its fp32 partial sums into
// `acc` ([k_split][M][Nout], acc_cap floats, no zeroing needed) and the last slice of a tile to arrive adds them in slice
// order and produces y.  Without tile_counters the slices add into `acc` ([M][Nout], zeroed by the caller) with vector
// red.add in slice order and slb_conv_finalize produces y.
struct BnbArgs { const void* y; const float *mean, *istd, *gamma, *beta; int relu, pool; };
struct PubArgs { uint32_t *ticket, *flag, *seq; };
static int conv_igemm_impl(const void* x, const void* w, void* y, const float* bias, float* col_sum, float* col_sumsq,
                           int B, int H, int W, int Ca, int Nout, int flip, int w_cin, int w_cout, int block_n, int k_split,
                           float* acc, long long acc_cap, uint32_t* tile_counters, const BnbArgs* bnb, int dtype, cudaStream_t st,
                           const PubArgs* pub = nullptr);

// conv / dgrad whose last CTA also publishes a mailbox flag (cut-head dgrad storing dX into the upstream stage's HBM)
int slb_conv3x3_igemm_pub(const void* x, const void* w, void* y, const float* bias, float* col_sum, float* col_sumsq,
                          int B, int H, int W, int Ca, int Nout, int flip, int w_cin, int w_cout, int block_n, int k_split,
                          float* acc, long long acc_cap, uint32_t* tile_counters, int dtype, uint32_t* pub_ticket, uint32_t* pub_flag,
                          uint32_t* pub_seq, cudaStream_t st) {
  if (k_split > 1 && tile_counters == nullptr) return -18;      // the flag must follow the *final* dX stores
  PubArgs pa = {pub_ticket, pub_flag, pub_seq};
  return conv_igemm_impl(x, w, y, bias, col_sum, col_sumsq, B, H, W, Ca, Nout, flip, w_cin, w_cout, block_n, k_split, acc,
                         acc_cap, tile_counters, nullptr, dtype, st, pub_flag != nullptr ? &pa : nullptr);
}

int slb_conv3x3_igemm(const void* x, const void* w, void* y, const float* bias, float* col_sum, float* col_sumsq,
                      int B, int H, int W, int Ca /*channels of A*/, int Nout /*output channels*/, int flip,
                      int w_cin /*Cin of the weight tensor*/, int w_cout, int block_n, int k_split, float* acc,
                      long long acc_cap, uint32_t* tile_counters, int dtype, cudaStream_t st) {
  return conv_igemm_impl(x, w, y, bias, col_sum, col_sumsq, B, H, W, Ca, Nout, flip, w_cin, w_cout, block_n, k_split, acc,
                         acc_cap, tile_counters, nullptr, dtype, st);
}

// dgrad whose epilogue also reduces the BatchNorm backward sums of the upstream block: dbeta / dgamma (zeroed by the
// caller) receive sum m*dX and sum m*dX*xhat; needs k_split == 1 or in-kernel finalisation (tile_counters).  bf16 only.
int slb_conv3x3_dgrad_bnstats(const void* dy, const void* w, void* dx, int B, int H, int W, int Ca, int Nout, int w_cin,
                              int w_cout, int block_n, int k_split, float* acc, long long acc_cap, uint32_t* tile_counters,
                              const void* up_y, const float* up_mean, const float* up_istd, const float* up_gamma,
                              const float* up_beta, int up_relu, int up_pool, float* dbeta, float* dgamma, cudaStream_t st) {
  if (k_split > 1 && tile_counters == nullptr) return -18;
  BnbArgs b = {up_y, up_mean, up_istd, up_gamma, up_beta, up_relu, up_pool};
  return conv_igemm_impl(dy, w, dx, nullptr, dbeta, dgamma, B, H, W, Ca, Nout, 1, w_cin, w_cout, block_n, k_split, acc,
                         acc_cap, tile_counters, &b, 0, st);
}

}  // extern "C"

static int conv_igemm_impl(const void* x, const void* w, void* y, const float* bias, float* col_sum, float* col_sumsq,
                           int B, int H, int W, int Ca, int Nout, int flip, int w_cin, int w_cout, int block_n, int k_split,
                           float* acc, long long acc_cap, uint32_t* tile_counters, const BnbArgs* bnb, int dtype, cudaStream_t st,
                           const PubArgs* pub) {
  const int KE = 128 / esize(dtype);
  if (Ca % KE != 0 || Nout % 32 != 0) return -10;
  const int M = B * H * W;
  if (B < 1 || H < 1 || W < 1 || W > 128) return -11;
  const bool rag = !pixel_box_exact(H, W, 128);
  if (rag) {
    // ragged tiles: single K slice, plain epilogue (split-K, BN statistics, fused BN-backward sums and the publish
    // are power-of-two-only options), bf16 only
    if (dtype != 0) return -13;
    if (k_split > 1 || col_sum != nullptr || col_sumsq != nullptr || bnb != nullptr || pub != nullptr) return -14;
  }
  int tb, th, tw;
  if (rag) padded_box(H, W, 128, &tb, &th, &tw);
  else pixel_box(H, W, 128, &tb, &th, &tw);
  if (tw * th * tb != 128) return -12;
  int bn = block_n > 0 ? block_n : (Nout >= 256 ? 256 : Nout);   // 32, 64, 128, 256
  if (bn > Nout) bn = Nout;
  if (Nout % bn) return -16;
  if (flip && bn < KE) return -4;                                  // MN-major B needs whole 128-byte groups
  CUtensorMap ta, tbm;
  int r = tmap_nhwc(&ta, x, B, H, W, Ca, tb, th, tw, dtype);
  if (r) return r;
  if (!flip) r = tmap_2d(&tbm, w, (uint64_t)9 * w_cin, w_cout, (uint64_t)9 * w_cin, KE, bn, dtype);
  else       r = tmap_2d(&tbm, w, (uint64_t)9 * w_cin, w_cout, (uint64_t)9 * w_cin, KE, KE, dtype, 1);
  if (r) return r;
  GemmParams p = {};
  p.M = M; p.N = Nout; p.k_iters = 9 * (Ca / KE);
  if (k_split < 1) k_split = 1;
  if (k_split > p.k_iters) k_split = p.k_iters;
  {  // no empty K slices (the tile semaphore counts exactly k_split arrivals)
    const int per = (p.k_iters + k_split - 1) / k_split;
    k_split = (p.k_iters + per - 1) / per;
  }
  p.k_split = k_split;
  p.a_mn = 0; p.b_mn = flip ? 1 : 0; p.ldo = Nout;
  if (k_split > 1) {
    if (acc == nullptr) return -17;
    // in-kernel finalisation: k_split partial tile sets [k_split][M][Nout]; otherwise one zeroed [M][Nout] accumulator
    if (acc_cap < (tile_counters != nullptr ? (long long)k_split : 1LL) * M * Nout) return -19;
    p.epi = EPI_F32_ATOMIC; p.out = acc;
    if (tile_counters != nullptr) {       // in-kernel finalisation by the last K-slice of every tile
      p.tile_counters = tile_counters; p.fin_out = y; p.fin_ld = Nout;
      p.bias = bias; p.col_sum = col_sum; p.col_sumsq = col_sumsq;
    }
  } else {
    p.epi = EPI_BF16; p.out = y;
    p.bias = bias; p.col_sum = col_sum; p.col_sumsq = col_sumsq;
  }
  p.C = Ca; p.tw = tw; p.th = th; p.tb = tb; p.H = H; p.W = W; p.flip = flip; p.b_row_stride = w_cin;
  if (bnb != nullptr) {
    p.bnb_y = reinterpret_cast<const __nv_bfloat16*>(bnb->y);
    p.bnb_mean = bnb->mean; p.bnb_istd = bnb->istd; p.bnb_gamma = bnb->gamma; p.bnb_beta = bnb->beta; p.bnb_relu = bnb->relu; p.bnb_pool = bnb->pool;
  }
  p.trace = g_gemm_trace;
  if (pub != nullptr) { p.pub_ticket = pub->ticket; p.pub_flag = pub->flag; p.pub_seq = pub->seq; }
  if (rag) {
    dim3 grid(((B + tb - 1) / tb) * ((H + th - 1) / th), Nout / bn, 1);
    return dispatch_bn<MODE_CONV, true>(bn, dtype, ta, tbm, p, grid, st);
  }
  dim3 grid((M + 127) / 128, Nout / bn, k_split);
  return dispatch_bn<MODE_CONV>(bn, dtype, ta, tbm, p, grid, st);
}

extern "C" {

// debugging aid: device buffer of 16 int64 that CTA (0,0,0) of the conv / wgrad kernels fills with clock64() stamps
void slb_set_gemm_trace(long long* buf) { g_gemm_trace = buf; }

// dw[Cout][3][3][Cin] (fp32, accumulated with red.add; caller zeroes) += sum_pixels dy (x) x ; x / dy typed by dtype
int slb_conv3x3_wgrad(const void* x, const void* dy, float* dw, int B, int H, int W, int Cin, int Cout, int k_split,
                      int block_n, int dtype, cudaStream_t st) {
  const int KE = 128 / esize(dtype);
  if (Cin % KE != 0 || Cout % KE != 0) return -10;
  const int pixels = B * H * W;
  if (B < 1 || H < 1 || W < 1 || W > KE) return -11;
  const bool rag = !pixel_box_exact(H, W, KE);     // ragged: one K step = one padded box (bf16 only)
  if (rag && dtype != 0) return -13;
  int tb, th, tw;
  if (rag) padded_box(H, W, KE, &tb, &th, &tw);
  else pixel_box(H, W, KE, &tb, &th, &tw);
  if (tw * th * tb != KE) return -12;
  int bn = block_n > 0 ? block_n : (Cin >= 128 ? 128 : Cin);
  if (bn > Cin) bn = Cin;
  if (Cin % bn || bn % KE) return -16;
  CUtensorMap ta, tbm;
  int r = tmap_nhwc(&ta, dy, B, H, W, Cout, tb, th, tw, dtype, 1);
  if (r) return r;
  r = tmap_nhwc(&tbm, x, B, H, W, Cin, tb, th, tw, dtype, 1);
  if (r) return r;
  GemmParams p = {};
  const int rows = 9 * Cout;
  p.M = ((rows + 127) / 128) * 128; p.N = Cin; p.k_iters = (pixels + KE - 1) / KE;   // tail pixels are TMA zero-fill
  if (rag) p.k_iters = ((B + tb - 1) / tb) * ((H + th - 1) / th);
  const int m_tiles = p.M / 128, n_tiles = Cin / bn;
  if (k_split <= 0) {
    int sms = 0, dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
    k_split = (sms + m_tiles * n_tiles - 1) / (m_tiles * n_tiles);
    const int cap = p.k_iters / 4 > 1 ? p.k_iters / 4 : 1;      // keep >= 4 K iterations per CTA
    if (k_split > cap) k_split = cap;
    if (k_split < 1) k_split = 1;
  }
  if (k_split > p.k_iters) k_split = p.k_iters;
  {
    const int per = (p.k_iters + k_split - 1) / k_split;
    k_split = (p.k_iters + per - 1) / per;
  }
  p.k_split = k_split;
  // a single K slice owns its output tile: plain stores (no zero-fill, no atomics)
  p.a_mn = 1; p.b_mn = 1; p.epi = k_split > 1 ? EPI_F32_ATOMIC : EPI_F32_STORE; p.out = dw; p.ldo = Cin;
  p.rmod = Cout; p.rmul1 = (long long)9 * Cin; p.rmul2 = Cin; p.m_valid_mod = 9;
  p.C = Cout; p.tw = tw; p.th = th; p.tb = tb; p.H = H; p.W = W; p.Cout = Cout;
  p.trace = g_gemm_trace;
  dim3 grid(m_tiles, n_tiles, k_split);
  if (rag) return dispatch_bn<MODE_WGRAD, true>(bn, dtype, ta, tbm, p, grid, st);
  return dispatch_bn<MODE_WGRAD>(bn, dtype, ta, tbm, p, grid, st);
}

// Generic bf16 GEMM:  D[M,N] = A x B  with fp32 result.
//   A: a_mn==0 -> stored [M][K] (K contiguous, lda); a_mn==1 -> stored [K][M] (M contiguous, lda)
//   B: b_mn==0 -> stored [N][K];                     b_mn==1 -> stored [K][N]
//   epi: 1 = atomic add into out[M][ldo], 2 = atomic add into transposed out[N][ldo], 3 = plain store out[M][ldo]
int slb_gemm_bf16(const void* A, const void* Bm, float* out, int M, int N, int K, int a_mn, int b_mn, long long lda,
                  long long ldb, long long ldo, int epi, int k_split, int block_n, cudaStream_t st) {
  if (block_n != 32 && block_n != 64 && block_n != 128 && block_n != 256) return -3;
  CUtensorMap ta, tbm;
  int r;
  if (!a_mn) r = tmap_2d(&ta, A, K, M, lda, 64, 128);
  else       r = tmap_2d(&ta, A, M, K, lda, 64, 64);
  if (r) return r;
  if (!b_mn) r = tmap_2d(&tbm, Bm, K, N, ldb, 64, block_n);
  else       r = tmap_2d(&tbm, Bm, N, K, ldb, 64, 64);
  if (r) return r;
  if (b_mn && block_n < 64) return -4;
  GemmParams p = {};
  p.M = M; p.N = N; p.k_iters = (K + 63) / 64;
  if (k_split < 1) k_split = 1;
  if (k_split > p.k_iters) k_split = p.k_iters;
  if (epi == EPI_F32_STORE) k_split = 1;
  {  // no empty K slices: every slice takes its turn
    const int per = (p.k_iters + k_split - 1) / k_split;
    k_split = (p.k_iters + per - 1) / per;
  }
  p.k_split = k_split; p.a_mn = a_mn; p.b_mn = b_mn; p.epi = epi; p.out = out; p.ldo = ldo;
  dim3 grid((M + 127) / 128, (N + block_n - 1) / block_n, k_split);
  return dispatch_bn<MODE_GEMM>(block_n, 0, ta, tbm, p, grid, st);
}

// Transformer GEMM: out_bf16[M][ldo] = act(A * B + bias + residual), optional pre-activation copy in `aux`.
// Same operand-major options as slb_gemm_bf16; no split-K (token counts give >= 1 wave of 128 x block_n tiles).
int slb_gemm_bf16_act(const void* A, const void* Bm, void* out, int M, int N, int K, int a_mn, int b_mn, long long lda,
                      long long ldb, long long ldo, int block_n, const float* bias, int act, void* aux,
                      const void* residual, cudaStream_t st) {
  if (block_n != 32 && block_n != 64 && block_n != 128 && block_n != 256) return -3;
  if (b_mn && block_n < 64) return -4;
  CUtensorMap ta, tbm;
  int r;
  if (!a_mn) r = tmap_2d(&ta, A, K, M, lda, 64, 128);
  else       r = tmap_2d(&ta, A, M, K, lda, 64, 64);
  if (r) return r;
  if (!b_mn) r = tmap_2d(&tbm, Bm, K, N, ldb, 64, block_n);
  else       r = tmap_2d(&tbm, Bm, N, K, ldb, 64, 64);
  if (r) return r;
  GemmParams p = {};
  p.M = M; p.N = N; p.k_iters = (K + 63) / 64; p.k_split = 1;
  p.a_mn = a_mn; p.b_mn = b_mn; p.epi = EPI_BF16; p.out = out; p.ldo = ldo;
  p.bias = bias; p.act = act; p.aux_out = reinterpret_cast<__nv_bfloat16*>(aux);
  p.residual = reinterpret_cast<const __nv_bfloat16*>(residual);
  dim3 grid((M + 127) / 128, (N + block_n - 1) / block_n, 1);
  return dispatch_bn<MODE_GEMM>(block_n, 0, ta, tbm, p, grid, st);
}

// Classifier head with fp32 output: out_f32[M][ldo] = A[M][K] * B[N][K]^T + bias (both operands K-major, plain store,
// no split-K).  The logits go straight to the loss / accuracy kernel without a bf16 rounding or a cast.
int slb_gemm_bf16_bias_f32(const void* A, const void* Bm, float* out, int M, int N, int K, long long lda, long long ldb,
                           long long ldo, int block_n, const float* bias, cudaStream_t st) {
  if (block_n != 32 && block_n != 64 && block_n != 128 && block_n != 256) return -3;
  if (M < 1 || N < 1 || K < 1 || K % 8 || lda < K || ldb < K || ldo < N || (lda | ldb) & 7) return -4;
  if (!A || !Bm || !out || !bias || (reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(Bm)) & 15 ||
      (reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(bias)) & 3)
    return -5;
  CUtensorMap ta, tbm;
  int r;
  if ((r = tmap_2d(&ta, A, K, M, lda, 64, 128))) return r;
  if ((r = tmap_2d(&tbm, Bm, K, N, ldb, 64, block_n))) return r;
  GemmParams p = {};
  p.M = M; p.N = N; p.k_iters = (K + 63) / 64; p.k_split = 1;
  p.a_mn = 0; p.b_mn = 0; p.epi = EPI_F32_STORE; p.out = out; p.ldo = ldo; p.bias = bias;
  dim3 grid((M + 127) / 128, (N + block_n - 1) / block_n, 1);
  return dispatch_bn<MODE_GEMM>(block_n, 0, ta, tbm, p, grid, st);
}

}  // extern "C"
