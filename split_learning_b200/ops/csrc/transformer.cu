// Encoder-block kernels for the token-model families (KWT / ViT / BERT; SURVEY §2.7 G11):
//
//   attn_fwd_kernel / attn_bwd_kernel
//       dense softmax attention for S <= 128, one CTA (one warpgroup) per (batch, head), everything on wgmma:
//       S = Q K^T and O = P V (forward), S / dP / dV / dQ / dK (backward) are 128-row tiles computed as two 64-row
//       wgmma halves whose operands are TMA boxes of the *packed* projection output (no head split / transpose
//       copies exist); the softmax runs on the register accumulators (a row spans the 4 threads of a quad) and
//       writes P / dS back to shared memory in the 128B-swizzled layout, so the same bytes serve as the K-major A
//       operand (P V, dS K) and as the MN-major A operand (P^T dO, dS^T Q).  Probability dropout is a counter
//       hash, regenerated in the backward pass; the key-padding bias is optional.
//       (reference math: src/model/BERT_AGNEWS.py:56-80, nn.MultiheadAttention in src/model/KWT_SPEECHCOMMANDS.py:5-23)
//   ln_fwd_kernel / ln_bwd_kernel      LayerNorm with a fused (dropout(x) + residual) prologue
//   act_bwd_kernel, colsum_kernel      GELU / tanh / ReLU backward, bias gradient
//   dropout_bf16_kernel                hash dropout (same kernel re-applies the mask in backward)
//   embed3_fwd_kernel / embed3_bwd_kernel   word + position + token-type embedding gather / scatter-add
#include "sm90.cuh"

namespace slb {

// ----------------------------------------------------------------------------- helpers
__device__ __forceinline__ uint32_t fmix32(uint32_t h) {
  h ^= h >> 16; h *= 0x85ebca6bu; h ^= h >> 13; h *= 0xc2b2ae35u; h ^= h >> 16;
  return h;
}
// keep-scale of element `idx` under dropout probability p: 0 or 1/(1-p)
__device__ __forceinline__ float drop_scale(uint32_t seed, uint32_t idx, float p, float inv_keep) {
  const uint32_t r = fmix32(idx * 0x9E3779B9u + seed) >> 8;            // 24 random bits
  return (static_cast<float>(r) * (1.f / 16777216.f) >= p) ? inv_keep : 0.f;
}
__device__ __forceinline__ uint32_t mix_seed(uint32_t seed, const uint32_t* ofs) {
  return ofs ? seed + __ldg(ofs) * 0x9E3779B9u : seed;
}

// byte offset of the 16-byte chunk holding columns [c8*8, c8*8+8) of row r inside a [128 rows][128 cols] bf16 tile
// stored as two 64-column panels of 128-byte rows with the 128B swizzle (what TMA writes for a {64, 128} box).
__device__ __forceinline__ uint32_t sw128_chunk(int r, int c8) {
  const int panel = c8 >> 3, cc = c8 & 7;
  return static_cast<uint32_t>(panel * 16384 + r * 128 + ((cc ^ (r & 7)) << 4));
}

struct AttnParams {
  int B, S, H, Dh;                 // Dh in {32, 64}; S <= 128
  int q_col, k_col, v_col, do_col; // first column of head 0 inside the Q / K / V / dO tensors
  float scale;                     // 1 / sqrt(Dh)
  const float* key_bias;           // [B][S] additive bias on the logits, or nullptr
  float p_drop;
  uint32_t seed;
  const uint32_t* seed_ofs;        // optional device counter mixed into the seed (fresh masks per CUDA-graph replay)
  __nv_bfloat16* out;              // forward: O [B*S][ldo], head h at column h*Dh
  long long ldo;
  float* lse;                      // [B*H][128] log-sum-exp of the scaled logits
  __nv_bfloat16 *dq, *dk, *dv;     // backward outputs, head h at column d?_col + h*Dh
  long long lddq, lddk, lddv;
  int dq_col, dk_col, dv_col;
};

static constexpr int ATT_TILE = 16384;                       // one [128][64] bf16 box
static constexpr int ATT_FWD_SMEM = 5 * ATT_TILE + 1024 + 1024;   // Q, K, V, P -> 2 CTAs per SM
static constexpr int ATT_BWD_SMEM = 4 * ATT_TILE + 2 * 32768 + 1024 + 1024;

// Rows of a thread inside a warpgroup's 64-row wgmma fragment: r and r + 8 (plus 64 for the second half of the tile);
// element d[4i + e] sits in column 8i + 2 * (lane % 4) + (e & 1).
__device__ __forceinline__ int frag_row(int half) { return 64 * half + 16 * (threadIdx.x >> 5) + (lane_id() >> 2); }
__device__ __forceinline__ int frag_col(int i) { return 8 * i + 2 * (lane_id() & 3); }
// sum / max over the four threads that share a row of the fragment
__device__ __forceinline__ float quad_sum(float x) {
  x += __shfl_xor_sync(0xffffffffu, x, 1);
  return x + __shfl_xor_sync(0xffffffffu, x, 2);
}
__device__ __forceinline__ float quad_max(float x) {
  x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 1));
  return fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 2));
}
// two adjacent bf16 values at (row, col) of a [128][128] tile in the two-panel 128B-swizzled layout (col even)
__device__ __forceinline__ void st_tile_pair(uint8_t* tile, int row, int col, float lo, float hi) {
  *reinterpret_cast<uint32_t*>(tile + sw128_chunk(row, col >> 3) + (col & 7) * 2) = pack_bf16x2(lo, hi);
}

// Write one head's slice of a 64 x 64 accumulator fragment (rows [64 * half, 64 * half + 64) of the tile): columns
// [n_off, n_off + Dh) go to dst[row * ld + col - n_off] for rows < S, scaled by mul[0] / mul[1] (rows r / r + 8).
__device__ __forceinline__ void store_head_frag(const float (&o)[32], int half, __nv_bfloat16* dst, long long ld, int n_off,
                                                int Dh, int S, const float (&mul)[2]) {
  const int r = frag_row(half);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int col = frag_col(i);
    if (col < n_off || col >= n_off + Dh) continue;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int row = r + 8 * hh;
      if (row < S)
        *reinterpret_cast<uint32_t*>(dst + row * ld + col - n_off) =
            pack_bf16x2(o[4 * i + 2 * hh] * mul[hh], o[4 * i + 2 * hh + 1] * mul[hh]);
    }
  }
}

// ----------------------------------------------------------------------------- attention forward
__global__ void __launch_bounds__(128, 2)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = smem + ATT_TILE;
  uint8_t* sV = smem + 2 * ATT_TILE;
  uint8_t* sP = smem + 3 * ATT_TILE;   // [128][128] bf16, two panels
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 5 * ATT_TILE);

  const int tid = threadIdx.x;
  const int b = blockIdx.x / p.H, h = blockIdx.x - b * p.H;
  const int qc = p.q_col + h * p.Dh, kc = p.k_col + h * p.Dh, vc = p.v_col + h * p.Dh;
  const int ksteps = p.Dh >> 4;

  if (tid == 0) {
    tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV);
    mbar_init(&bars[0], 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_expect_tx(&bars[0], 3 * ATT_TILE);
    tma_load_2d(sQ, &tmQ, &bars[0], qc & ~63, b * p.S);
    tma_load_2d(sK, &tmK, &bars[0], kc & ~63, b * p.S);
    tma_load_2d(sV, &tmV, &bars[0], vc & ~63, b * p.S);
  }
  mbar_wait(&bars[0], 0);

  const uint32_t qa = smem_u32(sQ) + ((qc & 63) >> 4) * 32, ka = smem_u32(sK) + ((kc & 63) >> 4) * 32;
  const float* kb = p.key_bias ? p.key_bias + static_cast<long long>(b) * p.S : nullptr;
  constexpr float LOG2E = 1.4426950408889634f;
  const uint32_t seed = mix_seed(p.seed, p.seed_ofs);
  const float inv_keep = p.p_drop > 0.f ? 1.f / (1.f - p.p_drop) : 1.f;
  float inv_sum[2][2];
  // ---- S = Q K^T and the softmax, one 64-row half of the tile at a time (fragment rows r, r + 8)
#pragma unroll 1
  for (int half = 0; half < 2; ++half) {
    float s[64];
    wgmma_fence();
    for (int k = 0; k < ksteps; ++k)
      wgmma_bf16_n128<0, 0>(s, wg_desc_sw128(qa + half * 8192 + k * 32, 16, 1024), wg_desc_sw128(ka + k * 32, 16, 1024), k != 0);
    wgmma_commit();
    wgmma_wait<0>();
    const int r = frag_row(half);
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < 16; ++i) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int col = frag_col(i) + (e & 1);
        const float x = col < p.S ? s[4 * i + e] * p.scale + (kb ? __ldg(kb + col) : 0.f) : -INFINITY;
        s[4 * i + e] = x;
        mx[e >> 1] = fmaxf(mx[e >> 1], x);
      }
    }
    mx[0] = quad_max(mx[0]);
    mx[1] = quad_max(mx[1]);
    float sum[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 16; ++i) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int row = r + 8 * hh;
        const uint32_t idx0 = (static_cast<uint32_t>(blockIdx.x) * 128u + row) * 128u;
        float e2[2];
#pragma unroll
        for (int t = 0; t < 2; ++t) {
          const int col = frag_col(i) + t;
          float x = 0.f;
          if (col < p.S) {
            x = exp2f((s[4 * i + 2 * hh + t] - mx[hh]) * LOG2E);
            sum[hh] += x;
            if (p.p_drop > 0.f) x *= drop_scale(seed, idx0 + col, p.p_drop, inv_keep);
          }
          e2[t] = x;
        }
        st_tile_pair(sP, row, frag_col(i), e2[0], e2[1]);
      }
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      sum[hh] = quad_sum(sum[hh]);
      inv_sum[half][hh] = 1.f / sum[hh];
      const int row = r + 8 * hh;
      if (row < p.S && (lane_id() & 3) == 0) p.lse[static_cast<long long>(blockIdx.x) * 128 + row] = mx[hh] + logf(sum[hh]);
    }
  }
  fence_proxy_async();                 // generic-proxy smem writes -> visible to the tensor core (async proxy)
  __syncthreads();
  // ---- O~ = P~ V  (A = P K-major, B = V MN-major), normalised by the row sums on the way out
  const uint32_t pa = smem_u32(sP), va = smem_u32(sV);
  __nv_bfloat16* dst = p.out + static_cast<long long>(b) * p.S * p.ldo + h * p.Dh;
#pragma unroll 1
  for (int half = 0; half < 2; ++half) {
    float o[32];
    wgmma_fence();
    for (int k = 0; k < 8; ++k)
      wgmma_bf16_n64<0, 1>(o, wg_desc_sw128(pa + half * 8192 + (k >> 2) * 16384 + (k & 3) * 32, 16, 1024),
                           wg_desc_sw128(va + k * 2048, 16384, 1024), k != 0);
    wgmma_commit();
    wgmma_wait<0>();
    store_head_frag(o, half, dst, p.ldo, vc & 63, p.Dh, p.S, inv_sum[half]);
  }
}

// ----------------------------------------------------------------------------- attention backward
__global__ void __launch_bounds__(128, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmDO,
                const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = smem + ATT_TILE;
  uint8_t* sV = smem + 2 * ATT_TILE;
  uint8_t* sdO = smem + 3 * ATT_TILE;
  uint8_t* sP = smem + 4 * ATT_TILE;                 // dropped probabilities  P~ = P * keep/(1-p)
  uint8_t* sdS = sP + 32768;                          // dS = P * (dP~ - D) * scale
  uint64_t* bars = reinterpret_cast<uint64_t*>(sdS + 32768);

  const int tid = threadIdx.x;
  const int b = blockIdx.x / p.H, h = blockIdx.x - b * p.H;
  const int qc = p.q_col + h * p.Dh, kc = p.k_col + h * p.Dh, vc = p.v_col + h * p.Dh, oc = p.do_col + h * p.Dh;
  const int ksteps = p.Dh >> 4;

  if (tid == 0) {
    tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV); tma_prefetch_desc(&tmDO);
    mbar_init(&bars[0], 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_expect_tx(&bars[0], 4 * ATT_TILE);
    tma_load_2d(sQ, &tmQ, &bars[0], qc & ~63, b * p.S);
    tma_load_2d(sK, &tmK, &bars[0], kc & ~63, b * p.S);
    tma_load_2d(sV, &tmV, &bars[0], vc & ~63, b * p.S);
    tma_load_2d(sdO, &tmDO, &bars[0], oc & ~63, b * p.S);
  }
  mbar_wait(&bars[0], 0);

  const float* kb = p.key_bias ? p.key_bias + static_cast<long long>(b) * p.S : nullptr;
  constexpr float LOG2E = 1.4426950408889634f;
  const uint32_t seed = mix_seed(p.seed, p.seed_ofs);
  const float inv_keep = p.p_drop > 0.f ? 1.f / (1.f - p.p_drop) : 1.f;
  {
    const uint32_t qa = smem_u32(sQ) + ((qc & 63) >> 4) * 32, ka = smem_u32(sK) + ((kc & 63) >> 4) * 32;
    const uint32_t va = smem_u32(sV) + ((vc & 63) >> 4) * 32, oa = smem_u32(sdO) + ((oc & 63) >> 4) * 32;
#pragma unroll 1
    for (int half = 0; half < 2; ++half) {
      float s[64], g[64];
      wgmma_fence();
      for (int k = 0; k < ksteps; ++k)                                   // S = Q K^T
        wgmma_bf16_n128<0, 0>(s, wg_desc_sw128(qa + half * 8192 + k * 32, 16, 1024), wg_desc_sw128(ka + k * 32, 16, 1024), k != 0);
      for (int k = 0; k < ksteps; ++k)                                   // dP = dO V^T
        wgmma_bf16_n128<0, 0>(g, wg_desc_sw128(oa + half * 8192 + k * 32, 16, 1024), wg_desc_sw128(va + k * 32, 16, 1024), k != 0);
      wgmma_commit();
      wgmma_wait<0>();
      const int r = frag_row(half);
      float lse[2], D[2] = {0.f, 0.f};
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
        lse[hh] = (r + 8 * hh) < p.S ? p.lse[static_cast<long long>(blockIdx.x) * 128 + r + 8 * hh] : 0.f;
      // P -> s, dP * mask -> g, P~ -> smem, D = rowsum(P~ * dP)
#pragma unroll
      for (int i = 0; i < 16; ++i) {
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int row = r + 8 * hh;
          const uint32_t idx0 = (static_cast<uint32_t>(blockIdx.x) * 128u + row) * 128u;
          float e2[2];
#pragma unroll
          for (int t = 0; t < 2; ++t) {
            const int col = frag_col(i) + t, j = 4 * i + 2 * hh + t;
            float x = 0.f, mk = 1.f;
            if (col < p.S && row < p.S) {
              x = exp2f((s[j] * p.scale + (kb ? __ldg(kb + col) : 0.f) - lse[hh]) * LOG2E);
              if (p.p_drop > 0.f) mk = drop_scale(seed, idx0 + col, p.p_drop, inv_keep);
            }
            s[j] = x;
            g[j] *= mk;
            D[hh] += x * g[j];
            e2[t] = x * mk;
          }
          st_tile_pair(sP, row, frag_col(i), e2[0], e2[1]);
        }
      }
      D[0] = quad_sum(D[0]);
      D[1] = quad_sum(D[1]);
      // dS = P * (dP * mask - D) * scale -> smem
#pragma unroll
      for (int i = 0; i < 16; ++i) {
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int j = 4 * i + 2 * hh;
          st_tile_pair(sdS, r + 8 * hh, frag_col(i), s[j] * (g[j] - D[hh]) * p.scale, s[j + 1] * (g[j + 1] - D[hh]) * p.scale);
        }
      }
    }
  }
  fence_proxy_async();
  __syncthreads();
  const uint32_t pa = smem_u32(sP), sa = smem_u32(sdS), qa = smem_u32(sQ), ka = smem_u32(sK), oa = smem_u32(sdO);
  const long long row0 = static_cast<long long>(b) * p.S;
  const float one[2] = {1.f, 1.f};
#pragma unroll 1
  for (int half = 0; half < 2; ++half) {
    float o[32];
    wgmma_fence();
    for (int k = 0; k < 8; ++k)        // dV[key][d] = sum_q P~[q][key] dO[q][d]   (A = P~ MN-major, B = dO MN-major)
      wgmma_bf16_n64<1, 1>(o, wg_desc_sw128(pa + half * 16384 + k * 2048, 16384, 1024), wg_desc_sw128(oa + k * 2048, 16384, 1024),
                           k != 0);
    wgmma_commit();
    wgmma_wait<0>();
    store_head_frag(o, half, p.dv + row0 * p.lddv + p.dv_col + h * p.Dh, p.lddv, oc & 63, p.Dh, p.S, one);
    wgmma_fence();
    for (int k = 0; k < 8; ++k)        // dQ[q][d] = sum_key dS[q][key] K[key][d]  (A = dS K-major, B = K MN-major)
      wgmma_bf16_n64<0, 1>(o, wg_desc_sw128(sa + half * 8192 + (k >> 2) * 16384 + (k & 3) * 32, 16, 1024),
                           wg_desc_sw128(ka + k * 2048, 16384, 1024), k != 0);
    wgmma_commit();
    wgmma_wait<0>();
    store_head_frag(o, half, p.dq + row0 * p.lddq + p.dq_col + h * p.Dh, p.lddq, kc & 63, p.Dh, p.S, one);
    wgmma_fence();
    for (int k = 0; k < 8; ++k)        // dK[key][d] = sum_q dS[q][key] Q[q][d]    (A = dS MN-major, B = Q MN-major)
      wgmma_bf16_n64<1, 1>(o, wg_desc_sw128(sa + half * 16384 + k * 2048, 16384, 1024), wg_desc_sw128(qa + k * 2048, 16384, 1024),
                           k != 0);
    wgmma_commit();
    wgmma_wait<0>();
    store_head_frag(o, half, p.dk + row0 * p.lddk + p.dk_col + h * p.Dh, p.lddk, qc & 63, p.Dh, p.S, one);
  }
}

// ----------------------------------------------------------------------------- LayerNorm
// y = LN(pre) * gamma + beta,  pre = drop(x) + res  (drop / res optional); one warp per row; D % 2 == 0.
__global__ void __launch_bounds__(256)
ln_fwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ res, const float* __restrict__ gamma,
              const float* __restrict__ beta, __nv_bfloat16* __restrict__ y, __nv_bfloat16* __restrict__ pre,
              float* __restrict__ mean, float* __restrict__ rstd, int rows, int D, float eps, float p_drop, uint32_t seed,
              const uint32_t* __restrict__ seed_ofs) {
  pdl_wait();
  seed = mix_seed(seed, seed_ofs);
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = lane_id(), D2 = D >> 1;
  const __nv_bfloat162* x2 = reinterpret_cast<const __nv_bfloat162*>(x + static_cast<long long>(row) * D);
  const __nv_bfloat162* r2 = res ? reinterpret_cast<const __nv_bfloat162*>(res + static_cast<long long>(row) * D) : nullptr;
  __nv_bfloat162* p2 = pre ? reinterpret_cast<__nv_bfloat162*>(pre + static_cast<long long>(row) * D) : nullptr;
  __nv_bfloat162* y2 = reinterpret_cast<__nv_bfloat162*>(y + static_cast<long long>(row) * D);
  const float inv_keep = p_drop > 0.f ? 1.f / (1.f - p_drop) : 1.f;
  float s1 = 0.f, s2 = 0.f;
  for (int i = lane; i < D2; i += 32) {
    float2 v = __bfloat1622float2(x2[i]);
    if (p_drop > 0.f) {
      const uint32_t idx = static_cast<uint32_t>(row) * D + 2 * i;
      v.x *= drop_scale(seed, idx, p_drop, inv_keep);
      v.y *= drop_scale(seed, idx + 1, p_drop, inv_keep);
    }
    if (r2) { const float2 r = __bfloat1622float2(r2[i]); v.x += r.x; v.y += r.y; }
    const __nv_bfloat162 hb = __floats2bfloat162_rn(v.x, v.y);      // statistics of the values the backward re-reads
    if (p2) p2[i] = hb;
    const float2 w = __bfloat1622float2(hb);
    s1 += w.x + w.y;
    s2 += w.x * w.x + w.y * w.y;
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
  const float mu = s1 / D, var = fmaxf(s2 / D - mu * mu, 0.f), rs = rsqrtf(var + eps);
  if (lane == 0) { mean[row] = mu; rstd[row] = rs; }
  __syncwarp();
  for (int i = lane; i < D2; i += 32) {
    float2 v;
    if (p2) v = __bfloat1622float2(p2[i]);
    else    v = __bfloat1622float2(x2[i]);                               // no prologue: pre == x
    const float2 g = reinterpret_cast<const float2*>(gamma)[i], bb = reinterpret_cast<const float2*>(beta)[i];
    y2[i] = __floats2bfloat162_rn((v.x - mu) * rs * g.x + bb.x, (v.y - mu) * rs * g.y + bb.y);
  }
}

// dpre = rstd * (g*dy - mean(g*dy) - xhat * mean(g*dy*xhat));  dgamma += dy*xhat, dbeta += dy.
// Each lane owns the column pairs lane, lane+32, ...; for D <= 1024 (16 pairs) the dgamma / dbeta partial sums of all the
// rows a warp visits stay in registers and reach shared memory once per warp (the first version did one shared-memory
// atomic per element: 0.14 of HBM bandwidth at 16 k tokens).
template <bool REGS>
__global__ void __launch_bounds__(256)
ln_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ pre, const float* __restrict__ gamma,
              const float* __restrict__ mean, const float* __restrict__ rstd, __nv_bfloat16* __restrict__ dpre,
              float* __restrict__ dgamma, float* __restrict__ dbeta, int rows, int D, int rows_per_block) {
  extern __shared__ float s_acc[];                 // [2][D]
  pdl_wait();
  for (int i = threadIdx.x; i < 2 * D; i += blockDim.x) s_acc[i] = 0.f;
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = lane_id(), nw = blockDim.x >> 5, D2 = D >> 1;
  const int r0 = blockIdx.x * rows_per_block, r1 = min(rows, r0 + rows_per_block);
  constexpr int MAXP = REGS ? 16 : 1;
  float2 ag[MAXP], ab[MAXP];
#pragma unroll
  for (int k = 0; k < MAXP; ++k) { ag[k] = make_float2(0.f, 0.f); ab[k] = make_float2(0.f, 0.f); }
  for (int row = r0 + warp; row < r1; row += nw) {
    const __nv_bfloat162* g2 = reinterpret_cast<const __nv_bfloat162*>(dy + static_cast<long long>(row) * D);
    const __nv_bfloat162* x2 = reinterpret_cast<const __nv_bfloat162*>(pre + static_cast<long long>(row) * D);
    __nv_bfloat162* o2 = reinterpret_cast<__nv_bfloat162*>(dpre + static_cast<long long>(row) * D);
    const float mu = mean[row], rs = rstd[row];
    float a = 0.f, bsum = 0.f;
    if constexpr (REGS) {
#pragma unroll
      for (int k = 0; k < MAXP; ++k) {
        const int i = lane + 32 * k;
        if (i < D2) {
          const float2 g = __bfloat1622float2(g2[i]), x = __bfloat1622float2(x2[i]);
          const float2 w = reinterpret_cast<const float2*>(gamma)[i];
          const float xh0 = (x.x - mu) * rs, xh1 = (x.y - mu) * rs;
          a += g.x * w.x + g.y * w.y;
          bsum += g.x * w.x * xh0 + g.y * w.y * xh1;
          ag[k].x += g.x * xh0; ag[k].y += g.y * xh1;
          ab[k].x += g.x;       ab[k].y += g.y;
        }
      }
    } else {
      for (int i = lane; i < D2; i += 32) {
        const float2 g = __bfloat1622float2(g2[i]), x = __bfloat1622float2(x2[i]);
        const float2 w = reinterpret_cast<const float2*>(gamma)[i];
        const float xh0 = (x.x - mu) * rs, xh1 = (x.y - mu) * rs;
        a += g.x * w.x + g.y * w.y;
        bsum += g.x * w.x * xh0 + g.y * w.y * xh1;
        if (dgamma) {
          atomicAdd(&s_acc[2 * i], g.x * xh0);
          atomicAdd(&s_acc[2 * i + 1], g.y * xh1);
          atomicAdd(&s_acc[D + 2 * i], g.x);
          atomicAdd(&s_acc[D + 2 * i + 1], g.y);
        }
      }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); bsum += __shfl_xor_sync(0xffffffffu, bsum, o); }
    a /= D; bsum /= D;
    for (int i = lane; i < D2; i += 32) {
      const float2 g = __bfloat1622float2(g2[i]), x = __bfloat1622float2(x2[i]);
      const float2 w = reinterpret_cast<const float2*>(gamma)[i];
      const float xh0 = (x.x - mu) * rs, xh1 = (x.y - mu) * rs;
      o2[i] = __floats2bfloat162_rn(rs * (g.x * w.x - a - xh0 * bsum), rs * (g.y * w.y - a - xh1 * bsum));
    }
  }
  if constexpr (REGS) {
    if (dgamma) {
#pragma unroll
      for (int k = 0; k < MAXP; ++k) {
        const int i = lane + 32 * k;
        if (i < D2) {
          atomicAdd(&s_acc[2 * i], ag[k].x);
          atomicAdd(&s_acc[2 * i + 1], ag[k].y);
          atomicAdd(&s_acc[D + 2 * i], ab[k].x);
          atomicAdd(&s_acc[D + 2 * i + 1], ab[k].y);
        }
      }
    }
  }
  __syncthreads();
  if (dgamma)
    for (int i = threadIdx.x; i < D; i += blockDim.x) {
      atomicAdd(dgamma + i, s_acc[i]);
      atomicAdd(dbeta + i, s_acc[D + i]);
    }
}

// ----------------------------------------------------------------------------- pointwise
// dz = dy * act'(.) ; kind 1 ReLU (ref = pre-activation), 2 GELU-erf (ref = pre-activation), 3 tanh (ref = output)
__global__ void __launch_bounds__(256)
act_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ ref, __nv_bfloat16* __restrict__ dz,
               long long n2, int kind) {
  pdl_wait();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n2;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float2 g = __bfloat1622float2(reinterpret_cast<const __nv_bfloat162*>(dy)[i]);
    const float2 z = __bfloat1622float2(reinterpret_cast<const __nv_bfloat162*>(ref)[i]);
    float d0, d1;
    if (kind == 1) { d0 = z.x > 0.f ? 1.f : 0.f; d1 = z.y > 0.f ? 1.f : 0.f; }
    else if (kind == 2) {
      d0 = 0.5f * (1.f + erff(z.x * 0.70710678f)) + z.x * 0.3989422804f * __expf(-0.5f * z.x * z.x);
      d1 = 0.5f * (1.f + erff(z.y * 0.70710678f)) + z.y * 0.3989422804f * __expf(-0.5f * z.y * z.y);
    } else { d0 = 1.f - z.x * z.x; d1 = 1.f - z.y * z.y; }
    reinterpret_cast<__nv_bfloat162*>(dz)[i] = __floats2bfloat162_rn(g.x * d0, g.y * d1);
  }
}

// out[c] += sum_r x[r][c]   (bias gradient); block = 32 x 8, each block reduces `rows_per_block` rows of 32 columns
__global__ void __launch_bounds__(256)
colsum_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ out, int rows, int cols, long long ld,
              int rows_per_block) {
  __shared__ float part[8][33];
  pdl_wait();
  const int c = blockIdx.x * 32 + threadIdx.x;
  const int r0 = blockIdx.y * rows_per_block, r1 = min(rows, r0 + rows_per_block);
  float s = 0.f;
  if (c < cols)
    for (int r = r0 + threadIdx.y; r < r1; r += 8) s += __bfloat162float(x[static_cast<long long>(r) * ld + c]);
  part[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && c < cols) {
#pragma unroll
    for (int i = 1; i < 8; ++i) s += part[i][threadIdx.x];
    atomicAdd(out + c, s);
  }
}

__global__ void __launch_bounds__(256)
dropout_bf16_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, long long n2, float p,
                    uint32_t seed, const uint32_t* __restrict__ seed_ofs) {
  pdl_wait();
  seed = mix_seed(seed, seed_ofs);
  const float inv_keep = 1.f / (1.f - p);
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n2;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float2 v = __bfloat1622float2(reinterpret_cast<const __nv_bfloat162*>(x)[i]);
    const uint32_t idx = static_cast<uint32_t>(2 * i);
    reinterpret_cast<__nv_bfloat162*>(y)[i] = __floats2bfloat162_rn(v.x * drop_scale(seed, idx, p, inv_keep),
                                                                    v.y * drop_scale(seed, idx + 1, p, inv_keep));
  }
}

// out[t][:] = word[ids[t]] + pos[t % S] + type[tt[t] or 0]      (fp32 tables -> bf16)
__global__ void __launch_bounds__(256)
embed3_fwd_kernel(const long long* __restrict__ ids, const long long* __restrict__ tts, const float* __restrict__ word,
                  const float* __restrict__ pos, const float* __restrict__ type, __nv_bfloat16* __restrict__ out,
                  int tokens, int S, int D) {
  pdl_wait();
  const int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (t >= tokens) return;
  const float2* w = reinterpret_cast<const float2*>(word + ids[t] * D);
  const float2* q = reinterpret_cast<const float2*>(pos + static_cast<long long>(t % S) * D);
  const float2* y = reinterpret_cast<const float2*>(type + (tts ? tts[t] : 0) * D);
  __nv_bfloat162* o = reinterpret_cast<__nv_bfloat162*>(out + static_cast<long long>(t) * D);
  for (int i = lane_id(); i < (D >> 1); i += 32) {
    const float2 a = w[i], b = q[i], c = y[i];
    o[i] = __floats2bfloat162_rn(a.x + b.x + c.x, a.y + b.y + c.y);
  }
}
__global__ void __launch_bounds__(256)
embed3_bwd_kernel(const long long* __restrict__ ids, const long long* __restrict__ tts, const __nv_bfloat16* __restrict__ g,
                  float* __restrict__ dword, float* __restrict__ dpos, float* __restrict__ dtype, int tokens, int S, int D,
                  long long pad_id) {
  pdl_wait();
  const int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (t >= tokens) return;
  const long long id = ids[t];
  float* w = dword + id * D;
  float* q = dpos + static_cast<long long>(t % S) * D;
  float* y = dtype + (tts ? tts[t] : 0) * D;
  const __nv_bfloat16* gr = g + static_cast<long long>(t) * D;
  for (int i = lane_id(); i < D; i += 32) {
    const float v = __bfloat162float(gr[i]);
    if (id != pad_id) atomicAdd(w + i, v);
    atomicAdd(q + i, v);
    atomicAdd(y + i, v);
  }
}

// ----------------------------------------------------------------------------- host side
typedef CUresult (*PFN_encodeTiled3)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                     const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                     CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled3 get_encode3() {
  // cuTensorMapEncodeTiled is a driver call: it needs a context bound to *this* thread.  Autograd worker threads may
  // reach us before any runtime call has bound the primary context (seen as CUresult 201) -> bind it once per thread.
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) { int d = 0; cudaGetDevice(&d); cudaSetDevice(d); ctx_bound = true; }   // capture-safe, unlike cudaFree(0)
  static PFN_encodeTiled3 fn = nullptr;
  if (!fn) {
    void* q = nullptr;
    cudaDriverEntryPointQueryResult r;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &q, cudaEnableDefault, &r) != cudaSuccess || !q) return nullptr;
    fn = reinterpret_cast<PFN_encodeTiled3>(q);
  }
  return fn;
}
// [rows][ld] bf16 tensor, box = 64 columns x 128 rows, 128B swizzle
static int tmap_rows(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t ld) {
  PFN_encodeTiled3 enc = get_encode3();
  if (!enc) return -1;
  cuuint64_t gdim[2] = {cols, rows}, gstr[1] = {ld * 2};
  cuuint32_t box[2] = {64, 128}, es[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstr, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -static_cast<int>(r) - 100;
}
static int check_launch() {
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : -static_cast<int>(e) - 2000;
}

extern "C" {

// q/k/v: bf16 [B*S][ld*]; head h of Q lives at columns q_col + h*Dh ...  out: [B*S][ldo]; lse: [B*H][128] fp32
int slb_attn_fwd(const void* q, const void* k, const void* v, long long ldq, long long ldk, long long ldv, int q_col,
                 int k_col, int v_col, void* out, long long ldo, float* lse, const float* key_bias, int B, int S, int H,
                 int Dh, float p_drop, unsigned seed, const unsigned* seed_ofs, cudaStream_t st) {
  if (S < 1 || S > 128 || (Dh != 32 && Dh != 64)) return -3;
  if ((q_col | k_col | v_col) & 31 || ((ldq | ldk | ldv | ldo) & 7)) return -4;
  CUtensorMap tq, tk, tv;
  const uint64_t rows = static_cast<uint64_t>(B) * S;
  int r;
  if ((r = tmap_rows(&tq, q, rows, ldq, ldq))) return r;
  if ((r = tmap_rows(&tk, k, rows, ldk, ldk))) return r;
  if ((r = tmap_rows(&tv, v, rows, ldv, ldv))) return r;
  AttnParams p = {};
  p.B = B; p.S = S; p.H = H; p.Dh = Dh; p.q_col = q_col; p.k_col = k_col; p.v_col = v_col;
  p.scale = 1.f / sqrtf(static_cast<float>(Dh)); p.key_bias = key_bias; p.p_drop = p_drop; p.seed = seed; p.seed_ofs = seed_ofs;
  p.out = reinterpret_cast<__nv_bfloat16*>(out); p.ldo = ldo; p.lse = lse;
  static bool attr = false;
  if (!attr) {
    if (cudaFuncSetAttribute(attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_FWD_SMEM) != cudaSuccess)
      return -1000;
    attr = true;
  }
  attn_fwd_kernel<<<B * H, 128, ATT_FWD_SMEM, st>>>(tq, tk, tv, p);
  return check_launch();
}

int slb_attn_bwd(const void* q, const void* k, const void* v, const void* dout, long long ldq, long long ldk,
                 long long ldv, long long lddo, int q_col, int k_col, int v_col, int do_col, void* dq, void* dk, void* dv,
                 long long lddq, long long lddk, long long lddv, int dq_col, int dk_col, int dv_col, const float* lse,
                 const float* key_bias, int B, int S, int H, int Dh, float p_drop, unsigned seed, const unsigned* seed_ofs,
                 cudaStream_t st) {
  if (S < 1 || S > 128 || (Dh != 32 && Dh != 64)) return -3;
  if ((q_col | k_col | v_col | do_col) & 31 || ((ldq | ldk | ldv | lddo | lddq | lddk | lddv) & 7) ||
      ((dq_col | dk_col | dv_col) & 7))
    return -4;
  CUtensorMap tq, tk, tv, tdo;
  const uint64_t rows = static_cast<uint64_t>(B) * S;
  int r;
  if ((r = tmap_rows(&tq, q, rows, ldq, ldq))) return r;
  if ((r = tmap_rows(&tk, k, rows, ldk, ldk))) return r;
  if ((r = tmap_rows(&tv, v, rows, ldv, ldv))) return r;
  if ((r = tmap_rows(&tdo, dout, rows, lddo, lddo))) return r;
  AttnParams p = {};
  p.B = B; p.S = S; p.H = H; p.Dh = Dh; p.q_col = q_col; p.k_col = k_col; p.v_col = v_col; p.do_col = do_col;
  p.scale = 1.f / sqrtf(static_cast<float>(Dh)); p.key_bias = key_bias; p.p_drop = p_drop; p.seed = seed; p.seed_ofs = seed_ofs;
  p.lse = const_cast<float*>(lse);
  p.dq = reinterpret_cast<__nv_bfloat16*>(dq); p.dk = reinterpret_cast<__nv_bfloat16*>(dk);
  p.dv = reinterpret_cast<__nv_bfloat16*>(dv);
  p.lddq = lddq; p.lddk = lddk; p.lddv = lddv; p.dq_col = dq_col; p.dk_col = dk_col; p.dv_col = dv_col;
  static bool attr = false;
  if (!attr) {
    if (cudaFuncSetAttribute(attn_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_BWD_SMEM) != cudaSuccess)
      return -1000;
    attr = true;
  }
  attn_bwd_kernel<<<B * H, 128, ATT_BWD_SMEM, st>>>(tq, tk, tv, tdo, p);
  return check_launch();
}

int slb_ln_fwd(const void* x, const void* res, const float* gamma, const float* beta, void* y, void* pre, float* mean,
               float* rstd, int rows, int D, float eps, float p_drop, unsigned seed, const unsigned* seed_ofs,
               cudaStream_t st) {
  if (D & 1) return -3;
  ln_fwd_kernel<<<(rows + 7) / 8, 256, 0, st>>>(
      reinterpret_cast<const __nv_bfloat16*>(x), reinterpret_cast<const __nv_bfloat16*>(res), gamma, beta,
      reinterpret_cast<__nv_bfloat16*>(y), reinterpret_cast<__nv_bfloat16*>(pre), mean, rstd, rows, D, eps, p_drop, seed,
      seed_ofs);
  return check_launch();
}
int slb_ln_bwd(const void* dy, const void* pre, const float* gamma, const float* mean, const float* rstd, void* dpre,
               float* dgamma, float* dbeta, int rows, int D, cudaStream_t st) {
  if (D & 1 || D > 4096) return -3;
  int rpb = (rows + 295) / 296;
  if (rpb < 8) rpb = 8;
  if (D <= 1024)
    ln_bwd_kernel<true><<<(rows + rpb - 1) / rpb, 256, 2 * D * sizeof(float), st>>>(
        reinterpret_cast<const __nv_bfloat16*>(dy), reinterpret_cast<const __nv_bfloat16*>(pre), gamma, mean, rstd,
        reinterpret_cast<__nv_bfloat16*>(dpre), dgamma, dbeta, rows, D, rpb);
  else
    ln_bwd_kernel<false><<<(rows + rpb - 1) / rpb, 256, 2 * D * sizeof(float), st>>>(
        reinterpret_cast<const __nv_bfloat16*>(dy), reinterpret_cast<const __nv_bfloat16*>(pre), gamma, mean, rstd,
        reinterpret_cast<__nv_bfloat16*>(dpre), dgamma, dbeta, rows, D, rpb);
  return check_launch();
}
int slb_act_bwd(const void* dy, const void* ref, void* dz, long long n, int kind, cudaStream_t st) {
  if (n & 1) return -3;
  const long long n2 = n / 2;
  int grid = static_cast<int>((n2 + 255) / 256);
  if (grid > 132 * 8) grid = 132 * 8;
  act_bwd_kernel<<<grid, 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(dy),
                                       reinterpret_cast<const __nv_bfloat16*>(ref),
                                       reinterpret_cast<__nv_bfloat16*>(dz), n2, kind);
  return check_launch();
}
int slb_colsum_bf16(const void* x, float* out, int rows, int cols, long long ld, cudaStream_t st) {
  int rpb = 256;
  dim3 grid((cols + 31) / 32, (rows + rpb - 1) / rpb);
  colsum_kernel<<<grid, dim3(32, 8), 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(x), out, rows, cols, ld, rpb);
  return check_launch();
}
int slb_dropout_bf16(const void* x, void* y, long long n, float p, unsigned seed, const unsigned* seed_ofs,
                     cudaStream_t st) {
  if (n & 1 || n >= (1ll << 32)) return -3;
  const long long n2 = n / 2;
  int grid = static_cast<int>((n2 + 255) / 256);
  if (grid > 132 * 8) grid = 132 * 8;
  dropout_bf16_kernel<<<grid, 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(x),
                                            reinterpret_cast<__nv_bfloat16*>(y), n2, p, seed, seed_ofs);
  return check_launch();
}
int slb_embed3_fwd(const long long* ids, const long long* tts, const float* word, const float* pos, const float* type,
                   void* out, int tokens, int S, int D, cudaStream_t st) {
  if (D & 1) return -3;
  embed3_fwd_kernel<<<(tokens + 7) / 8, 256, 0, st>>>(ids, tts, word, pos, type, reinterpret_cast<__nv_bfloat16*>(out),
                                                      tokens, S, D);
  return check_launch();
}
int slb_embed3_bwd(const long long* ids, const long long* tts, const void* g, float* dword, float* dpos, float* dtype,
                   int tokens, int S, int D, long long pad_id, cudaStream_t st) {
  embed3_bwd_kernel<<<(tokens + 7) / 8, 256, 0, st>>>(ids, tts, reinterpret_cast<const __nv_bfloat16*>(g), dword, dpos,
                                                      dtype, tokens, S, D, pad_id);
  return check_launch();
}

int slb_preload_transformer() {
  cudaFuncAttributes a;
  int bad = 0;
  bad |= cudaFuncGetAttributes(&a, attn_fwd_kernel) != cudaSuccess;
  bad |= cudaFuncGetAttributes(&a, attn_bwd_kernel) != cudaSuccess;
  bad |= cudaFuncGetAttributes(&a, ln_fwd_kernel) != cudaSuccess;
  bad |= cudaFuncGetAttributes(&a, ln_bwd_kernel<true>) != cudaSuccess;
  bad |= cudaFuncGetAttributes(&a, ln_bwd_kernel<false>) != cudaSuccess;
  bad |= cudaFuncGetAttributes(&a, act_bwd_kernel) != cudaSuccess;
  bad |= cudaFuncGetAttributes(&a, colsum_kernel) != cudaSuccess;
  bad |= cudaFuncGetAttributes(&a, dropout_bf16_kernel) != cudaSuccess;
  bad |= cudaFuncGetAttributes(&a, embed3_fwd_kernel) != cudaSuccess;
  bad |= cudaFuncGetAttributes(&a, embed3_bwd_kernel) != cudaSuccess;
  return bad ? -1 : 0;
}

}  // extern "C"
}  // namespace slb
