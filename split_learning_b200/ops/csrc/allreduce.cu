// FedAvg as one fused all-reduce over NVSwitch peer memory (SURVEY §2.7 G12, reference src/Utils.py:35-66 +
// src/Server.py:398-434):
//
//     p[i] = sum_q coef_q * nan_to_num(p_q[i]),   coef_q = w_q / (sum of w over q's cluster) / #clusters
//
// for every replica q that holds the segment — the reference's per-cluster weighted mean followed by the unweighted
// cross-cluster mean, collapsed into one set of coefficients.  Two-shot: participant r reduces slice r of the segment
// (reads that slice from every holder through peer loads: 1/R of the buffer per peer) and stores the result into the
// same slice of EVERY holder's buffer (peer stores), so each GPU moves (R-1)/R of the buffer in and out over NVLink
// instead of (R-1) buffers with an all-pull.  In place: slice r of every buffer is read and written by participant r
// only.  Weights, NaN votes and both barriers live in device memory (st.release.sys / ld.acquire.sys flags in each
// participant's exported sync block): no host message, pickle or NCCL call is involved in a round.
// Integer state (num_batches_tracked mirrors) is rounded to the nearest integer in the same pass.
#include "sm90.cuh"

namespace slb {

constexpr int AR_MAX = 16;

// One exported sync block per participant (u32 words):
//   [0, 16)  ready_from[q]   epoch of the last all-reduce for which q has published its buffer + weight
//   [16, 32) done_from[q]    epoch of the last all-reduce whose slice q has fully stored into my buffer
//   [32]     my weight (float bits)   [33] my ok vote   [34] CTA ticket   [35] result: 1 = aggregated, 0 = skipped
//   [36]     spin-timeout flag
struct ArParams {
  float* buf[AR_MAX];          // segment base inside holder q's buffer (local or peer-mapped)
  uint32_t* sync[AR_MAX];      // holder q's sync block
  int gid[AR_MAX];             // global participant index of holder q (flag slot)
  int cluster[AR_MAX];         // cluster id of holder q
  int nsrc, me;                // holders, my index among them
  int n_clusters;
  long long n4;                // segment length in float4
  long long round_lo4, round_hi4;   // float4 range holding integer-valued state (rounded after averaging)
  uint32_t epoch;
  float weight;                // my FedAvg weight (microbatch count)
  uint32_t ok;                 // my vote: 0 = NaN seen this round -> nobody aggregates (src/Server.py:162-170)
  unsigned long long max_spins;
};

__device__ __forceinline__ bool spin_until(const uint32_t* p, uint32_t epoch, unsigned long long max_spins) {
  unsigned long long spins = 0;
  while (static_cast<int32_t>(ld_acquire_sys(p) - epoch) < 0) {
    __nanosleep(100);
    if (++spins > max_spins) return false;
  }
  return true;
}

__global__ void __launch_bounds__(512) fedavg_allreduce_kernel(const ArParams p) {
  __shared__ float s_coef[AR_MAX];
  __shared__ int s_go;
  uint32_t* mine = p.sync[p.me];
  if (threadIdx.x == 0) {
    if (blockIdx.x == 0) {
      // publish my weight / vote, then tell every holder that my buffer is final for this epoch
      mine[32] = __float_as_uint(p.weight);
      mine[33] = p.ok;
      __threadfence_system();
      for (int q = 0; q < p.nsrc; ++q) st_release_sys(p.sync[q] + p.gid[p.me], p.epoch);
    }
    bool alive = true;
    for (int q = 0; q < p.nsrc && alive; ++q) alive = spin_until(mine + p.gid[q], p.epoch, p.max_spins);
    int go = alive ? 1 : 0;
    if (!alive) mine[36] = 1;
    float w[AR_MAX], tot[AR_MAX];
    for (int q = 0; q < p.nsrc && alive; ++q) {
      const volatile uint32_t* sq = p.sync[q];
      w[q] = __uint_as_float(sq[32]);
      if (sq[33] == 0) go = 0;
    }
    if (go) {
      for (int q = 0; q < p.nsrc; ++q) {
        float t = 0.f;
        for (int r = 0; r < p.nsrc; ++r)
          if (p.cluster[r] == p.cluster[q]) t += w[r];
        tot[q] = t;
        if (!(t > 0.f)) go = 0;
      }
    }
    for (int q = 0; q < p.nsrc; ++q) s_coef[q] = go ? w[q] / tot[q] / static_cast<float>(p.n_clusters) : 0.f;
    s_go = go;
  }
  __syncthreads();
  const int go = s_go;
  if (go) {
    const long long chunk = (p.n4 + p.nsrc - 1) / p.nsrc;
    const long long lo = chunk * p.me, hi = min(p.n4, lo + chunk);
    for (long long i = lo + blockIdx.x * (long long)blockDim.x + threadIdx.x; i < hi; i += (long long)gridDim.x * blockDim.x) {
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
      for (int q = 0; q < p.nsrc; ++q) {
        const float4 v = __ldcg(reinterpret_cast<const float4*>(p.buf[q]) + i);
        const float c = s_coef[q];
        acc.x += c * (v.x == v.x ? v.x : 0.f);
        acc.y += c * (v.y == v.y ? v.y : 0.f);
        acc.z += c * (v.z == v.z ? v.z : 0.f);
        acc.w += c * (v.w == v.w ? v.w : 0.f);
      }
      if (i >= p.round_lo4 && i < p.round_hi4) { acc.x = rintf(acc.x); acc.y = rintf(acc.y); acc.z = rintf(acc.z); acc.w = rintf(acc.w); }
#pragma unroll 4
      for (int q = 0; q < p.nsrc; ++q) reinterpret_cast<float4*>(p.buf[q])[i] = acc;
    }
  }
  // every CTA's peer stores are fenced; the last CTA tells every holder that my slice of its buffer is complete
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    const uint32_t t = atomicAdd(mine + 34, 1u);
    if (t == gridDim.x - 1) {
      mine[34] = 0;
      mine[35] = static_cast<uint32_t>(go);
      __threadfence_system();
      for (int q = 0; q < p.nsrc; ++q) st_release_sys(p.sync[q] + 16 + p.gid[p.me], p.epoch);
    }
  }
}

// Second half of the barrier: returns once every holder has stored its slice into my buffer.
__global__ void fedavg_allreduce_wait_kernel(const ArParams p) {
  uint32_t* mine = p.sync[p.me];
  for (int q = 0; q < p.nsrc; ++q)
    if (!spin_until(mine + 16 + p.gid[q], p.epoch, p.max_spins)) { mine[36] = 1; return; }
}

// ---------------------------------------------------------------------------------------------------------------
// Cross-GPU memory-ordering litmus (message passing, both directions) of the exact idiom every cut-edge kernel uses:
//   producer: payload stores by all threads -> bar.sync -> thread 0: fence.sys + st.release.sys flag
//   consumer: thread 0: ld.acquire.sys flag -> bar.sync -> all threads read the payload (L2 loads: a *new kernel* reads
//             the mailbox in the real pipeline, so L1 never holds an older copy; inside this persistent loop .cg does that)
// Two GPUs ping-pong `iters` messages; any payload word that does not carry the iteration number is counted.
__global__ void __launch_bounds__(256) litmus_pingpong_kernel(uint32_t* peer_payload, uint32_t* peer_flag, const uint32_t* my_payload,
                                                             const uint32_t* my_flag, int n_words, uint32_t iters, int role,
                                                             unsigned long long max_spins, uint32_t* result) {
  __shared__ int s_dead;
  uint32_t errors = 0;
  if (threadIdx.x == 0) s_dead = 0;
  __syncthreads();
  for (uint32_t it = 1; it <= iters; ++it) {
    if (role == 0) {
      for (int i = threadIdx.x; i < n_words; i += blockDim.x) peer_payload[i] = it * 2654435761u + i;
      __syncthreads();
      if (threadIdx.x == 0) { __threadfence_system(); st_release_sys(peer_flag, it); }
    }
    if (threadIdx.x == 0 && !spin_until(my_flag, it, max_spins)) s_dead = 1;
    __syncthreads();
    if (s_dead) break;
    for (int i = threadIdx.x; i < n_words; i += blockDim.x)
      if (__ldcg(my_payload + i) != it * 2654435761u + i) ++errors;
    if (role == 1) {
      __syncthreads();
      for (int i = threadIdx.x; i < n_words; i += blockDim.x) peer_payload[i] = it * 2654435761u + i;
      __syncthreads();
      if (threadIdx.x == 0) { __threadfence_system(); st_release_sys(peer_flag, it); }
    }
  }
  if (errors) atomicAdd(result, errors);
  if (threadIdx.x == 0 && s_dead) result[1] = 1;
}

}  // namespace slb
using namespace slb;

extern "C" int slb_litmus_pingpong(uint32_t* peer_payload, uint32_t* peer_flag, const uint32_t* my_payload, const uint32_t* my_flag,
                                   int n_words, uint32_t iters, int role, unsigned long long max_spins, uint32_t* result,
                                   cudaStream_t st) {
  litmus_pingpong_kernel<<<1, 256, 0, st>>>(peer_payload, peer_flag, my_payload, my_flag, n_words, iters, role, max_spins, result);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : -static_cast<int>(e) - 2000;
}

extern "C" {

int slb_preload_allreduce() {
  cudaFuncAttributes a;
  return (cudaFuncGetAttributes(&a, fedavg_allreduce_kernel) != cudaSuccess) + (cudaFuncGetAttributes(&a, fedavg_allreduce_wait_kernel) != cudaSuccess);
}

// bufs / syncs: host arrays of nsrc device pointers (segment base in every holder's buffer, holder's sync block).
// n: floats in the segment (multiple of 4); [round_lo, round_hi): float range holding integer-valued state.
int slb_fedavg_allreduce(float* const* bufs, uint32_t* const* syncs, const int* gids, const int* clusters, int nsrc, int me,
                         int n_clusters, long long n, long long round_lo, long long round_hi, uint32_t epoch, float weight,
                         int ok, unsigned long long max_spins, int grid, cudaStream_t st) {
  if (nsrc < 1 || nsrc > AR_MAX || n % 4 || round_lo % 4 || round_hi % 4 || me < 0 || me >= nsrc) return -1;
  ArParams p = {};
  for (int q = 0; q < nsrc; ++q) {
    p.buf[q] = bufs[q]; p.sync[q] = syncs[q]; p.gid[q] = gids[q]; p.cluster[q] = clusters[q];
    if (gids[q] < 0 || gids[q] >= AR_MAX) return -2;
  }
  p.nsrc = nsrc; p.me = me; p.n_clusters = n_clusters; p.n4 = n / 4; p.round_lo4 = round_lo / 4; p.round_hi4 = round_hi / 4;
  p.epoch = epoch; p.weight = weight; p.ok = ok ? 1u : 0u; p.max_spins = max_spins;
  if (grid < 1) grid = 1;
  const long long per = (p.n4 / nsrc + 511) / 512;
  if (grid > per && per >= 1) grid = static_cast<int>(per);
  fedavg_allreduce_kernel<<<grid, 512, 0, st>>>(p);
  fedavg_allreduce_wait_kernel<<<1, 1, 0, st>>>(p);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : -static_cast<int>(e) - 2000;
}

}  // extern "C"
