// Speech front-end kernels of the GPU-resident Speech Commands loader (data/gpu_loader.py, b200.gpu-loader):
//
//   mfcc_kernel            fp32 waveforms [n][L] -> fp32 MFCC features [n][ncoef][frames], computed in fp64 and rounded to
//                          fp32 once, step for step what data/speechcommands.py:mfcc() does on the host:
//                            pre-emphasis        p[0] = w[0], p[t] = w[t] - a * w[t-1]
//                            framing             frame f = p[f*hop, f*hop + win) * window   (zero-padded to nfft)
//                            power spectrum      |X_k|^2 / nfft, k < nfft/2 + 1, by a direct DFT whose twiddles come from
//                                                an nfft-entry (cos, sin) table indexed by (k * t) mod nfft
//                            mel + log           ln(max(fb @ power, floor))
//                            DCT                 dct @ mel, stored transposed as [ncoef][frames]
//                          The window, filterbank, DCT matrix and twiddle table are fp64 device tables built by the host
//                          from the same arrays mfcc() uses, and the frame geometry is a launch argument: the kernel holds
//                          no recipe constant of its own.  One CTA per (clip, group of MFCC_GROUP frames); one thread per
//                          frequency bin.  Clips whose valid byte is 0 (files the host could not read) get zero features.
//                          The template argument is the recipe (b200.speech-features).  MFCC_REFERENCE follows
//                          speechcommands.mfcc_reference() instead, in its two steps that differ:
//                            pre-emphasis        in fp32, p[t] = w[t] - (float)a * w[t-1] (each operation rounded), as NumPy
//                                                computes it on a float32 waveform; widened to fp64 for the window
//                            mel + log           20 log10(e), e = fb @ power, with e == 0 replaced by floor (eps)
//                          MFCC_ENGINE compiles to the code the kernel had before it took a recipe.
//   feature_batch_kernel   one training microbatch gathered from the resident features: out[b] = feat[idx[b]],
//                          y[b] = labels[idx[b]], 16-byte loads and stores.
#include "sm90.cuh"

namespace slb {

constexpr int MFCC_GROUP = 7;            // frames per CTA: 98 = 14 x 7; every twiddle load feeds 2 x 7 FMAs
constexpr int MFCC_XS = 8;               // row pitch (doubles) of the staged frame samples: 4 x 16-byte loads per sample
constexpr int MFCC_MAX_THREADS = 512;
enum MfccRecipe : int { MFCC_ENGINE = 0, MFCC_REFERENCE = 1 };   // the recipe argument of slb_mfcc

struct MfccArgs {
  const float* waves;
  const uint8_t* valid;                  // may be null: every clip valid
  const double* window;                  // [win]
  const double* fb;                      // [nmels][nbins]
  const double* dct;                     // [ncoef][nmels]
  const double2* twiddle;                // [nfft] (cos, sin) of 2 pi j / nfft
  float* out;                            // [n][ncoef][frames]
  int n, L, win, hop, frames, nfft, nbins, nmels, ncoef;
  int span;                              // floats of raw waveform staged per CTA (multiple of 4)
  double preemph, floor;                 // floor: lower clamp of the mel energies (engine), value of exact zeros (reference)
};

// dynamic shared memory of one CTA: twiddles, frame samples, raw fp32 span, power spectra, mel energies
static inline size_t mfcc_smem(int nfft, int win, int nbins, int nmels, int span) {
  return sizeof(double2) * nfft + sizeof(double) * (static_cast<size_t>(win) * MFCC_XS + MFCC_GROUP * nbins + MFCC_GROUP * nmels)
         + sizeof(float) * span;
}

template <MfccRecipe R>
__global__ void __launch_bounds__(MFCC_MAX_THREADS) mfcc_kernel(const MfccArgs a) {
  pdl_trigger();
  pdl_wait();
  const int groups = (a.frames + MFCC_GROUP - 1) / MFCC_GROUP;
  const int clip = blockIdx.x / groups;
  const int f0 = (blockIdx.x - clip * groups) * MFCC_GROUP;
  const int gf = min(MFCC_GROUP, a.frames - f0);
  const int tid = threadIdx.x, nt = blockDim.x;
  float* out = a.out + static_cast<long long>(clip) * a.ncoef * a.frames + f0;

  if (a.valid != nullptr && a.valid[clip] == 0) {
    for (int i = tid; i < a.ncoef * gf; i += nt) out[(i / gf) * a.frames + i % gf] = 0.f;
    return;
  }

  extern __shared__ __align__(16) unsigned char smem[];
  // every region read or written with 16-byte accesses sits at a multiple of 16 bytes: tw (16 nfft), xw (64 win), raw
  // (4 span, span % 4 == 0) come first; pw and mel, accessed as single doubles, follow
  double2* tw = reinterpret_cast<double2*>(smem);
  double* xw = reinterpret_cast<double*>(tw + a.nfft);            // [win][MFCC_XS] windowed frame samples
  float* raw = reinterpret_cast<float*>(xw + static_cast<size_t>(a.win) * MFCC_XS);
  double* pw = reinterpret_cast<double*>(raw + a.span);          // [MFCC_GROUP][nbins] power spectra
  double* mel = pw + MFCC_GROUP * a.nbins;                       // [MFCC_GROUP][nmels] log mel energies

  // raw waveform span [s0, s0 + span) covering every sample (and its predecessor) of this group's frames
  const float* w = a.waves + static_cast<long long>(clip) * a.L;
  const int s0 = max(f0 * a.hop - 1, 0) & ~3;
  const int s1 = min(s0 + a.span, a.L);
  for (int i = tid; 4 * i < s1 - s0; i += nt)
    reinterpret_cast<float4*>(raw)[i] = __ldg(reinterpret_cast<const float4*>(w + s0) + i);
  for (int j = tid; j < a.nfft; j += nt) tw[j] = a.twiddle[j];
  __syncthreads();

  // pre-emphasis and window in fp64, with the host's roundings (no contraction into an FMA)
  for (int i = tid; i < a.win * MFCC_XS; i += nt) {
    const int t = i / MFCC_XS, f = i - t * MFCC_XS;
    double v = 0.0;
    if (f < gf) {
      const int s = (f0 + f) * a.hop + t;
      double p;
      if constexpr (R == MFCC_ENGINE) {
        const double x = static_cast<double>(raw[s - s0]);
        p = s == 0 ? x : __dsub_rn(x, __dmul_rn(a.preemph, static_cast<double>(raw[s - 1 - s0])));
      } else {
        const float x = raw[s - s0];
        p = static_cast<double>(s == 0 ? x : __fsub_rn(x, __fmul_rn(static_cast<float>(a.preemph), raw[s - 1 - s0])));
      }
      v = __dmul_rn(p, a.window[t]);
    }
    xw[i] = v;
  }
  __syncthreads();

  // direct DFT: bin k of the GROUP frames at once, one twiddle load per sample
  for (int k = tid; k < a.nbins; k += nt) {
    double re[MFCC_GROUP], im[MFCC_GROUP];
#pragma unroll
    for (int f = 0; f < MFCC_GROUP; ++f) re[f] = im[f] = 0.0;
    int j = 0;                                                      // (k * t) mod nfft
#pragma unroll 2
    for (int t = 0; t < a.win; ++t) {
      const double2 c = tw[j];
      const double2* x2 = reinterpret_cast<const double2*>(xw + t * MFCC_XS);
      double x[MFCC_XS];
#pragma unroll
      for (int q = 0; q < MFCC_XS / 2; ++q) {
        const double2 v = x2[q];
        x[2 * q] = v.x;
        x[2 * q + 1] = v.y;
      }
#pragma unroll
      for (int f = 0; f < MFCC_GROUP; ++f) {
        re[f] = fma(x[f], c.x, re[f]);
        im[f] = fma(x[f], c.y, im[f]);
      }
      j += k;
      if (j >= a.nfft) j -= a.nfft;
    }
#pragma unroll
    for (int f = 0; f < MFCC_GROUP; ++f)
      if (f < gf) pw[f * a.nbins + k] = (re[f] * re[f] + im[f] * im[f]) / static_cast<double>(a.nfft);
  }
  __syncthreads();

  // mel energies: one warp per (frame, filter) row, lanes over bins, then a shuffle tree
  const int lane = tid & 31, warp = tid >> 5, nwarps = nt >> 5;
  for (int r = warp; r < gf * a.nmels; r += nwarps) {
    const int f = r / a.nmels, m = r - f * a.nmels;
    const double* fr = a.fb + static_cast<long long>(m) * a.nbins;
    const double* pr = pw + f * a.nbins;
    double s = 0.0;
    for (int k = lane; k < a.nbins; k += 32) s = fma(pr[k], __ldg(fr + k), s);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) {
      if constexpr (R == MFCC_ENGINE)
        mel[f * a.nmels + m] = log(fmax(s, a.floor));
      else
        mel[f * a.nmels + m] = 20.0 * log10(s == 0.0 ? a.floor : s);
    }
  }
  __syncthreads();

  // DCT, written [coef][frame]: consecutive threads store consecutive frames of one coefficient row
  for (int i = tid; i < a.ncoef * gf; i += nt) {
    const int c = i / gf, f = i - c * gf;
    const double* dr = a.dct + static_cast<long long>(c) * a.nmels;
    const double* mr = mel + f * a.nmels;
    double s = 0.0;
    for (int m = 0; m < a.nmels; ++m) s = fma(mr[m], __ldg(dr + m), s);
    out[c * a.frames + f] = __double2float_rn(s);
  }
}

// out[b][:] = feat[idx[b]][:], y[b] = labels[idx[b]]; rows of row4 float4s; blockIdx.y = b
__global__ void __launch_bounds__(256)
feature_batch_kernel(const float4* __restrict__ feat, const long long* __restrict__ labels, const long long* __restrict__ idx,
                     float4* __restrict__ out, long long* __restrict__ y, long long row4) {
  pdl_trigger();
  pdl_wait();
  const int b = blockIdx.y;
  const long long src = __ldg(idx + b);
  if (blockIdx.x == 0 && threadIdx.x == 0) y[b] = __ldg(labels + src);
  const float4* s = feat + src * row4;
  float4* d = out + static_cast<long long>(b) * row4;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < row4;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    d[i] = __ldg(s + i);
}

static bool misaligned(const void* ptr, uintptr_t bytes) {
  return ptr == nullptr || (reinterpret_cast<uintptr_t>(ptr) & (bytes - 1));
}
static int launch_status() {
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : -static_cast<int>(e) - 2000;
}

}  // namespace slb
using namespace slb;

extern "C" {

// Returns -3 (shape, recipe) or -4 (alignment) without launching anything.  L = win + hop * (frames - 1) and L % 4 == 0
// (16-byte waveform loads); win <= nfft, nfft even, nfft / 2 + 1 bins; waves 16-byte aligned, tables 8 (twiddle 16);
// recipe MFCC_ENGINE or MFCC_REFERENCE.  Dynamic shared memory (mfcc_smem): 55,880 B for the engine geometry (400 / 512),
// 59,912 B for the reference geometry (480 / 480).
int slb_mfcc(const float* waves, const uint8_t* valid, const double* window, const double* fb, const double* dct,
             const void* twiddle, float* out, int n, int L, int win, int hop, int frames, int nfft, int nmels, int ncoef,
             double preemph, double floor, int recipe, cudaStream_t st) {
  if (recipe != MFCC_ENGINE && recipe != MFCC_REFERENCE) return -3;
  if (n < 1 || win < 1 || hop < 1 || frames < 1 || nmels < 1 || ncoef < 1 || nfft < 2 || (nfft & 1) || win > nfft) return -3;
  if (static_cast<long long>(win) + static_cast<long long>(hop) * (frames - 1) != L || (L & 3)) return -3;
  const int groups = (frames + MFCC_GROUP - 1) / MFCC_GROUP;
  if (static_cast<long long>(n) * groups > INT32_MAX) return -3;
  if (misaligned(waves, 16) || misaligned(window, 8) || misaligned(fb, 8) || misaligned(dct, 8) || misaligned(twiddle, 16) ||
      misaligned(out, 4))
    return -4;
  MfccArgs a;
  a.waves = waves; a.valid = valid; a.window = window; a.fb = fb; a.dct = dct;
  a.twiddle = reinterpret_cast<const double2*>(twiddle); a.out = out;
  a.n = n; a.L = L; a.win = win; a.hop = hop; a.frames = frames; a.nfft = nfft; a.nbins = nfft / 2 + 1;
  a.nmels = nmels; a.ncoef = ncoef; a.preemph = preemph; a.floor = floor;
  a.span = ((MFCC_GROUP - 1) * hop + win + 1 + 3 + 3) & ~3;     // predecessor sample + alignment of both ends
  const size_t smem = mfcc_smem(nfft, win, a.nbins, nmels, a.span);
  if (smem > 227 * 1024) return -3;
  void (*kernel)(MfccArgs) = recipe == MFCC_ENGINE ? mfcc_kernel<MFCC_ENGINE> : mfcc_kernel<MFCC_REFERENCE>;
  if (smem > 48 * 1024 &&
      cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)) != cudaSuccess)
    return launch_status();
  const int threads = min(MFCC_MAX_THREADS, (a.nbins + 31) & ~31);
  launch_k(kernel, dim3(static_cast<unsigned>(n * groups)), dim3(threads), smem, st, a);
  return launch_status();
}

// feat fp32 [N][D], labels int64 [N], idx int64 [B] (each in [0, N)) -> out fp32 [B][D], y int64 [B].  D % 4 == 0.
int slb_feature_batch(const float* feat, const long long* labels, const long long* idx, float* out, long long* y, int N,
                      int B, long long D, cudaStream_t st) {
  if (N < 1 || B < 1 || B > 65535 || D < 4 || (D & 3)) return -3;
  if (misaligned(feat, 16) || misaligned(out, 16) || misaligned(labels, 8) || misaligned(idx, 8) || misaligned(y, 8)) return -4;
  const long long row4 = D / 4;
  const unsigned gx = static_cast<unsigned>(row4 > 64 * 256 ? 64 : (row4 + 255) / 256);
  launch_k(feature_batch_kernel, dim3(gx, static_cast<unsigned>(B)), dim3(256), 0, st, reinterpret_cast<const float4*>(feat),
           labels, idx, reinterpret_cast<float4*>(out), y, row4);
  return launch_status();
}

int slb_preload_audio() {
  cudaFuncAttributes a;
  int bad = 0;
  bad += cudaFuncGetAttributes(&a, mfcc_kernel<MFCC_ENGINE>) != cudaSuccess;
  bad += cudaFuncGetAttributes(&a, mfcc_kernel<MFCC_REFERENCE>) != cudaSuccess;
  bad += cudaFuncGetAttributes(&a, feature_batch_kernel) != cudaSuccess;
  return bad;
}

}  // extern "C"
