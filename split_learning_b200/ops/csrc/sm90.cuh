// sm_90a primitives used by every tensor-core kernel in this tree:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma.mma_async with shared-memory descriptors.
// Plain inline PTX; no CUTLASS dependency.  Bit layouts follow the PTX ISA "wgmma matrix
// descriptor" table.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

namespace slb {

// ----------------------------------------------------------------------------- misc
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ----------------------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded spin: a descriptor/pipeline bug must trap, not hang the GPU.
#ifndef SLB_SPIN_LIMIT
#define SLB_SPIN_LIMIT (1u << 24)
#endif
// No printf on the timeout path: any call in a kernel makes ptxas serialise its asynchronous wgmma MMAs.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > SLB_SPIN_LIMIT) {
      __trap();
    }
  }
}

// ----------------------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// ----------------------------------------------------------------------------- wgmma
// Shared-memory matrix descriptor of wgmma, 128-byte swizzle.
//   bits [0,14)  start address >> 4        bits [16,30) leading byte offset >> 4
//   bits [32,46) stride byte offset >> 4   bits [62,64) layout (1 = SWIZZLE_128B)
// K-major tile  = rows of 128 B (64 bf16 / 32 tf32 of K), 8-row swizzle atoms 1024 B apart -> SBO = 1024, LBO unused.
// MN-major tile = K-rows of 128 B (64 bf16 of M/N), 8-k atoms 1024 B apart (SBO = 1024),
//                 next 64-wide M/N group `lbo_bytes` further.
__device__ __forceinline__ uint64_t wg_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// generic-proxy shared-memory writes -> visible to the tensor core and TMA (async proxy)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// m64nNk16 (bf16, TA / TB: 1 = operand stored MN-major) and m64nNk8 (tf32, K-major operands only), fp32 accumulators
// in registers; acc == 0 overwrites d.  d[4i + e] holds row 16 * (warp % 4) + lane / 4 + 8 * (e >> 1),
// column 8i + 2 * (lane % 4) + (e & 1) of the warpgroup's 64 x N tile.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_n32(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
}
__device__ __forceinline__ void wgmma_tf32_n32(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a), "l"(b), "r"(acc));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_n64(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
}
__device__ __forceinline__ void wgmma_tf32_n64(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(acc));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_n128(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
}
__device__ __forceinline__ void wgmma_tf32_n128(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(acc));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_n256(float (&d)[128], uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, %131, %132;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
}
__device__ __forceinline__ void wgmma_tf32_n256(float (&d)[128], uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(a), "l"(b), "r"(acc));
}

template <typename T, int N> struct Wgmma;
#define SLB_WGMMA_DISPATCH(N)                                                                                           \
  template <> struct Wgmma<__nv_bfloat16, N> {                                                                          \
    static __device__ __forceinline__ void mma(float (&d)[N / 2], uint64_t a, uint64_t b, uint32_t acc, int a_mn,      \
                                               int b_mn) {                                                              \
      if (a_mn) { if (b_mn) wgmma_bf16_n##N<1, 1>(d, a, b, acc); else wgmma_bf16_n##N<1, 0>(d, a, b, acc); }            \
      else      { if (b_mn) wgmma_bf16_n##N<0, 1>(d, a, b, acc); else wgmma_bf16_n##N<0, 0>(d, a, b, acc); }            \
    }                                                                                                                   \
  };                                                                                                                    \
  template <> struct Wgmma<float, N> {                                                                                  \
    static __device__ __forceinline__ void mma(float (&d)[N / 2], uint64_t a, uint64_t b, uint32_t acc, int, int) {     \
      wgmma_tf32_n##N(d, a, b, acc);                                                                                    \
    }                                                                                                                   \
  };
SLB_WGMMA_DISPATCH(32)
SLB_WGMMA_DISPATCH(64)
SLB_WGMMA_DISPATCH(128)
SLB_WGMMA_DISPATCH(256)
#undef SLB_WGMMA_DISPATCH

// Operand-type traits of the GEMM pipelines: one K block is always one 128-byte swizzle row.
//   KE       elements per 128 bytes (= K elements per pipeline stage, = M/N elements per MN-major group)
template <typename T> struct OperandTraits;
template <> struct OperandTraits<__nv_bfloat16> {
  static constexpr int KE = 64;
  static constexpr bool TF32 = false;
};
template <> struct OperandTraits<float> {
  static constexpr int KE = 32;
  static constexpr bool TF32 = true;
};

// wgmma reads tf32 operands K-major only.  An fp32 operand stored MN-major (loaded by TMA without swizzle: groups of
// 32 M/N elements x 32 k-rows of 128 B, 4 KB apart) is transposed by the 256 consumer threads into a K-major
// 128B-swizzled tile of `rows` rows before the MMAs read it.
__device__ __forceinline__ void transpose_tf32_kmajor(uint8_t* dst, const uint8_t* src, int rows) {
  const float* s = reinterpret_cast<const float*>(src);
  for (int i = threadIdx.x; i < rows * 8; i += 256) {
    const int r = i & (rows - 1), c = i / rows;                    // row r, 16-byte chunk c (k = 4c .. 4c + 3)
    const float* col = s + (r >> 5) * 1024 + (4 * c) * 32 + (r & 31);
    *reinterpret_cast<float4*>(dst + r * 128 + ((c ^ (r & 7)) << 4)) = make_float4(col[0], col[32], col[64], col[96]);
  }
}

// Consumer side of a TMA -> wgmma ring, run by two warpgroups (threads 0..255) that own rows [0, 64) and [64, 128) of
// a 128 x BLOCK_N tile.  Stage s: A (128 x KE, at smem + s * stage_bytes) then B (BLOCK_N x KE, a_bytes further); K-major
// operands are 128-byte swizzled rows, bf16 MN-major operands are 64-wide groups of KE k-rows.  empty_bar[s] expects one
// arrival per warpgroup.  `stg` (fp32 only): 128 x 128 B + BLOCK_N x 128 B of K-major staging for MN-major operands.
template <typename T, int BLOCK_N>
__device__ __forceinline__ void wg_mainloop(uint8_t* smem, uint8_t* stg, int stage_bytes, int a_bytes, int stages,
                                            uint64_t* full_bar, uint64_t* empty_bar, int iters, int a_mn, int b_mn,
                                            float (&acc)[BLOCK_N / 2], int& stage, uint32_t& phase) {
  using OT = OperandTraits<T>;
  constexpr int GROUP_BYTES = OT::KE * 128;
  const uint32_t half = static_cast<uint32_t>(threadIdx.x >> 7) * 8192;   // 64 rows K-major == one MN-major group
  const bool transpose = OT::TF32 && (a_mn || b_mn);
  int prev = -1;
  for (int it = 0; it < iters; ++it) {
    mbar_wait(&full_bar[stage], phase);
    uint8_t* st = smem + stage * stage_bytes;
    uint32_t a_base = smem_u32(st), b_base = a_base + a_bytes;
    int amn = a_mn, bmn = b_mn;
    if (transpose) {
      wgmma_wait<0>();
      asm volatile("bar.sync 2, 256;" ::: "memory");               // both warpgroups are done with the staging tiles
      if (a_mn) transpose_tf32_kmajor(stg, st, 128);
      if (b_mn) transpose_tf32_kmajor(stg + 128 * 128, st + a_bytes, BLOCK_N);
      fence_proxy_async();
      asm volatile("bar.sync 2, 256;" ::: "memory");
      if (a_mn) { a_base = smem_u32(stg); amn = 0; }
      if (b_mn) { b_base = smem_u32(stg) + 128 * 128; bmn = 0; }
    }
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint64_t da = amn ? wg_desc_sw128(a_base + half + k * 2048, GROUP_BYTES, 1024)
                              : wg_desc_sw128(a_base + half + k * 32, 16, 1024);
      const uint64_t db = bmn ? wg_desc_sw128(b_base + k * 2048, GROUP_BYTES, 1024) : wg_desc_sw128(b_base + k * 32, 16, 1024);
      Wgmma<T, BLOCK_N>::mma(acc, da, db, (it | k) != 0 ? 1u : 0u, amn, bmn);
    }
    wgmma_commit();
    wgmma_wait<1>();                                                // the previous stage's MMAs have retired
    if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev]);
    prev = stage;
    if (++stage == stages) { stage = 0; phase ^= 1; }
  }
  wgmma_wait<0>();
  if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev]);
}

// The warpgroup's 64 x N accumulator fragment -> rows [0, 64) of an fp32 shared-memory tile with row pitch `ld` floats
// (the caller offsets `tile` to the warpgroup's first row).
template <int N>
__device__ __forceinline__ void wg_store_acc(float* tile, int ld, const float (&d)[N / 2]) {
  const int r = 16 * ((threadIdx.x >> 5) & 3) + (lane_id() >> 2), c = 2 * (lane_id() & 3);
#pragma unroll
  for (int i = 0; i < N / 8; ++i) {
    *reinterpret_cast<float2*>(tile + r * ld + 8 * i + c) = make_float2(d[4 * i], d[4 * i + 1]);
    *reinterpret_cast<float2*>(tile + (r + 8) * ld + 8 * i + c) = make_float2(d[4 * i + 2], d[4 * i + 3]);
  }
}
// 32 consecutive fp32 columns of one row of such a tile (ld % 4 == 0), as raw bits
__device__ __forceinline__ void acc_ld32(const float* tile, int ld, int row, int col, uint32_t (&v)[32]) {
  const float4* p = reinterpret_cast<const float4*>(tile + row * ld + col);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float4 t = p[j];
    v[4 * j] = __float_as_uint(t.x); v[4 * j + 1] = __float_as_uint(t.y);
    v[4 * j + 2] = __float_as_uint(t.z); v[4 * j + 3] = __float_as_uint(t.w);
  }
}

// ----------------------------------------------------------------------------- memory-model helpers
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_acquire_gpu(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_add_release_gpu(uint32_t* p, uint32_t v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// ----------------------------------------------------------------------------- programmatic dependent launch
// Every kernel of the stage programs is launched with programmaticStreamSerialization: it may begin (barrier init,
// descriptor prefetch, parameter loads) while its predecessor drains, and must execute pdl_wait()
// before touching global memory.  pdl_trigger() lets the *next* kernel start its own prologue early.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}

// 32 consecutive output columns of one row (fp32 accumulator values) -> bf16 (64 B) or fp32 (128 B), 16-byte stores
__device__ __forceinline__ void store_row32(__nv_bfloat16* o, const float (&f)[32]) {
  uint4* o4 = reinterpret_cast<uint4*>(o);
#pragma unroll
  for (int j = 0; j < 4; ++j)
    o4[j] = make_uint4(pack_bf16x2(f[8 * j], f[8 * j + 1]), pack_bf16x2(f[8 * j + 2], f[8 * j + 3]),
                       pack_bf16x2(f[8 * j + 4], f[8 * j + 5]), pack_bf16x2(f[8 * j + 6], f[8 * j + 7]));
}
__device__ __forceinline__ void store_row32(float* o, const float (&f)[32]) {
  float4* o4 = reinterpret_cast<float4*>(o);
#pragma unroll
  for (int j = 0; j < 8; ++j) o4[j] = make_float4(f[4 * j], f[4 * j + 1], f[4 * j + 2], f[4 * j + 3]);
}
__device__ __forceinline__ void store_row8(__nv_bfloat16* o, const float (&r)[8]) {
  *reinterpret_cast<uint4*>(o) = make_uint4(pack_bf16x2(r[0], r[1]), pack_bf16x2(r[2], r[3]), pack_bf16x2(r[4], r[5]), pack_bf16x2(r[6], r[7]));
}
__device__ __forceinline__ void store_row8(float* o, const float (&r)[8]) {
  reinterpret_cast<float4*>(o)[0] = make_float4(r[0], r[1], r[2], r[3]);
  reinterpret_cast<float4*>(o)[1] = make_float4(r[4], r[5], r[6], r[7]);
}
// the value a consumer will read back after the store (bf16 rounding is part of the stored activation)
__device__ __forceinline__ float stored_value(float x, const __nv_bfloat16*) { return __bfloat162float(__float2bfloat16(x)); }
__device__ __forceinline__ float stored_value(float x, const float*) { return x; }

// host: launch with the PDL attribute (SLB200_PDL=0 disables it; the device-side waits then are no-ops)
inline int pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("SLB200_PDL");
    v = (e && e[0] == '0') ? 0 : 1;
  }
  return v;
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = pdl_enabled();
  cfg.attrs = at;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// ----------------------------------------------------------------------------- run-to-run reproducible reductions
// Float atomics add in whatever order the blocks arrive, so sums differed in their last bits from run to run and a training
// run drifted apart.  Every cross-block float reduction goes through one of these two orders instead:
//   det_commit  many blocks: block m of a group stores its partial row, the last block to arrive sums the rows in m order;
//   turn_*      few slices (split-K): slice z adds its partial into the output after slice z - 1 has (a turn counter).
// Both rely on blocks of lower linear index being scheduled no later than higher ones.  Counters are zero at rest: the last
// participant resets them.  Scratch and counters belong to a stream (kernels of one stream never overlap their reductions).
struct Det {
  float* part;          // scratch for partial rows
  uint32_t* ctr;        // DET_COUNTERS zeroed counters
  long long cap;        // floats in `part`
};
constexpr int DET_COUNTERS = 4096;
constexpr int DET_TURN_BASE = 64;             // counters [0, 64): det_commit groups; [64, 4096): split-K turns
Det slb_det(cudaStream_t st);                 // elementwise.cu; part == nullptr when the scratch could not be allocated
void slb_det_release(cudaStream_t st);        // frees the stream's scratch (before the stream is destroyed)

__device__ __forceinline__ void st_release_gpu(uint32_t* p, uint32_t v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void turn_wait(const uint32_t* ctr, uint32_t my) {
  uint32_t spins = 0;
  while (ld_acquire_gpu(ctr) != my)
    if (++spins > (1u << 30)) __trap();
}
// after this participant's adds: make them visible, then hand the turn on (the last one resets the counter)
__device__ __forceinline__ void turn_pass(uint32_t* ctr, uint32_t my, uint32_t total) {
  __threadfence();
  st_release_gpu(ctr, my + 1 == total ? 0u : my + 1);
}
template <int BAR>            // BAR < 0: __syncthreads, else named barrier BAR over nthr threads
__device__ __forceinline__ void det_bar(int nthr) {
  if constexpr (BAR < 0) __syncthreads();
  else asm volatile("bar.sync %0, %1;" ::"n"(BAR), "r"(nthr) : "memory");
}
// Called by the nthr participating threads (tid 0..nthr-1) of every member block of group `grp`: adds the n values of
// s_vals (shared memory) into dst0[0, n0) and dst1[0, n - n0), summed over the members in member order.
template <int BAR>
__device__ __forceinline__ void det_commit(const Det& d, int grp, int member, int members, const float* s_vals, int n,
                                           float* dst0, int n0, float* dst1, int tid, int nthr) {
  __shared__ uint32_t s_last;
  float* rows = d.part + static_cast<long long>(grp) * members * n;
  for (int i = tid; i < n; i += nthr) rows[static_cast<long long>(member) * n + i] = s_vals[i];
  __threadfence();
  det_bar<BAR>(nthr);
  if (tid == 0) {
    const uint32_t t = atomicAdd(d.ctr + grp, 1u);
    s_last = (t == static_cast<uint32_t>(members) - 1u) ? 1u : 0u;
    if (s_last) d.ctr[grp] = 0;
  }
  det_bar<BAR>(nthr);
  if (!s_last) return;
  __threadfence();
  for (int i = tid; i < n; i += nthr) {
    float s = 0.f;
    for (int m = 0; m < members; ++m) s += __ldcg(rows + static_cast<long long>(m) * n + i);
    if (i < n0) dst0[i] += s;
    else dst1[i - n0] += s;
  }
}

}  // namespace slb
