// tng_ptx.cuh — the device helpers shared by the kernels of libtango_b200.so (sm_90a, Hopper H100):
//   * thin inline-PTX wrappers: mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA with shared-memory
//     descriptors), fences; hand-written PTX, no CUTLASS / CuTe dependency;
//   * the flash-attention online-softmax step on a wgmma score fragment;
//   * activations, warp / quad reductions, and bf16 I/O including the hi/lo split of the "split" precision.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/tango_b200.h"

namespace tng {

#ifndef TNG_SPIN_LIMIT
// Bounded spin on mbarriers: a protocol bug traps (visible error) instead of hanging the GPU box.
#define TNG_SPIN_LIMIT (1u << 28)
#endif

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// arrive only where `pred` holds, without a branch (a divergent branch while wgmma are in flight makes ptxas serialise them)
__device__ __forceinline__ void mbar_arrive_if(uint64_t* bar, bool pred) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %1, 0;\n\t@p mbarrier.arrive.shared::cta.b64 _, [%0];\n\t}"
      ::"r"(smem_u32(bar)), "r"((uint32_t)pred) : "memory");
}
// move registers between warpgroups (warp-specialised kernels: the producer gives, the consumers take)
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
__device__ __forceinline__ uint32_t mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok;
}
// No printf on the timeout path: a function call inside a wgmma pipeline makes ptxas serialise every wgmma of the kernel.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > TNG_SPIN_LIMIT) __trap();
  }
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];" ::"r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// ---------------------------------------------------------------- wgmma
// A warpgroup (4 consecutive warps, 128 threads) computes a 64 x N tile: warp w of the group owns rows [16w, 16w + 16);
// lane l holds, for every 8-column group j, d[4j + {0, 1}] = (row 16w + l/4, columns 8j + 2(l%4) + {0, 1}) and
// d[4j + {2, 3}] = the same columns of row 16w + l/4 + 8. The register A operand of an m64k16 step uses the same
// layout: the accumulator columns [16kk, 16kk + 16) of a previous wgmma, packed to bf16 pairs, are that operand.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accesses of accumulator registers across the asynchronous wgmma window
template <int R>
__device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Shared-memory matrix descriptor, SWIZZLE_128B, for tiles whose rows are 128 bytes (64 bf16), 1024-byte aligned atoms:
//   bits [0,14)  start address >> 4        bits [16,30) leading byte offset >> 4
//   bits [32,46) stride byte offset >> 4   bits [62,64) layout type (1 = SWIZZLE_128B)
// K-major operand (rows = M/N index, 64 K-elements per 128 B row): SBO = 1024 (8-row swizzle atom), LBO unused; the
//   16-element K steps inside the row advance the start address by 32 bytes (+2 in the address field).
// MN-major operand (rows = K index, 64 MN-elements per 128 B row): SBO = 1024 between 8-K-row groups,
//   LBO = byte distance between 64-wide MN atoms (unused when the operand is one atom wide).
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// D (+)= A * B^T, bf16 x bf16 -> fp32, both operands K-major in shared memory (scale_d = 0: D = A * B^T)
template <int N>
__device__ __forceinline__ void wgmma_ss(float (&d)[N / 2], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d);

template <>
__device__ __forceinline__ void wgmma_ss<32>(float (&d)[16], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a_desc), "l"(b_desc), "r"(scale_d));
}

template <>
__device__ __forceinline__ void wgmma_ss<64>(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a_desc), "l"(b_desc), "r"(scale_d));
}

template <>
__device__ __forceinline__ void wgmma_ss<128>(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a_desc), "l"(b_desc), "r"(scale_d));
}

template <>
__device__ __forceinline__ void wgmma_ss<160>(float (&d)[80], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %82, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n160k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79}, %80, %81, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79])
      : "l"(a_desc), "l"(b_desc), "r"(scale_d));
}

template <>
__device__ __forceinline__ void wgmma_ss<256>(float (&d)[128], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(a_desc), "l"(b_desc), "r"(scale_d));
}

// A from registers (the accumulator-shaped fragment of a previous wgmma), B MN-major (transposed) in shared memory
__device__ __forceinline__ void wgmma_rs_n64_tb(float (&d)[32], const uint32_t (&a)[4], uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(scale_d));
}

// ---------------------------------------------------------------- misc math
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// 2^x for x <= 0 on the FMA pipe instead of MUFU (which does 16 ex2 per clock per SM against 128 FMAs): x = n + f with
// n = floor(x) (a round-down add of 1.5 * 2^23 leaves n in the low mantissa bits of t), 2^f on [0, 1] by a degree-4
// minimax polynomial with p(0) = 1 in Horner form, then a multiply by 2^n built from t's bits. It agrees with
// ex2.approx.ftz at the edges the softmax reaches: -inf -> +0, x < -126 -> +0 (2^n is +0 for n = -127, the clamp),
// 0 -> exactly 1. Relative error <= 2^-18 over [-126, 0] (tests/test_attention_exp2_cpu.py states it in torch).
__device__ __forceinline__ float ex2_poly(float x) {
  x = fmaxf(x, -127.0f);
  const float t = __fadd_rd(x, 12582912.0f);
  const float f = x - (t - 12582912.0f);
  float p = fmaf(0x1.b7ea5cp-7f, f, 0x1.abfe7ep-5f);
  p = fmaf(p, f, 0x1.ee2374p-3f);
  p = fmaf(p, f, 0x1.62d6d0p-1f);
  p = fmaf(p, f, 1.0f);
  return p * __int_as_float((__float_as_int(t) << 23) + 0x3f800000);
}
__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// SiLU with the two MUFU approximations (ex2, rcp) and no range fix-ups: 5 instructions, relative error ~2e-7.
// x -> -inf gives x * rcp(inf) = -0, x -> +inf gives x * rcp(1) = x.
__device__ __forceinline__ float silu_f(float x) {
  return x * rcp_approx(1.0f + ex2_approx(x * -1.4426950408889634f));
}
// GELU (erf form, attention.py:431-433 / F.gelu default) as x * Phi(x), Phi(x) = 1 - q for x >= 0 and q otherwise,
// q = 0.5 * erfc(|x| / sqrt 2) by Abramowitz-Stegun 7.1.26 (|abs err| <= 1.5e-7 on erf, below the fp32 round-off of the
// surrounding arithmetic). The constants are folded so that the exponent argument is a single product:
// w = |x| * sqrt(log2(e) / 2)  =>  exp(-x^2/2) = 2^(-w*w),  t = 1 / (1 + p * |x| / sqrt 2) = 1 / (1 + (p / sqrt(log2 e)) * w),
// and the 0.5 is folded into the polynomial. ~14 instructions (2 MUFU) instead of the ~30 of erff().
__device__ __forceinline__ float gelu_erf_f(float x) {
  const float w = fabsf(x) * 0.84932180028801904272f;
  const float t = rcp_approx(fmaf(0.27273748088f, w, 1.0f));
  const float e = ex2_approx(w * -w);
  float poly = fmaf(0.5307027145f, t, -0.7265760135f);
  poly = fmaf(poly, t, 0.7107068705f);
  poly = fmaf(poly, t, -0.142248368f);
  poly = fmaf(poly, t, 0.127414796f);
  const float q = poly * t * e;
  const float phi = x >= 0.0f ? 1.0f - q : q;
  return x * phi;
}
// GELU, tanh form ("gelu_new" of the T5 v1.1 / FLAN-T5 gated feed-forward):
// 0.5 x (1 + tanh(u)) = x * sigmoid(2u), u = sqrt(2/pi) (x + 0.044715 x^3); 2 MUFU, relative error ~3e-7.
__device__ __forceinline__ float gelu_tanh_f(float x) {
  const float w = x * fmaf(x * x, 0.044715f, 1.0f);
  return x * rcp_approx(1.0f + ex2_approx(w * -2.3022081986f));   // 2 sqrt(2/pi) log2(e)
}
__device__ __forceinline__ float act_f(float x, int act, float p) {
  if (act == TNG_ACT_SILU) return silu_f(x);
  if (act == TNG_ACT_LRELU) return x > 0.f ? x : x * p;
  return x;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// over the four lanes that hold one row of a wgmma accumulator (lanes 4i .. 4i + 3)
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}
__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}

// ---------------------------------------------------------------- bf16 I/O
// The "split" precision stores an operand x as hi = bf16_rn(x) and, split_off elements further, lo = bf16_rn(bf16_lo(x)).
// The split GEMM and attention kernels rely on this exact residual; every writer of a lo half uses the helpers below.
__device__ __forceinline__ float bf16_lo(float v) { return v - __bfloat162float(__float2bfloat16_rn(v)); }
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ uint32_t pack_bf16_lo(float a, float b) { return pack_bf16(bf16_lo(a), bf16_lo(b)); }
__device__ __forceinline__ float4 load_bf16x4(const __nv_bfloat16* p) {
  const uint2 u = *reinterpret_cast<const uint2*>(p);
  const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.x));
  const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.y));
  return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ void store4_bf16(__nv_bfloat16* p, float4 v) {
  uint2 u;
  u.x = pack_bf16(v.x, v.y);
  u.y = pack_bf16(v.z, v.w);
  *reinterpret_cast<uint2*>(p) = u;
}
__device__ __forceinline__ void store4_bf16_lo(__nv_bfloat16* p, float4 v) {
  store4_bf16(p, make_float4(bf16_lo(v.x), bf16_lo(v.y), bf16_lo(v.z), bf16_lo(v.w)));
}
// hi at p and, when split_off > 0, lo at p + split_off
__device__ __forceinline__ void store4_split(__nv_bfloat16* p, float4 v, int split_off) {
  store4_bf16(p, v);
  if (split_off > 0) store4_bf16_lo(p + split_off, v);
}
__device__ __forceinline__ void store_bf16_split(__nv_bfloat16* p, float v, int split_off) {
  const __nv_bfloat16 hi = __float2bfloat16_rn(v);
  *p = hi;
  if (split_off > 0) p[split_off] = __float2bfloat16_rn(v - __bfloat162float(hi));
}

// ---------------------------------------------------------------- flash attention on wgmma fragments
// A 64 x 64 score tile in the accumulator layout of a warpgroup (see wgmma above): this thread holds rows r and r + 8
// of its warp's 16, s[4j + {0, 1}] of row r and s[4j + {2, 3}] of row r + 8. Index 0 / 1 of the per-row arrays below is
// row r / r + 8; l_run is this lane's partial sum (the quad's lanes are combined by softmax_inv).
//
// One online-softmax step in the log2 domain: s * scl are the scaled scores (masked keys at -inf) and s becomes the
// unnormalised probabilities 2^(s * scl - m), one FMA and one ex2 per score; m_run / l_run are updated; corr receives
// the factor by which everything accumulated over the previous tiles must be scaled. scl > 0, so the row maximum of
// s * scl is the maximum of s times scl; with scl = 1 the FMA is exactly s - m. A row whose scores are all -inf so far
// keeps m_run = -inf and gets probabilities 0 (instead of the NaN of -inf - -inf).
// POLY_EVERY > 0 moves every POLY_EVERY-th exponential of each row (a fixed set of registers) from MUFU to ex2_poly.
template <int POLY_EVERY = 0>
__device__ __forceinline__ void softmax_step(float (&s)[32], float scl, float (&m_run)[2], float (&l_run)[2],
                                             float (&corr)[2]) {
  auto ex2 = [](float x, int k) {
    if constexpr (POLY_EVERY > 0)
      if (k % POLY_EVERY == POLY_EVERY - 1) return ex2_poly(x);
    return ex2_approx(x);
  };
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int j = 0; j < 8; ++j) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      mx[0] = fmaxf(mx[0], s[4 * j + e]);
      mx[1] = fmaxf(mx[1], s[4 * j + 2 + e]);
    }
  }
  float m_use[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const float m_new = fmaxf(m_run[h], quad_max(mx[h]) * scl);
    m_use[h] = (m_new == -INFINITY) ? 0.f : m_new;
    corr[h] = ex2_approx(m_run[h] - m_use[h]);   // 0 on the first tile (m_run = -inf)
    m_run[h] = m_new;
    l_run[h] *= corr[h];
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      s[4 * j + e] = ex2(fmaf(s[4 * j + e], scl, -m_use[0]), 2 * j + e);
      s[4 * j + 2 + e] = ex2(fmaf(s[4 * j + 2 + e], scl, -m_use[1]), 16 + 2 * j + e);
      l_run[0] += s[4 * j + e];
      l_run[1] += s[4 * j + 2 + e];
    }
  }
}
// o: a [64 x 64] output accumulator in the same layout
__device__ __forceinline__ void rescale_rows(float (&o)[32], const float (&corr)[2]) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    o[4 * j] *= corr[0]; o[4 * j + 1] *= corr[0];
    o[4 * j + 2] *= corr[1]; o[4 * j + 3] *= corr[1];
  }
}
// P as the register A operand of O += P V: k-step kk (keys [16kk, 16kk + 16)) = accumulator registers [8kk, 8kk + 8).
// LO packs the bf16 residuals instead (the lo half of P in the split precision).
template <bool LO = false>
__device__ __forceinline__ void pack_p(uint32_t (&pa)[4][4], const float (&s)[32]) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk)
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const float x0 = s[8 * kk + 2 * r], x1 = s[8 * kk + 2 * r + 1];
      pa[kk][r] = LO ? pack_bf16_lo(x0, x1) : pack_bf16(x0, x1);
    }
}
// the final normalisation: 1 / (row sum) of both rows
__device__ __forceinline__ void softmax_inv(const float (&l_run)[2], float (&inv)[2]) {
#pragma unroll
  for (int h = 0; h < 2; ++h) inv[h] = 1.0f / quad_sum(l_run[h]);
}

}  // namespace tng
