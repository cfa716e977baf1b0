// Thin inline-PTX layer for sm_90a: mbarrier, bulk async copy, warpgroup MMA (wgmma) and its shared-memory descriptors.
// Bit layouts follow the PTX ISA "matrix descriptor" and "wgmma register fragment" sections; the kernels own their
// pipelines.
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>

namespace gmma {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier -------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// try_wait with a suspend-time hint: a waiting thread sleeps in hardware (no issue slots) until the phase completes
// or the hint expires, so role warps that mostly wait do not take issue slots from the gather warps.
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity), "r"(0x4000u)
      : "memory");
  return ok != 0;
}
#ifdef PASCO_HANG_TRAP
// debug build (PASCO_NVCC_FLAGS=-DPASCO_HANG_TRAP python -m pasco_b200.build --force): a wait that spins for ~1 s reports
// who waits on what and traps, so that a pipeline deadlock shows up as an error with a location instead of a hang
static __device__ __noinline__ void mbar_wait_report(uint32_t bar, uint32_t parity) {
  printf("HANG block %d thread %d (warp %d) waits on smem barrier 0x%x parity %u\n", blockIdx.x, threadIdx.x, threadIdx.x >> 5, bar, parity);
  __trap();
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  unsigned long long spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1ull << 17)) mbar_wait_report(bar, parity);
  }
}
#else
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
#endif

// ---- async-proxy visibility of generic st.shared writes ------------------------------------------------
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- 1-D bulk copy global → shared, completion on an mbarrier -------------------------------------------
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}

// named barrier over `nthreads` threads (whole warps), ids 1.. (0 is __syncthreads)
__device__ __forceinline__ void named_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// per-thread register budget of the executing warpgroup (all 4 warps execute it): the warpgroups that wait most of the
// time hand registers to the ones that hold accumulators
template <uint32_t R>
__device__ __forceinline__ void reg_alloc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <uint32_t R>
__device__ __forceinline__ void reg_dealloc() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

// ---- descriptors ---------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor, 128-byte swizzle.  Tiles are stored as rows of 128 bytes (64 bf16), 8 rows =
// one 1024-byte swizzle atom, 16-byte chunk c of row r lives at chunk (c ^ (r & 7)).
//   K-major  operand (rows = M/N index, 128 B = 64 K-elements): SBO = 1024 (next 8 rows), LBO unused (1);
//            the k-step of 16 elements (32 bytes) advances the start-address field by 2
//   MN-major operand (rows = K index,   128 B = 64 M/N-elements): SBO = 1024 (next 8 K-rows),
//            LBO = byte distance to the next 64 M/N elements; the k-step of 16 rows advances the start by 2048 bytes
__device__ __forceinline__ uint64_t make_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;  // SWIZZLE_128B
  return d;
}

// ---- wgmma ---------------------------------------------------------------------------------------------------
// Issued by a whole warpgroup (4 consecutive warps starting at a multiple of 4).  D[64 x N] fp32 lives in registers:
// thread t of the warpgroup (warp w = t / 32, lane l) holds d[i] at
//   row = 16 w + l / 4 + 8 ((i >> 1) & 1),   col = 8 (i >> 2) + 2 (l & 3) + (i & 1).
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ int frag_row(int i, int wq, int lane) { return 16 * wq + (lane >> 2) + 8 * ((i >> 1) & 1); }
__device__ __forceinline__ int frag_col(int i, int lane) { return 8 * (i >> 2) + 2 * (lane & 3) + (i & 1); }

// D[64 x 64] += A[64 x 16] · B[16 x 64], bf16 operands from shared memory; TA / TB: operand is MN-major
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.eq.u32 p, 1, 1;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, %34, %35;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "n"(TA), "n"(TB));
}
// D[64 x 128] += A[64 x 16] · B[16 x 128]: one instruction reads A once for 128 columns (two n64 MMAs on the same A read
// it twice); same fragment layout, d[0..31] = columns 0-63, d[32..63] = columns 64-127
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.eq.u32 p, 1, 1;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, %66, %67;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
        "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
        "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
        "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
        "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "n"(TA), "n"(TB));
}
// D[64 x 16] += A[64 x 16] · B[16 x 16], both operands K-major
__device__ __forceinline__ void wgmma_n16(float (&d)[8], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.eq.u32 p, 1, 1;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(adesc), "l"(bdesc));
}

// ---- bf16 split helpers -------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}
// x ≈ hi + lo with hi = bf16(x), lo = bf16(x − hi): 16 mantissa bits in total.  Packed conversions only
// (F2FP.BF16.PACK_AB, full-rate ALU) — the scalar F2F path is quarter rate and dominated the gather warps.
__device__ __forceinline__ void split4(const float4& x, uint2& hi, uint2& lo) {
  const uint32_t h01 = pack_bf16x2(x.x, x.y), h23 = pack_bf16x2(x.z, x.w);
  hi.x = h01;
  hi.y = h23;
  const float r0 = x.x - __uint_as_float(h01 << 16), r1 = x.y - __uint_as_float(h01 & 0xffff0000u);
  const float r2 = x.z - __uint_as_float(h23 << 16), r3 = x.w - __uint_as_float(h23 & 0xffff0000u);
  lo.x = pack_bf16x2(r0, r1);
  lo.y = pack_bf16x2(r2, r3);
}
__device__ __forceinline__ uint2 to_bf16x4(const float4& x) { return make_uint2(pack_bf16x2(x.x, x.y), pack_bf16x2(x.z, x.w)); }

}  // namespace gmma
