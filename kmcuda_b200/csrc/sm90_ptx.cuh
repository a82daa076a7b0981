// sm90_ptx.cuh -- thin inline-PTX wrappers for the Hopper (sm_90a) features the assignment kernel uses:
// mbarrier, TMA (cp.async.bulk[.tensor]) and warpgroup MMA (wgmma.mma_async).  Nothing here is CUTLASS;
// descriptor bit layouts follow the PTX ISA "asynchronous warpgroup level matrix" shared-memory descriptor.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace kmb {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---------------------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// named barrier `id` (1..15; 0 is __syncthreads) among `nthreads` threads of the CTA, a multiple of 32
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
// Bounded wait: a stuck pipeline must not hang the GPU.  The try_wait carries a suspend-time hint, so a waiting
// warp sleeps until the barrier's phase flips (or the hint expires) instead of competing for issue slots.
__device__ __forceinline__ bool mbar_try_wait(uint32_t addr, uint32_t parity, uint32_t hint_ns) {
  uint32_t done;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(done)
      : "r"(addr), "r"(parity), "r"(hint_ns)
      : "memory");
  return done != 0;
}
constexpr uint32_t WAIT_HINT_NS = 2000;   // suspend-time hint of the first probe of every wait
// Remainder of every wait: a tight polling loop (a hinted try_wait returns on every update of the barrier, not only
// when the phase flips, so the error word and the clock are checked only every 1024 probes).  Inlined: under setmaxnreg,
// ptxas cannot allocate a call made while wgmma accumulators are in flight.
// `site` names the waiting role; after ~2 s (or as soon as another thread has reported an error) the wait gives up
// and reports 0x1000 + site in *err: a stuck pipeline must not hang the GPU.
#ifndef KMB_SLOW_HINT_NS
#define KMB_SLOW_HINT_NS 20000
#endif
__device__ __forceinline__ void mbar_wait_slow(uint32_t addr, uint32_t parity, uint32_t* err, uint32_t site, uint32_t flag_u32) {
  // flag_u32: a word of this CTA's shared memory that is set once any wait of the CTA has given up; from then on every
  // wait returns at once, so a broken pipeline drains in milliseconds instead of timing out wait by wait
  uint32_t dead;
  asm volatile("ld.volatile.shared.u32 %0, [%1];" : "=r"(dead) : "r"(flag_u32));
  if (dead) return;
  const long long t0 = clock64();
  for (;;) {
    uint32_t done;
    asm volatile(
        "{\n\t.reg .pred p, q;\n\t.reg .b32 c;\n\t"
        "mov.u32 c, 0;\n"
        "KMB_WAIT_LOOP_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "@p bra KMB_WAIT_DONE_%=;\n\t"
        "add.u32 c, c, 1;\n\t"
        "setp.lt.u32 q, c, 1024;\n\t"
        "@q bra KMB_WAIT_LOOP_%=;\n"
        "KMB_WAIT_DONE_%=:\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(addr), "r"(parity), "r"(static_cast<uint32_t>(KMB_SLOW_HINT_NS))
        : "memory");
    if (done) return;
    asm volatile("ld.volatile.shared.u32 %0, [%1];" : "=r"(dead) : "r"(flag_u32));
    const bool lost = dead || *reinterpret_cast<volatile uint32_t*>(err);
    if (lost || clock64() - t0 > 4000000000ll) {
      if (!lost) atomicMax(err, 0x1000u + site);
      asm volatile("st.volatile.shared.u32 [%0], %1;" ::"r"(flag_u32), "r"(1u) : "memory");
      return;
    }
  }
}
// The inline part: one probe (with the suspend hint it may sleep up to the hint while the phase has not flipped).
__device__ __forceinline__ void mbar_wait(uint32_t addr, uint32_t parity, uint32_t* err, uint32_t site, uint32_t flag_u32) {
  if (!mbar_try_wait(addr, parity, WAIT_HINT_NS)) mbar_wait_slow(addr, parity, err, site, flag_u32);
}

// ---------------------------------------------------------------------------- fp32 pairs
// Two fp32 values carried in one 64-bit register pair.  Hopper has no packed fp32 instructions, so each helper is
// two scalar operations with the same IEEE rounding; the pair form keeps the callers' arithmetic in one place.
__device__ __forceinline__ uint64_t pack2(float lo, float hi) {
  uint64_t r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
  return r;
}
__device__ __forceinline__ void unpack2(uint64_t v, float& lo, float& hi) {
  asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
__device__ __forceinline__ uint64_t fadd2(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1;
  unpack2(a, a0, a1);
  unpack2(b, b0, b1);
  return pack2(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
__device__ __forceinline__ uint64_t fsub2(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1;
  unpack2(a, a0, a1);
  unpack2(b, b0, b1);
  return pack2(__fsub_rn(a0, b0), __fsub_rn(a1, b1));
}
__device__ __forceinline__ uint64_t ffma2(uint64_t a, uint64_t b, uint64_t c) {
  float a0, a1, b0, b1, c0, c1;
  unpack2(a, a0, a1);
  unpack2(b, b0, b1);
  unpack2(c, c0, c1);
  return pack2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
// maximum of three; NaN operands are ignored like fmaxf
__device__ __forceinline__ float fmax3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }

// generic-proxy writes to shared memory -> visible to the async proxy (wgmma / TMA reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---------------------------------------------------------------------------- TMA
__device__ __forceinline__ void prefetch_tmap(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
// 2-D tiled load: coordinates {c0 (innermost), c1}
__device__ __forceinline__ void tma_load_2d(void* dst, const void* tmap, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// 1-D bulk copy global -> shared (size multiple of 16, both 16-byte aligned)
__device__ __forceinline__ void bulk_load(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// ---------------------------------------------------------------------------- wgmma
// shared-memory matrix descriptor (PTX ISA, wgmma "matrix descriptor"):
//   [0,14)  start address >> 4        [16,30) leading-dim byte offset >> 4
//   [32,46) stride-dim byte offset >> 4   [49,52) base offset = 0   [62,64) swizzle: 0 none, 1 128B, 2 64B, 3 32B
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes,
                                                   uint32_t swizzle) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr >> 4) & 0x3FFF);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(swizzle & 3) << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of the accumulator registers across an asynchronous wgmma
template <int N>
__device__ __forceinline__ void wgmma_fence_acc(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; i++) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64 x 64] (+)= A[64 x 16] * B[64 x 16]^T, the same fragment layout as below with j < 8:
// d[j*4 + h*2 + e] = (row warp*16 + h*8 + lane/4, column 8j + 2*(lane%4) + e)
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(accumulate)
      : "memory");
}
// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T, fp16 operands from shared memory (both K-major), fp32 accumulators in
// the registers of the warpgroup: d[j*4 + h*2 + e] = (row warp*16 + h*8 + lane/4, column 8j + 2*(lane%4) + e)
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate)
      : "memory");
}

// per-warpgroup register budget (every warp of the warpgroup executes it): .dec hands registers back to the CTA's pool,
// .inc waits until the pool can grant the new count
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

__device__ __forceinline__ float4 ldg_nc_f4(const float* p) {
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p));
  return v;
}

}  // namespace ptx
}  // namespace kmb
