// wgmma / mbarrier / bulk-copy primitives shared by the tensor-core kernels (sm_90a inline PTX).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "wgmma.cuh"

namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// generic-proxy shared-memory writes -> visible to the async proxy (wgmma operand reads, bulk copies)
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// 1-D bulk copy global -> shared (TMA engine), completion signalled on an mbarrier
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   dst_smem),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}

// K-major SWIZZLE_128B operand descriptor: 8-row groups of 128-byte rows, 1024 bytes apart.
// A k-step inside the 128-byte row advances the start address by its byte offset.
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);   // start address
  d |= (uint64_t)1 << 16;                         // leading byte offset (unused for SW128 K-major)
  d |= (uint64_t)(1024 >> 4) << 32;               // stride byte offset: next 8-row group
  d |= (uint64_t)1 << 62;                         // SWIZZLE_128B
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int kPending>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(kPending) : "memory");
}
// pins the accumulator registers in place across wgmma_wait: no read may be hoisted above it
template <int R>
__device__ __forceinline__ void fence_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

__device__ __forceinline__ void red_add_v2(float* addr, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ float tf32_round(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

// split one float4 into a TF32 "hi" part (round to nearest) and the exact fp32 residual "lo"
// (the tensor core truncates lo to TF32: 2^-21 relative overall) and store both 16-byte pieces
__device__ __forceinline__ void split_store(float4 v, unsigned char* hi_tile, unsigned char* lo_tile, uint32_t off) {
  float4 h, l;
  h.x = tf32_round(v.x); h.y = tf32_round(v.y); h.z = tf32_round(v.z); h.w = tf32_round(v.w);
  l.x = v.x - h.x; l.y = v.y - h.y; l.z = v.z - h.z; l.w = v.w - h.w;
  *reinterpret_cast<float4*>(hi_tile + off) = h;
  *reinterpret_cast<float4*>(lo_tile + off) = l;
}

// 3xFP16 split: fp16 carries the same 11 significant bits as TF32 at half the bytes and twice the tensor
// rate.  x is first scaled by a power of two `sx` (exact) that maps the tensor's absolute maximum into
// [2^14, 2^15) - below fp16's 65504, far above its 2^-14 normal floor - then split into hi = fp16(x'),
// lo = fp16(x' - hi): the same hi*hi + lo*hi + hi*lo products as 3xTF32, 2^-21 relative (an element more
// than 2^17 below the tensor's maximum loses bits of its lo part: <= 2^-39 of the maximum).
__device__ __forceinline__ void split_store_f16(float4 a, float4 b, float sx, unsigned char* hi_tile,
                                                unsigned char* lo_tile, uint32_t off) {
  const float x[8] = {a.x * sx, a.y * sx, a.z * sx, a.w * sx, b.x * sx, b.y * sx, b.z * sx, b.w * sx};
  uint32_t h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const __half2 hh = __floats2half2_rn(x[2 * i], x[2 * i + 1]);
    const float2 hf = __half22float2(hh);
    const __half2 ll = __floats2half2_rn(x[2 * i] - hf.x, x[2 * i + 1] - hf.y);
    h[i] = *reinterpret_cast<const uint32_t*>(&hh);
    l[i] = *reinterpret_cast<const uint32_t*>(&ll);
  }
  *reinterpret_cast<uint4*>(hi_tile + off) = make_uint4(h[0], h[1], h[2], h[3]);
  *reinterpret_cast<uint4*>(lo_tile + off) = make_uint4(l[0], l[1], l[2], l[3]);
}
// power of two that maps `amax` into [2^14, 2^15); 1 for amax == 0 / non-finite
__device__ __forceinline__ float f16_scale_for(float amax) {
  const uint32_t b = __float_as_uint(amax);
  const int e = (int)((b >> 23) & 255u);
  if (e == 0 || e == 255) return 1.f;
  int se = 14 - (e - 127) + 127;
  se = se < 1 ? 1 : (se > 254 ? 254 : se);
  return __uint_as_float((uint32_t)se << 23);
}

// One 128-byte K chunk (4 k-steps of 32 bytes) of a warpgroup's D[64, N] += A . B^T.
// kPasses = 3: hi*hi + lo*hi + hi*lo (split operands, fp32-accurate); kPasses = 1: hi*hi only.
template <int N, bool kF16, int kPasses>
__device__ __forceinline__ void mma_chunk(float (&d)[N / 2], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi,
                                          uint32_t b_lo) {
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    const uint32_t ko = ks * 32;
    const uint64_t dbh = wgmma_desc(b_hi + ko);
    Wgmma<N, kF16>::mma(d, wgmma_desc(a_hi + ko), dbh);
    if (kPasses == 3) {
      Wgmma<N, kF16>::mma(d, wgmma_desc(a_lo + ko), dbh);
      Wgmma<N, kF16>::mma(d, wgmma_desc(a_hi + ko), wgmma_desc(b_lo + ko));
    }
  }
}

}  // namespace tc
