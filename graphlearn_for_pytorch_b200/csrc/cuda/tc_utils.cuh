// wgmma / TMA / mbarrier PTX wrappers shared by the sm_90a tensor-core kernels
// (sage_tc.cu: fused gather+aggregate+GEMM; tc_gemm.cu: TMA-fed dense GEMMs of the engine).
#pragma once
#include "device_utils.cuh"

namespace glt {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}\n" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
      "l"(src), "r"(bytes), "r"(bar)
      : "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// Shared-memory matrix descriptor of wgmma, SWIZZLE_128B, K-major (LBO unused) -- 8-row groups 1024 B apart.
__device__ __forceinline__ uint64_t make_sw128_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;   // SWIZZLE_128B
  return d;
}

// warpgroup MMA (wgmma.mma_async): all 128 threads of a 4-warp-aligned warpgroup issue it together; the fp32
// accumulator fragment of m64nN lives in registers: d[4 j + 2 h + e] is row 16 (warp % 4) + lane / 4 + 8 h,
// column 8 j + 2 (lane % 4) + e.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

#define GLT_ACC16(d, o)                                                                                        \
  "+f"(d[o + 0]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), "+f"(d[o + 6]), \
      "+f"(d[o + 7]), "+f"(d[o + 8]), "+f"(d[o + 9]), "+f"(d[o + 10]), "+f"(d[o + 11]), "+f"(d[o + 12]),          \
      "+f"(d[o + 13]), "+f"(d[o + 14]), "+f"(d[o + 15])

// D[64 x 64] (+)= A[64 x 16] . B[64 x 16]^T, bf16 in, fp32 accumulate; TA / TB: operand is MN-major in smem
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64k16_bf16(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, %35, %36;\n"
      "}\n"
      : GLT_ACC16(d, 0), GLT_ACC16(d, 16)
      : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
}
// D[64 x 32] (+)= A[64 x 16] . B[32 x 16]^T, both K-major; d[0..16) is the fragment
__device__ __forceinline__ void wgmma_m64n32k16_bf16(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n"
      "}\n"
      : GLT_ACC16(d, 0)
      : "l"(da), "l"(db), "r"(accumulate));
}
#undef GLT_ACC16

// explicit shared-window accesses (the aligned smem base is an integer-cast pointer, which the
// compiler would otherwise address through the slower generic path)
__device__ __forceinline__ uint64_t lds64(uint32_t addr) {
  uint64_t v;
  asm volatile("ld.shared.b64 %0, [%1];" : "=l"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ int32_t lds32(uint32_t addr) {
  int32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts64(uint32_t addr, uint64_t v) {
  asm volatile("st.shared.b64 [%0], %1;" ::"r"(addr), "l"(v) : "memory");
}
__device__ __forceinline__ void sts32(uint32_t addr, int32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void sts128(uint32_t addr, const uint4& v) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}


// ---- additions used by the TMA-fed GEMMs ----------------------------------------------------
// 2-D tensor-map load: box -> shared memory, completion counted on an mbarrier (SASS: UTMALDG)
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const void* tmap, int c0, int c1, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      ::"r"(dst), "l"(tmap), "r"(c0), "r"(c1), "r"(bar)
      : "memory");
}
// 2-D tensor-map store: shared memory -> global box, bulk-group completion (SASS: UTMASTG)
__device__ __forceinline__ void tma_store_2d(const void* tmap, int c0, int c1, uint32_t src) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%1, %2}], [%3];" ::"l"(tmap), "r"(c0),
               "r"(c1), "r"(src)
               : "memory");
}
__device__ __forceinline__ void tma_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_wait_group_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_wait_group() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// Shared-memory matrix descriptor of wgmma, SWIZZLE_128B, either operand major-ness (canonical layouts as in
// CUTLASS cute/atom/mma_traits_sm90_gmma.hpp make_gmma_desc):
//   K-major : rows of 128 B (64 bf16 along K); 8-row groups SBO bytes apart; LBO unused (16)
//   MN-major: rows of 128 B (64 bf16 along M/N) indexed by K; 8-row K groups SBO bytes apart; the next 64
//             M/N elements LBO bytes further
__device__ __forceinline__ uint64_t make_sw128_desc_lbo(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(1) << 62;   // SWIZZLE_128B
  return d;
}

}  // namespace tc
}  // namespace glt
