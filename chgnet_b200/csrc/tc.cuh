// Hopper tensor-core / mbarrier / bulk-copy primitives for sm_90a (inline PTX; no CUTLASS dependency).
//
// Precision: the model needs fp32-level products (DESIGN.md §4), so every GEMM is issued as
// a 3xTF32 split:  a = a_hi + a_lo with a_hi = a with its 13 low mantissa bits cleared
// (exactly a TF32 number) and a_lo = a - a_hi (exact in fp32), likewise b;
//   a.b ~= a_hi.b_hi + a_lo.b_hi + a_hi.b_lo          (error ~2^-21 relative)
// accumulated in fp32 in the registers of the issuing warpgroup (wgmma.mma_async, m64nNk8).
//
// Operand layouts: B (and A in the shared-memory form) are K-major no-swizzle images of 8-row x
// 16-byte core matrices (kmajor_offset); A in the register form is the m16n8k8 tf32 fragment per
// warp.  Accumulator fragment of a m64nN product, warp w of the warpgroup, lane l (g = l / 4,
// c = l % 4):  d[4j + 0 / 1] = D[16w + g][8j + 2c + 0 / 1],  d[4j + 2 / 3] = D[16w + g + 8][8j + 2c + 0 / 1].
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace chg {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// generic-proxy writes to shared memory -> visible to the async proxy (tensor core operand reads, TMA stores)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- mbarrier -------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// bounded spin: a lost arrive traps instead of hanging the GPU
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  for (uint32_t spin = 0; spin < (1u << 26); ++spin) {
    uint32_t done;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
    if (done) return;
  }
  __trap();
}

// ---- wgmma ----------------------------------------------------------------------------------
// shared-memory matrix descriptor, K-major, no swizzle: lbo = byte distance between the two core
// matrices one k8 step consumes along K, sbo = byte distance between 8-row groups
// (cute: ((8,m),(T,2)):((1T,SBO),(1,LBO)))
__device__ __forceinline__ uint64_t smem_desc_kmajor(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  return d;  // base_offset 0, layout_type 0 = no swizzle
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// D[64 x N] += A . B^T, one warpgroup; A from registers (tf32 fragment), B from shared memory
__device__ __forceinline__ void wgmma_tf32_m64n64(float (&d)[32], const uint32_t (&a)[4], uint64_t b_desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.eq.u32 p, 1, 1;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
      "{%32,%33,%34,%35}, %36, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc)
      : "memory");
}
__device__ __forceinline__ void wgmma_tf32_m64n128(float (&d)[64], const uint32_t (&a)[4], uint64_t b_desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.eq.u32 p, 1, 1;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, "
      "{%64,%65,%66,%67}, %68, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc)
      : "memory");
}
__device__ __forceinline__ void wgmma_tf32_ss_m64n64(float (&d)[32], uint64_t a_desc, uint64_t b_desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.eq.u32 p, 1, 1;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
      "%32, %33, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a_desc), "l"(b_desc)
      : "memory");
}
template <int N>
__device__ __forceinline__ void wgmma_tf32(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t b_desc) {
  if constexpr (N == 64) wgmma_tf32_m64n64(d, a, b_desc);
  else wgmma_tf32_m64n128(d, a, b_desc);
}

// ---- 3xTF32 split -----------------------------------------------------------------------------
__device__ __forceinline__ void split_tf32(float a, uint32_t& hi, uint32_t& lo) {
  hi = __float_as_uint(a) & 0xFFFFE000u;
  lo = __float_as_uint(a - __uint_as_float(hi));
}

// byte offset of element (row, k) inside a no-swizzle K-major operand image with K columns
__host__ __device__ constexpr uint32_t kmajor_offset(int row, int k, int K) {
  return (uint32_t)((row >> 3) * (K / 4) * 128 + (k >> 2) * 128 + (row & 7) * 16 + (k & 3) * 4);
}

// d[64 x N] += A[64 x 64] . B^T as 3xTF32 on one warpgroup (all 128 threads call it).
// A: fp32, element (r, k) of this warpgroup's 64-row block read from shared memory as a_at(r, k);
// B: hi / lo images (byte addresses of the slice's first k) of N rows x K, sbo = byte stride of 8 rows.
// Returns with the products complete (A may be overwritten).
template <int N, class AFn>
__device__ __forceinline__ void wg_gemm_k64(float (&d)[N / 2], AFn a_at, uint32_t bhi, uint32_t blo, uint32_t sbo) {
  const int lane = threadIdx.x & 31;
  const int r = 16 * ((threadIdx.x >> 5) & 3) + (lane >> 2), c = lane & 3;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    uint32_t ahi[4][4], alo[4][4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = (h * 4 + j) * 8 + c;
      split_tf32(a_at(r, k), ahi[j][0], alo[j][0]);
      split_tf32(a_at(r + 8, k), ahi[j][1], alo[j][1]);
      split_tf32(a_at(r, k + 4), ahi[j][2], alo[j][2]);
      split_tf32(a_at(r + 8, k + 4), ahi[j][3], alo[j][3]);
    }
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint32_t koff = (uint32_t)(h * 4 + j) * 256;
      const uint64_t bh = smem_desc_kmajor(bhi + koff, 128, sbo), bl = smem_desc_kmajor(blo + koff, 128, sbo);
      wgmma_tf32<N>(d, ahi[j], bh);
      wgmma_tf32<N>(d, alo[j], bh);
      wgmma_tf32<N>(d, ahi[j], bl);
    }
    wgmma_commit();
    wgmma_wait<0>();
  }
}

// this thread's accumulator element i of a m64nN fragment: (row, col) inside the 64 x N block
__device__ __forceinline__ int frag_row(int i) { return 16 * ((threadIdx.x >> 5) & 3) + ((threadIdx.x & 31) >> 2) + ((i >> 1) & 1) * 8; }
__device__ __forceinline__ int frag_col(int i) { return (i >> 2) * 8 + 2 * (threadIdx.x & 3) + (i & 1); }

// named barrier for one warpgroup (ids 1..15; 0 is __syncthreads)
__device__ __forceinline__ void wg_barrier(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

}  // namespace tc
}  // namespace chg

// ---- TMA completion and bulk-group bookkeeping -------------------------------------------------
namespace chg {
namespace tc {
// one thread: this phase of `bar` completes after `bytes` more bytes have landed (plus 1 arrival)
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// wait until at most N of this thread's bulk groups still READ their shared-memory source
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait_all() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
}  // namespace tc
}  // namespace chg
