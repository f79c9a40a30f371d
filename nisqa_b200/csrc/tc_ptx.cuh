// tc_ptx.cuh - PTX wrappers shared by the tensor-core conv kernels (mbarrier, cp.async.bulk, ldmatrix, Hopper
// wgmma with the A operand in registers and B through a shared-memory matrix descriptor) and the two-term fp16 split.
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

namespace nisqa {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// Waits with a watchdog: a protocol bug (wrong parity, missing arrive) must end as a trapped kernel that the host sees as a
// CUDA error, never as a hung GPU (try_wait itself sleeps in hardware for a bounded time per call; ~2^26 calls is
// seconds - far beyond any legitimate wait in these kernels).
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  uint32_t spins = 0;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    if (!done && ++spins > (1u << 26)) __trap();
  } while (!done);
}
// one arrival (release semantics: this thread's earlier shared-memory accesses are ordered before the phase completes)
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
// generic-proxy accesses of this thread -> ordered before later async-proxy (bulk copy) accesses of the same memory
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

// four 8x8 b16 matrices; lane l supplies the row address of matrix l / 8, row l % 8
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr) : "memory");
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// barrier ID among the first N threads that reach it (N a multiple of 32; ID 0 is __syncthreads)
template <int ID, int N> __device__ __forceinline__ void named_bar_sync() { asm volatile("bar.sync %0, %1;" ::"n"(ID), "n"(N) : "memory"); }
// the same with a warp-uniform run-time ID
template <int N> __device__ __forceinline__ void named_bar_sync(uint32_t id) { asm volatile("bar.sync %0, %1;" ::"r"(id), "n"(N) : "memory"); }

// per-thread register budget of the calling warpgroup, raised (waits for registers released by others) or lowered
template <int N> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }

// wait until at most N committed wgmma groups of this warpgroup are still pending
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// B operand: K-major, no swizzle: core matrices of 8 rows x 16 bytes, rows 16 B apart, 8-row groups SBO = 128 B apart
// along N, K-adjacent core matrices LBO bytes apart
__device__ __forceinline__ uint64_t make_desc_b(uint32_t saddr, uint32_t lbo_bytes) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo_bytes >> 4) << 16) | ((uint64_t)(128u >> 4) << 32);
}

// D[64 x N] (fp32, registers of the warpgroup) += A[64 x 16] (fp16, registers: the mma.m16n8k16 A fragment of the
// warp's 16 rows) * B[16 x N] (fp16, shared memory descriptor)
template <int N>
__device__ __forceinline__ void wgmma_rs(float* d, const uint32_t (&a)[4], uint64_t b_desc);
template <> __device__ __forceinline__ void wgmma_rs<16>(float* d, const uint32_t (&a)[4], uint64_t b_desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7}, {%8,%9,%10,%11}, %12, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(1));
}
template <>__device__ __forceinline__ void wgmma_rs<32>(float* d, const uint32_t (&a)[4], uint64_t b_desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
      "{"
      "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15"
      "}, {%16,%17,%18,%19}, %20, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(1));
}

template <> __device__ __forceinline__ void wgmma_rs<64>(float* d, const uint32_t (&a)[4], uint64_t b_desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{"
      "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31"
      "}, {%32,%33,%34,%35}, %36, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(1));
}


// two-term fp16 split of 8 consecutive channels -> two 16-byte rows.  hi + lo keeps 22 significant bits of x while
// 2^-3 <= x <= 60000; below 2^-3 lo is subnormal (absolute error <= 2^-25), above 60000 the value is clamped.  The
// producing layer's weights and bias carry 2^-e_c for each output channel c (pack_weights), with e_c chosen from that
// channel's folded BatchNorm (E_c = |beta_c| + 3 |gamma_c| maps to [2.8, 5.7)), so x is the channel's value times 2^-e_c
// and the window is 1e4 times the channel's own BN output estimate, whatever the other channels' ranges.
// split4: the same for 4 consecutive channels (one 8-byte half of a row chunk); split8 is two of them.
__device__ __forceinline__ void split4(const float4& a, uint2& hi, uint2& lo) {
  const float x[4] = {a.x, a.y, a.z, a.w};
  uint32_t h[2], l[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    // post-ReLU inputs (>= 0)
    const float x0 = fminf(x[2 * i], 60000.f), x1 = fminf(x[2 * i + 1], 60000.f);
    const __half h0 = __float2half_rn(x0), h1 = __float2half_rn(x1);
    const __half l0 = __float2half_rn(x0 - __half2float(h0)), l1 = __float2half_rn(x1 - __half2float(h1));
    h[i] = (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
    l[i] = (uint32_t)__half_as_ushort(l0) | ((uint32_t)__half_as_ushort(l1) << 16);
  }
  hi = make_uint2(h[0], h[1]);
  lo = make_uint2(l[0], l[1]);
}
__device__ __forceinline__ void split8(const float4& a, const float4& b, uint4& hi, uint4& lo) {
  uint2 ha, la, hb, lb;
  split4(a, ha, la);
  split4(b, hb, lb);
  hi = make_uint4(ha.x, ha.y, hb.x, hb.y);
  lo = make_uint4(la.x, la.y, lb.x, lb.y);
}

}  // namespace nisqa
