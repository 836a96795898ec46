// Thin inline-PTX wrappers for the sm_90a features the kernels use:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma (fence / commit / wait; the MMAs themselves are in wgmma.cuh),
// setmaxnreg and named barriers.
// The bit layout of the matrix descriptor follows the PTX ISA "wgmma matrix descriptor" table.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "wgmma.cuh"

namespace fresco {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// The single thread of a warp that issues TMA.  Selecting it with elect.sync (and not with `lane == 0`) lets the
// compiler keep the tensor-map and barrier addresses in uniform registers.
#define FRESCO_ISSUER_THREAD(lane) (::fresco::elect_one())

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// try_wait suspends the thread until the phase completes or a time limit passes.  The hint asks for up to
// FRESCO_TRYWAIT_NS before giving up, so a waiting warp does not take issue slots from the warps that have work;
// completion still wakes the thread at once.
#ifndef FRESCO_TRYWAIT_NS
#define FRESCO_TRYWAIT_NS 2000
#endif
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2, %3;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "n"(FRESCO_TRYWAIT_NS)
      : "memory");
  return ok != 0;
}
// non-blocking probe (try_wait may suspend the thread for a system-dependent time when the phase is not complete)
__device__ __forceinline__ bool mbar_test_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Watchdog: a lost arrival would otherwise hang the GPU until the driver's own limit.  After ~2^22 failed
// polls (seconds) the waiter reports which barrier it was stuck on and traps, turning a hang into an error.
#ifndef FRESCO_WATCHDOG_POLLS
#define FRESCO_WATCHDOG_POLLS (1u << 22)          /* each failed try_wait may block up to FRESCO_TRYWAIT_NS */
#endif
static __device__ __noinline__ void mbar_timeout(const uint64_t* bar, uint32_t parity, int tag) {
  printf("fresco_b200 watchdog: block (%d,%d,%d) thread %d stuck on mbarrier smem+0x%x parity %u tag %d\n",
         blockIdx.x, blockIdx.y, blockIdx.z, threadIdx.x, smem_u32(bar), parity, tag);
  __trap();
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, int tag = 0) {
  uint32_t polls = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++polls > FRESCO_WATCHDOG_POLLS) mbar_timeout(bar, parity, tag);
  }
}
// Wait for threads that share a scheduler with busy math warps (TMA producer, MMA issuer): back off between probes
// so the polling loop does not steal issue slots from them.
__device__ __forceinline__ void mbar_wait_backoff(uint64_t* bar, uint32_t parity, uint32_t ns, int tag = 0) {
  uint32_t polls = 0;
  while (!mbar_try_wait(bar, parity)) {
    __nanosleep(ns);
    if (++polls > FRESCO_WATCHDOG_POLLS) mbar_timeout(bar, parity, tag);
  }
}
// Kernels that issue wgmma use these instead: ptxas serialises every wgmma of a kernel that contains a call to a function
// that is not inlined (mbar_timeout and its printf), so their watchdog traps without a report.
__device__ __forceinline__ void mbar_wait_mma(uint64_t* bar, uint32_t parity) {
  uint32_t polls = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++polls > FRESCO_WATCHDOG_POLLS) __trap();
  }
}
__device__ __forceinline__ void mbar_wait_mma_backoff(uint64_t* bar, uint32_t parity, uint32_t ns) {
  uint32_t polls = 0;
  while (!mbar_try_wait(bar, parity)) {
    __nanosleep(ns);
    if (++polls > FRESCO_WATCHDOG_POLLS) __trap();
  }
}
// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1,
                                            int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
      "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
      "r"(c2)
      : "memory");
}

// ---------------------------------------------------------------- wgmma
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// ---------------------------------------------------------------- warpgroup scheduling
// setmaxnreg: every warp of a warpgroup executes the same one; the kernel needs __launch_bounds__ so ptxas knows the
// register count it starts from.  The values are multiples of 8 in [24, 256].
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
// named barriers (id 0 is __syncthreads'): a barrier completes when `threads` threads have arrived; bar.sync arrives
// and waits, bar.arrive only arrives.
__device__ __forceinline__ void named_bar_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(int id, int threads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
// mbar_wait_mma for a warpgroup that raised its register budget with setmaxnreg.inc: ptxas holds every region from
// which a trap is reachable to the launch-time register count, so the watchdog first drops back to LAUNCH_REGS.
template <int LAUNCH_REGS>
__device__ __forceinline__ void mbar_wait_mma_raised(uint64_t* bar, uint32_t parity) {
  uint32_t polls = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++polls > FRESCO_WATCHDOG_POLLS) {
      setmaxnreg_dec<LAUNCH_REGS>();
      __trap();
    }
  }
}
// keeps the compiler from moving reads or writes of accumulator registers across an asynchronous wgmma
template <int N>
__device__ __forceinline__ void reg_fence(float (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}

// ---------------------------------------------------------------- descriptors
// wgmma shared-memory matrix descriptor (64 bit):
//   [0,14) start address >> 4   [16,30) leading byte offset >> 4   [32,46) stride byte offset >> 4
//   [49,52) base offset  [62,64) layout (1 = 128B swizzle)
// K-major operands: SBO = 1024 (eight 128-byte rows), LBO unused.  MN-major operands: LBO = distance between 64-element
// column blocks, SBO = 1024.  A K step of 16 inside a K-major 128B-swizzled atom adds 32 bytes to the start address.
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes,
                                                         uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// (row, column) inside a warpgroup's 64 x N wgmma accumulator of accumulator register i (see wgmma.cuh)
__device__ __forceinline__ int acc_row(int i) { return 16 * ((threadIdx.x >> 5) & 3) + ((threadIdx.x & 31) >> 2) + 8 * ((i >> 1) & 1); }
__device__ __forceinline__ int acc_col(int i) { return 8 * (i >> 2) + 2 * (threadIdx.x & 3) + (i & 1); }

__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
  __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}

// One warp fills a [128 rows x 64 fp16] K-major atom of src[row, k] (row stride ld elements) in the layout a
// SWIZZLE_128B TMA box gives it (16-byte chunk c of row r at r * 128 + ((c ^ (r & 7)) << 4)), zero outside
// rows < n_rows, k < n_k.  For an operand whose row stride is not a multiple of 16 bytes, which no tensor map can
// describe: its rows may be only 2-byte aligned, so the loads are per element.  The caller fences the generic-proxy
// stores (fence_proxy_async_smem) before it signals the atom to wgmma.
__device__ __forceinline__ void fill_kmajor_atom_sw128(uint8_t* dst, const __half* src, size_t ld, int row0, int k0,
                                                       int n_rows, int n_k, int lane) {
  const unsigned short* s = reinterpret_cast<const unsigned short*>(src);
#pragma unroll 4
  for (int t = lane; t < 128 * 8; t += 32) {
    const int r = t >> 3, c = t & 7;
    const int gr = row0 + r, gk = k0 + c * 8;
    uint32_t w[4];
#pragma unroll
    for (int e = 0; e < 8; e += 2) {
      const size_t off = (size_t)gr * ld + gk + e;
      const uint32_t lo = (gr < n_rows && gk + e < n_k) ? __ldg(s + off) : 0u;
      const uint32_t hi = (gr < n_rows && gk + e + 1 < n_k) ? __ldg(s + off + 1) : 0u;
      w[e >> 1] = lo | (hi << 16);
    }
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(smem_u32(dst + r * 128 + ((c ^ (r & 7)) << 4))),
                 "r"(w[0]), "r"(w[1]), "r"(w[2]), "r"(w[3])
                 : "memory");
  }
}

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// sign of r as -1, 0 or +1 (0 for a zero residual), the derivative L1 losses use
__device__ __forceinline__ float sgnf(float r) { return r > 0.f ? 1.f : (r < 0.f ? -1.f : 0.f); }

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

}  // namespace fresco
