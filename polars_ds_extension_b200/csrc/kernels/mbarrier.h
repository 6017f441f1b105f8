// mbarrier and bulk-copy helpers (sm_90) shared by the ring kernels: the wgmma moments kernel (k2_gram_wgmma.cu) and
// the frame predict kernel (k4_predict.cu).  A producer lane arms a "full" barrier with the bytes it expects and
// issues asynchronous copies that complete against it; consumers release the slot on an "empty" barrier.
#pragma once
#include <cstdint>

namespace pdsb {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  // bounded wait (4 s of %globaltimer): a protocol bug must surface as a trapped kernel (an error the host reports),
  // never as a hung GPU.  First a plain non-blocking test, then try_wait with a suspend-time hint, which lets the
  // hardware park the warp until the phase flips instead of re-issuing the poll.
  uint32_t done = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P1;\n\t"
      "}" : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  if (done) return;
  uint64_t t0;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  while (!done) {
    asm volatile(
        "{\n\t"
        ".reg .pred P1;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, P1;\n\t"
        "}" : "=r"(done) : "r"(smem_u32(bar)), "r"(parity), "r"(0x989680u) : "memory");
    if (!done) {
      uint64_t t1;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
      if (t1 - t0 > 4000000000ull) __trap();          // 4 s: no legitimate wait of these kernels comes near it
    }
  }
}
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}" : "=r"(pred));
  return pred != 0;
}
// 1-D bulk copy global -> shared of `bytes` (a multiple of 16; both addresses 16-byte aligned), completing on `bar`
__device__ __forceinline__ void bulk_load(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
      ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

}  // namespace pdsb
