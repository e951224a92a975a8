// Device-side building blocks shared by the Hopper tensor-core kernels (conv1d_tc.cu, conv1d_gp.cu, resblock_gp.cu,
// attention_tc.cu): mbarrier / bulk-copy wrappers, the no-swizzle K-major shared-memory descriptor, warpgroup MMA (wgmma)
// with fp32 accumulators in registers, and the accumulator fragment layout.  Internal header.
#pragma once
#include <type_traits>
#include "ev_common.cuh"

namespace ev {
namespace tc {

constexpr int BM = 128;              // rows (time steps) per accumulator tile: two consumer warpgroups x 64 rows
constexpr int NCONS = 256;           // warps 0-7: two consumer warpgroups (issue the MMAs, own the accumulators, run the epilogue)
constexpr int NPRODUCER = 192;       // warps 8-13: stage A
constexpr int W_WLOAD = (NCONS + NPRODUCER) / 32;      // warp 14: weight loader
constexpr int NTHREADS = NCONS + NPRODUCER + 32;
constexpr int ACC_REGS = 64;         // fp32 accumulator registers per consumer thread: MT x BN <= 2 * ACC_REGS columns x 64 rows
constexpr int A_LD = 8;              // float4 loads in flight per producer thread and batch
constexpr int MAX_A_STAGES = 8, MAX_B_STAGES = 8;
constexpr int NPWARPS = NPRODUCER / 32;   // producer warps are split into `ngroups` groups; group g stages A stage a_cnt when
                                          // a_cnt % ngroups == g, so `ngroups` stages are being filled concurrently instead of one
                                          // stop-and-go stage.  SAFETY: the parity wait on a_empty can only tell consecutive
                                          // phases apart, so a group must never run two uses of a ring slot ahead of the
                                          // consumer; that holds iff ngroups <= a_stages (see make_plan).

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

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
      "{\n\t"
      ".reg .pred p;\n\t"
      "LAB_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE;\n\t"
      "bra LAB_WAIT;\n\t"
      "DONE:\n\t"
      "}" ::"r"(bar), "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// named barrier over the `n` threads of some warps (id 0 is __syncthreads)
__device__ __forceinline__ void bar_sync(uint32_t id, uint32_t n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// two fp32 -> packed bf16x2 (round to nearest even); `lo` lands in the low half = lower address
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
// no-swizzle K-major shared-memory matrix descriptor (wgmma): [0,14) start>>4 | [16,30) LBO>>4 (stride between the two 16-B K
// granules of one MMA) | [32,46) SBO>>4 (stride between 8-row groups) | [62,64) layout = 0 (no swizzle).  With SBO = 128 B
// consecutive rows are 16 B apart for the whole tile, so a start address advanced by whole rows is again a valid operand.
__device__ __forceinline__ uint64_t make_desc(uint32_t addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return (uint64_t)((addr >> 4) & 0x3FFFu) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) |
         ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32);
}
// descriptor with the start address field advanced by `bytes` (the 14-bit field holds address >> 4; shared memory is < 256 KB)
__device__ __forceinline__ uint64_t desc_advance(uint64_t desc, uint32_t bytes) { return desc + (uint64_t)(bytes >> 4); }
__device__ __forceinline__ float to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

// ---- warpgroup MMA: D (64 x N fp32, registers of the 128 threads) (+)= A (64 x K, shared) * B (K x N, shared), both K-major.
// tf32: K = 8 per instruction; bf16: K = 16.  `acc` = 0 overwrites D.  The accumulator fragment of thread t (warp w = t/32 of
// the warpgroup, lane l): register i holds row 16 w + l/4 + 8 ((i/2) & 1), column 8 (i/4) + 2 (l%4) + (i&1).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ int frag_row(int i, int lane, int wl) { return wl * 16 + (lane >> 2) + 8 * ((i >> 1) & 1); }
__device__ __forceinline__ int frag_col(int i, int lane) { return (i >> 2) * 8 + (lane & 3) * 2 + (i & 1); }

// The granule-planar epilogues (conv1d_gp.cu, resblock_gp.cu) read and write one accumulator register pair at a time: two adjacent
// channels of one row, a float2 of an fp32 tensor or one bf16x2 word.  They walk the pairs in chunks and issue all of a chunk's
// global loads before its first store: the output may alias the residual, so the compiler cannot hoist a load above an earlier
// store by itself, and one pair at a time every pair would wait a full global-load latency.
template <bool BF16>
using pair_t = std::conditional_t<BF16, uint32_t, float2>;
template <bool BF16>
__device__ __forceinline__ pair_t<BF16> load_pair(const void* t, size_t e) {      // elements e, e+1
  if constexpr (BF16) return *reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint16_t*>(t) + e);
  else return *reinterpret_cast<const float2*>(reinterpret_cast<const float*>(t) + e);
}
__device__ __forceinline__ float2 unpack_pair(float2 v) { return v; }
__device__ __forceinline__ float2 unpack_pair(uint32_t v) { return make_float2(__uint_as_float(v << 16), __uint_as_float(v & 0xffff0000u)); }
template <bool BF16>
__device__ __forceinline__ void store_pair(void* t, size_t e, float v0, float v1) {
  if constexpr (BF16) *reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(t) + e) = pack_bf16(v0, v1);
  else *reinterpret_cast<float2*>(reinterpret_cast<float*>(t) + e) = make_float2(v0, v1);
}

__device__ __forceinline__ void wgmma_tf32_n16(float* d, uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
               : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_tf32_n32(float* d, uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
               : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_tf32_n48(float* d, uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n48k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23}, %24, %25, p, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
               : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_tf32_n64(float* d, uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
               : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_tf32_n80(float* d, uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %42, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n80k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39}, %40, %41, p, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
               : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_tf32_n96(float* d, uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n96k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47}, %48, %49, p, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
               : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_tf32_n112(float* d, uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %58, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n112k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55}, %56, %57, p, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55])
               : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_tf32_n128(float* d, uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
               : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_bf16_n16(float* d, uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
               : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_bf16_n32(float* d, uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
               : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_bf16_n48(float* d, uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23}, %24, %25, p, 1, 1, 0, 0;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
               : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_bf16_n64(float* d, uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
               : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_bf16_n80(float* d, uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %42, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n80k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39}, %40, %41, p, 1, 1, 0, 0;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
               : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_bf16_n96(float* d, uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47}, %48, %49, p, 1, 1, 0, 0;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
               : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_bf16_n112(float* d, uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %58, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n112k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55}, %56, %57, p, 1, 1, 0, 0;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55])
               : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void wgmma_bf16_n128(float* d, uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
               : "l"(a), "l"(b), "r"(acc));
}

// D = A * B with the instruction's N fixed at compile time (a multiple of 16 up to 2 * NA).  Every convolution kernel fixes N
// this way: with N chosen at run time each MMA went through a jump table, and ptxas fenced it with its own warpgroup.arrive.
template <bool BF16, int N, int NA>
__device__ __forceinline__ void wgmma_fixed(float (&d)[NA], uint64_t a, uint64_t b, uint32_t acc) {
  static_assert(N % 16 == 0 && N >= 16 && N <= 128 && N <= 2 * NA, "N tile must be a multiple of 16 up to 128 and fit the accumulator");
  if constexpr (N == 16) { if constexpr (BF16) wgmma_bf16_n16(d, a, b, acc); else wgmma_tf32_n16(d, a, b, acc); }
  else if constexpr (N == 32) { if constexpr (BF16) wgmma_bf16_n32(d, a, b, acc); else wgmma_tf32_n32(d, a, b, acc); }
  else if constexpr (N == 48) { if constexpr (BF16) wgmma_bf16_n48(d, a, b, acc); else wgmma_tf32_n48(d, a, b, acc); }
  else if constexpr (N == 64) { if constexpr (BF16) wgmma_bf16_n64(d, a, b, acc); else wgmma_tf32_n64(d, a, b, acc); }
  else if constexpr (N == 80) { if constexpr (BF16) wgmma_bf16_n80(d, a, b, acc); else wgmma_tf32_n80(d, a, b, acc); }
  else if constexpr (N == 96) { if constexpr (BF16) wgmma_bf16_n96(d, a, b, acc); else wgmma_tf32_n96(d, a, b, acc); }
  else if constexpr (N == 112) { if constexpr (BF16) wgmma_bf16_n112(d, a, b, acc); else wgmma_tf32_n112(d, a, b, acc); }
  else { if constexpr (BF16) wgmma_bf16_n128(d, a, b, acc); else wgmma_tf32_n128(d, a, b, acc); }
}

// One K step of the convolution kernels' modes into one accumulator, N fixed at compile time.  MODE 0: one tf32 MMA; 2: one bf16
// MMA; 1 ("3xTF32") / 3 ("bf16x3"): operands split into hi + lo, a*b ~= a_lo*b_hi + a_hi*b_lo + a_hi*b_hi (small terms first, the
// dropped lo*lo term is below fp32 rounding), three MMAs into the same fp32 accumulator.  Every MMA is one wgmma, so the MMAs of a
// whole channel block form one unbroken chain between a fence and a commit.
template <int MODE, int N, int NA>
__device__ __forceinline__ void mma_step_fixed(float (&d)[NA], uint64_t a_hi, uint64_t a_lo, uint64_t b_hi, uint64_t b_lo, uint32_t acc) {
  constexpr bool OP16 = MODE >= 2;
  if constexpr (MODE == 1 || MODE == 3) {
    wgmma_fixed<OP16, N>(d, a_lo, b_hi, acc);
    wgmma_fixed<OP16, N>(d, a_hi, b_lo, 1u);
    wgmma_fixed<OP16, N>(d, a_hi, b_hi, 1u);
  } else {
    wgmma_fixed<OP16, N>(d, a_hi, b_hi, acc);
  }
}

// One K step k of a tap into the MT accumulators (one weight tile feeds all of them).  a: the A descriptor at this tap and
// warpgroup; a_step: A bytes per K step; a_lo: offset of the A lo operand; b: the weight stage's descriptor (N columns, so 2 N
// granules per K step); b_lo: offset of its lo plane.  cbj = channel block | tap: 0 on a tile's first tap, whose first MMAs
// overwrite the accumulators.
template <int MODE, int N, int MT, int NA>
__device__ __forceinline__ void tap_k_step(float (&acc)[MT][NA], uint64_t a, uint32_t a_step, uint32_t a_lo, uint64_t b, uint32_t b_lo,
                                           int cbj, int k) {
  const uint64_t b_hi = desc_advance(b, (uint32_t)k * (2u * N * 16u));
  const uint64_t b_lo_k = desc_advance(b_hi, b_lo);
  const uint64_t a_k = desc_advance(a, (uint32_t)k * a_step);
  const uint32_t first = (cbj | k) != 0 ? 1u : 0u;
#pragma unroll
  for (int mt = 0; mt < MT; ++mt) {
    const uint64_t a_hi = desc_advance(a_k, (uint32_t)(mt * BM) * 16u);
    mma_step_fixed<MODE, N>(acc[mt], a_hi, desc_advance(a_hi, a_lo), b_hi, b_lo_k, first);
  }
}

// Consumers of the convolution kernels (conv1d_tc.cu, conv1d_gp.cu, resblock_gp.cu), one tap over a full channel block: NK K steps
// x MT accumulators of mma_step_fixed as one chain between a fence and a commit (arguments: tap_k_step).
//
// A C_in that is not a multiple of the block (conv_pre's 80 channels, any such C_in at the conv1d_tc C ABI) ends in a short block:
// tap_chain_short.  The kernel picks one of the two per channel block and runs its wgmma_wait<1>() inside the same branch.  Where
// the two paths join before the commit instead, the commit opens a second commit group at the join, which ptxas closes with an
// empty no-op HGMMA (gsb0): each tap is then two groups, and `wgmma.wait_group 1` after it waits for the tap's real MMAs, so every
// tap drained the tensor core before the next one was queued.  Where they join between commit and wait, the compiler copies the
// wait into both paths anyway; writing it there keeps the source's wait sites equal to the WARPGROUP.DEPBAR in the SASS.
template <int MODE, int N, int NK, int MT, int NA>
__device__ __forceinline__ void tap_chain(float (&acc)[MT][NA], uint64_t a, uint32_t a_step, uint32_t a_lo, uint64_t b, uint32_t b_lo, int cbj) {
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < NK; ++k) tap_k_step<MODE, N>(acc, a, a_step, a_lo, b, b_lo, cbj, k);
  wgmma_commit();
}

// The short last block: nk K steps (1 <= nk < NK) in a run-time loop, a fence on every trip (a wgmma after a loop head with no fence
// of its own gets a warpgroup.arrive injected by ptxas, warning C7519), one commit.
template <int MODE, int N, int MT, int NA>
__device__ __forceinline__ void tap_chain_short(float (&acc)[MT][NA], uint64_t a, uint32_t a_step, uint32_t a_lo, uint64_t b, uint32_t b_lo,
                                                int cbj, int nk) {
#pragma unroll 1
  for (int k = 0; k < nk; ++k) {
    wgmma_fence();
    tap_k_step<MODE, N>(acc, a, a_step, a_lo, b, b_lo, cbj, k);
  }
  wgmma_commit();
}

}  // namespace tc
}  // namespace ev
