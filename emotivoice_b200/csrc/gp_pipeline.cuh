// The granule-planar convolution pipeline shared by conv1d_gp.cu and resblock_gp.cu (sm_90a).  Internal header.
//
// Roles (448 threads) and the mbarrier ring they hand stages over with:
//   warp 12, one lane     x loader: a tile's rows [row0, row0 + rows) clipped to [0, len), one bulk copy per 16-byte granule plane of
//                         a channel block, into an x stage -> a_full
//   warps 8-11            transform: an in-place pass over the landed stage (LeakyReLU, zeros outside [0, len), the MODE's tf32
//                         rounding or hi / lo split), fence.proxy.async -> a_ready
//   warp 13, one lane     weight loader: one weight stage per (channel block, tap), in the order the consumers read them -> b_full
//   warps 0-7             consumers: per tap one wgmma chain over a channel block (tc::tap_chain), then -- one tap behind, once wgmma.wait_group 1 has
//                         seen the previous chain complete -- that chain's weight stage -> b_empty and, after a block's last tap, its
//                         x stage -> a_empty
// Every role walks the same tiles and channel blocks and counts stages the same way (slot = count % stages, parity = count /
// stages & 1), so the rings stay in step; tests/test_tc_protocol_sim.py models this protocol.
#pragma once
#include "tc_common.cuh"

namespace ev {
namespace gpl {

using namespace tc;

constexpr int NCW = 8;                       // consumer warps (two warpgroups)
constexpr int NTW = 4;                       // transform warps
constexpr int W_XFORM = NCW;                 // warps 8..11
constexpr int W_ALOAD = W_XFORM + NTW;       // 12
constexpr int W_BLOAD = W_ALOAD + 1;         // 13
constexpr int THREADS = (W_BLOAD + 1) * 32;  // 448
constexpr int MAX_B = 8;                     // weight stages
constexpr int SMEM_HEAD = 1024;              // barriers
constexpr int XF_UNROLL = 4;                 // rows per transform thread loaded before any of them is transformed

// LeakyReLU for 0 <= slope <= 1 as max(v, v*slope): two instructions (FMUL + FMNMX) instead of compare / multiply / select; same bits
__device__ __forceinline__ float lrelu_f(float v, float slope) { return fmaxf(v, v * slope); }

// The barriers at the head of shared memory: a_full / a_ready / a_empty of up to MAX_A x stages, b_full / b_empty of up to MAX_B
// weight stages.
template <int MAX_A>
struct Ring {
  uint32_t base;
  __device__ __forceinline__ uint32_t a_full(int s) const { return base + 8u * s; }
  __device__ __forceinline__ uint32_t a_ready(int s) const { return base + 8u * (MAX_A + s); }
  __device__ __forceinline__ uint32_t a_empty(int s) const { return base + 8u * (2 * MAX_A + s); }
  __device__ __forceinline__ uint32_t b_full(int s) const { return base + 8u * (3 * MAX_A + s); }
  __device__ __forceinline__ uint32_t b_empty(int s) const { return base + 8u * (3 * MAX_A + MAX_B + s); }
  // one thread, then __syncthreads
  __device__ __forceinline__ void init(int a_stages, int b_stages) const {
    for (int s = 0; s < a_stages; ++s) { mbar_init(a_full(s), 1); mbar_init(a_ready(s), NTW * 32); mbar_init(a_empty(s), NCW); }
    for (int s = 0; s < b_stages; ++s) { mbar_init(b_full(s), 1); mbar_init(b_empty(s), NCW); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
};

// Stage counts for a plan: the weight ring turns over K times per x stage, so first up to 4 weight stages, then up to 4 x stages
// (they prefetch ACROSS tiles: the ring is not bounded by the channel blocks of one tile), then whatever still fits.  False when
// two of each (fewer weight stages if b_max < 2) do not fit `budget` bytes.
__host__ __device__ inline bool grow_stages(int a_bytes, int b_bytes, int budget, int a_max, int b_max, int* a_stages, int* b_stages) {
  auto fits = [&](int a, int b) { return a * a_bytes + b * b_bytes <= budget; };
  int a = 2, b = b_max < 2 ? b_max : 2;
  if (!fits(a, b)) return false;
  while (b < b_max && b < 4 && fits(a, b + 1)) ++b;
  while (a < 4 && fits(a + 1, b)) ++a;
  while (b < b_max && fits(a, b + 1)) ++b;
  while (a < a_max && fits(a + 1, b)) ++a;
  *a_stages = a;
  *b_stages = b;
  return true;
}

// Launch order of a grouped launch's n <= 3 members (anything with a tap count K): heaviest first, so that with static round-robin
// tiles the CTAs that take a second (third) tile take a light one.
template <class P>
inline void heaviest_first(const P* ps, int n, int order[3]) {
  order[0] = 0; order[1] = 1; order[2] = 2;
  for (int i = 0; i < n; ++i)
    for (int j = i + 1; j < n; ++j)
      if (ps[order[j]].K > ps[order[i]].K) { const int t = order[i]; order[i] = order[j]; order[j] = t; }
}

// x loader, one tile: rows [row0, row0 + rows) of item b of x (C channels, L rows per granule plane) into consecutive stages,
// channel block after channel block.  Rows outside [0, len) are not copied; the transform writes them as zeros.
template <int CPG, int KBG, int MAX_A>
__device__ __forceinline__ void load_x_tile(Ring<MAX_A> ring, int& a_cnt, int a_stages, uint8_t* x_tiles, int stage_bytes, int rows_pad,
                                            const void* x, int b, int C, int L, int row0, int rows, int len) {
  constexpr int KB = CPG * KBG;
  const int n_cb = (C + KB - 1) / KB;
  const int r_lo = max(row0, 0);
  const int r_hi = min(row0 + rows, len);      // len <= L: never past the plane
  const uint32_t nbytes = (uint32_t)(r_hi - r_lo) * 16u, roff = (uint32_t)(r_lo - row0) * 16u;
  const uint8_t* xb = reinterpret_cast<const uint8_t*>(x) + ((size_t)b * (C / CPG) * L + r_lo) * 16;
  for (int cb = 0; cb < n_cb; ++cb, ++a_cnt) {
    const int s = a_cnt % a_stages;
    const int ngran = min(KB, C - cb * KB) / CPG;
    mbar_wait(ring.a_empty(s), ((a_cnt / a_stages) & 1) ^ 1);
    mbar_expect_tx(ring.a_full(s), (uint32_t)ngran * nbytes);
    const uint32_t dst = smem_u32(x_tiles + s * stage_bytes) + roff;
    const uint8_t* src = xb + (size_t)(cb * KBG) * L * 16;
    for (int g = 0; g < ngran; ++g) bulk_g2s(dst + (uint32_t)(g * rows_pad * 16), src + (size_t)g * L * 16, nbytes, ring.a_full(s));
  }
}

// Transform warps, one tile: the in-place pass over each landed stage of the tile, shared memory to shared memory, conflict-free
// (consecutive threads = consecutive 16 B); xt = this thread's index among the NTW * 32.  Stage row r is sequence row row0 + r.
// MODE 0: round to nearest tf32 (the MMA would otherwise truncate the low 13 mantissa bits); 1: tf32 hi + lo in the plane
// plane_bytes further on; 2: bf16 in, bf16 out; 3: fp32 in, the granule pair (2q, 2q+1) = 8 channels becomes [bf16 hi of the 8 |
// bf16 lo of the 8], so the hi plane is the even granule slots and the lo plane the odd ones (descriptor LBO = two slots).
template <int MODE, int KBG, int MAX_A>
__device__ __forceinline__ void transform_tile(Ring<MAX_A> ring, int& a_cnt, int a_stages, uint8_t* x_tiles, int stage_bytes, int plane_bytes,
                                               int rows_pad, int C, int row0, int rows, int len, bool lrelu, float slope, int xt) {
  constexpr bool SPLIT3 = (MODE == 1), BF16 = (MODE == 2), X3B = (MODE == 3);
  constexpr int CPG = BF16 ? 8 : 4;
  constexpr int KB = CPG * KBG;
  const int n_cb = (C + KB - 1) / KB;
  for (int cb = 0; cb < n_cb; ++cb, ++a_cnt) {
    const int s = a_cnt % a_stages;
    const int ngran = min(KB, C - cb * KB) / CPG;
    uint8_t* base = x_tiles + s * stage_bytes;
    mbar_wait(ring.a_full(s), (a_cnt / a_stages) & 1);
    if (X3B) {
      for (int q = 0; q < ngran / 2; ++q) {
        uint8_t* g0 = base + (size_t)(2 * q) * rows_pad * 16;
        uint8_t* g1 = g0 + (size_t)rows_pad * 16;
        for (int r = xt; r < rows; r += NTW * 32) {
          const int row = row0 + r;
          float4 u = make_float4(0.f, 0.f, 0.f, 0.f), w = u;
          if (row >= 0 && row < len) { u = *reinterpret_cast<const float4*>(g0 + r * 16); w = *reinterpret_cast<const float4*>(g1 + r * 16); }
          float f[8] = {u.x, u.y, u.z, u.w, w.x, w.y, w.z, w.w};
          uint32_t hi[4], lo[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            float a0 = f[2 * e], a1 = f[2 * e + 1];
            if (lrelu) { a0 = lrelu_f(a0, slope); a1 = lrelu_f(a1, slope); }
            hi[e] = pack_bf16(a0, a1);
            lo[e] = pack_bf16(a0 - __uint_as_float(hi[e] << 16), a1 - __uint_as_float(hi[e] & 0xffff0000u));
          }
          *reinterpret_cast<uint4*>(g0 + r * 16) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
          *reinterpret_cast<uint4*>(g1 + r * 16) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
        }
      }
    }
    for (int g = 0; g < (X3B ? 0 : ngran); ++g) {
      uint8_t* gb = base + (size_t)g * rows_pad * 16;
      for (int r0 = 0; r0 < rows; r0 += NTW * 32 * XF_UNROLL) {
        uint4 v[XF_UNROLL];
#pragma unroll
        for (int u = 0; u < XF_UNROLL; ++u) {
          const int r = r0 + u * (NTW * 32) + xt;
          const int row = row0 + r;
          v[u] = make_uint4(0u, 0u, 0u, 0u);
          if (r < rows && row >= 0 && row < len) v[u] = *reinterpret_cast<const uint4*>(gb + r * 16);
        }
#pragma unroll
        for (int u = 0; u < XF_UNROLL; ++u) {
          const int r = r0 + u * (NTW * 32) + xt;
          if (r >= rows) continue;
          if (BF16) {
            if (lrelu) {
              uint32_t w4[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const float lo = lrelu_f(__uint_as_float(w4[e] << 16), slope);
                const float hi = lrelu_f(__uint_as_float(w4[e] & 0xffff0000u), slope);
                w4[e] = pack_bf16(lo, hi);
              }
              v[u] = make_uint4(w4[0], w4[1], w4[2], w4[3]);
            }
            *reinterpret_cast<uint4*>(gb + r * 16) = v[u];
          } else {
            float4 t = make_float4(__uint_as_float(v[u].x), __uint_as_float(v[u].y), __uint_as_float(v[u].z), __uint_as_float(v[u].w));
            if (lrelu) { t.x = lrelu_f(t.x, slope); t.y = lrelu_f(t.y, slope); t.z = lrelu_f(t.z, slope); t.w = lrelu_f(t.w, slope); }
            const float4 h = make_float4(to_tf32(t.x), to_tf32(t.y), to_tf32(t.z), to_tf32(t.w));
            *reinterpret_cast<float4*>(gb + r * 16) = h;
            if (SPLIT3) {
              const float4 l = make_float4(to_tf32(t.x - h.x), to_tf32(t.y - h.y), to_tf32(t.z - h.z), to_tf32(t.w - h.w));
              *reinterpret_cast<float4*>(gb + plane_bytes + r * 16) = l;
            }
          }
        }
      }
    }
    fence_proxy_async();      // generic-proxy smem writes -> visible to the tensor core (async proxy)
    mbar_arrive(ring.a_ready(s));
  }
}

// Weight loader, one convolution of one tile: a stage per (channel block, tap), in the consumers' order.  w: [plane (hi, lo)][N tile
// of bnp = the packing tile][tap][C_in / WCPG granules][bnp][16 bytes], already advanced to the tile's first column; a stage holds
// N columns of the block's granules: one bulk copy per plane when N is the packing tile, else one per granule.
template <int MODE, int KBG, int N, int MAX_A>
__device__ __forceinline__ void load_w_tile(Ring<MAX_A> ring, int& b_cnt, int b_stages, uint8_t* b_tiles, int stage_bytes, int plane_bytes,
                                            const float* wt, int K, int Cin, int Cout, int bnp) {
  constexpr int PLANES = (MODE == 1 || MODE == 3) ? 2 : 1;
  constexpr int CPG = MODE == 2 ? 8 : 4;       // channels per granule of the activations
  constexpr int WCPG = MODE >= 2 ? 8 : 4;      // ... of the weights
  constexpr int KB = CPG * KBG;
  constexpr int KBGW = KBG * CPG / WCPG;       // weight granules per stage
  const int n_cb = (Cin + KB - 1) / KB;
  const int win = Cin / WCPG;                  // weight granules along C_in
  const size_t plane = (size_t)K * win * Cout * 4;      // 4-byte words per plane
  for (int cb = 0; cb < n_cb; ++cb) {
    const int ngran = min(KB, Cin - cb * KB) / WCPG;
    for (int j = 0; j < K; ++j, ++b_cnt) {
      const int sb = b_cnt % b_stages;
      mbar_wait(ring.b_empty(sb), ((b_cnt / b_stages) & 1) ^ 1);
      mbar_expect_tx(ring.b_full(sb), (uint32_t)(PLANES * ngran * N * 16));
      const uint32_t dst = smem_u32(b_tiles + sb * stage_bytes);
      const float* src = wt + ((size_t)j * win + (size_t)cb * KBGW) * bnp * 4;
      if (N == bnp) {
        bulk_g2s(dst, src, (uint32_t)(ngran * N * 16), ring.b_full(sb));
        if (PLANES == 2) bulk_g2s(dst + (uint32_t)plane_bytes, src + plane, (uint32_t)(ngran * N * 16), ring.b_full(sb));
      } else {
        for (int g = 0; g < ngran; ++g) {
          bulk_g2s(dst + (uint32_t)(g * N * 16), src + (size_t)g * bnp * 4, (uint32_t)(N * 16), ring.b_full(sb));
          if (PLANES == 2) bulk_g2s(dst + (uint32_t)(plane_bytes + g * N * 16), src + plane + (size_t)g * bnp * 4, (uint32_t)(N * 16), ring.b_full(sb));
        }
      }
    }
  }
}

// Consumers: each tap is one tc::tap_chain (tc_common.cuh), and a tap's stages go back one tap behind its issue.  After a tap_chain
// that read weight stage sb (and x stage sa >= 0 on a channel block's last tap) the kernel runs wgmma_wait<1>() -- the PREVIOUS chain has completed, so its operands are no longer read --
// then step(sb, sa), which hands the previous chain's stages back and remembers this one's.  After a tile's last chain: the
// epilogue's first loads, wgmma_wait<0>(), then drain().  The waits stay in each kernel's own source, where its wgmma.wait_group
// sites -- the bound tests/test_wgmma_pipeline_sass.py puts on its WARPGROUP.DEPBAR count -- can be read.
template <int MAX_A>
struct OneBehind {
  Ring<MAX_A> ring;
  int lane;
  int sb = -1, sa = -1;
  __device__ __forceinline__ void release() const {
    __syncwarp();
    if (lane == 0) {
      mbar_arrive(ring.b_empty(sb));
      if (sa >= 0) mbar_arrive(ring.a_empty(sa));
    }
  }
  __device__ __forceinline__ void step(int sb_now, int sa_now) {      // after wgmma_wait<1>()
    if (sb >= 0) release();
    sb = sb_now;
    sa = sa_now;
  }
  __device__ __forceinline__ void drain() const { release(); }         // after wgmma_wait<0>()
};

}  // namespace gpl
}  // namespace ev
