// Multi-head self-attention on the Hopper tensor cores (sm_90a): S = Q K^T and O = P V are wgmma (tf32 operands from shared
// memory, fp32 accumulators in registers); the softmax runs on the S accumulator fragments, so no (L x L) tensor is ever stored.
// Replaces encoder.py:84-109 (scores = q k^T / sqrt(d_k); key-padding mask; softmax; p v) for d_k = 48 (EmotiVoice: 384 / 8).
//
// One CTA = 128 queries of one (batch item, head), two consumer warpgroups of 64 query rows each; keys are walked ONCE in tiles of
// 64 with a lazily rescaled online softmax:
//   S_j = Q K_j^T  ->  P_j = exp(S_j / sqrt(d_k) - m), l += rowsum(P_j), O += P_j V_j
// m is the running row maximum; it only moves (and O, l are only rescaled by exp(m_old - m_new)) when a tile's maximum exceeds it
// by more than 8: until then P_j <= e^8, harmless in fp32 and in the relative precision of the tf32 operand.  Softmax is shift
// invariant, so the result is the reference's up to rounding.  Final: ctx = O / l.  A row's 64 scores of a tile are spread over
// the four lanes of a quad (16 each): row maxima and sums take two xor-shuffles.
//
// Operands are staged in shared memory in the no-swizzle K-major layout of conv1d_tc.cu (element (row r, 16-byte
// granule g) at (g * rows_pad + r) * 16):  Q [12 granules][128 rows], K_j [12][64 rows] (B operand of S), V_j^T [16 key
// granules][48 rows = d] (B operand of O: the loader warps transpose 4x4 blocks in registers), P_j [16 key granules][128 rows]
// (A operand of O, written by each consumer warpgroup for its own 64 rows).
// MODE 1 = 3xTF32 fp32 emulation (x = hi + lo, three MMAs per K step): the duration-critical encoder prefix and the "fp32"
// precision; MODE 0 = one tf32 MMA per K step (operands rounded to nearest).
//
// Roles (384 threads): warps 0-7 consumers (MMA issue, softmax, output), warps 8-11 loaders.  mbarriers: q_ready,
// kv_full / kv_empty[2] (K and V^T double buffered: the loads of tile j+1 run under the MMAs and softmax of tile j).
#include "ev_common.cuh"
#include "tc_common.cuh"

namespace ev {
namespace atc {

using namespace tc;

constexpr int BQ = 128, BKT = 64;
constexpr int NCW = 8, NLW = 4;                  // consumer warps, loader warps
constexpr int W_LOAD = NCW;
constexpr int ATC_THREADS = (NCW + NLW) * 32;    // 384
constexpr int QPAD = BQ + 1, KPAD = BKT + 1;     // rows_pad == 1 (mod 8): granule-fastest 16-byte stores are conflict free

template <int DK>
struct Smem {
  static constexpr int G = DK / 4;               // channel granules of Q / K
  static constexpr int GK = BKT / 4;             // key granules of V^T / P
  static constexpr int VPAD = DK + 1;
  static constexpr int q_plane = G * QPAD * 16;
  static constexpr int k_plane = G * KPAD * 16;
  static constexpr int v_plane = GK * VPAD * 16;
  static constexpr int p_plane = GK * BQ * 16;
  static constexpr int head = 256;
  static constexpr int total(int planes) { return head + planes * (q_plane + 2 * k_plane + 2 * v_plane + p_plane); }
};

template <int DK, int MODE>
__global__ void __launch_bounds__(ATC_THREADS, 1) attention_tc_kernel(const float* __restrict__ qkv, const int32_t* __restrict__ key_lens,
                                                                      float* __restrict__ ctx, int L, int H) {
  constexpr bool SPLIT3 = (MODE == 1);
  constexpr int PL = SPLIT3 ? 2 : 1;
  using S = Smem<DK>;
  constexpr int G = S::G, GK = S::GK, VPAD = S::VPAD;
  constexpr int NS = BKT / 2, NO = DK / 2;        // accumulator registers per thread: S tile, O
  extern __shared__ __align__(128) uint8_t smem_raw[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * BQ;
  const size_t ld = (size_t)3 * H;
  const float* base = qkv + (size_t)b * L * ld;

  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw);
  uint8_t* q_s = smem_raw + S::head;                       // [plane][G][QPAD][16]
  uint8_t* k_s = q_s + PL * S::q_plane;                    // [stage][plane][G][KPAD][16]
  uint8_t* v_s = k_s + 2 * PL * S::k_plane;                // [stage][plane][GK][VPAD][16]
  uint8_t* p_s = v_s + 2 * PL * S::v_plane;                // [plane][GK][BQ][16]
  const uint32_t bar_base = smem_u32(bars);
  const uint32_t q_ready = bar_base;
  auto kv_full = [&](int s) { return bar_base + 32u + 8u * s; };
  auto kv_empty = [&](int s) { return bar_base + 48u + 8u * s; };

  if (tid == 0) {
    mbar_init(q_ready, NLW * 32);
    for (int s = 0; s < 2; ++s) { mbar_init(kv_full(s), NLW * 32); mbar_init(kv_empty(s), NCW); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  // Programmatic dependent launch: the set-up above ran under the predecessor's tail; EVERY thread now waits for the preceding grids
  // before anything is read -- including key_lens, which in the encoder is written by validate_inputs_kernel a few launches upstream
  // (a role that decoded its tile count from stale lengths would desynchronise the pipeline).
  asm volatile("griddepcontrol.launch_dependents;\n\tgriddepcontrol.wait;" ::: "memory");
  const int klen = key_lens ? min(L, key_lens[b]) : L;
  const int nkt = (klen + BKT - 1) / BKT;

  if (warp < NCW) {
    // ================================ consumers: warpgroup wg owns query rows [64 wg, 64 wg + 64) ============================
    const int wg = warp >> 2, wl = warp & 3;
    const uint32_t wg_bar = 2u + (uint32_t)wg;            // named barrier of the warpgroup (P tile hand-over)
    constexpr uint32_t q_lbo = QPAD * 16, k_lbo = KPAD * 16, v_lbo = VPAD * 16, p_lbo = BQ * 16;
    const uint64_t q_desc = make_desc(smem_u32(q_s) + (uint32_t)(wg * 64) * 16u, q_lbo, 128u);
    const uint64_t p_desc = make_desc(smem_u32(p_s) + (uint32_t)(wg * 64) * 16u, p_lbo, 128u);
    const uint64_t k_desc0 = make_desc(0u, k_lbo, 128u), v_desc0 = make_desc(0u, v_lbo, 128u);
    const float inv_sqrt_dk = 1.0f / sqrtf((float)DK);
    constexpr float RESCALE_AT = 8.0f;
    float sacc[NS], oacc[NO];
#pragma unroll
    for (int i = 0; i < NS; ++i) sacc[i] = 0.f;
#pragma unroll
    for (int i = 0; i < NO; ++i) oacc[i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};     // per fragment row (h = 0: row l/4, h = 1: row l/4 + 8); l: this thread's columns
    mbar_wait(q_ready, 0);
    for (int j = 0; j < nkt; ++j) {
      const int s = j & 1;
      mbar_wait(kv_full(s), (j >> 1) & 1);
      // ---- S_j = Q K_j^T
      const uint64_t k_desc = desc_advance(k_desc0, smem_u32(k_s + (size_t)s * PL * S::k_plane));
      wgmma_fence();
#pragma unroll
      for (int k8 = 0; k8 < G / 2; ++k8) {
        const uint64_t a_hi = desc_advance(q_desc, (uint32_t)(2 * k8) * q_lbo);
        const uint64_t b_hi = desc_advance(k_desc, (uint32_t)(2 * k8) * k_lbo);
        if (SPLIT3) {
          wgmma_tf32_n64(sacc, desc_advance(a_hi, (uint32_t)S::q_plane), b_hi, k8 ? 1u : 0u);
          wgmma_tf32_n64(sacc, a_hi, desc_advance(b_hi, (uint32_t)S::k_plane), 1u);
          wgmma_tf32_n64(sacc, a_hi, b_hi, 1u);
        } else {
          wgmma_tf32_n64(sacc, a_hi, b_hi, k8 ? 1u : 0u);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      // ---- online softmax on the fragments
      const int nvalid = min(BKT, klen - j * BKT);
      float mt[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int i = 0; i < NS; ++i) {
        sacc[i] *= inv_sqrt_dk;
        if (frag_col(i, lane) < nvalid) mt[(i >> 1) & 1] = fmaxf(mt[(i >> 1) & 1], sacc[i]);
      }
      float f[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        mt[r] = fmaxf(mt[r], __shfl_xor_sync(0xffffffffu, mt[r], 1));
        mt[r] = fmaxf(mt[r], __shfl_xor_sync(0xffffffffu, mt[r], 2));
        const bool need = (j > 0) && (mt[r] > m[r] + RESCALE_AT);
        if (j == 0) m[r] = mt[r];
        f[r] = 1.0f;
        if (need) { f[r] = __expf(m[r] - mt[r]); m[r] = mt[r]; l[r] *= f[r]; }
      }
      if (f[0] != 1.0f || f[1] != 1.0f) {
#pragma unroll
        for (int i = 0; i < NO; ++i) oacc[i] *= f[(i >> 1) & 1];
      }
      // the PV MMAs of tile j-1 of the whole warpgroup have completed (every warp passed its wait): P may be overwritten
      bar_sync(wg_bar, 128);
#pragma unroll
      for (int i = 0; i < NS; i += 2) {
        const int c = frag_col(i, lane), hr = (i >> 1) & 1;
        const float p0 = c < nvalid ? __expf(sacc[i] - m[hr]) : 0.f;          // ex2.approx: relative error 2^-22; x <= 8
        const float p1 = c + 1 < nvalid ? __expf(sacc[i + 1] - m[hr]) : 0.f;
        const float2 hi = make_float2(to_tf32(p0), to_tf32(p1));
        // the denominator sums exactly what the tensor core multiplies: p (= hi + lo) in the 3xTF32 mode, the rounded hi otherwise
        l[hr] += SPLIT3 ? (p0 + p1) : (hi.x + hi.y);
        const int r = wg * 64 + frag_row(i, lane, wl);
        uint8_t* d = p_s + ((size_t)(c >> 2) * BQ + r) * 16 + (c & 3) * 4;
        *reinterpret_cast<float2*>(d) = hi;
        if (SPLIT3) *reinterpret_cast<float2*>(d + S::p_plane) = make_float2(to_tf32(p0 - hi.x), to_tf32(p1 - hi.y));
      }
      fence_proxy_async();
      bar_sync(wg_bar, 128);           // the warpgroup's P rows are complete
      // ---- O += P_j V_j
      const uint64_t v_desc = desc_advance(v_desc0, smem_u32(v_s + (size_t)s * PL * S::v_plane));
      wgmma_fence();
#pragma unroll
      for (int k8 = 0; k8 < GK / 2; ++k8) {
        const uint64_t a_hi = desc_advance(p_desc, (uint32_t)(2 * k8) * p_lbo);
        const uint64_t b_hi = desc_advance(v_desc, (uint32_t)(2 * k8) * v_lbo);
        const uint32_t acc = (j | k8) ? 1u : 0u;
        if (SPLIT3) {
          wgmma_tf32_n48(oacc, desc_advance(a_hi, (uint32_t)S::p_plane), b_hi, acc);
          wgmma_tf32_n48(oacc, a_hi, desc_advance(b_hi, (uint32_t)S::v_plane), 1u);
          wgmma_tf32_n48(oacc, a_hi, b_hi, 1u);
        } else {
          wgmma_tf32_n48(oacc, a_hi, b_hi, acc);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(kv_empty(s));     // K_j and V_j have been read
    }
    // ctx = O / l   (an item without keys -- rejected by the module's input validation -- yields zeros instead of a hang)
    float inv[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float lr = l[r];
      lr += __shfl_xor_sync(0xffffffffu, lr, 1);
      lr += __shfl_xor_sync(0xffffffffu, lr, 2);
      inv[r] = nkt > 0 ? 1.0f / lr : 0.f;
    }
#pragma unroll
    for (int i = 0; i < NO; i += 2) {
      const int row = q0 + wg * 64 + frag_row(i, lane, wl);
      if (row < L) {
        const float iv = inv[(i >> 1) & 1];
        *reinterpret_cast<float2*>(ctx + ((size_t)b * L + row) * H + h * DK + frag_col(i, lane)) = make_float2(oacc[i] * iv, oacc[i + 1] * iv);
      }
    }
  } else {
    // ================================ loaders =====================================================================
    const int lt = (warp - W_LOAD) * 32 + lane;        // 0..127
    // Every tile is loaded in batches of independent 16-byte loads issued back to back (memory-level parallelism: one latency
    // per batch instead of one per element), then rounded / split and stored in operand layout.
    auto store_split = [&](uint8_t* dst, int plane_bytes, const float4& t) {
      const float4 hi = make_float4(to_tf32(t.x), to_tf32(t.y), to_tf32(t.z), to_tf32(t.w));
      *reinterpret_cast<float4*>(dst) = hi;
      if (SPLIT3) {
        const float4 lo = make_float4(to_tf32(t.x - hi.x), to_tf32(t.y - hi.y), to_tf32(t.z - hi.z), to_tf32(t.w - hi.w));
        *reinterpret_cast<float4*>(dst + plane_bytes) = lo;
      }
    };
    constexpr int NT = NLW * 32;
    constexpr int QB = 6;                                  // loads in flight per thread
    static_assert((BQ * G) % (NT * QB) == 0 && (BKT * G) == NT * QB, "loader batching assumes d_k = 48, 128 loader threads");
    // Q tile: (row, granule) pairs, granule fastest -> coalesced 192-byte head rows; rows >= L are zeros
    for (int base_idx = 0; base_idx < BQ * G; base_idx += NT * QB) {
      float4 t[QB];
#pragma unroll
      for (int u = 0; u < QB; ++u) {
        const int idx = base_idx + u * NT + lt;
        const int r = idx / G, g = idx - r * G;
        const int row = q0 + r;
        t[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (row < L) t[u] = __ldg(reinterpret_cast<const float4*>(base + (size_t)row * ld + h * DK + g * 4));
      }
#pragma unroll
      for (int u = 0; u < QB; ++u) {
        const int idx = base_idx + u * NT + lt;
        const int r = idx / G, g = idx - r * G;
        store_split(q_s + ((size_t)g * QPAD + r) * 16, S::q_plane, t[u]);
      }
    }
    fence_proxy_async();
    mbar_arrive(q_ready);
    for (int j = 0; j < nkt; ++j) {
      const int s = j & 1;
      const int k0 = j * BKT;
      // all global loads of the tile first (K: 6 per thread; V: one or two 4-key x 4-channel blocks = 4 or 8 per thread) ...
      float4 kt[QB];
#pragma unroll
      for (int u = 0; u < QB; ++u) {
        const int idx = u * NT + lt;
        const int r = idx / G, g = idx - r * G;
        const int row = k0 + r;
        kt[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (row < klen) kt[u] = __ldg(reinterpret_cast<const float4*>(base + (size_t)row * ld + H + h * DK + g * 4));
      }
      constexpr int VB = (GK * G + NT - 1) / NT;         // blocks per thread (2 for d_k = 48; the second only for lt < 64)
      float4 vt[VB][4];
#pragma unroll
      for (int u = 0; u < VB; ++u) {
        const int idx = u * NT + lt;
        const int gk = idx / G, d4 = idx - gk * G;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int row = k0 + 4 * gk + i;
          vt[u][i] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (idx < GK * G && row < klen) vt[u][i] = __ldg(reinterpret_cast<const float4*>(base + (size_t)row * ld + 2 * H + h * DK + d4 * 4));
        }
      }
      // ... then wait for the ring slot and store
      mbar_wait(kv_empty(s), ((j >> 1) & 1) ^ 1);
      uint8_t* kd = k_s + (size_t)s * PL * S::k_plane;
#pragma unroll
      for (int u = 0; u < QB; ++u) {
        const int idx = u * NT + lt;
        const int r = idx / G, g = idx - r * G;
        store_split(kd + ((size_t)g * KPAD + r) * 16, S::k_plane, kt[u]);
      }
      // V_j^T: a 4 keys x 4 channels block per (key granule gk, channel group d4), transposed in registers
      uint8_t* vd = v_s + (size_t)s * PL * S::v_plane;
#pragma unroll
      for (int u = 0; u < VB; ++u) {
        const int idx = u * NT + lt;
        if (idx < GK * G) {
          const int gk = idx / G, d4 = idx - gk * G;
          const float4* t = vt[u];
          store_split(vd + ((size_t)gk * VPAD + d4 * 4 + 0) * 16, S::v_plane, make_float4(t[0].x, t[1].x, t[2].x, t[3].x));
          store_split(vd + ((size_t)gk * VPAD + d4 * 4 + 1) * 16, S::v_plane, make_float4(t[0].y, t[1].y, t[2].y, t[3].y));
          store_split(vd + ((size_t)gk * VPAD + d4 * 4 + 2) * 16, S::v_plane, make_float4(t[0].z, t[1].z, t[2].z, t[3].z));
          store_split(vd + ((size_t)gk * VPAD + d4 * 4 + 3) * 16, S::v_plane, make_float4(t[0].w, t[1].w, t[2].w, t[3].w));
        }
      }
      fence_proxy_async();
      mbar_arrive(kv_full(s));
    }
  }
}

}  // namespace atc

template <int DK, int MODE>
static int launch_atc(const float* qkv, const int32_t* key_lens, float* ctx, int B, int L, int H, int heads, cudaStream_t st) {
  const int smem = atc::Smem<DK>::total(MODE == 1 ? 2 : 1);
  static std::atomic<uint64_t> attr_devs{0};
  if (first_use_on_device(attr_devs))
    cudaFuncSetAttribute(atc::attention_tc_kernel<DK, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  dim3 grid((L + atc::BQ - 1) / atc::BQ, heads, B);
  return launch("attention_tc_kernel", atc::attention_tc_kernel<DK, MODE>, grid, atc::ATC_THREADS, (size_t)smem, st, qkv, key_lens, ctx, L, H);
}

void preload_attention_tc() {      // see preload_conv1d_gp
  cudaFuncSetAttribute(atc::attention_tc_kernel<48, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, atc::Smem<48>::total(1));
  cudaFuncSetAttribute(atc::attention_tc_kernel<48, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, atc::Smem<48>::total(2));
  cudaGetLastError();
}

// tc_mode 1: 3xTF32 (fp32-accurate), 0: one tf32 MMA per K step.  Supported head size: 48.
int launch_attention_tc(const float* qkv, const int32_t* key_lens, float* ctx, int B, int L, int H, int heads, int tc_mode, cudaStream_t st) {
  EV_CHECK_ARG(B > 0 && L > 0 && heads > 0 && H % heads == 0 && H / heads == 48, "attention_tc: needs d_k = 48 (B=%d L=%d H=%d heads=%d)", B, L, H, heads);
  EV_CHECK_ARG(B <= 65535 && heads <= 65535, "attention_tc: grid too large");
  return tc_mode == 1 ? launch_atc<48, 1>(qkv, key_lens, ctx, B, L, H, heads, st) : launch_atc<48, 0>(qkv, key_lens, ctx, B, L, H, heads, st);
}

}  // namespace ev
