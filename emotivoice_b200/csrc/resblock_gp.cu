// One ResBlock1 layer of HiFi-GAN as ONE kernel on granule-planar activations (sm_90a):
//     out = [acc]( x + c2( lrelu( c1( lrelu(x), dilation d ) ), dilation 1 ) )            (hifigan/models.py:50-57)
// The intermediate xt = c1(lrelu(x)) never leaves the SM: c1's epilogue writes lrelu(acc1 + b1) -- rounded / split exactly like
// conv1d_gp.cu's transform warps would after a round trip through HBM -- straight from the accumulator registers into a
// shared-memory tile that already has the K-major operand layout, and c2's taps are descriptor shifts over that tile.
// Per layer the activation traffic drops from 5 passes (x, xt write, xt read, x residual, out) to 2 (x, out; the residual
// re-read hits L2) and the launches halve.  Same reduction orders and roundings as two conv1d_gp launches: BITWISE equal to them.
//
// Tile = R = 128*MT - (K-1) output rows.  c1 computes MT accumulators for the 128*MT xt rows [t0 - (K-1)/2, ...) from a staged x
// tile of 128*MT + (K-1)*d rows (the x loader and transform warps of gp_pipeline.cuh); c2 computes MT accumulators from the xt
// tile (its last K-1 rows per tile are surplus and discarded).  xt rows outside [0, len) are written as zeros: the reference
// pads c2's input with zeros, it does not convolve c1 over the padding.
//
// The roles and their code are gp_pipeline.cuh's, shared with conv1d_gp.cu: the consumer warpgroups run, per tile, c1 (one wgmma
// chain per tap, accumulators acc1 in registers), epi1 into the xt tile, a named barrier over both warpgroups, c2 over the xt tile
// into a second accumulator set acc2 (the same chains and one-behind release, with no x stage to hand back), then c1 of their
// next tile with epi2 (+ b2 + x, accumulate modes) of this one to HBM in chunks under its taps; the weight loader streams w1 then
// w2 of every tile, the order the consumers read them.  The x ring and the weight ring prefetch across tiles, so the loads of
// tile i+1 run under c2 of tile i, and the tensor core runs c1 of tile i+1 while epi2 of tile i waits on L2.
#include "ev_common.cuh"
#include "gp_pipeline.cuh"

namespace ev {
namespace gpp {

using namespace gpl;

constexpr int MAX_A = 6;                     // x stages
// The fused kernel launches 512 threads: gp_pipeline.cuh's 448 and two idle warps that complete warp 12-13's warpgroup, because
// setmaxnreg acts on whole warpgroups.  At launch every thread has 65536 / 512 = 128 registers; the two consumer warpgroups then
// take cons_regs(MT * C) each (both accumulator sets and an epilogue chunk) from what the transform and loader warpgroups give
// back.  With full accumulators (MT * C = 128) the consumers need 216 and the other warps fit 40; with fewer, 208 and 48 (the
// 3xTF32 transform needs more than 40).
constexpr int PAIR_THREADS = 512;
__host__ __device__ constexpr int cons_regs(int acc_cols) { return acc_cols == 2 * ACC_REGS ? 216 : 208; }
__host__ __device__ constexpr int prod_regs(int acc_cols) { return (65536 / 128 - 2 * cons_regs(acc_cols)) / 2; }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
// tc_common.cuh's load_pair / store_pair as predicated instructions (no branch); a load that is off returns zeros
template <bool BF16>
__device__ __forceinline__ pair_t<BF16> load_pair_if(bool on, const void* t, size_t e) {
  if constexpr (BF16) {
    uint32_t v = 0u;
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %2, 0;\n\t@p ld.global.b32 %0, [%1];\n\t}"
                 : "+r"(v) : "l"(reinterpret_cast<const uint16_t*>(t) + e), "r"((int)on));
    return v;
  } else {
    float2 v = make_float2(0.f, 0.f);
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %3, 0;\n\t@p ld.global.v2.f32 {%0, %1}, [%2];\n\t}"
                 : "+f"(v.x), "+f"(v.y) : "l"(reinterpret_cast<const float*>(t) + e), "r"((int)on));
    return v;
  }
}
template <bool BF16>
__device__ __forceinline__ void store_pair_if(bool on, void* t, size_t e, float v0, float v1) {
  if constexpr (BF16)
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %2, 0;\n\t@p st.global.b32 [%0], %1;\n\t}"
                 :: "l"(reinterpret_cast<uint16_t*>(t) + e), "r"(pack_bf16(v0, v1)), "r"((int)on) : "memory");
  else
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %3, 0;\n\t@p st.global.v2.f32 [%0], {%1, %2};\n\t}"
                 :: "l"(reinterpret_cast<float*>(t) + e), "f"(v0), "f"(v1), "r"((int)on) : "memory");
}

struct PPlan {
  int mt, kbg;
  int rows1_pad, rows2_pad, R;
  int x_plane_bytes, x_stage_bytes, a2_plane_bytes, a2_bytes, b_plane_bytes, b_stage_bytes;
  int a_stages, b_stages;
  int acc_cols;        // MT * C <= 2 * ACC_REGS
  int tiles_m, total_tiles;
  int smem_total;
};

// span1 = (K-1)*dil of the widest member and kmax = the most taps of a grouped launch (-1 / 0: p's own)
__host__ __device__ inline bool make_pplan(const GpPairParams& p, int mode, int mt, int kbg, PPlan* o, int span1 = -1, int kmax = 0) {
  if (span1 < 0) span1 = (p.K - 1) * p.dil;
  if (kmax <= 0) kmax = p.K;
  PPlan q;
  q.mt = mt; q.kbg = kbg;
  const int C = p.C;
  if (C > 128 || C % 32 || mt * C > 2 * ACC_REGS) return false;
  const int cpg = mode == 2 ? 8 : 4;            // activation granule (HBM / x tile)
  const int ocpg = mode >= 2 ? 8 : 4;           // operand granule of the xt tile and the weights
  const int xplanes = mode == 1 ? 2 : 1;
  const int splitp = (mode == 1 || mode == 3) ? 2 : 1;
  q.R = BM * mt - (p.K - 1);
  if (BM * mt - (kmax - 1) < 32) return false;
  const int rows1 = BM * mt + span1;
  q.rows1_pad = (rows1 + 7) / 8 * 8;
  q.rows2_pad = (BM * mt + (kmax - 1) + 7) / 8 * 8;
  q.x_plane_bytes = kbg * q.rows1_pad * 16;
  q.x_stage_bytes = xplanes * q.x_plane_bytes;
  q.a2_plane_bytes = (C / ocpg) * q.rows2_pad * 16;
  q.a2_bytes = splitp * q.a2_plane_bytes;
  q.b_plane_bytes = (kbg * cpg / ocpg) * C * 16;
  q.b_stage_bytes = splitp * q.b_plane_bytes;
  const int budget = 227 * 1024 - SMEM_HEAD - q.a2_bytes;
  if (!grow_stages(q.x_stage_bytes, q.b_stage_bytes, budget, MAX_A, MAX_B, &q.a_stages, &q.b_stages)) return false;
  q.acc_cols = mt * C;
  q.tiles_m = (p.L + q.R - 1) / q.R;
  q.total_tiles = p.B * q.tiles_m;
  q.smem_total = SMEM_HEAD + q.a2_bytes + q.a_stages * q.x_stage_bytes + q.b_stages * q.b_stage_bytes;
  *o = q;
  return true;
}

// MODE as conv1d_gp.cu: 0 tf32, 1 3xTF32, 2 bf16 activations + operands, 3 bf16x3 on fp32 activations.  C = p.C, the channels.
template <int MODE, int MT, int KBG, int C>
__global__ void __launch_bounds__(PAIR_THREADS, 1) resblock_gp_kernel(const __grid_constant__ GpPairParams p, const __grid_constant__ PPlan pl,
                                                                     const __grid_constant__ GpPairGroups gs) {
  constexpr bool SPLIT3 = (MODE == 1), BF16 = (MODE == 2), X3B = (MODE == 3);
  constexpr bool OP16 = BF16 || X3B;
  constexpr int CPG = BF16 ? 8 : 4;
  constexpr int OCPG = OP16 ? 8 : 4;
  constexpr int KB = CPG * KBG;
  constexpr int KBGW = KBG * CPG / OCPG;        // operand granules (weights, xt tile) per channel block
  constexpr int NA = ACC_REGS / MT;
  constexpr int NQ = C / 8;                     // column groups (8 columns, 4 accumulator registers per thread and MT) = epi2 chunks
  // C and KB are powers of two: every channel block is full (or the only one), so its MMA K steps are a constant
  constexpr int NK = (C < KB ? C : KB) / (2 * OCPG);
  static_assert(C % KB == 0 || C < KB, "every channel block has NK K steps");
  static_assert(!X3B || KBG % 4 == 0, "bf16x3 consumes four fp32 granules per MMA K step");
  static_assert(MT * C <= 2 * ACC_REGS, "accumulators of the tile exceed the register budget");
  extern __shared__ __align__(128) uint8_t smem_raw[];
  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);   // provably warp-uniform: ptxas serialises every wgmma on a path it cannot prove uniform

  uint8_t* a2_tile = smem_raw + SMEM_HEAD;
  uint8_t* x_tiles = a2_tile + pl.a2_bytes;
  uint8_t* b_tiles = x_tiles + pl.a_stages * pl.x_stage_bytes;
  const Ring<MAX_A> ring{smem_u32(smem_raw)};
  if (tid == 0) ring.init(pl.a_stages, pl.b_stages);
  __syncthreads();
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if (warp < NCW) setmaxnreg_inc<cons_regs(MT * C)>();
  else setmaxnreg_dec<prod_regs(MT * C)>();

  const int n_cb = (C + KB - 1) / KB;
  const int gC = C / CPG;                      // activation granule planes per item
  // A launch carries up to three layers of one shape (the same-index layers of HiFi-GAN's parallel ResBlocks: their own taps,
  // dilation, weights, tensors, hence their own rows per tile and tile count); tiles are numbered member after member.
  auto group_of = [&](int tile) { return (gs.ng > 1 && tile >= gs.g[1].tile0) ? ((gs.ng > 2 && tile >= gs.g[2].tile0) ? 2 : 1) : 0; };
  auto tile_len = [&](int tile, int& gi, int& b, int& t0) {
    gi = group_of(tile);
    const int local = tile - gs.g[gi].tile0;
    b = local / gs.g[gi].tiles_m;
    t0 = (local - b * gs.g[gi].tiles_m) * gs.g[gi].R;
    return p.lens ? min(p.L, p.lens[b] * p.lens_mul) : p.L;
  };
  auto active = [&](int tile) { int gi, b, t0; const int len = tile_len(tile, gi, b, t0); return t0 < len; };
  auto next_active = [&](int tile) {      // first active tile of this CTA at or after `tile` (stride gridDim.x); >= total when none
    while (tile < pl.total_tiles && !active(tile)) tile += gridDim.x;
    return tile;
  };

  if (warp < NCW) {
    // ============================ consumers: c1 -> epi1 (xt tile) -> c2, then the next tile's c1 under epi2 ==================
    // c1 accumulates in acc1 and c2 in acc2, so the next tile's c1 can run while this tile's epi2 waits on L2: each tap of
    // c1(i+1) issues its chain, waits for the previous one (wgmma_wait<1>), hands its stages back, then runs one chunk of epi2(i)
    // while the chain just issued executes.  The stages are consumed in the order of one tile at a time (x(i+1) and w1(i+1) after
    // w2(i)), so the loaders, the transform warps and the mbarrier protocol are those of conv1d_gp.  (The chunk goes after the
    // wait: with two chains in flight ptxas cannot tell acc2 from the accumulators they write, and waits for both.)
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const int wg = warp >> 2, wl = warp & 3;
    const float slope = p.slope;
    const uint32_t x_lbo = (uint32_t)pl.rows1_pad * 16u, a2_lbo = (uint32_t)pl.rows2_pad * 16u, b_lbo = (uint32_t)C * 16u;
    const uint64_t x_desc0 = make_desc(0u, X3B ? 2u * x_lbo : x_lbo, 128u), b_desc0 = make_desc(0u, b_lbo, 128u);
    const uint64_t a2_desc0 = make_desc(smem_u32(a2_tile) + (uint32_t)(wg * 64) * 16u, a2_lbo, 128u);
    const uint32_t x_k = (X3B ? 4u : 2u) * x_lbo, x_lo_off = X3B ? x_lbo : (uint32_t)pl.x_plane_bytes;
    float acc1[MT][NA], acc2[MT][NA];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int i = 0; i < NA; ++i) {
        acc1[mt][i] = 0.f;
        // a zero of its own: were acc2 a copy of acc1's zero, ptxas would see epi2's reads of acc2 as reads of the acc1 registers
        // that c1's MMAs are writing, and wait for them
        asm volatile("mov.b32 %0, 0;" : "=f"(acc2[mt][i]));
      }
    int a_cnt = 0, b_cnt = 0;
    // ---- epi2 of tile e_tile (acc2 + b2 + x (+ accumulate) -> out), one chunk per call: column group q (8 columns, one b2), pairs
    // i = 4 q + 2 h of every accumulator mt at tile row rl0 + mt * BM + 8 h.  q is a run-time index, so the pairs are picked from
    // acc2 with selects (indexing acc2 by q would put it in local memory).  A chunk issues all its loads (b2, the residual x, `out`
    // in the accumulate modes) before its stores.  out != x (plan_pair), and in the accumulate modes every element of out is loaded
    // and stored by exactly one thread, load first.
    int e_tile = -1, e_gi = 0, e_b = 0, e_t0 = 0, e_len = 0;
    const int rl0 = wg * 64 + frag_row(0, lane, wl);
    auto epi2_chunk = [&](int q, auto div) {      // div: std::true_type where the chunk may run ACC_ADD_DIV's division
      const GpPairGroup& E = gs.g[e_gi];
      const int c = frag_col(4 * q, lane);
      const size_t ec = ((size_t)e_b * gC + c / CPG) * p.L * CPG + (c % CPG);      // element index at row 0
      const float2 ebias = __ldg(reinterpret_cast<const float2*>(E.b2 + c));
      const bool accm = p.acc != EV_ACC_STORE;
      // Rows past R or len are predicated off, not branched around: a divergent branch between two tap chains makes ptxas
      // serialise every wgmma of the kernel (C7518).
      pair_t<BF16> eres[MT][2], eout[MT][2];
#pragma unroll
      for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int rl = rl0 + mt * BM + 8 * h, row = e_t0 + rl;
          const bool ok = rl < E.R && row < e_len;
          const size_t e = ec + (size_t)row * CPG;
          eres[mt][h] = load_pair_if<BF16>(ok, E.x, e);      // the residual: L2 hit
          eout[mt][h] = load_pair_if<BF16>(ok && accm, E.out, e);
        }
#pragma unroll
      for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int rl = rl0 + mt * BM + 8 * h, row = e_t0 + rl;
          const bool ok = rl < E.R && row < e_len;
          float a0 = acc2[mt][2 * h], a1 = acc2[mt][2 * h + 1];
#pragma unroll
          for (int g = 1; g < NQ; ++g) {
            a0 = g == q ? acc2[mt][4 * g + 2 * h] : a0;
            a1 = g == q ? acc2[mt][4 * g + 2 * h + 1] : a1;
          }
          float v0 = a0 + ebias.x, v1 = a1 + ebias.y;
          const float2 r = unpack_pair(eres[mt][h]);
          v0 += r.x; v1 += r.y;
          const float2 o = unpack_pair(eout[mt][h]);
          v0 = accm ? v0 + o.x : v0;
          v1 = accm ? v1 + o.y : v1;
          if constexpr (decltype(div)::value)
            if (p.acc == EV_ACC_ADD_DIV) { v0 /= p.div; v1 /= p.div; }
          store_pair_if<BF16>(ok, E.out, ec + (size_t)row * CPG, v0, v1);
        }
    };
    for (int tile = next_active(blockIdx.x);; tile = next_active(tile + gridDim.x)) {
      const bool live = tile < pl.total_tiles;      // else only the previous tile's epi2 is left
      int gi = 0, b = 0, t0 = 0, len = 0;
      if (live) len = tile_len(tile, gi, b, t0);
      const GpPairGroup& G = gs.g[gi];
      const int K = G.K, dil = G.dil;
      const int h2 = (K - 1) / 2;
      // epi1 in parts of B1Q column groups (pair i = 4 q + 2 h of every accumulator lies in column group q: 8 columns, one b1): a
      // part's b1 loads are all issued ahead of its shared-memory stores, the first part's under c1's last MMAs
      constexpr int B1Q = 2;
      float2 bias1[B1Q];
      auto load_b1 = [&](int part) {
#pragma unroll
        for (int q = 0; q < B1Q; ++q) {
          const int c = frag_col(4 * (part * B1Q + q), lane);
          if (c < C) bias1[q] = __ldg(reinterpret_cast<const float2*>(G.b1 + c));
        }
      };
      // ---- c1 over the staged x tile -> acc1, one chunk of the previous tile's epi2 under each tap
      {
        if (!live) {          // this CTA has no tile left: the last epi2 on its own
#pragma unroll 1
          for (int q = e_tile >= 0 ? 0 : NQ; q < NQ; ++q) epi2_chunk(q, std::true_type{});
          break;
        }
        // The division's slow path is a subroutine call, and ptxas serialises every wgmma of a kernel that makes a call while MMAs
        // are in flight: in ACC_ADD_DIV mode (a solo launch, never the grouped ones) epi2 waits for c1 to complete.
        const bool under = e_tile >= 0 && p.acc != EV_ACC_ADD_DIV;
        int q = under ? 0 : NQ;
        OneBehind<MAX_A> rel{ring, lane};
        // Not unrolled, not peeled: with C and the K steps constants the compiler would otherwise copy the channel-block and tap
        // loops, and every copy adds a wgmma.wait_group site (tests/test_wgmma_pipeline_sass.py counts them).
#pragma unroll 1
        for (int cb = 0; cb < n_cb; ++cb, ++a_cnt) {
          const int sa = a_cnt % pl.a_stages;
          mbar_wait(ring.a_ready(sa), (a_cnt / pl.a_stages) & 1);
          const uint64_t x0 = desc_advance(x_desc0, smem_u32(x_tiles + sa * pl.x_stage_bytes) + (uint32_t)(wg * 64) * 16u);
#pragma unroll 1
          for (int j = 0; j < K; ++j, ++b_cnt) {
            const int sb = b_cnt % pl.b_stages;
            mbar_wait(ring.b_full(sb), (b_cnt / pl.b_stages) & 1);
            const uint64_t b0 = desc_advance(b_desc0, smem_u32(b_tiles + sb * pl.b_stage_bytes));
            tap_chain<MODE, C, NK>(acc1, desc_advance(x0, (uint32_t)(j * dil) * 16u), x_k, x_lo_off, b0, (uint32_t)pl.b_plane_bytes, cb | j);
            wgmma_wait<1>();          // the previous tap's chain has completed: its stages may be refilled
            rel.step(sb, j == K - 1 ? sa : -1);
            if (q < NQ) epi2_chunk(q++, std::false_type{});      // while this tap's chain runs
          }
        }
#pragma unroll 1
        for (; q < NQ; ++q) epi2_chunk(q, std::false_type{});      // c1 had fewer taps than epi2 has chunks: under its last one
        load_b1(0);
        wgmma_wait<0>();
        rel.drain();
        if (e_tile >= 0 && !under)
#pragma unroll 1
          for (q = 0; q < NQ; ++q) epi2_chunk(q, std::true_type{});
      }
      // ---- epi1: acc1 + b1 -> lrelu -> operand format -> xt tile.  Both warpgroups' c2 of the previous tile read the whole
      // ---- xt tile (their taps overlap the other's rows), so the tile is only rewritten once both have finished it.
      bar_sync(1, NCW * 32);
#pragma unroll
      for (int part = 0; part < NA / 4 / B1Q; ++part) {
        if (part > 0) load_b1(part);
#pragma unroll
        for (int q = 0; q < B1Q; ++q)
#pragma unroll
          for (int mt = 0; mt < MT; ++mt)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int i = 4 * (part * B1Q + q) + 2 * h;
              const int c = frag_col(i, lane);
              if (c >= C) continue;
              const int r2 = mt * BM + wg * 64 + frag_row(i, lane, wl);
              const int row = t0 - h2 + r2;
              const bool ok = row >= 0 && row < len;            // xt outside the sequence is c2's ZERO padding
              float v0 = acc1[mt][i] + bias1[q].x, v1 = acc1[mt][i + 1] + bias1[q].y;
              if (BF16) {      // the unfused path stores xt as bf16 before activating it
                v0 = __uint_as_float(pack_bf16(v0, 0.f) << 16);
                v1 = __uint_as_float(pack_bf16(v1, 0.f) << 16);
              }
              v0 = ok ? lrelu_f(v0, slope) : 0.f;
              v1 = ok ? lrelu_f(v1, slope) : 0.f;
              uint8_t* d = a2_tile + ((size_t)(c / OCPG) * pl.rows2_pad + r2) * 16 + (c % OCPG) * (OP16 ? 2 : 4);
              if (OP16) {
                const uint32_t hi = pack_bf16(v0, v1);
                *reinterpret_cast<uint32_t*>(d) = hi;
                if (X3B) *reinterpret_cast<uint32_t*>(d + pl.a2_plane_bytes) = pack_bf16(v0 - __uint_as_float(hi << 16), v1 - __uint_as_float(hi & 0xffff0000u));
              } else {
                const float2 t = make_float2(to_tf32(v0), to_tf32(v1));
                *reinterpret_cast<float2*>(d) = t;
                if (SPLIT3) *reinterpret_cast<float2*>(d + pl.a2_plane_bytes) = make_float2(to_tf32(v0 - t.x), to_tf32(v1 - t.y));
              }
            }
      }
      fence_proxy_async();          // generic-proxy smem writes -> visible to the tensor core
      bar_sync(1, NCW * 32);        // the whole xt tile is written
      // ---- c2 over the xt tile -> acc2
      {
        OneBehind<MAX_A> rel{ring, lane};
#pragma unroll 1                            // as in c1
        for (int cb = 0; cb < n_cb; ++cb) {
          const uint64_t a0 = desc_advance(a2_desc0, (uint32_t)(cb * KBGW) * a2_lbo);
#pragma unroll 1
          for (int j = 0; j < K; ++j, ++b_cnt) {
            const int sb = b_cnt % pl.b_stages;
            mbar_wait(ring.b_full(sb), (b_cnt / pl.b_stages) & 1);
            const uint64_t b0 = desc_advance(b_desc0, smem_u32(b_tiles + sb * pl.b_stage_bytes));
            tap_chain<MODE, C, NK>(acc2, desc_advance(a0, (uint32_t)j * 16u), 2u * a2_lbo, (uint32_t)pl.a2_plane_bytes, b0, (uint32_t)pl.b_plane_bytes, cb | j);
            wgmma_wait<1>();          // the previous tap's chain has completed: its stages may be refilled
            rel.step(sb, -1);
          }
        }
        wgmma_wait<0>();
        rel.drain();
      }
      e_tile = tile; e_gi = gi; e_b = b; e_t0 = t0; e_len = len;
    }
  } else if (warp < W_ALOAD) {
    // ============================ transform warps ========================================================================
    const int xt = (warp - W_XFORM) * 32 + lane;
    int a_cnt = 0;
    for (int tile = next_active(blockIdx.x); tile < pl.total_tiles; tile = next_active(tile + gridDim.x)) {
      int gi, b, t0;
      const int len = tile_len(tile, gi, b, t0);
      const int span = (gs.g[gi].K - 1) * gs.g[gi].dil;
      transform_tile<MODE, KBG>(ring, a_cnt, pl.a_stages, x_tiles, pl.x_stage_bytes, pl.x_plane_bytes, pl.rows1_pad, C,
                                t0 - (gs.g[gi].K - 1) / 2 - span / 2, BM * MT + span, len, true, p.slope, xt);
    }
  } else if (warp == W_ALOAD) {
    // ============================ x loader ===============================================================================
    if (lane == 0) {
      asm volatile("griddepcontrol.wait;" ::: "memory");
      int a_cnt = 0;
      for (int tile = next_active(blockIdx.x); tile < pl.total_tiles; tile = next_active(tile + gridDim.x)) {
        int gi, b, t0;
        const int len = tile_len(tile, gi, b, t0);
        const int span = (gs.g[gi].K - 1) * gs.g[gi].dil;
        load_x_tile<CPG, KBG>(ring, a_cnt, pl.a_stages, x_tiles, pl.x_stage_bytes, pl.rows1_pad, gs.g[gi].x, b, C, p.L,
                              t0 - (gs.g[gi].K - 1) / 2 - span / 2, BM * MT + span, len);
      }
    }
    __syncwarp();
  } else if (warp == W_BLOAD) {
    // ============================ weight loader: the consumers' order  w1(i), w2(i), w1(i+1), ... ====================
    if (lane == 0) {
      int b_cnt = 0;
      for (int tile = next_active(blockIdx.x); tile < pl.total_tiles; tile = next_active(tile + gridDim.x)) {
        const GpPairGroup& G = gs.g[group_of(tile)];
        load_w_tile<MODE, KBG, C>(ring, b_cnt, pl.b_stages, b_tiles, pl.b_stage_bytes, pl.b_plane_bytes, G.w1, G.K, C, C, C);
        load_w_tile<MODE, KBG, C>(ring, b_cnt, pl.b_stages, b_tiles, pl.b_stage_bytes, pl.b_plane_bytes, G.w2, G.K, C, C, C);
      }
    }
    __syncwarp();
  }
}

}  // namespace gpp

// K granules per stage: conv1d_gp.cu's function of the layer shape (it fixes the reduction order, and the fused layer must stay
// bitwise equal to the two launches it replaces).
static int pair_shape_kbg(const GpPairParams& p, int mode) {
  GpConvParams q{};
  q.Cin = p.C; q.Cout = p.C; q.K = p.K; q.dil = p.dil; q.rate = 1;
  return gp_shape_kbg(q, mode);
}

static bool plan_pair(const GpPairParams& p, int mode, gpp::PPlan* out) {
  if (mode < 0 || mode > 3 || p.B <= 0 || p.L <= 0 || (p.C != 32 && p.C != 64 && p.C != 128) || !(p.K & 1) || p.dil < 1) return false;
  if (mode >= 2 && p.C % 16) return false;
  if (p.x == p.out) return false;
  const int kbg = pair_shape_kbg(p, mode);
  const int nsm = sm_count();
  // most accumulators per tile (the K-1 surplus rows and the halo are amortised) that still leave about a tile per SM
  for (int mt = 4; mt >= 1; mt >>= 1) {
    gpp::PPlan pl;
    if (!gpp::make_pplan(p, mode, mt, kbg, &pl)) continue;
    if (mt > 1 && pl.total_tiles < nsm) {
      gpp::PPlan smaller;
      if (gpp::make_pplan(p, mode, mt / 2, kbg, &smaller)) continue;
    }
    *out = pl;
    return true;
  }
  return false;
}

// What the ENGINE fuses: shapes whose tile keeps at least two accumulators (R >= 246 of 256 rows).  With one accumulator the K-1
// surplus rows of c2 and the halo re-reads of c1 cost ~9 % of a tile, which the compute-bound 128-channel layers do not win back.
bool gp_pair_supported(const GpPairParams& p, int mode) {
  gpp::PPlan pl;
  return plan_pair(p, mode, &pl) && pl.mt >= 2;
}

int debug_gp_pair_plan(const GpPairParams& p, int mode, int* v) {
  gpp::PPlan pl;
  if (!plan_pair(p, mode, &pl)) { set_error("resblock_gp: shape not supported (C=%d K=%d dil=%d mode=%d)", p.C, p.K, p.dil, mode); return EV_EINVAL; }
  v[0] = pl.mt; v[1] = pl.kbg; v[2] = pl.a_stages; v[3] = pl.b_stages; v[4] = gpp::NTW; v[5] = pl.acc_cols; v[6] = pl.smem_total;
  v[7] = pl.total_tiles; v[8] = pl.R; v[9] = pl.rows1_pad; v[10] = pl.rows2_pad;
  return EV_OK;
}

// The instantiations: every (MODE, KBG) of pair_shape_kbg times every tile plan_pair can return, C in {32, 64, 128} with MT * C <= 128.
using PairKernel = void (*)(GpPairParams, gpp::PPlan, GpPairGroups);
template <int MODE, int KBG>
static PairKernel pair_kernel_tile(int mt, int c) {
  switch (c) {
    case 128: return mt == 1 ? gpp::resblock_gp_kernel<MODE, 1, KBG, 128> : nullptr;
    case 64: return mt == 2 ? gpp::resblock_gp_kernel<MODE, 2, KBG, 64> : mt == 1 ? gpp::resblock_gp_kernel<MODE, 1, KBG, 64> : nullptr;
    case 32: return mt == 4 ? gpp::resblock_gp_kernel<MODE, 4, KBG, 32> : mt == 2 ? gpp::resblock_gp_kernel<MODE, 2, KBG, 32>
                  : mt == 1 ? gpp::resblock_gp_kernel<MODE, 1, KBG, 32> : nullptr;
    default: return nullptr;
  }
}
static PairKernel pair_kernel(int mode, int kbg, int mt, int c) {
  if (mode == 1) return kbg == 4 ? pair_kernel_tile<1, 4>(mt, c) : nullptr;
  if (mode == 3) return kbg == 8 ? pair_kernel_tile<3, 8>(mt, c) : pair_kernel_tile<3, 4>(mt, c);
  if (mode == 2) return kbg == 8 ? pair_kernel_tile<2, 8>(mt, c) : pair_kernel_tile<2, 4>(mt, c);
  return kbg == 8 ? pair_kernel_tile<0, 8>(mt, c) : pair_kernel_tile<0, 4>(mt, c);
}

static int dispatch_pair(const GpPairParams& p, const gpp::PPlan& pl, const GpPairGroups& gs, int mode, cudaStream_t st) {
  static std::atomic<uint64_t> attr_devs{0};
  if (first_use_on_device(attr_devs)) preload_resblock_gp();
  const PairKernel k = pair_kernel(mode, pl.kbg, pl.mt, p.C);
  EV_CHECK_ARG(k, "resblock_gp: no kernel for mode %d, KBG %d, MT %d, C %d", mode, pl.kbg, pl.mt, p.C);
  const int nsm = sm_count();
  const int grid = pl.total_tiles < nsm ? pl.total_tiles : nsm;
  return launch("resblock_gp_kernel", k, (unsigned)grid, gpp::PAIR_THREADS, pl.smem_total, st, p, pl, gs);
}

void preload_resblock_gp() {      // see preload_conv1d_gp
  for (int mode = 0; mode < 4; ++mode)
    for (int kbg = 4; kbg <= 8; kbg += 4)
      for (int c = 32; c <= 128; c *= 2)
        for (int mt = 1; mt * c <= 128; mt *= 2)
          if (const PairKernel k = pair_kernel(mode, kbg, mt, c)) cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
  cudaGetLastError();
}

int launch_gp_pair(const GpPairParams& p, int mode, cudaStream_t st) {
  gpp::PPlan pl;
  if (!plan_pair(p, mode, &pl)) { set_error("resblock_gp: shape not supported (C=%d K=%d dil=%d mode=%d)", p.C, p.K, p.dil, mode); return EV_EINVAL; }
  GpPairGroups gs{};
  gs.ng = 1;
  gs.g[0] = GpPairGroup{p.x, p.w1, p.b1, p.w2, p.b2, p.out, p.K, p.dil, pl.R, pl.tiles_m, 0};
  return dispatch_pair(p, pl, gs, mode, st);
}

int gp_pair_solo_tiles(const GpPairParams& p, int mode) {
  gpp::PPlan pl;
  return plan_pair(p, mode, &pl) ? pl.total_tiles : 0;
}

// ---- grouped launch: members ordered heaviest first; one MT for all (the smallest any member's own plan takes, >= 2), stage sizes from
// ---- the widest halos; each member keeps its own rows per tile R = 128*MT - (K-1) and tile count ------------------------------------
static bool plan_pair_group(const GpPairParams* ps, int n, int mode, GpPairGroups* gs, gpp::PPlan* out) {
  if (!ps || n < 1 || n > 3) return false;
  const GpPairParams& a = ps[0];
  int kbg = 0, span1 = 0, kmax = 0;
  for (int i = 0; i < n; ++i) {
    const GpPairParams& q = ps[i];
    if (q.B != a.B || q.L != a.L || q.C != a.C || q.lens != a.lens || q.lens_mul != a.lens_mul || q.slope != a.slope || q.acc != EV_ACC_STORE) return false;
    if (!q.x || !q.out || !q.w1 || !q.w2 || !q.b1 || !q.b2 || q.x == q.out) return false;
    for (int j = 0; j < n; ++j)
      if (j != i && (ps[j].out == q.out || ps[j].out == q.x)) return false;       // a member's output is nobody's input
    gpp::PPlan solo;
    if (!plan_pair(q, mode, &solo) || solo.mt < 2) return false;
    if (i == 0) kbg = solo.kbg;
    else if (solo.kbg != kbg) return false;
    span1 = (q.K - 1) * q.dil > span1 ? (q.K - 1) * q.dil : span1;
    kmax = q.K > kmax ? q.K : kmax;
  }
  int order[3];
  gpl::heaviest_first(ps, n, order);
  const int nsm = sm_count();
  for (int mt = 4; mt >= 2; mt >>= 1) {
    gpp::PPlan pl;
    if (!gpp::make_pplan(a, mode, mt, kbg, &pl, span1, kmax)) continue;
    int total = 0;
    gs->ng = n;
    for (int i = 0; i < n; ++i) {
      const GpPairParams& q = ps[order[i]];
      const int R = tc::BM * mt - (q.K - 1);
      const int tm = (q.L + R - 1) / R;
      gs->g[i] = GpPairGroup{q.x, q.w1, q.b1, q.w2, q.b2, q.out, q.K, q.dil, R, tm, total};
      total += q.B * tm;
    }
    if (mt > 2 && total < 2 * nsm) continue;          // keep about two tiles per SM: prefer the smaller tile
    pl.total_tiles = total;
    *out = pl;
    return true;
  }
  return false;
}
int debug_gp_pair_group_plan(const GpPairParams* ps, int n, int mode, int* v) {      // v[16]
  GpPairGroups gs{};
  gpp::PPlan pl;
  if (!plan_pair_group(ps, n, mode, &gs, &pl)) { set_error("resblock_gp group: the %d layers do not share a launch shape", n); return EV_EINVAL; }
  v[0] = pl.mt; v[1] = pl.kbg; v[2] = pl.total_tiles; v[3] = pl.rows1_pad; v[4] = pl.rows2_pad; v[5] = pl.smem_total; v[6] = pl.acc_cols;
  for (int i = 0; i < 3; ++i) {
    v[7 + 3 * i] = i < gs.ng ? gs.g[i].K : 0;
    v[8 + 3 * i] = i < gs.ng ? gs.g[i].tiles_m : 0;
    v[9 + 3 * i] = i < gs.ng ? gs.g[i].tile0 : 0;
  }
  return EV_OK;
}
bool gp_pair_group_supported(const GpPairParams* ps, int n, int mode) {
  GpPairGroups gs{};
  gpp::PPlan pl;
  return plan_pair_group(ps, n, mode, &gs, &pl);
}
int launch_gp_pair_group(const GpPairParams* ps, int n, int mode, cudaStream_t st) {
  GpPairGroups gs{};
  gpp::PPlan pl;
  if (!plan_pair_group(ps, n, mode, &gs, &pl)) { set_error("resblock_gp group: the %d layers do not share a launch shape", n); return EV_EINVAL; }
  return dispatch_pair(ps[0], pl, gs, mode, st);
}

}  // namespace ev
