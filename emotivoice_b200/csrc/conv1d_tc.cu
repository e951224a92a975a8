// Time-major 1-D convolution as an implicit GEMM on the Hopper tensor cores (sm_90a):
// wgmma (tf32 or bf16 operands from shared memory, fp32 accumulators in registers), weights streamed
// by bulk async copies (cp.async.bulk -> mbarrier complete_tx).  Same contract as conv1d_tm.cu (see ev_common.cuh):
//
//   out[b,t,co] = epi( bias[co] + sum_j sum_ci w[j][ci][co] * act_in( x[b, t + (j-(K-1)/2)*dil, ci] ) )
//
// GEMM view: M = time (128 rows per accumulator tile, MT tiles per CTA tile), N = C_out tile (<= 128),
// K = taps x C_in.
//
// * ONE activation fetch per tile for all k taps: the A operand lives in shared memory in the
//   no-swizzle K-major layout with the 8-row-group stride (SBO) set to 128 B, i.e. element
//   (row r, 16-byte K-granule g) sits at  A + (g * rows_pad + r) * 16 bytes.  Consecutive rows are
//   16 B apart for the whole tile, so tap j of a dilated convolution is the same staged tile with the
//   descriptor start address advanced by j*dil rows, and accumulator mt by 128*mt rows.  The producer
//   warps apply the LeakyReLU prologue, the zero padding at the sequence ends, the tf32 rounding /
//   hi-lo split and the layout change while staging, so activations stay plain fp32 time-major in HBM
//   and no tensor map is needed.
// * One weight tile from L2 feeds MT accumulators (MT x fewer weight bytes per output row).
// * Persistent CTAs (one per SM) loop over tiles.
//
// Roles (480 threads): warps 0-7 are two consumer warpgroups: warpgroup w issues the wgmma for rows [64 w, 64 w + 64) of every
// 128-row accumulator, keeps those accumulators in registers and stores them; warps 8-13 stage A; warp 14's first lane streams
// the weight tiles.  mbarrier pipelines: A ring (a_full/a_empty), B ring (b_full/b_empty); a consumer warp releases a stage once
// wgmma.wait_group has seen the MMAs that read it complete (one step behind the issue, so the tensor core always has the next
// step queued).
#include <cstdio>
#include <cstdlib>

#include "ev_common.cuh"
#include "tc_common.cuh"

namespace ev {

namespace tc {

struct Plan {
  int BN, mt, kbg, planes;
  int rows_pad;        // staged rows per A granule; == 8/kbg (mod 8) -> conflict-free 16 B stores
  int a_plane_bytes, b_plane_bytes, a_stage_bytes, b_stage_bytes;
  int a_stages, b_stages;
  int ngroups;         // producer groups: largest of {6,3,2,1} that is <= a_stages
  int ksplit;          // K-split factor S: S CTAs share one output tile, each reducing a slice of the C_in blocks
                       // into a private partial buffer; splitk_reduce_kernel sums them in a fixed order
  int acc_cols;        // accumulator columns per consumer thread's 64-row slices: MT * BN <= 2 * ACC_REGS
  int tiles_m, tiles_n, total_tiles;
  int smem_total;
};

// smem map: [0,256) barriers | 1024: A ring | B ring
__host__ __device__ inline bool make_plan(const ConvParams& p, int mode, int BN, int mt, int kbg, int min_b_stages, Plan* o, int b_target = 4) {
  Plan q;
  q.planes = (mode == 1 || mode == 3) ? 2 : 1;
  const int cpg = mode >= 2 ? 8 : 4;      // channels per 16-byte operand granule (bf16 : tf32)
  q.kbg = kbg;
  q.mt = mt;
  q.BN = BN;
  if (mt * q.BN > 2 * ACC_REGS) return false;
  q.acc_cols = mt * q.BN;
  const int rows = BM * mt + (p.K - 1) * p.dil;
  q.rows_pad = ((rows + 7) / 8) * 8 + 8 / q.kbg;
  q.a_plane_bytes = q.kbg * q.rows_pad * 16;
  q.b_plane_bytes = q.kbg * q.BN * 16;
  q.a_stage_bytes = q.planes * q.a_plane_bytes;
  q.b_stage_bytes = q.planes * q.b_plane_bytes;
  const int budget = 227 * 1024 - 1024;
  const int n_cb = (p.Cin + cpg * q.kbg - 1) / (cpg * q.kbg);
  // at least 2 + 2 stages; then grow the weight ring first (it turns over K times per A stage)
  if (min_b_stages > n_cb * p.K) min_b_stages = n_cb * p.K;
  if (min_b_stages < 2) min_b_stages = 2;
  if (2 * q.a_stage_bytes + min_b_stages * q.b_stage_bytes > budget) return false;
  q.a_stages = 2;
  q.b_stages = 2;
  while (q.b_stages < MAX_B_STAGES && q.b_stages < n_cb * p.K &&
         q.a_stages * q.a_stage_bytes + (q.b_stages + 1) * q.b_stage_bytes <= budget && q.b_stages < b_target) ++q.b_stages;
  while (q.a_stages < MAX_A_STAGES && q.a_stages < n_cb &&
         (q.a_stages + 1) * q.a_stage_bytes + q.b_stages * q.b_stage_bytes <= budget && q.a_stages < 6) ++q.a_stages;
  while (q.b_stages < MAX_B_STAGES && q.b_stages < n_cb * p.K &&
         q.a_stages * q.a_stage_bytes + (q.b_stages + 1) * q.b_stage_bytes <= budget) ++q.b_stages;
  while (q.a_stages < MAX_A_STAGES && q.a_stages < n_cb &&
         (q.a_stages + 1) * q.a_stage_bytes + q.b_stages * q.b_stage_bytes <= budget) ++q.a_stages;
  q.ngroups = q.a_stages >= 6 ? 6 : (q.a_stages >= 3 ? 3 : (q.a_stages >= 2 ? 2 : 1));
  q.tiles_m = (p.L + BM * mt - 1) / (BM * mt);
  q.tiles_n = (p.Cout + q.BN - 1) / q.BN;
  q.ksplit = 1;
  q.total_tiles = p.B * q.tiles_m * q.tiles_n;
  q.smem_total = 1024 + q.a_stages * q.a_stage_bytes + q.b_stages * q.b_stage_bytes;
  *o = q;
  return true;
}

// out[e..e+3] = epi( sum_z partial[z][e..e+3] ): the slices added in the fixed order z = 0..S-1 starting from zero (deterministic,
// batch invariant), then bias / activation / residual / accumulate exactly like the fused epilogue; rows >= len are zeros.
__device__ __forceinline__ void splitk_reduce_store(const ConvParams& p, int S, size_t per, size_t e, int b, int row, int col, int len) {
  float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
  if (row < len) {
    for (int z = 0; z < S; ++z) {
      const float4 v = *reinterpret_cast<const float4*>(p.splitk_ws + (size_t)z * per + e);
      o.x += v.x; o.y += v.y; o.z += v.z; o.w += v.w;
    }
    if (p.bias) {
      const float4 b4 = __ldg(reinterpret_cast<const float4*>(p.bias + (size_t)b * p.bias_bs + col));
      o.x += b4.x; o.y += b4.y; o.z += b4.z; o.w += b4.w;
    }
    if (p.out_act != EV_ACT_NONE) {
      o.x = act_apply(o.x, p.out_act, 0.f); o.y = act_apply(o.y, p.out_act, 0.f);
      o.z = act_apply(o.z, p.out_act, 0.f); o.w = act_apply(o.w, p.out_act, 0.f);
    }
    if (p.res) {
      const float4 r4 = *reinterpret_cast<const float4*>(p.res + e);
      o.x += r4.x; o.y += r4.y; o.z += r4.z; o.w += r4.w;
    }
    if (p.acc != EV_ACC_STORE) {
      const float4 q4 = *reinterpret_cast<const float4*>(p.out + e);
      o.x += q4.x; o.y += q4.y; o.z += q4.z; o.w += q4.w;
      if (p.acc == EV_ACC_ADD_DIV) { o.x /= p.div; o.y /= p.div; o.z /= p.div; o.w /= p.div; }
    }
  }
  *reinterpret_cast<float4*>(p.out + e) = o;
}

// MODE 0: one tf32 MMA per K step (operands rounded to nearest tf32).
// MODE 2: bf16 operands (rounded to nearest even by the producers / the host), 8 channels per granule.
// MODE 3: "bf16x3" fp32-class emulation: x = hi + lo with hi = bf16(x), lo = bf16(x - hi) (16 significant bits), three bf16 MMAs per
//                 K = 16 step: ~1e-5 relative at half the tensor-core / weight-stream cost of 3xTF32.
// MODE 1: "3xTF32" fp32 emulation: x = hi + lo with hi = tf32(x), lo = tf32(x - hi), three MMAs per K step into the same fp32
//                 accumulator.  Weights arrive pre-split (two planes, packing.to_tc_layout); activations are split by the producer warps.
// MT: 128-row accumulator tiles per CTA tile.  KBG: 16-byte K granules (4 tf32 or 8 bf16 channels each) per pipeline stage.
// BN = pl.BN, the N tile: fixed at compile time, so a tap of a full channel block is one unbroken wgmma chain (tc::tap_chain).
template <int MODE, int MT, int KBG, int BN>
__global__ void __launch_bounds__(NTHREADS, 1) conv1d_tc_kernel(ConvParams p, Plan pl) {
  constexpr bool SPLIT3 = (MODE == 1);
  constexpr bool X3B = (MODE == 3);       // "bf16x3": fp32 operands split into bf16 hi + lo planes, three bf16 MMAs per K = 16 step
  constexpr bool BF16 = (MODE == 2) || X3B;      // the staged operands are bf16 (8 channels per granule)
  constexpr int PLANES = (SPLIT3 || X3B) ? 2 : 1;
  constexpr int CPG = BF16 ? 8 : 4;       // channels per 16-byte granule
  constexpr int KB = CPG * KBG;
  constexpr int NK8 = KBG / 2;            // MMA K steps of a full channel block: two 16-byte granules each
  constexpr int GSH = (KBG == 8 ? 3 : 2);
  constexpr int NA = BN / 2;              // accumulator registers per 128-row tile: BN columns x 64 rows over 128 threads
  constexpr int NCW = NCONS / 32;         // consumer warps: every one of them releases each stage
  static_assert(BN % 16 == 0 && MT * BN <= 2 * ACC_REGS, "accumulators of the tile exceed the register budget");
  extern __shared__ __align__(128) uint8_t smem_raw[];
  const int tid = threadIdx.x;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);   // provably warp-uniform: ptxas serialises every wgmma on a path it cannot prove uniform
  const int lane = tid & 31;

  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw);
  uint8_t* a_tiles = smem_raw + 1024;
  uint8_t* b_tiles = a_tiles + pl.a_stages * pl.a_stage_bytes;
  const uint32_t bar_base = smem_u32(bars);
  auto a_full = [&](int s) { return bar_base + 8u * s; };
  auto a_empty = [&](int s) { return bar_base + 8u * (MAX_A_STAGES + s); };
  auto b_full = [&](int s) { return bar_base + 8u * (2 * MAX_A_STAGES + s); };
  auto b_empty = [&](int s) { return bar_base + 8u * (2 * MAX_A_STAGES + MAX_B_STAGES + s); };

  if (tid == 0) {
    for (int s = 0; s < pl.a_stages; ++s) { mbar_init(a_full(s), (NPWARPS / pl.ngroups) * 32); mbar_init(a_empty(s), NCW); }
    for (int s = 0; s < pl.b_stages; ++s) { mbar_init(b_full(s), 1); mbar_init(b_empty(s), NCW); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // Programmatic dependent launch (ev_common.cuh).  The grid is persistent (<= one CTA per SM, all resident), so it lets the NEXT
  // launch in the stream start as soon as SMs free up: that kernel's CTAs run their set-up (barriers) while this grid's tail is
  // still running.  Every role, the weight loader included, executes griddepcontrol.wait before it reads p.lens or activations:
  // p.lens may come from a grid that is still running TWO launches upstream (validate_inputs_kernel writes the int32 lengths,
  // LayerNorm starts early and waits, this kernel starts early too), and a role that decoded tiles from stale lengths would walk
  // a different tile sequence than the others and the pipeline would deadlock.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  const int n_cb = (p.Cin + KB - 1) / KB;
  const int halo = ((p.K - 1) / 2) * p.dil;
  const int rows_a = BM * MT + (p.K - 1) * p.dil;
  const int tiles_per_b = pl.tiles_m * pl.tiles_n;

  // tile -> (b, t0, n0, nt, len); every role walks the same sequence
  int z_cur = 0;     // K-split slice of the tile most recently decoded by this thread
  auto decode = [&](int tile, int& b, int& t0, int& n0, int& nt, int& len) {
    z_cur = tile % pl.ksplit;
    tile /= pl.ksplit;
    b = tile / tiles_per_b;
    const int r = tile - b * tiles_per_b;
    const int tm = r / pl.tiles_n, tn = r - tm * pl.tiles_n;
    t0 = tm * (BM * MT);
    n0 = tn * BN;
    nt = min(BN, p.Cout - n0);
    len = p.lens ? min(p.L, p.lens[b] * p.lens_mul) : p.L;
  };

  if (warp < NCW) {
    // ============================ consumers: MMA issue + epilogue ==================================
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const int wg = warp >> 2, wl = warp & 3;
    const bool split = pl.ksplit > 1;           // K-split: raw partial sums, the fused epilogue runs in the reduce kernel
    const bool has_res = p.res != nullptr && !split;
    const int oact = split ? EV_ACT_NONE : p.out_act, accm = split ? EV_ACC_STORE : p.acc;
    const uint32_t a_lbo = (uint32_t)pl.rows_pad * 16u, b_lbo = (uint32_t)BN * 16u;
    const uint64_t a_desc0 = make_desc(0u, a_lbo, 128u), b_desc0 = make_desc(0u, b_lbo, 128u);
    const uint32_t a_tap = (uint32_t)p.dil * 16u, a_k8 = 2u * a_lbo;
    float acc[MT][NA];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int i = 0; i < NA; ++i) acc[mt][i] = 0.f;
    auto release = [&](int sb, int sa) {
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(b_empty(sb));
        if (sa >= 0) mbar_arrive(a_empty(sa));
      }
    };
    int a_cnt = 0, b_cnt = 0;
    for (int tile = blockIdx.x; tile < pl.total_tiles; tile += gridDim.x) {
      int b, t0, n0, nt, len;
      decode(tile, b, t0, n0, nt, len);
      float* ob = (split ? p.splitk_ws + (size_t)z_cur * p.B * p.L * p.Cout : p.out) + (size_t)b * p.L * p.Cout;   // may alias p.res
      const float* rb = has_res ? p.res + (size_t)b * p.L * p.Cout : nullptr;
      const bool active = t0 < len;      // padding tile: the batch-invariant contract stores zeros (no MMA work is issued)
      if (active) {
        const int cb_lo = (z_cur * n_cb) / pl.ksplit, cb_hi = ((z_cur + 1) * n_cb) / pl.ksplit;
        int prev_sb = -1, prev_sa = -1;
        for (int cb = cb_lo; cb < cb_hi; ++cb, ++a_cnt) {
          const int sa = a_cnt % pl.a_stages;
          const int nk8 = min(KB, p.Cin - cb * KB) / (2 * CPG);   // MMA K steps: two 16-byte granules each
          mbar_wait(a_full(sa), (a_cnt / pl.a_stages) & 1);
          const uint64_t a_hi0 = desc_advance(a_desc0, smem_u32(a_tiles + sa * pl.a_stage_bytes) + (uint32_t)(wg * 64) * 16u);
          for (int j = 0; j < p.K; ++j, ++b_cnt) {
            const int sb = b_cnt % pl.b_stages;
            mbar_wait(b_full(sb), (b_cnt / pl.b_stages) & 1);
            const uint64_t b_hi0 = desc_advance(b_desc0, smem_u32(b_tiles + sb * pl.b_stage_bytes));
            // the tap's nk8 K steps x MT accumulators as one chain; the K-split slice's first tap overwrites the accumulators.  The
            // wait inside each branch: joined before it, the paths would leave the tap as two commit groups (tc::tap_chain)
            const uint64_t a_j = desc_advance(a_hi0, (uint32_t)j * a_tap);
            if (nk8 == NK8) {
              tap_chain<MODE, BN, NK8>(acc, a_j, a_k8, (uint32_t)pl.a_plane_bytes, b_hi0, (uint32_t)pl.b_plane_bytes, (cb - cb_lo) | j);
              wgmma_wait<1>();        // the previous step's MMAs have completed: its stages may be refilled
            } else {
              tap_chain_short<MODE, BN>(acc, a_j, a_k8, (uint32_t)pl.a_plane_bytes, b_hi0, (uint32_t)pl.b_plane_bytes, (cb - cb_lo) | j, nk8);
              wgmma_wait<1>();
            }
            if (prev_sb >= 0) release(prev_sb, prev_sa);
            prev_sb = sb;
            prev_sa = j == p.K - 1 ? sa : -1;
          }
        }
        wgmma_wait<0>();
        release(prev_sb, prev_sa);
      }
      // epilogue straight from the accumulator fragments: two adjacent columns per register pair (8-byte accesses)
      const float* __restrict__ bias = (p.bias && !split) ? p.bias + (size_t)b * p.bias_bs + n0 : nullptr;
#pragma unroll
      for (int mt = 0; mt < MT; ++mt) {
#pragma unroll
        for (int i = 0; i < NA; i += 2) {
          const int c = frag_col(i, lane);
          const int row = t0 + mt * BM + wg * 64 + frag_row(i, lane, wl);
          if (c >= nt || row >= p.L) continue;
          const size_t off = (size_t)row * p.Cout + n0 + c;
          float2 o = make_float2(0.f, 0.f);
          if (active && row < len) {
            o = make_float2(acc[mt][i], acc[mt][i + 1]);
            if (bias) {
              const float2 b2 = __ldg(reinterpret_cast<const float2*>(bias + c));
              o.x += b2.x; o.y += b2.y;
            }
            if (oact != EV_ACT_NONE) { o.x = act_apply(o.x, oact, 0.f); o.y = act_apply(o.y, oact, 0.f); }
            if (has_res) {
              const float2 r2 = *reinterpret_cast<const float2*>(rb + off);
              o.x += r2.x; o.y += r2.y;
            }
            if (accm != EV_ACC_STORE) {
              const float2 q2 = *reinterpret_cast<const float2*>(ob + off);
              o.x += q2.x; o.y += q2.y;
              if (accm == EV_ACC_ADD_DIV) { o.x /= p.div; o.y /= p.div; }
            }
          }
          *reinterpret_cast<float2*>(ob + off) = o;
        }
      }
    }
  } else if (warp < W_WLOAD) {
    // ============================ A producers ===================================================
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const int pwarp = warp - NCW;
    const int wpg = NPWARPS / pl.ngroups;          // warps per group
    const int grp = pwarp / wpg;
    const int gt = (pwarp - grp * wpg) * 32 + lane;  // thread index inside the group
    const int GT = wpg * 32;
    const bool lrelu = (p.in_act == EV_ACT_LRELU);
    const float slope = p.in_slope;
    const int total = rows_a * KBG;   // (row, granule) pairs; granule fastest -> coalesced row segments
    int a_cnt = 0;
    for (int tile = blockIdx.x; tile < pl.total_tiles; tile += gridDim.x) {
      int b, t0, n0, nt, len;
      decode(tile, b, t0, n0, nt, len);
      if (t0 >= len) continue;
      const float* __restrict__ xb = p.x + (size_t)b * p.L * p.Cin;
      const int cb_lo = (z_cur * n_cb) / pl.ksplit, cb_hi = ((z_cur + 1) * n_cb) / pl.ksplit;
      for (int cb = cb_lo; cb < cb_hi; ++cb, ++a_cnt) {
        if (a_cnt % pl.ngroups != grp) continue;       // this stage belongs to another producer group
        const int s = a_cnt % pl.a_stages;
        const int c0 = cb * KB;
        const int ngran = min(KB, p.Cin - c0) / CPG;
        uint8_t* dst = a_tiles + s * pl.a_stage_bytes;
        constexpr int ALD = BF16 ? A_LD / 2 : A_LD;     // (row, granule) pairs per thread and batch
        constexpr int NW = BF16 ? 2 : 1;                // float4 loads per pair (8 : 4 channels)
        for (int base = 0; base < total; base += GT * ALD) {
          // a batch of global loads is issued before anything else (memory-level parallelism)
          float4 v[ALD * NW];
#pragma unroll
          for (int u = 0; u < ALD; ++u) {
            const int idx = base + u * GT + gt;
            const int r = idx >> GSH, g = idx & (KBG - 1);
            const int row = t0 - halo + r;
            const bool ok = idx < total && g < ngran && row >= 0 && row < len;
            const float* src = xb + (size_t)row * p.Cin + c0 + g * CPG;
#pragma unroll
            for (int w = 0; w < NW; ++w)
              v[u * NW + w] = ok ? __ldg(reinterpret_cast<const float4*>(src + 4 * w)) : make_float4(0.f, 0.f, 0.f, 0.f);
          }
          if (base == 0) mbar_wait(a_empty(s), ((a_cnt / pl.a_stages) & 1) ^ 1);
#pragma unroll
          for (int u = 0; u < ALD; ++u) {
            const int idx = base + u * GT + gt;
            const int r = idx >> GSH, g = idx & (KBG - 1);
            if (idx < total && g < ngran) {
#pragma unroll
              for (int w = 0; w < NW; ++w) {
                float4& t = v[u * NW + w];
                if (lrelu) {
                  t.x = t.x > 0.f ? t.x : t.x * slope;
                  t.y = t.y > 0.f ? t.y : t.y * slope;
                  t.z = t.z > 0.f ? t.z : t.z * slope;
                  t.w = t.w > 0.f ? t.w : t.w * slope;
                }
              }
              uint8_t* d = dst + ((size_t)g * pl.rows_pad + r) * 16;
              if (BF16) {
                const float4 t0 = v[u * NW], t1 = v[u * NW + NW - 1];
                uint4 q;
                q.x = pack_bf16(t0.x, t0.y); q.y = pack_bf16(t0.z, t0.w);
                q.z = pack_bf16(t1.x, t1.y); q.w = pack_bf16(t1.z, t1.w);
                *reinterpret_cast<uint4*>(d) = q;
                if (X3B) {      // lo plane: what the bf16 rounding dropped (8 more significant bits)
                  uint4 l;
                  l.x = pack_bf16(t0.x - __uint_as_float(q.x << 16), t0.y - __uint_as_float(q.x & 0xffff0000u));
                  l.y = pack_bf16(t0.z - __uint_as_float(q.y << 16), t0.w - __uint_as_float(q.y & 0xffff0000u));
                  l.z = pack_bf16(t1.x - __uint_as_float(q.z << 16), t1.y - __uint_as_float(q.z & 0xffff0000u));
                  l.w = pack_bf16(t1.z - __uint_as_float(q.w << 16), t1.w - __uint_as_float(q.w & 0xffff0000u));
                  *reinterpret_cast<uint4*>(d + pl.a_plane_bytes) = l;
                }
              } else {
                const float4 t = v[u * NW];
                // round-to-nearest tf32 (the MMA would otherwise truncate the low 13 mantissa bits)
                const float4 h = make_float4(to_tf32(t.x), to_tf32(t.y), to_tf32(t.z), to_tf32(t.w));
                *reinterpret_cast<float4*>(d) = h;
                if (SPLIT3) {
                  const float4 l = make_float4(to_tf32(t.x - h.x), to_tf32(t.y - h.y), to_tf32(t.z - h.z), to_tf32(t.w - h.w));
                  *reinterpret_cast<float4*>(d + pl.a_plane_bytes) = l;
                }
              }
            }
          }
        }
        fence_proxy_async();      // generic-proxy smem writes -> visible to the tensor core (async proxy)
        mbar_arrive(a_full(s));
      }
    }
  } else {
    // ============================ weight loader ==================================================
    if (lane == 0) {
      asm volatile("griddepcontrol.wait;" ::: "memory");      // p.lens (see the note after the set-up)
      // w_tc layout: [plane (hi, lo)][N tile of BNp = min(Cout,128)][tap][Cin/CPG granules][BNp][16 bytes]
      // (4 fp32 or 8 bf16 per granule; granule-major inside a tile)
      const int cin4 = p.Cin / CPG;
      const int bnp = p.Cout < 128 ? p.Cout : 128;
      const size_t plane = (size_t)p.K * cin4 * p.Cout * 4;         // 4-byte words per plane (fp32 or packed bf16 granules)
      const size_t tile_stride = (size_t)p.K * cin4 * bnp * 4;      // floats per packed N tile
      int b_cnt = 0;
      for (int tile = blockIdx.x; tile < pl.total_tiles; tile += gridDim.x) {
        int b, t0, n0, nt, len;
        decode(tile, b, t0, n0, nt, len);
        if (t0 >= len) continue;
        const float* wt = p.w + (size_t)(n0 / bnp) * tile_stride + (size_t)(n0 % bnp) * 4;
        const int cb_lo = (z_cur * n_cb) / pl.ksplit, cb_hi = ((z_cur + 1) * n_cb) / pl.ksplit;
        for (int cb = cb_lo; cb < cb_hi; ++cb) {
          const int ngran = min(KB, p.Cin - cb * KB) / CPG;
          for (int j = 0; j < p.K; ++j, ++b_cnt) {
            const int sb = b_cnt % pl.b_stages;
            mbar_wait(b_empty(sb), ((b_cnt / pl.b_stages) & 1) ^ 1);
            mbar_expect_tx(b_full(sb), (uint32_t)(PLANES * ngran * nt * 16));
            const uint32_t dst = smem_u32(b_tiles + sb * pl.b_stage_bytes);
            const float* src = wt + ((size_t)j * cin4 + (size_t)cb * KBG) * bnp * 4;
            if (nt == bnp) {
              // the CTA's N tile is a whole packed tile: the stage's granules are adjacent in memory -> ONE bulk copy per plane
              bulk_g2s(dst, src, (uint32_t)(ngran * nt * 16), b_full(sb));
              if (PLANES == 2) bulk_g2s(dst + (uint32_t)pl.b_plane_bytes, src + plane, (uint32_t)(ngran * nt * 16), b_full(sb));
            } else {
              for (int g = 0; g < ngran; ++g) {
                bulk_g2s(dst + (uint32_t)(g * BN * 16), src + (size_t)g * bnp * 4, (uint32_t)(nt * 16), b_full(sb));
                if (PLANES == 2) bulk_g2s(dst + (uint32_t)(pl.b_plane_bytes + g * BN * 16), src + plane + (size_t)g * bnp * 4, (uint32_t)(nt * 16), b_full(sb));
              }
            }
          }
        }
      }
    }
    __syncwarp();
  }
}

// Second half of a K-split convolution: out = epi( sum_z partial[z] ) with the slices added in the
// fixed order z = 0..S-1 (deterministic, batch invariant), then bias / activation / residual /
// accumulate exactly like the fused epilogue.  One float4 per thread.
__global__ void __launch_bounds__(256) splitk_reduce_kernel(ConvParams p, int S) {
  pdl_entry();
  const size_t per = (size_t)p.B * p.L * p.Cout;
  const size_t i4 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i4 * 4 >= per) return;
  const size_t e = i4 * 4;
  const int col = (int)(e % p.Cout);
  const size_t rowg = e / p.Cout;
  const int b = (int)(rowg / p.L), row = (int)(rowg % p.L);
  const int len = p.lens ? min(p.L, p.lens[b] * p.lens_mul) : p.L;
  splitk_reduce_store(p, S, per, e, b, row, col, len);
}

}  // namespace tc

// The instantiations: every (MODE, KBG) the shape rule tc_shape_kbg gives (KBG = 4 in 3xTF32) times every tile plan_conv1d_tc can
// return.  BN starts at min(C_out, 128) and halves while it stays a multiple of 16 (so any multiple of 16 up to 128), MT halves until
// MT * BN <= 128: 14 tiles per (MODE, KBG), 98 kernels.
using TcKernel = void (*)(ConvParams, tc::Plan);
template <int MODE, int KBG>
static TcKernel tc_kernel_tile(int mt, int bn) {
  using namespace tc;
  switch (bn) {
    case 128: return mt == 1 ? conv1d_tc_kernel<MODE, 1, KBG, 128> : nullptr;
    case 112: return mt == 1 ? conv1d_tc_kernel<MODE, 1, KBG, 112> : nullptr;
    case 96: return mt == 1 ? conv1d_tc_kernel<MODE, 1, KBG, 96> : nullptr;
    case 80: return mt == 1 ? conv1d_tc_kernel<MODE, 1, KBG, 80> : nullptr;
    case 64: return mt == 2 ? conv1d_tc_kernel<MODE, 2, KBG, 64> : mt == 1 ? conv1d_tc_kernel<MODE, 1, KBG, 64> : nullptr;
    case 48: return mt == 2 ? conv1d_tc_kernel<MODE, 2, KBG, 48> : mt == 1 ? conv1d_tc_kernel<MODE, 1, KBG, 48> : nullptr;
    case 32: return mt == 4 ? conv1d_tc_kernel<MODE, 4, KBG, 32> : mt == 2 ? conv1d_tc_kernel<MODE, 2, KBG, 32>
                  : mt == 1 ? conv1d_tc_kernel<MODE, 1, KBG, 32> : nullptr;
    case 16: return mt == 4 ? conv1d_tc_kernel<MODE, 4, KBG, 16> : mt == 2 ? conv1d_tc_kernel<MODE, 2, KBG, 16>
                  : mt == 1 ? conv1d_tc_kernel<MODE, 1, KBG, 16> : nullptr;
    default: return nullptr;
  }
}
static TcKernel tc_kernel(int mode, int kbg, int mt, int bn) {
  if (mode == 1) return kbg == 4 ? tc_kernel_tile<1, 4>(mt, bn) : nullptr;
  if (mode == 3) return kbg == 8 ? tc_kernel_tile<3, 8>(mt, bn) : tc_kernel_tile<3, 4>(mt, bn);
  if (mode == 2) return kbg == 8 ? tc_kernel_tile<2, 8>(mt, bn) : tc_kernel_tile<2, 4>(mt, bn);
  return kbg == 8 ? tc_kernel_tile<0, 8>(mt, bn) : tc_kernel_tile<0, 4>(mt, bn);
}

// Load every instantiation's code now and set the shared-memory attribute (see conv1d_gp.cu: preload_conv1d_gp), on exactly the
// instantiations dispatch_tc can launch.
void preload_conv1d_tc() {
  for (int mode = 0; mode < 4; ++mode)
    for (int kbg = 4; kbg <= 8; kbg += 4)
      for (int bn = 16; bn <= 128; bn += 16)
        for (int mt = 1; mt <= 4 && mt * bn <= 128; mt *= 2)
          if (const TcKernel k = tc_kernel(mode, kbg, mt, bn)) cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
  cudaFuncAttributes fa;
  cudaFuncGetAttributes(&fa, tc::splitk_reduce_kernel);
  cudaGetLastError();
}

static int validate_conv1d_tc(const ConvParams& p, int mode) {
  EV_CHECK_ARG(p.B > 0 && p.L > 0, "conv1d_tc: bad problem B=%d L=%d", p.B, p.L);
  EV_CHECK_ARG(p.Cin % (mode >= 2 ? 16 : 8) == 0, "conv1d_tc: Cin=%d must be a multiple of %d", p.Cin, mode >= 2 ? 16 : 8);
  EV_CHECK_ARG(p.Cout % 16 == 0 && (p.Cout <= 128 || p.Cout % 128 == 0), "conv1d_tc: Cout=%d must be a multiple of 16, and of 128 above 128", p.Cout);
  EV_CHECK_ARG(p.K >= 1 && (p.K & 1) && p.dil >= 1, "conv1d_tc: K=%d must be odd, dil=%d >= 1", p.K, p.dil);
  EV_CHECK_ARG(p.in_act == EV_ACT_NONE || p.in_act == EV_ACT_LRELU, "conv1d_tc: unsupported input activation");
  return EV_OK;
}

// K granules per stage decide how the (channel block, tap) reduction is ordered, so they must be a function
// of the layer shape alone: 8 if a (widest-N, one-accumulator) tile fits with them in 1x mode, else 4.
int tc_shape_kbg(const ConvParams& p, int mode) {
  tc::Plan pl;
  const int bn_max = p.Cout <= 128 ? p.Cout : 128;
  return (mode != 1 && tc::make_plan(p, mode, bn_max, 1, 8, 4, &pl)) ? 8 : 4;
}

// K-split: a long reduction at few output tiles (the acoustic model's GEMMs at batch 1; the conv-FFN's second
// conv has K = 3*1536) is one long serial chain per tile; share it among S CTAs with private partial buffers
// + a fixed-order reduce kernel.  S is requested per LAYER by the engine (never derived from batch or
// length), so the summation order -- and therefore every output bit -- is the same for a B=1 call and for
// the same utterance inside any batch.
static int apply_ksplit(const ConvParams& p, int mode, tc::Plan* pl) {
  const size_t per = (size_t)p.B * p.L * p.Cout;
  if (p.ksplit > 1 && (p.splitk_ws || p.splitk_cap == (size_t)-1)) {
    int S = p.ksplit;
    const int cpg = mode >= 2 ? 8 : 4;
    const int n_cb = (p.Cin + cpg * pl->kbg - 1) / (cpg * pl->kbg);
    if (S > n_cb) S = n_cb;
    if ((size_t)S * per > p.splitk_cap) { set_error("conv1d_tc: split-K scratch too small (%zu < %zu floats)", p.splitk_cap, (size_t)S * per); return EV_EWORKSPACE; }
    if (S > 1) {
      pl->ksplit = S;
      pl->total_tiles *= S;
    }
  }
  return EV_OK;
}

// Tile / pipeline plan of one launch (pure host arithmetic; also exported as ev_debug_tc_plan so the CPU tests
// can check the invariants the kernel's barrier protocol and the batch-invariance contract rely on).
static int plan_conv1d_tc(const ConvParams& p, int mode, tc::Plan* out) {
  EV_TRY(validate_conv1d_tc(p, mode));
  // Tile shape.  None of these choices changes the order in which any output element's K reduction is
  // summed, so results are bitwise independent of batch size / sequence length (batch-invariant contract).
  //  * N tile: min(C_out, 128) (the weight packing tile: one bulk copy per stage); halved (down to 32) only for
  //    launches with a handful of tiles (measured: finer N splitting costs more in per-granule copies and
  //    replicated A staging than it gains in parallelism).
  //  * rows per tile: as many 128-row accumulators as still leave about one tile per SM (every weight tile
  //    fetched from L2 then feeds MT MMAs), limited by the accumulator registers (MT x BN <= 128) and smem.
  const int bn_thresh = 24, mt_thresh = 120;     // tuning constants (tile shape only: results are unaffected)
  const long long tiles128 = (long long)((p.L + tc::BM - 1) / tc::BM) * p.B;
  int BN = p.Cout <= 128 ? p.Cout : 128;          // == the packing tile of packing.to_tc_layout
  while (BN >= 64 && (BN / 2) % 16 == 0 && tiles128 * ((p.Cout + BN - 1) / BN) < bn_thresh) BN /= 2;
  int mt = tiles128 >= 4 * mt_thresh ? 4 : (tiles128 >= 2 * mt_thresh ? 2 : 1);
  tc::Plan pl;
  const int kbg = tc_shape_kbg(p, mode);
  for (;; mt >>= 1) {
    if (tc::make_plan(p, mode, BN, mt, kbg, 4, &pl)) break;
    if (tc::make_plan(p, mode, BN, mt, kbg, 2, &pl)) break;
    if (mt == 1) { set_error("conv1d_tc: tile does not fit in shared memory / accumulator registers (K=%d dil=%d Cout=%d)", p.K, p.dil, p.Cout); return EV_EINVAL; }
  }
  EV_TRY(apply_ksplit(p, mode, &pl));
  *out = pl;
  return EV_OK;
}

int debug_tc_plan(const ConvParams& p, int mode, int* v) {
  tc::Plan pl;
  const int rc = plan_conv1d_tc(p, mode, &pl);
  if (rc != EV_OK) return rc;
  v[0] = pl.BN; v[1] = pl.mt; v[2] = pl.kbg; v[3] = pl.a_stages; v[4] = pl.b_stages; v[5] = pl.ngroups;
  v[6] = pl.ksplit; v[7] = pl.acc_cols; v[8] = pl.smem_total; v[9] = pl.total_tiles; v[10] = pl.rows_pad;
  return EV_OK;
}

static int dispatch_tc(const ConvParams& p, int mode, const tc::Plan& pl, cudaStream_t st) {
  static std::atomic<uint64_t> attr_devs{0};   // function attributes are per device
  if (first_use_on_device(attr_devs)) preload_conv1d_tc();
  const TcKernel k = tc_kernel(mode, pl.kbg, pl.mt, pl.BN);
  EV_CHECK_ARG(k, "conv1d_tc: no kernel for mode %d, KBG %d, MT %d, BN %d", mode, pl.kbg, pl.mt, pl.BN);
  const int grid = pl.total_tiles < sm_count() ? pl.total_tiles : sm_count();
  return launch("conv1d_tc_kernel", k, (unsigned)grid, tc::NTHREADS, pl.smem_total, st, p, pl);
}

// p.w must be in the tensor-core layout [plane][Cout/BNp][K][Cin/4][BNp][4] (packing.py: to_tc_layout);
// mode 0: 1xTF32, 1: 3xTF32 fp32 emulation (reads both planes), 2: bf16 operands (p.w in the bf16 tc layout).
int launch_conv1d_tc(const ConvParams& p, int mode, cudaStream_t st) {
  tc::Plan pl;
  EV_TRY(plan_conv1d_tc(p, mode, &pl));
  const size_t per = (size_t)p.B * p.L * p.Cout;
  const int rc = dispatch_tc(p, mode, pl, st);
  if (rc != EV_OK || pl.ksplit == 1) return rc;
  const size_t n4 = per / 4;
  return launch("splitk_reduce_kernel", tc::splitk_reduce_kernel, (unsigned)((n4 + 255) / 256), 256, 0, st, p, pl.ksplit);
}

}  // namespace ev
