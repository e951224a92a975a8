// HiFi-GAN convolutions on "granule-planar" activations (sm_90a): wgmma implicit GEMM whose A operand is fed by bulk async
// copies (cp.async.bulk -> mbarrier complete_tx) instead of a register round trip, and whose epilogue stores straight from the
// accumulator fragments -- no shared-memory transpose on either side.
//
// Layout (GP): an activation tensor (B, L, C) is stored as [b][g = C / cpg][l][cpg] with 16-byte granules
// (cpg = 4 fp32 or 8 bf16 channels): every granule is a contiguous plane of L x 16 bytes.  That is exactly the no-swizzle
// K-major operand layout of conv1d_tc.cu (element (row r, granule g) at (g * rows_pad + r) * 16), so
//   * the A stage of a tile = KBG contiguous runs of `rows x 16 B`  -> KBG bulk copies issued by ONE thread, as many stages
//     in flight as shared memory holds;
//   * tap j of a dilated convolution is still the same staged tile with the descriptor start advanced by j*dil rows;
//   * an accumulator register pair is two adjacent channels of one row: one 8-byte (fp32) or 4-byte (bf16) store, and the four
//     lanes of a quad together with the eight rows of a warp cover whole 128-byte granule runs.
// What still has to touch the operand between the copy and the MMA -- LeakyReLU of the input, zeroing of rows outside
// [0, len) (the convolution's zero padding and the batch-invariant contract), round-to-nearest tf32 and the hi/lo split of
// the 3xTF32 fp32 emulation -- is an IN-PLACE pass over the staged tile by four "transform" warps.
// HBM therefore holds plain activation values (fp32, or bf16 in the bf16 mode): residuals stay exact, one copy per tensor.
//
// The roles, their mbarrier ring and their code (x loader, transform warps, weight loader, the consumers' per-tap wgmma chain and
// one-behind release) are gp_pipeline.cuh, shared with resblock_gp.cu; this kernel adds the tile order and the epilogue (consumer
// warps: rows [64 w, 64 w + 64) of every 128-row accumulator, fp32 accumulators in registers).  Persistent CTAs, static
// round-robin tile order.
//
// out[b, m*rate + n / CoutR, n % CoutR] = epi( bias[n] + sum_j sum_ci w[j][ci][n] * act_in(x[b, m + (j-(K-1)/2)*dil, ci]) )
// rate > 1 is the polyphase form of ConvTranspose1d (packing.polyphase_pack): the GEMM's N = rate * CoutR columns are the
// `rate` output phases of each input row.  Replaces hifigan/models.py:50-57 (ResBlock1 convs), :116 (conv_pre), :118-119 (ups).
#include "ev_common.cuh"
#include "gp_pipeline.cuh"

namespace ev {
namespace gp {

using namespace gpl;

constexpr int MAX_A = 8;                     // x stages

struct GPlan {
  int BN, mt, kbg, planes;
  int rows_pad;
  int a_plane_bytes, b_plane_bytes, a_stage_bytes, b_stage_bytes;
  int a_stages, b_stages;
  int acc_cols;        // MT * BN <= 2 * ACC_REGS
  int tiles_m, tiles_n, total_tiles;
  int smem_total;
};

// span = (K-1)*dil of the widest member and kmin = the fewest taps of a grouped launch (ng convolutions); -1 / 0: p's own
__host__ __device__ inline bool make_gplan(const GpConvParams& p, int mode, int BN, int mt, int kbg, GPlan* o, int span = -1, int kmin = 0, int ng = 1) {
  if (span < 0) span = (p.K - 1) * p.dil;
  if (kmin <= 0) kmin = p.K;
  GPlan q;
  q.planes = mode == 1 ? 2 : 1;          // A planes in shared memory (mode 3 keeps hi / lo interleaved in ONE plane, in place)
  const int b_planes = (mode == 1 || mode == 3) ? 2 : 1;
  const int cpg = mode == 2 ? 8 : 4;     // channels per 16-byte granule of the ACTIVATIONS
  const int wcpg = mode >= 2 ? 8 : 4;    // channels per 16-byte granule of the WEIGHTS (bf16 operands: 8)
  q.kbg = kbg; q.mt = mt; q.BN = BN;
  if (mt * BN > 2 * ACC_REGS) return false;
  q.acc_cols = mt * BN;
  const int rows = BM * mt + span;
  q.rows_pad = (rows + 7) / 8 * 8;
  q.a_plane_bytes = kbg * q.rows_pad * 16;
  q.b_plane_bytes = (kbg * cpg / wcpg) * BN * 16;
  q.a_stage_bytes = q.planes * q.a_plane_bytes;
  q.b_stage_bytes = b_planes * q.b_plane_bytes;
  const int budget = 227 * 1024 - SMEM_HEAD;
  const int n_cb = (p.Cin + cpg * kbg - 1) / (cpg * kbg);
  const int b_max = n_cb * kmin < MAX_B ? n_cb * kmin : MAX_B;
  if (!grow_stages(q.a_stage_bytes, q.b_stage_bytes, budget, MAX_A, b_max, &q.a_stages, &q.b_stages)) return false;
  q.tiles_m = (p.L + BM * mt - 1) / (BM * mt);
  q.tiles_n = (p.Cout + BN - 1) / BN;
  q.total_tiles = ng * p.B * q.tiles_m * q.tiles_n;
  q.smem_total = SMEM_HEAD + q.a_stages * q.a_stage_bytes + q.b_stages * q.b_stage_bytes;
  *o = q;
  return true;
}

// MODE 0: one tf32 MMA per K step; 1: 3xTF32 fp32 emulation (hi/lo planes, three MMAs per K step); 2: bf16 operands,
// bf16 activations in HBM (8 channels per granule); 3: "bf16x3": fp32 activations in HBM, every operand split
// into bf16 hi + lo (16 significant bits), three bf16 MMAs per K = 16 step -- an fp32-class result (~1e-5 relative) at
// half the tensor-core and shared-memory cost of 3xTF32.  Accumulation is fp32 in every mode.  BN = pl.BN, the N tile.
template <int MODE, int MT, int KBG, int BN>
__global__ void __launch_bounds__(THREADS, 1) conv1d_gp_kernel(const __grid_constant__ GpConvParams p, const __grid_constant__ GPlan pl,
                                                               const __grid_constant__ GpGroups gs) {
  constexpr bool BF16 = (MODE == 2);       // bf16 activations in HBM, bf16 operands
  constexpr bool X3B = (MODE == 3);        // fp32 activations in HBM, operands split into bf16 hi + lo: three bf16 MMAs per K=16 step
  constexpr bool OP16 = BF16 || X3B;       // the MMA operands are bf16
  constexpr int CPG = BF16 ? 8 : 4;        // channels per 16-byte granule of the activations (HBM and the staged tile)
  constexpr int WCPG = OP16 ? 8 : 4;       // channels per 16-byte granule of the weights
  constexpr int KB = CPG * KBG;
  constexpr int NA = ACC_REGS / MT;
  constexpr int NK8 = KB / (2 * WCPG);     // MMA K steps of a full channel block
  static_assert(!X3B || KBG % 4 == 0, "bf16x3 consumes four fp32 granules (16 channels) per MMA K step");
  static_assert(MT * BN <= 2 * ACC_REGS, "accumulators of the tile exceed the register budget");
  extern __shared__ __align__(128) uint8_t smem_raw[];
  const int tid = threadIdx.x;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);   // provably warp-uniform: ptxas serialises every wgmma on a path it cannot prove uniform
  const int lane = tid & 31;

  uint8_t* a_tiles = smem_raw + SMEM_HEAD;
  uint8_t* b_tiles = a_tiles + pl.a_stages * pl.a_stage_bytes;
  const Ring<MAX_A> ring{smem_u32(smem_raw)};
  if (tid == 0) ring.init(pl.a_stages, pl.b_stages);
  __syncthreads();

  // Programmatic dependent launch: harmless without the launch attribute.  With it, the next kernel in the stream may start
  // its set-up (barriers, first weight stages) while this grid's tail is still running; everything that touches
  // activations executes griddepcontrol.wait first (returns once the preceding grid has completed and flushed).
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  const int n_cb = (p.Cin + KB - 1) / KB;
  const int tiles_per_b = pl.tiles_m * pl.tiles_n;
  const int tiles_per_g = p.B * tiles_per_b;  // a launch may carry up to three convolutions of one shape (different taps, dilations,
                                              // weights and tensors): tile -> (convolution, item, row tile, column tile)

  auto decode = [&](int tile, int& gi, int& b, int& t0, int& n0, int& len) {
    gi = tile / tiles_per_g;
    tile -= gi * tiles_per_g;
    b = tile / tiles_per_b;
    const int r = tile - b * tiles_per_b;
    const int tm = r / pl.tiles_n, tn = r - tm * pl.tiles_n;
    t0 = tm * (BM * MT);
    n0 = tn * BN;
    len = p.lens ? min(p.L, p.lens[b] * p.lens_mul) : p.L;
  };

  if (warp < NCW) {
    // ============================ consumers: MMA issue + epilogue ==============================================
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const int wg = warp >> 2, wl = warp & 3;
    const int coutR = p.Cout / p.rate;
    const int gout = coutR / CPG;              // output granule planes per item
    const size_t Lout = (size_t)p.L * p.rate;
    const int accm = p.acc;
    const uint32_t a_lbo = (uint32_t)pl.rows_pad * 16u, b_lbo = (uint32_t)BN * 16u;
    // bf16x3: the two K granules of one MMA are two slots apart (hi in the even slots, lo in the odd ones), one K step = 4 slots
    const uint64_t a_desc0 = make_desc(0u, X3B ? 2u * a_lbo : a_lbo, 128u), b_desc0 = make_desc(0u, b_lbo, 128u);
    const uint32_t a_k8 = (X3B ? 4u : 2u) * a_lbo;   // bytes per K step
    const uint32_t a_lo_off = X3B ? a_lbo : (uint32_t)pl.a_plane_bytes;
    float acc[MT][NA];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int i = 0; i < NA; ++i) acc[mt][i] = 0.f;
    int a_cnt = 0, b_cnt = 0;
    for (int tile = blockIdx.x; tile < pl.total_tiles; tile += gridDim.x) {
      int gi, b, t0, n0, len;
      decode(tile, gi, b, t0, n0, len);
      if (t0 >= len) continue;                 // padding tile: no MMA work is issued, nothing is stored (rows >= len are undefined)
      const GpGroup& G = gs.g[gi];
      const int K = G.K;
      const uint32_t a_tap = (uint32_t)G.dil * 16u;          // bytes per tap shift
      OneBehind<MAX_A> rel{ring, lane};
      for (int cb = 0; cb < n_cb; ++cb, ++a_cnt) {
        const int sa = a_cnt % pl.a_stages;
        const int nk8 = min(KB, p.Cin - cb * KB) / (2 * WCPG);  // MMA K steps: two 16-byte operand granules each
        mbar_wait(ring.a_ready(sa), (a_cnt / pl.a_stages) & 1);
        const uint64_t a_hi0 = desc_advance(a_desc0, smem_u32(a_tiles + sa * pl.a_stage_bytes) + (uint32_t)(wg * 64) * 16u);
        for (int j = 0; j < K; ++j, ++b_cnt) {
          const int sb = b_cnt % pl.b_stages;
          mbar_wait(ring.b_full(sb), (b_cnt / pl.b_stages) & 1);
          const uint64_t b_hi0 = desc_advance(b_desc0, smem_u32(b_tiles + sb * pl.b_stage_bytes));
          const uint64_t a_j = desc_advance(a_hi0, (uint32_t)j * a_tap);
          // the wait inside each branch: joined before it, the paths would leave the tap as two commit groups (tc::tap_chain)
          if (nk8 == NK8) {
            tap_chain<MODE, BN, NK8>(acc, a_j, a_k8, a_lo_off, b_hi0, (uint32_t)pl.b_plane_bytes, cb | j);
            wgmma_wait<1>();        // the previous tap's chain has completed: its stages may be refilled
          } else {
            tap_chain_short<MODE, BN>(acc, a_j, a_k8, a_lo_off, b_hi0, (uint32_t)pl.b_plane_bytes, cb | j, nk8);
            wgmma_wait<1>();
          }
          rel.step(sb, j == K - 1 ? sa : -1);
        }
      }

      // epilogue: register pair i, i+1 = channels n, n+1 of one row (one granule).  Pair i = 4 q + 2 h of accumulator mt lies in
      // column group q (8 columns: the same bias for every mt and h) and row row0 + mt * BM + 8 h.  The pairs are walked in chunks
      // of EQ column groups, 4 pairs (8 at MT = 4: one column group; larger chunks spill at MT = 1, 2).  A chunk issues all its
      // loads (bias, residual, `out` in the accumulate modes) before its arithmetic and stores, and the first chunk's loads run
      // under the tile's last MMAs.  In place (out == res, or out read by the accumulate modes) this stays correct: every output
      // element is loaded and stored by exactly one thread, once per launch, and that thread loads it before it stores it.
      constexpr int EQ = MT == 1 ? 2 : 1;
      const bool has_res = G.res != nullptr;
      const int row0 = t0 + wg * 64 + frag_row(0, lane, wl);   // GEMM rows = input-resolution time steps
      float2 ebias[EQ];
      pair_t<BF16> eres[EQ][MT][2], eout[EQ][MT][2];
      auto column = [&](int q, int& n) {
        n = n0 + frag_col(4 * q, lane);
        const int phase = n / coutR, co = n - phase * coutR;
        return (((size_t)b * gout + co / CPG) * Lout + phase) * CPG + (co % CPG);     // element index at row 0
      };
      auto epi_load = [&](int ch) {         // chunk ch = column groups [ch * EQ, ch * EQ + EQ)
#pragma unroll
        for (int q = 0; q < EQ; ++q) {
          int n;
          const size_t ec = column(ch * EQ + q, n);
          if (n - n0 >= BN) continue;
          if (G.bias) ebias[q] = __ldg(reinterpret_cast<const float2*>(G.bias + n));
#pragma unroll
          for (int mt = 0; mt < MT; ++mt)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int row = row0 + mt * BM + 8 * h;
              if (row >= len) continue;
              const size_t e = ec + (size_t)row * p.rate * CPG;
              if (has_res) eres[q][mt][h] = load_pair<BF16>(G.res, e);
              if (accm != EV_ACC_STORE) eout[q][mt][h] = load_pair<BF16>(G.out, e);
            }
        }
      };
      auto epi_store = [&](int ch) {
#pragma unroll
        for (int q = 0; q < EQ; ++q) {
          int n;
          const size_t ec = column(ch * EQ + q, n);
          if (n - n0 >= BN) continue;
#pragma unroll
          for (int mt = 0; mt < MT; ++mt)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int row = row0 + mt * BM + 8 * h;
              if (row >= len) continue;
              const int i = 4 * (ch * EQ + q) + 2 * h;
              float v0 = acc[mt][i], v1 = acc[mt][i + 1];
              if (G.bias) { v0 += ebias[q].x; v1 += ebias[q].y; }
              if (has_res) {
                const float2 r = unpack_pair(eres[q][mt][h]);
                v0 += r.x; v1 += r.y;
              }
              if (accm != EV_ACC_STORE) {
                const float2 o = unpack_pair(eout[q][mt][h]);
                v0 += o.x; v1 += o.y;
                if (accm == EV_ACC_ADD_DIV) { v0 /= p.div; v1 /= p.div; }
              }
              store_pair<BF16>(G.out, ec + (size_t)row * p.rate * CPG, v0, v1);
            }
        }
      };
      epi_load(0);
      wgmma_wait<0>();
      rel.drain();
#pragma unroll
      for (int ch = 0; ch < NA / 4 / EQ; ++ch) {
        if (ch > 0) epi_load(ch);
        epi_store(ch);
      }
    }
  } else if (warp < W_ALOAD) {
    // ============================ transform warps ========================================================================
    const int xt = (warp - W_XFORM) * 32 + lane;      // 0..127
    int a_cnt = 0;
    for (int tile = blockIdx.x; tile < pl.total_tiles; tile += gridDim.x) {
      int gi, b, t0, n0, len;
      decode(tile, gi, b, t0, n0, len);
      if (t0 >= len) continue;
      const int span = (gs.g[gi].K - 1) * gs.g[gi].dil;
      transform_tile<MODE, KBG>(ring, a_cnt, pl.a_stages, a_tiles, pl.a_stage_bytes, pl.a_plane_bytes, pl.rows_pad, p.Cin, t0 - span / 2,
                                           BM * MT + span, len, p.in_act == EV_ACT_LRELU, p.in_slope, xt);
    }
  } else if (warp == W_ALOAD) {
    // ============================ x loader ===============================================================================
    if (lane == 0) {
      asm volatile("griddepcontrol.wait;" ::: "memory");
      int a_cnt = 0;
      for (int tile = blockIdx.x; tile < pl.total_tiles; tile += gridDim.x) {
        int gi, b, t0, n0, len;
        decode(tile, gi, b, t0, n0, len);
        if (t0 >= len) continue;
        const int span = (gs.g[gi].K - 1) * gs.g[gi].dil;
        load_x_tile<CPG, KBG>(ring, a_cnt, pl.a_stages, a_tiles, pl.a_stage_bytes, pl.rows_pad, gs.g[gi].x, b, p.Cin, p.L, t0 - span / 2,
                              BM * MT + span, len);
      }
    }
    __syncwarp();
  } else {
    // ============================ weight loader (weights are constants: no dependency wait) ========================
    if (lane == 0) {
      const int bnp = p.Cout < 128 ? p.Cout : 128;                   // the packing tile
      const int win = p.Cin / WCPG;
      int b_cnt = 0;
      for (int tile = blockIdx.x; tile < pl.total_tiles; tile += gridDim.x) {
        int gi, b, t0, n0, len;
        decode(tile, gi, b, t0, n0, len);
        if (t0 >= len) continue;
        const int K = gs.g[gi].K;
        const size_t tile_stride = (size_t)K * win * bnp * 4;       // 4-byte words per packed N tile
        const float* wt = gs.g[gi].w + (size_t)(n0 / bnp) * tile_stride + (size_t)(n0 % bnp) * 4;
        load_w_tile<MODE, KBG, BN>(ring, b_cnt, pl.b_stages, b_tiles, pl.b_stage_bytes, pl.b_plane_bytes, wt, K, p.Cin, p.Cout, bnp);
      }
    }
    __syncwarp();
  }
}

// ---- layout conversion at the vocoder's boundary ---------------------------------------------------------------------
// in[b*sb + t*st + c*sc] fp32 (time-major (B,F,C): st = C, sc = 1; channels-first (B,C,F): st = 1, sc = F)  ->  GP.
template <bool BF16>
__global__ void __launch_bounds__(256) to_gp_kernel(const float* __restrict__ in, long long sb, long long st_, long long sc, void* __restrict__ out,
                                                    int B, int L, int C) {
  asm volatile("griddepcontrol.launch_dependents;\n\tgriddepcontrol.wait;" ::: "memory");
  constexpr int CPG = BF16 ? 8 : 4;
  const int G = C / CPG;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;      // (b, g, t), t fastest
  if (i >= (size_t)B * G * L) return;
  const int t = (int)(i % L);
  const int g = (int)((i / L) % G);
  const int b = (int)(i / ((size_t)L * G));
  const float* src = in + (size_t)b * sb + (size_t)t * st_ + (size_t)(g * CPG) * sc;
  float v[CPG];
#pragma unroll
  for (int e = 0; e < CPG; ++e) v[e] = src[(size_t)e * sc];
  uint4 o;
  if (BF16) {
    o.x = pack_bf16(v[0], v[1]); o.y = pack_bf16(v[2], v[3]); o.z = pack_bf16(v[CPG - 4], v[CPG - 3]); o.w = pack_bf16(v[CPG - 2], v[CPG - 1]);
  } else {
    o.x = __float_as_uint(v[0]); o.y = __float_as_uint(v[1]); o.z = __float_as_uint(v[2]); o.w = __float_as_uint(v[3]);
  }
  reinterpret_cast<uint4*>(out)[i] = o;
}

// out = ((b + a) [+ c]) / div over whole fp32 granule-planar tensors: the `xs += ...; x = xs / n` of a HiFi-GAN stage
// (hifigan/models.py:120-126) when the three ResBlocks' last layers ran as one grouped launch into their own tensors.  Same additions
// in the same order as the accumulate modes of the epilogue (a stored, then b + a, then c + that, then / div): identical bits.
template <int N>
__global__ void __launch_bounds__(256) gp_sum_div_kernel(const float4* __restrict__ a, const float4* __restrict__ b, const float4* __restrict__ c,
                                                         float4* __restrict__ out, size_t n4, float div) {
  asm volatile("griddepcontrol.launch_dependents;\n\tgriddepcontrol.wait;" ::: "memory");
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const float4 va = a[i], vb = b[i];
  float4 t = make_float4(vb.x + va.x, vb.y + va.y, vb.z + va.z, vb.w + va.w);
  if (N == 3) {
    const float4 vc = c[i];
    t = make_float4(vc.x + t.x, vc.y + t.y, vc.z + t.z, vc.w + t.w);
  }
  out[i] = make_float4(t.x / div, t.y / div, t.z / div, t.w / div);
}

// wav[b,t] = tanh( bias + sum_j sum_c w[j][c] * lrelu(x[b, t+j-(K-1)/2, c]) ) on a GP input (hifigan/models.py:127-129:
// F.leaky_relu default slope 0.01, Conv1d(C,1,7,pad 3), tanh).  HBM-bound: each CTA stages (256 + K - 1) rows once, already
// activated; rows >= len read as zero padding and are written as zeros.  Same summation order as conv_post_kernel.  Generic shapes;
// HiFi-GAN's own (K = 7, C <= 48) run conv_post_gp4_kernel below.
constexpr int GPP_BT = 256;
template <bool BF16>
__global__ void __launch_bounds__(GPP_BT) conv_post_gp_kernel(const void* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                                              const int32_t* __restrict__ lens, int lens_mul, int L, int C, int K, float slope,
                                                              float* __restrict__ wav) {
  asm volatile("griddepcontrol.launch_dependents;\n\tgriddepcontrol.wait;" ::: "memory");
  constexpr int CPG = BF16 ? 8 : 4;
  extern __shared__ __align__(16) float gpp_smem[];
  const int rows = GPP_BT + K - 1;
  float* xs = gpp_smem;                 // [C][rows] channel-major: conflict-free for consecutive rows
  float* ws = gpp_smem + (size_t)C * rows;   // [K][C]
  const int b = blockIdx.y, t0 = blockIdx.x * GPP_BT;
  const int len = lens ? min(L, lens[b] * lens_mul) : L;
  const int halo = (K - 1) / 2;
  const int G = C / CPG;
  const uint4* xb = reinterpret_cast<const uint4*>(x) + (size_t)b * G * L;
  for (int i = threadIdx.x; i < G * rows; i += GPP_BT) {
    const int g = i / rows, r = i - g * rows;
    const int row = t0 - halo + r;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (row >= 0 && row < len) v = xb[(size_t)g * L + row];
    float f[CPG];
    if (BF16) {
      const uint32_t w4[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) { f[2 * e] = __uint_as_float(w4[e] << 16); f[2 * e + 1] = __uint_as_float(w4[e] & 0xffff0000u); }
    } else {
      f[0] = __uint_as_float(v.x); f[1] = __uint_as_float(v.y); f[2] = __uint_as_float(v.z); f[3] = __uint_as_float(v.w);
    }
#pragma unroll
    for (int e = 0; e < CPG; ++e) xs[(size_t)(g * CPG + e) * rows + r] = lrelu_f(f[e], slope);
  }
  for (int i = threadIdx.x; i < K * C; i += GPP_BT) ws[i] = w[i];
  __syncthreads();
  const int t = t0 + threadIdx.x;
  if (t >= L) return;
  float acc = 0.f;
  for (int c = 0; c < C; ++c) {       // channel-major reduction order (all three conv_post kernels share it)
    const float* xr = xs + (size_t)c * rows + threadIdx.x;
    for (int j = 0; j < K; ++j) acc = fmaf(xr[j], ws[j * C + c], acc);
  }
  wav[(size_t)b * L + t] = t < len ? tanhf(acc + bias[0]) : 0.f;
}

// The same operator for the shapes HiFi-GAN has (K = 7, C = 32): 128 threads x 4 consecutive outputs.  Per channel a thread reads its
// 4 + K - 1 inputs (three LDS.128) and the K taps (two broadcast LDS.128) for 4 K FMAs -- the one-output kernel above spends two
// shared-memory loads per FMA and measured 14x over its HBM time.  Tiles past the item's length only store zeros.  Same sums, same order.
constexpr int GP4_T = 128, GP4_O = 4, GP4_ROWS = GP4_T * GP4_O;
template <bool BF16, int K>
__global__ void __launch_bounds__(GP4_T) conv_post_gp4_kernel(const void* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                                              const int32_t* __restrict__ lens, int lens_mul, int L, int C, float slope,
                                                              float* __restrict__ wav) {
  asm volatile("griddepcontrol.launch_dependents;\n\tgriddepcontrol.wait;" ::: "memory");
  constexpr int CPG = BF16 ? 8 : 4;
  constexpr int HALO = (K - 1) / 2;
  constexpr int NW = (GP4_O + K - 1 + 3) / 4;          // float4 loads per input window
  constexpr int RS = GP4_ROWS + (NW - 1) * 4;          // staged rows per channel (the last thread's window ends at 4*127 + 4*NW)
  constexpr int KP = (K + 3) / 4 * 4;
  extern __shared__ __align__(16) float gpp_smem[];
  float* xs = gpp_smem;                       // [C][RS]
  float* ws = gpp_smem + (size_t)C * RS;      // [C][KP]
  const int b = blockIdx.y, t0 = blockIdx.x * GP4_ROWS;
  const int len = lens ? min(L, lens[b] * lens_mul) : L;
  const int t = t0 + GP4_O * threadIdx.x;
  float* out = wav + (size_t)b * L + t;
  const bool vec = (L & 3) == 0 && t + GP4_O <= L;
  if (t0 >= len) {                            // padding tile
    if (vec) *reinterpret_cast<float4*>(out) = make_float4(0.f, 0.f, 0.f, 0.f);
    else for (int o = 0; o < GP4_O; ++o) if (t + o < L) out[o] = 0.f;
    return;
  }
  const int G = C / CPG;
  const uint4* xb = reinterpret_cast<const uint4*>(x) + (size_t)b * G * L;
#pragma unroll 4
  for (int i = threadIdx.x; i < G * RS; i += GP4_T) {
    const int g = i / RS, r = i - g * RS;
    const int row = t0 - HALO + r;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (row >= 0 && row < len) v = __ldg(xb + (size_t)g * L + row);
    float f[CPG];
    if (BF16) {
      const uint32_t w4[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) { f[2 * e] = __uint_as_float(w4[e] << 16); f[2 * e + 1] = __uint_as_float(w4[e] & 0xffff0000u); }
    } else {
      f[0] = __uint_as_float(v.x); f[1] = __uint_as_float(v.y); f[2] = __uint_as_float(v.z); f[3] = __uint_as_float(v.w);
    }
#pragma unroll
    for (int e = 0; e < CPG; ++e) xs[(size_t)(g * CPG + e) * RS + r] = lrelu_f(f[e], slope);
  }
  for (int i = threadIdx.x; i < C * KP; i += GP4_T) {
    const int c = i / KP, j = i - c * KP;
    ws[i] = j < K ? w[j * C + c] : 0.f;
  }
  __syncthreads();
  float acc[GP4_O];
#pragma unroll
  for (int o = 0; o < GP4_O; ++o) acc[o] = 0.f;
  for (int c = 0; c < C; ++c) {
    float xw[NW * 4], wv[KP];
    const float4* xr = reinterpret_cast<const float4*>(xs + (size_t)c * RS + GP4_O * threadIdx.x);
    const float4* wr = reinterpret_cast<const float4*>(ws + c * KP);
#pragma unroll
    for (int q = 0; q < NW; ++q) { const float4 v = xr[q]; xw[4 * q] = v.x; xw[4 * q + 1] = v.y; xw[4 * q + 2] = v.z; xw[4 * q + 3] = v.w; }
#pragma unroll
    for (int q = 0; q < KP / 4; ++q) { const float4 v = wr[q]; wv[4 * q] = v.x; wv[4 * q + 1] = v.y; wv[4 * q + 2] = v.z; wv[4 * q + 3] = v.w; }
#pragma unroll
    for (int j = 0; j < K; ++j)
#pragma unroll
      for (int o = 0; o < GP4_O; ++o) acc[o] = fmaf(xw[o + j], wv[j], acc[o]);
  }
  const float b0 = bias[0];
  float r[GP4_O];
#pragma unroll
  for (int o = 0; o < GP4_O; ++o) r[o] = t + o < len ? tanhf(acc[o] + b0) : 0.f;
  if (vec) *reinterpret_cast<float4*>(out) = make_float4(r[0], r[1], r[2], r[3]);
  else for (int o = 0; o < GP4_O; ++o) if (t + o < L) out[o] = r[o];
}

}  // namespace gp

static int validate_gp(const GpConvParams& p, int mode) {
  EV_CHECK_ARG(p.B > 0 && p.L > 0, "conv1d_gp: bad problem B=%d L=%d", p.B, p.L);
  EV_CHECK_ARG(mode >= 0 && mode <= 3, "conv1d_gp: mode %d", mode);
  EV_CHECK_ARG(p.Cin % (mode >= 2 ? 16 : 8) == 0, "conv1d_gp: Cin=%d must be a multiple of %d", p.Cin, mode >= 2 ? 16 : 8);
  EV_CHECK_ARG(p.Cout % 32 == 0 && (p.Cout <= 128 || p.Cout % 128 == 0), "conv1d_gp: Cout=%d must be a multiple of 32, and of 128 above 128", p.Cout);
  EV_CHECK_ARG(p.rate >= 1 && p.Cout % p.rate == 0 && (p.Cout / p.rate) % 32 == 0, "conv1d_gp: rate=%d does not split Cout=%d into multiples of 32", p.rate, p.Cout);
  EV_CHECK_ARG(p.K >= 1 && (p.K & 1) && p.dil >= 1, "conv1d_gp: K=%d must be odd, dil=%d >= 1", p.K, p.dil);
  EV_CHECK_ARG(p.in_act == EV_ACT_NONE || p.in_act == EV_ACT_LRELU, "conv1d_gp: unsupported input activation");
  EV_CHECK_ARG(p.rate == 1 || (!p.res && p.acc == EV_ACC_STORE), "conv1d_gp: residual / accumulate need rate == 1");
  EV_CHECK_ARG((long long)p.L * p.rate < (1ll << 31), "conv1d_gp: output too long");
  return EV_OK;
}

// K granules per stage decide the order of the (channel block, tap, k-step) reduction, so they are a function of the layer
// shape alone (never of batch or length): 8 outside the 3xTF32 mode if a one-accumulator tile fits with them, else 4.
int gp_shape_kbg(const GpConvParams& p, int mode) {
  gp::GPlan pl;
  const int bn_max = p.Cout <= 128 ? p.Cout : 128;
  return (mode != 1 && gp::make_gplan(p, mode, bn_max, 1, 8, &pl)) ? 8 : 4;
}

// Tile shape: none of these choices changes the order in which any output element's K reduction is summed, so results are
// bitwise independent of batch size / sequence length (batch-invariant contract) and the shape can be picked by a cost model.
// Per tile of MT x 128 rows and BN columns, three engines run concurrently and the slowest one sets the pace:
//   tensor core + its shared-memory operand reads:  MT * m * max(BN/2, 32 + BN/4) cycles per (tap, 8 channels)   (m = 3 MMAs in 3xTF32; bf16: 16 channels)
//   weight stream L2 -> shared memory:              planes * 32 B * BN per (tap, 8 channels) at ~42 B/cycle/SM (6.3 KB/cycle chip-wide)
//   activations HBM -> shared memory -> HBM:        MT * 128 rows * (Cin + 2 Cout) * esize at ~23 B/cycle/SM
// plus a fixed pipeline fill / drain per tile; the launch takes ceil(tiles / SMs) such tile times.  More accumulators per tile
// (MT) amortise the weight stream and the halo rows, a narrower N tile fills idle SMs (HiFi-GAN stage 1 at batch 1).
// A grouped launch (ng convolutions of one shape, ksum = the sum of their taps, span / kmin as in make_gplan) is planned like one
// convolution with the mean number of taps and ng times the tiles; kbg must be the members' own (checked by the caller).
static int plan_gp(const GpConvParams& p, int mode, gp::GPlan* out, int ng = 1, int ksum = 0, int span = -1, int kmin = 0, int kbg_forced = 0,
                   const int* gK = nullptr) {
  EV_TRY(validate_gp(p, mode));
  const int nsm = sm_count();
  const int kbg = kbg_forced ? kbg_forced : gp_shape_kbg(p, mode);
  if (ksum <= 0) ksum = p.K;
  if (span < 0) span = (p.K - 1) * p.dil;
  const double kc8 = (double)ksum / ng * p.Cin / 8.0;
  const double n_mma = ((mode == 1 || mode == 3) ? 3.0 : 1.0) * (mode >= 2 ? 0.5 : 1.0) * kc8;     // MMA instructions per accumulator and tile
  const double w_per_n = ((mode == 1 || mode == 3) ? 2.0 : 1.0) * (mode >= 2 ? 16.0 : 32.0) / 42.0;
  const double esize = mode == 2 ? 2.0 : 4.0;
  double best = 1e300;
  bool found = false;
  gp::GPlan best_pl;
  const int bn_max = p.Cout <= 128 ? p.Cout : 128;
  // N tile = the weight packing tile (min(C_out, 128)): ONE bulk copy per weight stage and plane.  Narrower tiles would fill idle SMs
  // at batch 1 (stage 1: 68 tiles) but need one 1-KB copy per granule issued by a single thread -- measured 1.5x slower.
  for (int BN = bn_max; BN >= bn_max; BN /= 2) {
    if (p.Cout % BN || BN % 32) continue;
    for (int mt = 4; mt >= 1; mt >>= 1) {
      gp::GPlan pl;
      if (!gp::make_gplan(p, mode, BN, mt, kbg, &pl, span, kmin, ng)) continue;
      // per MMA instruction: BN/2 tensor cycles, but both operands come from shared memory (128 B/cycle): (128 + BN) rows x 32 B
      // = 32 + BN/4 cycles -- the binding term below BN = 128 (a 64-wide tile costs 1.5x per FLOP, a 32-wide one 2.5x)
      double c_mma = BN / 2.0;
      if (32.0 + BN / 4.0 > c_mma) c_mma = 32.0 + BN / 4.0;
      const double t_mma = mt * n_mma * c_mma;
      const double t_w = w_per_n * BN * kc8;
      const double t_hbm = (double)mt * tc::BM * ((double)p.Cin * (mt * tc::BM + span) / (mt * tc::BM) + 2.0 * BN) * esize / 23.0;
      double t = t_mma > t_w ? t_mma : t_w;
      if (t_hbm > t) t = t_hbm;
      double cost;
      if (ng > 1 && gK) {
        // grouped launch: the members' tiles cost in proportion to their taps and are dealt round-robin in member order (heaviest
        // first); the launch takes as long as its busiest CTA
        const int tg = pl.total_tiles / ng;
        const int ncta = pl.total_tiles < nsm ? pl.total_tiles : nsm;
        cost = 0.0;
        for (int c = 0; c < ncta; ++c) {
          double sum = 0.0;
          for (int i = c; i < pl.total_tiles; i += nsm) sum += t * gK[i / tg] * ng / (double)ksum + 3000.0;
          if (sum > cost) cost = sum;
        }
      } else {
        const double waves = (double)((pl.total_tiles + nsm - 1) / nsm);
        cost = waves * (t + 3000.0);
      }
      if (cost < best * 0.97) { best = cost; best_pl = pl; found = true; }     // widest N / most accumulators first; 3 % hysteresis
    }
  }
  if (!found) { set_error("conv1d_gp: tile does not fit in shared memory / accumulator registers (K=%d dil=%d Cout=%d)", p.K, p.dil, p.Cout); return EV_EINVAL; }
  *out = best_pl;
  return EV_OK;
}

int gp_solo_tiles(const GpConvParams& p, int mode) {
  gp::GPlan pl;
  return plan_gp(p, mode, &pl) == EV_OK ? pl.total_tiles : 0;
}

int debug_gp_plan(const GpConvParams& p, int mode, int* v) {
  gp::GPlan pl;
  const int rc = plan_gp(p, mode, &pl);
  if (rc != EV_OK) return rc;
  v[0] = pl.BN; v[1] = pl.mt; v[2] = pl.kbg; v[3] = pl.a_stages; v[4] = pl.b_stages; v[5] = gp::NTW;
  v[6] = pl.planes; v[7] = pl.acc_cols; v[8] = pl.smem_total; v[9] = pl.total_tiles; v[10] = pl.rows_pad;
  return EV_OK;
}

// The instantiations: every (MODE, KBG) the shape rule gp_shape_kbg gives (KBG = 4 in 3xTF32) times every tile plan_gp can return,
// BN = min(C_out, 128) in {32, 64, 96, 128} (validate_gp) with MT * BN <= 128.
using GpKernel = void (*)(GpConvParams, gp::GPlan, GpGroups);
template <int MODE, int KBG>
static GpKernel gp_kernel_tile(int mt, int bn) {
  switch (bn) {
    case 128: return mt == 1 ? gp::conv1d_gp_kernel<MODE, 1, KBG, 128> : nullptr;
    case 96: return mt == 1 ? gp::conv1d_gp_kernel<MODE, 1, KBG, 96> : nullptr;
    case 64: return mt == 2 ? gp::conv1d_gp_kernel<MODE, 2, KBG, 64> : mt == 1 ? gp::conv1d_gp_kernel<MODE, 1, KBG, 64> : nullptr;
    case 32: return mt == 4 ? gp::conv1d_gp_kernel<MODE, 4, KBG, 32> : mt == 2 ? gp::conv1d_gp_kernel<MODE, 2, KBG, 32>
                  : mt == 1 ? gp::conv1d_gp_kernel<MODE, 1, KBG, 32> : nullptr;
    default: return nullptr;
  }
}
static GpKernel gp_kernel(int mode, int kbg, int mt, int bn) {
  if (mode == 1) return kbg == 4 ? gp_kernel_tile<1, 4>(mt, bn) : nullptr;
  if (mode == 3) return kbg == 8 ? gp_kernel_tile<3, 8>(mt, bn) : gp_kernel_tile<3, 4>(mt, bn);
  if (mode == 2) return kbg == 8 ? gp_kernel_tile<2, 8>(mt, bn) : gp_kernel_tile<2, 4>(mt, bn);
  return kbg == 8 ? gp_kernel_tile<0, 8>(mt, bn) : gp_kernel_tile<0, 4>(mt, bn);
}

static int dispatch_gp(const GpConvParams& p, const gp::GPlan& pl, const GpGroups& gs, int mode, cudaStream_t st) {
  static std::atomic<uint64_t> attr_devs{0};
  if (first_use_on_device(attr_devs)) preload_conv1d_gp();
  const GpKernel k = gp_kernel(mode, pl.kbg, pl.mt, pl.BN);
  EV_CHECK_ARG(k, "conv1d_gp: no kernel for mode %d, KBG %d, MT %d, BN %d", mode, pl.kbg, pl.mt, pl.BN);
  const int nsm = sm_count();
  const int grid = pl.total_tiles < nsm ? pl.total_tiles : nsm;
  return launch("conv1d_gp_kernel", k, (unsigned)grid, gpl::THREADS, pl.smem_total, st, p, pl, gs);
}

int launch_conv1d_gp(const GpConvParams& p, int mode, cudaStream_t st) {
  gp::GPlan pl;
  EV_TRY(plan_gp(p, mode, &pl));
  GpGroups gs{};
  gs.ng = 1;
  gs.g[0] = GpGroup{p.x, p.w, p.bias, p.res, p.out, p.K, p.dil};
  return dispatch_gp(p, pl, gs, mode, st);
}

// ---- grouped launch ------------------------------------------------------------------------------------------------------
static bool group_shapes_match(const GpConvParams* ps, int n, int mode, int* kbg) {
  if (n < 1 || n > 3) return false;
  const GpConvParams& a = ps[0];
  int kb = 0;
  for (int i = 0; i < n; ++i) {
    const GpConvParams& q = ps[i];
    if (q.B != a.B || q.L != a.L || q.Cin != a.Cin || q.Cout != a.Cout || q.rate != 1 || q.lens != a.lens || q.lens_mul != a.lens_mul ||
        q.in_act != a.in_act || q.in_slope != a.in_slope || q.acc != EV_ACC_STORE || !q.x || !q.w || !q.out)
      return false;
    if (q.K < 1 || !(q.K & 1) || q.dil < 1) return false;
    for (int j = 0; j < i; ++j)
      if (ps[j].out == q.out) return false;                 // every member writes its own tensor
    const int k = gp_shape_kbg(q, mode);                    // the reduction order of each member must be its own launch's
    if (i == 0) kb = k;
    else if (k != kb) return false;
  }
  *kbg = kb;
  return true;
}
bool gp_group_supported(const GpConvParams* ps, int n, int mode) {
  int kbg = 0;
  if (mode < 0 || mode > 3 || !group_shapes_match(ps, n, mode, &kbg)) return false;
  return validate_gp(ps[0], mode) == EV_OK;
}
static int plan_group(const GpConvParams* ps, int n, int mode, GpGroups* gs_out, gp::GPlan* pl_out);
int debug_gp_group_plan(const GpConvParams* ps, int n, int mode, int* v) {
  GpGroups gs{};
  gp::GPlan pl;
  EV_TRY(plan_group(ps, n, mode, &gs, &pl));
  v[0] = pl.BN; v[1] = pl.mt; v[2] = pl.kbg; v[3] = pl.a_stages; v[4] = pl.b_stages; v[5] = gp::NTW;
  v[6] = pl.planes; v[7] = pl.acc_cols; v[8] = pl.smem_total; v[9] = pl.total_tiles; v[10] = pl.rows_pad;
  return EV_OK;
}
int launch_conv1d_gp_group(const GpConvParams* ps, int n, int mode, cudaStream_t st) {
  GpGroups gs{};
  gp::GPlan pl;
  EV_TRY(plan_group(ps, n, mode, &gs, &pl));
  return dispatch_gp(ps[0], pl, gs, mode, st);
}
static int plan_group(const GpConvParams* ps, int n, int mode, GpGroups* gs_out, gp::GPlan* pl_out) {
  GpGroups& gs = *gs_out;
  gp::GPlan& pl = *pl_out;
  int kbg = 0;
  EV_CHECK_ARG(ps && group_shapes_match(ps, n, mode, &kbg), "conv1d_gp group: the %d convolutions do not share a launch shape", n);
  int order[3];
  gpl::heaviest_first(ps, n, order);
  gs = GpGroups{};
  gs.ng = n;
  int ksum = 0, span = 0, kmin = 1 << 30;
  for (int i = 0; i < n; ++i) {
    const GpConvParams& q = ps[order[i]];
    gs.g[i] = GpGroup{q.x, q.w, q.bias, q.res, q.out, q.K, q.dil};
    ksum += q.K;
    span = (q.K - 1) * q.dil > span ? (q.K - 1) * q.dil : span;
    kmin = q.K < kmin ? q.K : kmin;
  }
  int gK[3] = {0, 0, 0};
  for (int i = 0; i < n; ++i) gK[i] = gs.g[i].K;
  return plan_gp(ps[0], mode, &pl, n, ksum, span, kmin, kbg, gK);
}

// Load every instantiation's code now (CUDA loads kernels lazily, at their first launch: tens of milliseconds for a kernel of this
// size, which would otherwise hit whichever utterance first needs a new tile shape) and set the shared-memory attribute -- on
// exactly the instantiations dispatch_gp can launch.
void preload_conv1d_gp() {
  for (int mode = 0; mode < 4; ++mode)
    for (int kbg = 4; kbg <= 8; kbg += 4)
      for (int bn = 32; bn <= 128; bn += 32)
        for (int mt = 1; mt * bn <= 128; mt *= 2)
          if (const GpKernel k = gp_kernel(mode, kbg, mt, bn)) cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
  cudaFuncSetAttribute(gp::conv_post_gp_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
  cudaFuncSetAttribute(gp::conv_post_gp_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
  cudaFuncSetAttribute(gp::conv_post_gp4_kernel<false, 7>, cudaFuncAttributeMaxDynamicSharedMemorySize, 112 * 1024);
  cudaFuncSetAttribute(gp::conv_post_gp4_kernel<true, 7>, cudaFuncAttributeMaxDynamicSharedMemorySize, 112 * 1024);
  cudaFuncAttributes fa;
  cudaFuncGetAttributes(&fa, gp::to_gp_kernel<false>);
  cudaFuncGetAttributes(&fa, gp::to_gp_kernel<true>);
  cudaGetLastError();
}

int launch_to_gp(const float* in, long long sb, long long st_, long long sc, void* out, int B, int L, int C, int bf16, cudaStream_t st) {
  EV_CHECK_ARG(B > 0 && L > 0 && C % (bf16 ? 8 : 4) == 0, "to_gp: B=%d L=%d C=%d", B, L, C);
  const size_t n = (size_t)B * (C / (bf16 ? 8 : 4)) * L;
  const unsigned grid = (unsigned)((n + 255) / 256);
  return launch("to_gp_kernel", bf16 ? gp::to_gp_kernel<true> : gp::to_gp_kernel<false>, grid, 256, 0, st, in, sb, st_, sc, out, B, L, C);
}

int launch_gp_sum_div(const float* a, const float* b, const float* c, float* out, size_t n_floats, float div, cudaStream_t st) {
  EV_CHECK_ARG(a && b && out && n_floats % 4 == 0, "gp_sum_div: bad arguments");
  const size_t n4 = n_floats / 4;
  const unsigned grid = (unsigned)((n4 + 255) / 256);
  const float4 *a4 = reinterpret_cast<const float4*>(a), *b4 = reinterpret_cast<const float4*>(b), *c4 = reinterpret_cast<const float4*>(c);
  float4* o4 = reinterpret_cast<float4*>(out);
  return launch("gp_sum_div_kernel", c ? gp::gp_sum_div_kernel<3> : gp::gp_sum_div_kernel<2>, grid, 256, 0, st, a4, b4, c4, o4, n4, div);
}

int launch_conv_post_gp(const void* x, int bf16, const float* w, const float* bias, const int32_t* lens, int lens_mul, int B, int L, int C, int K,
                        float slope, float* wav, cudaStream_t st) {
  EV_CHECK_ARG(C % (bf16 ? 8 : 4) == 0 && C <= 128 && K <= 15 && (K & 1), "conv_post_gp: C=%d K=%d", C, K);
  EV_CHECK_ARG(B > 0 && B <= 65535 && L > 0, "conv_post_gp: bad shape");
  const size_t smem = (size_t)(C * (gp::GPP_BT + K - 1) + K * C) * sizeof(float);
  static std::atomic<uint64_t> attr_devs{0};
  if (first_use_on_device(attr_devs)) {
    cudaFuncSetAttribute(gp::conv_post_gp_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
    cudaFuncSetAttribute(gp::conv_post_gp_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
    cudaFuncSetAttribute(gp::conv_post_gp4_kernel<false, 7>, cudaFuncAttributeMaxDynamicSharedMemorySize, 112 * 1024);
    cudaFuncSetAttribute(gp::conv_post_gp4_kernel<true, 7>, cudaFuncAttributeMaxDynamicSharedMemorySize, 112 * 1024);
  }
  if (K == 7 && C <= 48) {
    constexpr int RS = gp::GP4_ROWS + 8;
    const size_t smem4 = (size_t)C * (RS + 8) * sizeof(float);
    dim3 grid4((L + gp::GP4_ROWS - 1) / gp::GP4_ROWS, B);
    return launch("conv_post_gp4_kernel", bf16 ? gp::conv_post_gp4_kernel<true, 7> : gp::conv_post_gp4_kernel<false, 7>, grid4, gp::GP4_T, smem4,
                  st, x, w, bias, lens, lens_mul, L, C, slope, wav);
  }
  dim3 grid((L + gp::GPP_BT - 1) / gp::GPP_BT, B);
  return launch("conv_post_gp_kernel", bf16 ? gp::conv_post_gp_kernel<true> : gp::conv_post_gp_kernel<false>, grid, gp::GPP_BT, smem, st, x, w,
                bias, lens, lens_mul, L, C, K, slope, wav);
}

}  // namespace ev
