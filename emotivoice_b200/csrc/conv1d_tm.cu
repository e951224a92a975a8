// Generic time-major 1-D convolution as an implicit GEMM, fp32 FFMA path (sm_90a).
//
//   out[b,t,co] = epi( bias[co] + sum_j sum_ci w[j][ci][co] * act_in( x[b, t + (j-(K-1)/2)*dil, ci] ) )
//
// M = time, N = C_out, K = taps x C_in.  The K taps of one input-channel chunk are ROW-SHIFTED
// VIEWS of a single shared-memory tile (BM + (K-1)*dil rows), so every activation is fetched from
// L2/HBM once per (m-tile, n-tile) regardless of the kernel size; weights stream through a
// double-buffered (16 x BN) tile.  The same kernel serves nn.Linear (K=1), the conv-FFN,
// the predictor convs, conv_pre, every ResBlock1 conv and (with polyphase-packed weights) the
// transposed convolutions of the HiFi-GAN generator.
//
// Reference semantics: torch.nn.Conv1d cross-correlation with "same" zero padding
// (encoder.py:31-52, variance.py:17-31, hifigan/models.py:23-57,96-116).
#include "ev_common.cuh"

namespace ev {

constexpr int KC = 16;          // input channels per smem chunk
constexpr int NTHREADS = 256;

// TXN: threads along N (8 or 16); NV: float4 column groups per thread (1 or 2); TM: rows per thread.
//   BN = TXN*4*NV,  BM = (256/TXN)*TM.
template <int TXN, int NV, int TM>
__global__ void __launch_bounds__(NTHREADS) conv1d_tm_kernel(ConvParams p, int a_ld) {
  pdl_entry();
  constexpr int TYN = NTHREADS / TXN;   // threads along M
  constexpr int BM = TYN * TM;
  constexpr int BN = TXN * 4 * NV;
  constexpr int TN = 4 * NV;
  constexpr int B_F4 = KC * BN / 4;                          // float4 per weight tile
  constexpr int B_PER_T = (B_F4 + NTHREADS - 1) / NTHREADS;  // per thread

  extern __shared__ __align__(16) float smem[];
  float* As = smem;                    // [2][KC][a_ld]   (transposed: channel-major, rows contiguous)
  float* Bs = smem + 2 * KC * a_ld;    // [2][KC][BN]

  const int tid = threadIdx.x;
  const int tx = tid % TXN;
  const int ty = tid / TXN;
  const int b = blockIdx.z;
  const int t0 = blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;

  const int len = p.lens ? min(p.L, p.lens[b] * p.lens_mul) : p.L;
  const int halo = ((p.K - 1) / 2) * p.dil;
  const int rows_a = BM + (p.K - 1) * p.dil;

  const float* __restrict__ xb = p.x + (size_t)b * p.L * p.Cin;
  float* ob = p.out   /* may alias p.res (in-place residual) */ + (size_t)b * p.L * p.Cout;

  if (t0 >= len) {
    // whole tile is padding: the batch-invariant contract stores zeros there.
    for (int i = 0; i < TM; ++i) {
      const int row = t0 + ty + TYN * i;
      if (row >= p.L) continue;
#pragma unroll
      for (int v = 0; v < NV; ++v) {
        const int col = n0 + v * (TXN * 4) + tx * 4;
        if (col < p.Cout) *reinterpret_cast<float4*>(ob + (size_t)row * p.Cout + col) = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    return;
  }

  const int n_chunks = p.Cin / KC;
  const int n_it = n_chunks * p.K;
  const int a_f4 = rows_a * (KC / 4);   // float4 loads per A tile
  constexpr int A_PER_T_MAX = 6;        // rows_a <= 384 enforced by the launcher

  float4 a_reg[A_PER_T_MAX];
  float4 b_reg[B_PER_T];

  auto load_a = [&](int chunk) {
#pragma unroll
    for (int i = 0; i < A_PER_T_MAX; ++i) {
      const int idx = tid + i * NTHREADS;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (idx < a_f4) {
        const int r = idx >> 2, c4 = idx & 3;
        const int row = t0 - halo + r;
        if (row >= 0 && row < len)
          v = __ldg(reinterpret_cast<const float4*>(xb + (size_t)row * p.Cin + chunk * KC + c4 * 4));
      }
      a_reg[i] = v;
    }
  };
  auto store_a = [&](int buf) {
    float* dst = As + buf * KC * a_ld;
#pragma unroll
    for (int i = 0; i < A_PER_T_MAX; ++i) {
      const int idx = tid + i * NTHREADS;
      if (idx < a_f4) {
        const int r = idx >> 2, c4 = idx & 3;
        float4 v = a_reg[i];
        if (p.in_act == EV_ACT_LRELU) {
          v.x = v.x > 0.f ? v.x : v.x * p.in_slope;
          v.y = v.y > 0.f ? v.y : v.y * p.in_slope;
          v.z = v.z > 0.f ? v.z : v.z * p.in_slope;
          v.w = v.w > 0.f ? v.w : v.w * p.in_slope;
        }
        dst[(c4 * 4 + 0) * a_ld + r] = v.x;
        dst[(c4 * 4 + 1) * a_ld + r] = v.y;
        dst[(c4 * 4 + 2) * a_ld + r] = v.z;
        dst[(c4 * 4 + 3) * a_ld + r] = v.w;
      }
    }
  };
  auto load_b = [&](int it) {
    const int chunk = it / p.K, tap = it - chunk * p.K;
    const float* __restrict__ wt = p.w + ((size_t)tap * p.Cin + (size_t)chunk * KC) * p.Cout;
#pragma unroll
    for (int i = 0; i < B_PER_T; ++i) {
      const int idx = tid + i * NTHREADS;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (idx < B_F4) {
        const int kk = idx / (BN / 4), c4 = idx % (BN / 4);
        const int col = n0 + c4 * 4;
        if (col < p.Cout) v = __ldg(reinterpret_cast<const float4*>(wt + (size_t)kk * p.Cout + col));
      }
      b_reg[i] = v;
    }
  };
  auto store_b = [&](int buf) {
    float* dst = Bs + buf * KC * BN;
#pragma unroll
    for (int i = 0; i < B_PER_T; ++i) {
      const int idx = tid + i * NTHREADS;
      if (idx < B_F4) *reinterpret_cast<float4*>(dst + idx * 4) = b_reg[i];
    }
  };

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  load_a(0);
  load_b(0);
  store_a(0);
  store_b(0);
  __syncthreads();

  int chunk = 0, tap = 0;
  for (int it = 0; it < n_it; ++it) {
    const int nit = it + 1;
    const bool has_next = nit < n_it;
    const bool next_new_chunk = has_next && (tap + 1 == p.K);
    if (has_next) load_b(nit);
    if (next_new_chunk) load_a(chunk + 1);

    const float* a_s = As + (chunk & 1) * KC * a_ld + ty + tap * p.dil;
    const float* b_s = Bs + (it & 1) * KC * BN + tx * 4;
#pragma unroll
    for (int kk = 0; kk < KC; ++kk) {
      float a[TM];
      float bv[TN];
#pragma unroll
      for (int i = 0; i < TM; ++i) a[i] = a_s[kk * a_ld + TYN * i];
#pragma unroll
      for (int v = 0; v < NV; ++v) {
        const float4 t4 = *reinterpret_cast<const float4*>(b_s + kk * BN + v * (TXN * 4));
        bv[v * 4 + 0] = t4.x; bv[v * 4 + 1] = t4.y; bv[v * 4 + 2] = t4.z; bv[v * 4 + 3] = t4.w;
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], bv[j], acc[i][j]);
    }

    if (has_next) store_b(nit & 1);
    if (next_new_chunk) store_a((chunk + 1) & 1);
    __syncthreads();
    if (++tap == p.K) { tap = 0; ++chunk; }
  }

  // ---- epilogue: bias, activation, residual, accumulate, pad rows -> 0 -----------------------
  const float* __restrict__ bias = p.bias ? p.bias + (size_t)b * p.bias_bs : nullptr;
  const float* rb = p.res ? p.res + (size_t)b * p.L * p.Cout : nullptr;
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int row = t0 + ty + TYN * i;
    if (row >= p.L) continue;
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      const int col = n0 + v * (TXN * 4) + tx * 4;
      if (col >= p.Cout) continue;
      float4 o;
      if (row < len) {
        float r[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float t = acc[i][v * 4 + j];
          if (bias) t += __ldg(bias + col + j);
          r[j] = act_apply(t, p.out_act, 0.f);
        }
        if (rb) {
          const float4 q = *reinterpret_cast<const float4*>(rb + (size_t)row * p.Cout + col);
          r[0] += q.x; r[1] += q.y; r[2] += q.z; r[3] += q.w;
        }
        if (p.acc != EV_ACC_STORE) {
          const float4 q = *reinterpret_cast<const float4*>(ob + (size_t)row * p.Cout + col);
          r[0] += q.x; r[1] += q.y; r[2] += q.z; r[3] += q.w;
          if (p.acc == EV_ACC_ADD_DIV) { r[0] /= p.div; r[1] /= p.div; r[2] /= p.div; r[3] /= p.div; }
        }
        o = make_float4(r[0], r[1], r[2], r[3]);
      } else {
        o = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      *reinterpret_cast<float4*>(ob + (size_t)row * p.Cout + col) = o;
    }
  }
}

// The launch of one convolution: the template variant, its tile, the A tile's rows and leading dimension, shared memory and grid.
struct Conv1dPlan {
  int TXN, NV, TM, BM, BN, rows_a, a_ld;
  size_t smem;
  int grid_x, grid_y;
};
constexpr size_t kSmemAttr = 96 * 1024;   // the dynamic shared-memory attribute every variant is given

// Argument checks and the variant choice of launch_conv1d (pure host arithmetic; also exported as ev_debug_conv1d_plan).  Every
// variant sums each output in the same (chunk, tap, kk) order as one fmaf chain, so the choice changes no result bit.
static int plan_conv1d(const ConvParams& p, Conv1dPlan* pl) {
  EV_CHECK_ARG(p.B > 0 && p.L > 0, "conv1d: empty problem B=%d L=%d", p.B, p.L);
  EV_CHECK_ARG(p.Cin > 0 && p.Cin % KC == 0, "conv1d: Cin=%d must be a positive multiple of %d", p.Cin, KC);
  EV_CHECK_ARG(p.Cout > 0 && p.Cout % 4 == 0, "conv1d: Cout=%d must be a positive multiple of 4", p.Cout);
  EV_CHECK_ARG(p.K >= 1 && (p.K & 1) && p.dil >= 1, "conv1d: K=%d must be odd, dil=%d >= 1", p.K, p.dil);
  EV_CHECK_ARG(p.in_act == EV_ACT_NONE || p.in_act == EV_ACT_LRELU, "conv1d: unsupported input activation");
  EV_CHECK_ARG(p.B <= 65535, "conv1d: B too large");
  // tile selection: wide N -> 128x128 (8x8 per thread); N<=64 -> 128x64; N<=32 -> 256x32;
  // small problems (few CTAs) -> 64x64 so that more SMs get work.
  int txn, nv, tm;
  const long long m_tiles = (p.L + 127) / 128;
  if (p.Cout <= 32) {
    txn = 8; nv = 1; tm = 8;
  } else if (p.Cout <= 64) {
    if (m_tiles * p.B < sm_count()) { txn = 16; nv = 1; tm = 4; } else { txn = 16; nv = 1; tm = 8; }
  } else if (m_tiles * ((p.Cout + 127) / 128) * p.B < sm_count()) {
    txn = 16; nv = 1; tm = 4;
  } else {
    txn = 16; nv = 2; tm = 8;
  }
  Conv1dPlan r;
  r.TXN = txn; r.NV = nv; r.TM = tm;
  r.BM = (NTHREADS / txn) * tm;
  r.BN = txn * 4 * nv;
  const long long rows_a = r.BM + (long long)(p.K - 1) * p.dil;
  EV_CHECK_ARG(rows_a <= 6 * NTHREADS / 4, "conv1d: receptive field too wide for the tile (rows_a=%lld)", rows_a);
  r.rows_a = (int)rows_a;
  r.a_ld = ((r.rows_a + 7) / 8) * 8 + 2;   // == 2 (mod 8): conflict-free transposed stores
  r.smem = (size_t)(2 * KC * r.a_ld + 2 * KC * r.BN) * sizeof(float);
  EV_CHECK_ARG(r.smem <= kSmemAttr, "conv1d: smem %zu too large", r.smem);
  r.grid_x = (p.L + r.BM - 1) / r.BM;
  r.grid_y = (p.Cout + r.BN - 1) / r.BN;
  *pl = r;
  return EV_OK;
}

int debug_conv1d_plan(const ConvParams& p, int* v) {
  Conv1dPlan pl;
  EV_TRY(plan_conv1d(p, &pl));
  v[0] = pl.TXN; v[1] = pl.NV; v[2] = pl.TM; v[3] = pl.BM; v[4] = pl.BN; v[5] = pl.rows_a; v[6] = pl.a_ld;
  v[7] = (int)pl.smem; v[8] = pl.grid_x; v[9] = pl.grid_y;
  return EV_OK;
}

template <int TXN, int NV, int TM>
static int launch_variant(const ConvParams& p, const Conv1dPlan& pl, cudaStream_t st) {
  static std::atomic<uint64_t> attr_devs{0};   // per instantiation
  if (first_use_on_device(attr_devs))
    cudaFuncSetAttribute(conv1d_tm_kernel<TXN, NV, TM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemAttr);
  dim3 grid(pl.grid_x, pl.grid_y, p.B);
  return launch("conv1d_tm_kernel", conv1d_tm_kernel<TXN, NV, TM>, grid, NTHREADS, pl.smem, st, p, pl.a_ld);
}

int launch_conv1d(const ConvParams& p, cudaStream_t st) {
  Conv1dPlan pl;
  EV_TRY(plan_conv1d(p, &pl));
  if (pl.TXN == 8) return launch_variant<8, 1, 8>(p, pl, st);
  if (pl.NV == 2) return launch_variant<16, 2, 8>(p, pl, st);
  if (pl.TM == 4) return launch_variant<16, 1, 4>(p, pl, st);
  return launch_variant<16, 1, 8>(p, pl, st);
}

}  // namespace ev
