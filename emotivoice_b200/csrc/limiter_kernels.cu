// True-peak limiter of output waveforms (ev_limit): a look-ahead limiter that holds each listed item, scaled by its loudness
// pre-gain g, at or below a ceiling C in dBTP.  Everything runs at the items' own rate; per item of n valid samples:
//   detector   p[s] = max(|x[s]|, |sum_j bank[ph][j] * x[s + c - j]| over the bank's phases), c = (taps - 1) / 2, x zero outside
//              [0, n): the oversampled (interpolated, and for a lower output rate also low-passed) waveform around s.  fp32, one
//              chain per value in tap order (tp_detect, true_peak.cuh, which ev_meter's true peak runs too).
//   required   r[s] = min(0, C - 20 log10(g p[s])) in fp64, clamped at -1000 dB and rounded DOWN to the grid Q = 2^-32 dB; 0 outside
//              the item.
//   hold       m[s] = min r over [s - M, s + L + M] (look-ahead L, hold M), for s in [-L, n).
//   release    G1[s] = min(m[s], G1[s - 1] + rho), G1[-L - 1] = 0, i.e. G1[s] = min(0, rho i + min_{k <= i} (m[k] - rho k)) with
//              i = s + L the extended index.  rho is on the grid Q, so every term is an integer multiple of Q below 2^53 Q and the
//              prefix minimum is exact in fp64: the same bits whatever the tiling, the batch or the CTA order.
//   attack     G[s] = (sum of G1 over [s - L, s]) / (L + 1).  The partial sums are exact too (|G1| <= 1000, L <= 1024), so the
//              sliding sum below equals the sum in index order.  Every window [j - M, j + L + M], j in [s - L, s], holds s, so
//              G[s] <= r[s].
//   apply      out[s] = fp32(x[s] * g * 10^(G[s] / 20)).
// g = 10^((T - lufs0) / 20) * 10^((T - lufs1) / 20), each factor 1 when its pointer is null or its loudness is -inf.
//
// Three launches.  lim_detect_kernel: one CTA per (tile of LM_TILE extended indices, listed item) stages the bank and x over the
// tile's span, computes r, then m, and writes v[i] = m[i - L] - rho i and the tile's minimum.  lim_tiles_kernel: one CTA per
// item, the exclusive prefix minimum over its tiles.  lim_apply_kernel: one CTA per (tile of LM_TILE output samples, item) scans v
// over two tiles from the carried minimum, forms G1, G and the output.
#include <math.h>

#include "ev_common.cuh"
#include "true_peak.cuh"

namespace ev {

constexpr int LM_THREADS = 256, LM_TILE = 1024, LM_PER = LM_TILE / LM_THREADS;
constexpr int LM_MAX_PHASES = 64, LM_MAX_TAPS = 255, LM_MAX_BANK = 16384;
constexpr int LM_MAX_LOOKAHEAD = LM_TILE, LM_MAX_HOLD = 1024;   // the apply kernel's two tiles hold a tile and its look-ahead
constexpr double LM_Q = 4294967296.0;       // grid of the envelope: 2^-32 dB
constexpr double LM_FLOOR_DB = -1000.0;
constexpr double LM_EXACT_DB = 1048576.0;   // 2^20 dB: rho * (extended length) must stay below, so 2^53 Q is never reached

__device__ __forceinline__ double lim_pregain(const float* lufs0, const float* lufs1, double target, int k) {
  double g = 1.0;
  if (lufs0) {
    const double L0 = lufs0[k];
    if (L0 > -INFINITY) g = pow(10.0, (target - L0) / 20.0);
    if (lufs1) {
      const double L1 = lufs1[k];
      if (L1 > -INFINITY) g *= pow(10.0, (target - L1) / 20.0);
    }
  }
  return g;
}

__device__ __forceinline__ long long lim_n(const int64_t* n_in, const int64_t* items, int k, long long item_stride, long long* b) {
  *b = items ? items[k] : k;
  return min((long long)n_in[*b], item_stride);
}

__global__ void __launch_bounds__(LM_THREADS) lim_detect_kernel(const float* __restrict__ wav, long long item_stride,
                                                                const int64_t* __restrict__ n_in, const int64_t* __restrict__ items,
                                                                const float* __restrict__ lufs0, const float* __restrict__ lufs1,
                                                                double target, double ceiling, const float* __restrict__ bank,
                                                                int phases, int taps, int L, int M, double rho, long long max_tiles,
                                                                double* __restrict__ v, double* __restrict__ tile_min) {
  pdl_entry();
  extern __shared__ __align__(16) unsigned char lm_smem[];
  const int k = blockIdx.y;
  long long b;
  const long long n = lim_n(n_in, items, k, item_stride, &b);
  const long long E = n + L;                                  // extended indices i = s + L, s in [-L, n)
  const long long i0 = (long long)blockIdx.x * LM_TILE;
  if (i0 >= E) return;
  const int c = (taps - 1) / 2;
  const int rspan = LM_TILE + L + 2 * M;                      // r over samples [i0 - L - M, i0 + LM_TILE - 1 + M]
  const int xspan = rspan + 2 * c;
  double* rs = reinterpret_cast<double*>(lm_smem);
  float* hs = reinterpret_cast<float*>(rs + rspan);
  float* xs = hs + phases * taps;
  const long long r0 = i0 - L - M;                            // sample of rs[0]
  const float* x = wav + b * item_stride;
  for (int i = threadIdx.x; i < phases * taps; i += LM_THREADS) hs[i] = bank[i];
  for (int i = threadIdx.x; i < xspan; i += LM_THREADS) {
    const long long s = r0 - c + i;
    xs[i] = (s >= 0 && s < n) ? x[s] : 0.f;
  }
  __syncthreads();
  const double g = lim_pregain(lufs0, lufs1, target, k);
  for (int q = threadIdx.x; q < rspan; q += LM_THREADS) {
    const long long s = r0 + q;
    double r = 0.0;
    if (s >= 0 && s < n) {
      const float p = tp_detect(xs + q, hs, phases, taps);      // xs[q + c] = x[s]
      const double gp = g * (double)p;
      if (gp > 0.0) r = fmax(fmin(0.0, ceiling - 20.0 * log10(gp)), LM_FLOOR_DB);
      if (!(r == r)) r = LM_FLOOR_DB;                          // a NaN sample: as loud as can be
      r = floor(r * LM_Q) / LM_Q;
    }
    rs[q] = r;
  }
  __syncthreads();
  // m at extended index i0 + q reads rs[q .. q + W - 1], W = L + 2M + 1; LM_PER consecutive outputs per thread share the core
  const int W = L + 2 * M + 1;
  const int q0 = threadIdx.x * LM_PER;
  double core = 0.0;
  for (int j = q0 + LM_PER - 1; j < q0 + W; ++j) core = fmin(core, rs[j]);
  double lo = INFINITY;
  double* vk = v + (size_t)k * (size_t)(max_tiles * LM_TILE);
  for (int t = 0; t < LM_PER; ++t) {
    const int q = q0 + t;
    double m = core;
    for (int j = q; j < q0 + LM_PER - 1; ++j) m = fmin(m, rs[j]);
    for (int j = q0 + W; j < q + W; ++j) m = fmin(m, rs[j]);
    const long long i = i0 + q;
    if (i < E) {
      const double vi = m - rho * (double)i;                  // exact: both on the grid, below 2^53 Q
      vk[i] = vi;
      lo = fmin(lo, vi);
    }
  }
  for (int o = 16; o > 0; o >>= 1) lo = fmin(lo, __shfl_xor_sync(0xffffffffu, lo, o));
  __shared__ double wmin[LM_THREADS / 32];
  if ((threadIdx.x & 31) == 0) wmin[threadIdx.x >> 5] = lo;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < LM_THREADS / 32; ++w) lo = fmin(lo, wmin[w]);
    tile_min[(size_t)k * max_tiles + blockIdx.x] = lo;
  }
}

// block-wide inclusive minimum scan of one value per thread (min is exact, so the order is free)
__device__ __forceinline__ double block_min_scan(double a, double* sh) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int o = 1; o < 32; o <<= 1) {
    const double y = __shfl_up_sync(0xffffffffu, a, o);
    if (lane >= o) a = fmin(a, y);
  }
  if (lane == 31) sh[w] = a;
  __syncthreads();
  if (w == 0) {
    double t = lane < (int)(blockDim.x >> 5) ? sh[lane] : INFINITY;
    for (int o = 1; o < 32; o <<= 1) {
      const double y = __shfl_up_sync(0xffffffffu, t, o);
      if (lane >= o) t = fmin(t, y);
    }
    sh[lane] = t;
  }
  __syncthreads();
  if (w > 0) a = fmin(a, sh[w - 1]);
  __syncthreads();
  return a;
}

__global__ void __launch_bounds__(LM_THREADS) lim_tiles_kernel(long long item_stride, const int64_t* __restrict__ n_in,
                                                               const int64_t* __restrict__ items, int L, long long max_tiles,
                                                               const double* __restrict__ tile_min, double* __restrict__ before) {
  pdl_entry();
  __shared__ double sh[32];
  __shared__ double last;
  const int k = blockIdx.x;
  long long b;
  const long long n = lim_n(n_in, items, k, item_stride, &b);
  const long long tiles = (n + L + LM_TILE - 1) / LM_TILE;
  const double* tm = tile_min + (size_t)k * max_tiles;
  double* bf = before + (size_t)k * max_tiles;
  double carry = INFINITY;
  for (long long t0 = 0; t0 < tiles; t0 += LM_THREADS) {
    const long long t = t0 + threadIdx.x;
    const double a = t < tiles ? tm[t] : INFINITY;
    const double inc = block_min_scan(a, sh);
    double ex = __shfl_up_sync(0xffffffffu, inc, 1);
    if ((threadIdx.x & 31) == 0) ex = threadIdx.x ? sh[(threadIdx.x >> 5) - 1] : INFINITY;
    if (t < tiles) bf[t] = fmin(carry, ex);
    if (threadIdx.x == LM_THREADS - 1) last = inc;
    __syncthreads();
    carry = fmin(carry, last);
    __syncthreads();
  }
}

__global__ void __launch_bounds__(LM_THREADS) lim_apply_kernel(const float* __restrict__ wav, long long item_stride,
                                                               const int64_t* __restrict__ n_in, const int64_t* __restrict__ items,
                                                               const float* __restrict__ lufs0, const float* __restrict__ lufs1,
                                                               double target, int L, double rho, long long max_tiles,
                                                               const double* __restrict__ v, const double* __restrict__ before,
                                                               float* __restrict__ out, long long out_stride) {
  pdl_entry();
  __shared__ double g1[2 * LM_TILE];
  __shared__ double sh[32];
  const int k = blockIdx.y;
  long long b;
  const long long n = lim_n(n_in, items, k, item_stride, &b);
  const long long s0 = (long long)blockIdx.x * LM_TILE;       // output samples [s0, s0 + LM_TILE): extended [s0, s0 + LM_TILE + L]
  if (s0 >= n) return;
  const long long E = n + L;
  const double* vk = v + (size_t)k * (size_t)(max_tiles * LM_TILE);
  // G1 over extended [s0, s0 + 2 LM_TILE): each thread scans 2 LM_PER consecutive values, then the block scan carries across
  constexpr int P2 = 2 * LM_PER;
  double a[P2];
  double run = before[(size_t)k * max_tiles + blockIdx.x];
  const long long e0 = s0 + (long long)threadIdx.x * P2;
  double loc = INFINITY;
  for (int t = 0; t < P2; ++t) {
    a[t] = e0 + t < E ? vk[e0 + t] : INFINITY;
    loc = fmin(loc, a[t]);
  }
  const double inc = block_min_scan(loc, sh);
  double ex = __shfl_up_sync(0xffffffffu, inc, 1);
  if ((threadIdx.x & 31) == 0) ex = threadIdx.x ? sh[(threadIdx.x >> 5) - 1] : INFINITY;
  run = fmin(run, ex);
  for (int t = 0; t < P2; ++t) {
    run = fmin(run, a[t]);
    g1[threadIdx.x * P2 + t] = fmin(0.0, rho * (double)(e0 + t) + run);
  }
  __syncthreads();
  const double g = lim_pregain(lufs0, lufs1, target, k);
  const float* x = wav + b * item_stride;
  float* y = out + (size_t)k * out_stride;
  const int q0 = threadIdx.x * LM_PER;
  double sum = 0.0;
  for (int j = q0; j <= q0 + L; ++j) sum += g1[j];
  for (int t = 0; t < LM_PER; ++t) {
    const long long s = s0 + q0 + t;
    if (t) sum += g1[q0 + t + L] - g1[q0 + t - 1];           // exact: every partial sum is a multiple of Q below 2^53 Q
    if (s < n) y[s] = (float)((double)x[s] * g * exp10(sum / (double)(L + 1) / 20.0));
  }
}

static long long lim_tiles(long long max_n, int L) { return (max_n + L + LM_TILE - 1) / LM_TILE; }

static size_t lim_ws_bytes(int n_items, long long max_n, int L) {
  const size_t t = (size_t)lim_tiles(max_n, L);
  return (size_t)n_items * t * (LM_TILE + 2) * sizeof(double);
}

static bool lim_args_ok(int n_items, long long max_n, int L) {
  return n_items >= 1 && n_items <= 65535 && max_n >= 1 && L >= 0 && L <= LM_MAX_LOOKAHEAD;
}

}  // namespace ev

using namespace ev;

extern "C" {

size_t ev_limit_workspace_bytes(int n_items, long long max_n, int lookahead) {
  return lim_args_ok(n_items, max_n, lookahead) ? lim_ws_bytes(n_items, max_n, lookahead) : 0;
}

int ev_limit(const float* wav, long long item_stride, const int64_t* n_in, const int64_t* items, int n_items, int sample_rate,
             const float* lufs0, const float* lufs1, float target_lufs, float ceiling_dbtp, const float* bank, int phases, int taps,
             int lookahead, int hold, double release_db_per_sample, float* out, long long out_stride, void* ws, size_t ws_bytes,
             void* stream) {
  EV_CHECK_ARG(wav && n_in && bank && out && ws, "ev_limit: null argument");
  EV_CHECK_ARG(lufs0 || !lufs1, "ev_limit: lufs1 needs lufs0");
  EV_CHECK_ARG(n_items >= 1 && n_items <= 65535, "ev_limit: n_items=%d must lie in [1, 65535]", n_items);
  EV_CHECK_ARG(item_stride >= 1 && out_stride >= item_stride, "ev_limit: item_stride=%lld must be at least 1 and out_stride=%lld at least "
               "item_stride", item_stride, out_stride);
  EV_CHECK_ARG(sample_rate >= 4000 && sample_rate <= 192000, "ev_limit: sample_rate=%d must lie in [4000, 192000]", sample_rate);
  EV_CHECK_ARG(!lufs0 || (target_lufs >= -70.f && target_lufs <= 0.f), "ev_limit: target_lufs=%g must lie in [-70, 0]",
               (double)target_lufs);
  EV_CHECK_ARG(ceiling_dbtp >= -20.f && ceiling_dbtp <= 0.f, "ev_limit: ceiling_dbtp=%g must lie in [-20, 0]", (double)ceiling_dbtp);
  EV_CHECK_ARG(phases >= 1 && phases <= LM_MAX_PHASES && taps >= 1 && taps <= LM_MAX_TAPS && taps % 2 == 1 &&
               phases * taps <= LM_MAX_BANK, "ev_limit: a bank of %d phases of %d taps (odd taps, at most %d phases, %d taps, %d in all)",
               phases, taps, LM_MAX_PHASES, LM_MAX_TAPS, LM_MAX_BANK);
  EV_CHECK_ARG(lookahead >= 0 && lookahead <= LM_MAX_LOOKAHEAD, "ev_limit: lookahead=%d must lie in [0, %d]", lookahead, LM_MAX_LOOKAHEAD);
  EV_CHECK_ARG(lookahead + 2 * hold + 1 >= LM_PER, "ev_limit: lookahead=%d and hold=%d span fewer than %d samples", lookahead, hold, LM_PER);
  EV_CHECK_ARG(hold >= (taps - 1) / 2 && hold <= LM_MAX_HOLD, "ev_limit: hold=%d must lie in [%d (the bank's half-span), %d]", hold,
               (taps - 1) / 2, LM_MAX_HOLD);
  const double rq = release_db_per_sample * LM_Q;
  EV_CHECK_ARG(release_db_per_sample > 0.0 && release_db_per_sample <= 1.0 && rq == floor(rq),
               "ev_limit: release_db_per_sample=%.17g must lie in (0, 1] on the 2^-32 dB grid", release_db_per_sample);
  EV_CHECK_ARG(release_db_per_sample * (double)(item_stride + lookahead) < LM_EXACT_DB,
               "ev_limit: item_stride=%lld is too long for an exact release at %.17g dB per sample", item_stride, release_db_per_sample);
  const size_t need = lim_ws_bytes(n_items, item_stride, lookahead);
  EV_CHECK_ARG(ws_bytes >= need, "ev_limit: workspace of %zu bytes, %zu needed", ws_bytes, need);
  const long long max_tiles = lim_tiles(item_stride, lookahead);
  const long long out_tiles = (item_stride + LM_TILE - 1) / LM_TILE;
  EV_CHECK_ARG(max_tiles <= 0x7fffffffll, "ev_limit: item_stride=%lld is too long", item_stride);
  EV_TRY(use_device_of(wav));
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int rspan = LM_TILE + lookahead + 2 * hold;
  const size_t smem = (size_t)rspan * sizeof(double) + (size_t)(phases * taps + rspan + (taps - 1)) * sizeof(float);
  static std::atomic<uint64_t> attr_devs{0};
  if (first_use_on_device(attr_devs))
    cudaFuncSetAttribute(lim_detect_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  double* v = static_cast<double*>(ws);
  double* tile_min = v + (size_t)n_items * (size_t)max_tiles * LM_TILE;
  double* before = tile_min + (size_t)n_items * (size_t)max_tiles;
  const double target = (double)target_lufs, ceiling = (double)ceiling_dbtp;
  EV_TRY(launch("lim_detect_kernel", lim_detect_kernel, dim3((unsigned)max_tiles, n_items), LM_THREADS, smem, st, wav, item_stride, n_in,
                items, lufs0, lufs1, target, ceiling, bank, phases, taps, lookahead, hold, release_db_per_sample, max_tiles, v, tile_min));
  EV_TRY(launch("lim_tiles_kernel", lim_tiles_kernel, dim3(n_items), LM_THREADS, 0, st, item_stride, n_in, items, lookahead, max_tiles,
                (const double*)tile_min, before));
  return launch("lim_apply_kernel", lim_apply_kernel, dim3((unsigned)out_tiles, n_items), LM_THREADS, 0, st, wav, item_stride, n_in,
                items, lufs0, lufs1, target, lookahead, release_db_per_sample, max_tiles, (const double*)v, (const double*)before, out,
                out_stride);
}

}  // extern "C"
