// Loudness meter of waveform items (ev_meter, EBU R128 / ITU-R BS.1770-4, one channel): integrated loudness, momentary and
// short-term loudness and their maxima, loudness range (EBU Tech 3342) and true peak.  Per item of n samples at sr Hz:
//   sub-blocks  e[j]: the K-weighted sum of squares of the j-th 100 ms sub-block (S = sr / 10 samples), ev_loudness's
//               loud_subblock_kernel; only the n / S full sub-blocks count.
//   momentary   M[k] = -0.691 + 10 log10((((e[k] + e[k+1]) + e[k+2]) + e[k+3]) / (4 S)), k < n / S - 3: ev_loudness's gating
//               blocks, ungated.
//   short-term  S[k] = -0.691 + 10 log10((e[k] + ... + e[k+29], summed left to right) / (30 S)), k < n / S - 29.
//   integrated  I: ev_loudness's loud_gate_kernel on the same sub-blocks, so bitwise its lufs.
//   range       LRA (Tech 3342): the values S > -70 (absolute gate); of those, the values above 10 log10(mean 10^(S/10)) - 20
//               (relative gate; the power mean is taken over the absolute-gated mean squares, fp64 in a fixed order); of the n
//               values left, v[round(0.95 (n - 1))] - v[round(0.10 (n - 1))] in ascending order, round half away from zero,
//               each v selected exactly; NaN when n = 0.
//   true peak   20 log10 max_s p[s], p the detector of ev_limit (true_peak.cuh) with the bank of audio.true_peak_bank(sr): all R
//               phases of the limiter's interpolator (the limiter skips phase 0), so p reads resample_poly(x, R, 1) and |x|.
//
// Four launches.  loud_subblock_kernel and loud_gate_kernel as in ev_loudness, with the items at their start offsets.
// meter_peak_kernel: one CTA per (tile of MP_TILE samples, item) stages the bank and the tile's samples with their halo and
// writes the tile's largest p (max is exact: any order gives the same bits).  meter_range_kernel: one CTA per item forms the M
// and S series and their maxima, the two gates and LRA, and the item's true peak from its tiles.  The selection is an MSB-first
// radix select over the 64-bit patterns of the short-term mean squares (positive doubles order as their bit patterns; the map
// to loudness is monotone, so it commutes with order statistics), 8 passes of 8 bits with integer histograms: the rejected
// values are written as 0 and ranked below every kept one, so no compaction and no length cap.
#include <math.h>

#include "ev_common.cuh"
#include "true_peak.cuh"

namespace ev {

constexpr int MP_THREADS = 256, MP_TILE = 2048;
constexpr int MR_THREADS = 512, MR_WARPS = MR_THREADS / 32;
constexpr int MR_MOMENTARY = 4, MR_SHORT = 30;              // sub-blocks per momentary (400 ms) and short-term (3 s) window
constexpr int MT_MAX_PHASES = 64, MT_MAX_TAPS = 255, MT_MAX_BANK = 16384;
constexpr int MT_MIN_RATE = 4000, MT_MAX_RATE = 192000;

__global__ void __launch_bounds__(MP_THREADS) meter_peak_kernel(const float* __restrict__ wav, const int64_t* __restrict__ start,
                                                                const int64_t* __restrict__ n_in, long long max_n,
                                                                const float* __restrict__ bank, int phases, int taps,
                                                                long long max_tiles, float* __restrict__ tile_max) {
  pdl_entry();
  extern __shared__ __align__(16) float mp_smem[];
  const int k = blockIdx.y;
  const long long n = min((long long)n_in[k], max_n);
  const long long s0 = (long long)blockIdx.x * MP_TILE;
  if (s0 >= n) return;                                      // past the item: the range kernel reads only its own tiles
  const int c = (taps - 1) / 2;
  float* hs = mp_smem;
  float* xs = hs + phases * taps;                           // xs[i] = x[s0 - c + i]
  const float* x = wav + start[k];
  for (int i = threadIdx.x; i < phases * taps; i += MP_THREADS) hs[i] = bank[i];
  for (int i = threadIdx.x; i < MP_TILE + 2 * c; i += MP_THREADS) {
    const long long s = s0 - c + i;
    xs[i] = (s >= 0 && s < n) ? x[s] : 0.f;
  }
  __syncthreads();
  float pk = 0.f;
  for (int q = threadIdx.x; q < MP_TILE && s0 + q < n; q += MP_THREADS) pk = fmaxf(pk, tp_detect(xs + q, hs, phases, taps));
  for (int o = 16; o > 0; o >>= 1) pk = fmaxf(pk, __shfl_xor_sync(0xffffffffu, pk, o));
  __shared__ float wmax[MP_THREADS / 32];
  if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = pk;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < MP_THREADS / 32; ++w) pk = fmaxf(pk, wmax[w]);
    tile_max[(size_t)k * max_tiles + blockIdx.x] = pk;
  }
}

__device__ __forceinline__ double meter_loudness(double ms) { return -0.691 + 10.0 * log10(ms); }

// fixed-order CTA sum of one (sum, count) pair per thread: a tree over the threads, so the result does not depend on the batch
__device__ __forceinline__ void meter_sum(double& s, double& cnt, double* red) {
  red[threadIdx.x] = s;
  red[MR_THREADS + threadIdx.x] = cnt;
  __syncthreads();
  for (int h = MR_THREADS / 2; h > 0; h >>= 1) {
    if ((int)threadIdx.x < h) {
      red[threadIdx.x] += red[threadIdx.x + h];
      red[MR_THREADS + threadIdx.x] += red[MR_THREADS + threadIdx.x + h];
    }
    __syncthreads();
  }
  s = red[0];
  cnt = red[MR_THREADS];
  __syncthreads();
}

// CTA maximum of two values per thread (exact, any order)
__device__ __forceinline__ void meter_max(double& a, double& b, double* red) {
  for (int o = 16; o > 0; o >>= 1) {
    a = fmax(a, __shfl_xor_sync(0xffffffffu, a, o));
    b = fmax(b, __shfl_xor_sync(0xffffffffu, b, o));
  }
  if ((threadIdx.x & 31) == 0) {
    red[threadIdx.x >> 5] = a;
    red[MR_WARPS + (threadIdx.x >> 5)] = b;
  }
  __syncthreads();
  for (int w = 0; w < MR_WARPS; ++w) {
    a = fmax(a, red[w]);
    b = fmax(b, red[MR_WARPS + w]);
  }
  __syncthreads();
}

__global__ void __launch_bounds__(MR_THREADS) meter_range_kernel(const int64_t* __restrict__ n_in, long long max_n, int S,
                                                                 long long max_sub, const double* __restrict__ energy,
                                                                 double* __restrict__ keys, long long max_tiles,
                                                                 const float* __restrict__ tile_max, float* __restrict__ results,
                                                                 int n_items, float* __restrict__ momentary,
                                                                 float* __restrict__ short_term, long long series_stride) {
  pdl_entry();
  __shared__ double red[2 * MR_THREADS];
  __shared__ unsigned int hist[2][256];
  __shared__ unsigned long long sel[2];
  __shared__ long long rank[2];
  const int k = blockIdx.x;
  const long long n = min((long long)n_in[k], max_n);
  const long long n_full = n / S;
  const long long n_m = n_full >= MR_MOMENTARY ? n_full - (MR_MOMENTARY - 1) : 0;
  const long long n_s = n_full >= MR_SHORT ? n_full - (MR_SHORT - 1) : 0;
  const double* e = energy + (size_t)k * max_sub;
  double* key = keys + (size_t)k * max_sub;
  // momentary series and its maximum
  double max_m = -INFINITY;
  const double inv_m = 1.0 / (4.0 * S), inv_s = 1.0 / (30.0 * S);
  for (long long j = threadIdx.x; j < n_m; j += MR_THREADS) {
    const double l = meter_loudness((((e[j] + e[j + 1]) + e[j + 2]) + e[j + 3]) * inv_m);
    max_m = fmax(max_m, l);
    if (momentary) momentary[(size_t)k * series_stride + j] = (float)l;
  }
  // short-term series, its maximum, and the absolute gate of the range
  double max_s = -INFINITY, s1 = 0.0, c1 = 0.0;
  for (long long j = threadIdx.x; j < n_s; j += MR_THREADS) {
    double z = 0.0;
    for (int i = 0; i < MR_SHORT; ++i) z += e[j + i];
    z *= inv_s;
    const double l = meter_loudness(z);
    max_s = fmax(max_s, l);
    if (short_term) short_term[(size_t)k * series_stride + j] = (float)l;
    key[j] = z;
    if (l > -70.0) { s1 += z; c1 += 1.0; }
  }
  if (momentary)
    for (long long j = n_m + threadIdx.x; j < series_stride; j += MR_THREADS) momentary[(size_t)k * series_stride + j] = NAN;
  if (short_term)
    for (long long j = n_s + threadIdx.x; j < series_stride; j += MR_THREADS) short_term[(size_t)k * series_stride + j] = NAN;
  meter_max(max_m, max_s, red);
  meter_sum(s1, c1, red);
  // relative gate: the kept values become their mean square, the others 0, which ranks below every kept value
  double c2 = 0.0;
  if (c1 > 0.0) {
    const double rel = meter_loudness(s1 / c1) - 20.0;
    double unused = 0.0;
    for (long long j = threadIdx.x; j < n_s; j += MR_THREADS) {
      const double z = key[j];
      const double l = meter_loudness(z);
      const bool keep = l > -70.0 && l > rel;
      key[j] = keep ? z : 0.0;
      c2 += keep ? 1.0 : 0.0;
    }
    meter_sum(unused, c2, red);
  }
  const long long kept = (long long)c2;
  if (kept > 0) {
    if (threadIdx.x == 0) {
      sel[0] = sel[1] = 0ull;
      rank[0] = (n_s - kept) + llround((double)(kept - 1) * 0.10);
      rank[1] = (n_s - kept) + llround((double)(kept - 1) * 0.95);
    }
    for (int shift = 56; shift >= 0; shift -= 8) {
      for (int i = threadIdx.x; i < 2 * 256; i += MR_THREADS) (&hist[0][0])[i] = 0u;
      __syncthreads();
      const unsigned long long hi_mask = shift == 56 ? 0ull : ~0ull << (shift + 8);
      const unsigned long long p0 = sel[0], p1 = sel[1];
      for (long long j = threadIdx.x; j < n_s; j += MR_THREADS) {
        const unsigned long long u = (unsigned long long)__double_as_longlong(key[j]);
        const unsigned d = (unsigned)(u >> shift) & 255u;
        if ((u & hi_mask) == p0) atomicAdd(&hist[0][d], 1u);
        if ((u & hi_mask) == p1) atomicAdd(&hist[1][d], 1u);
      }
      __syncthreads();
      const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
      if (w < 2) {                                           // warp w picks the digit of selection w
        unsigned loc = 0u;
        for (int i = 0; i < 8; ++i) loc += hist[w][lane * 8 + i];
        unsigned inc = loc;
        for (int o = 1; o < 32; o <<= 1) {
          const unsigned y = __shfl_up_sync(0xffffffffu, inc, o);
          if (lane >= o) inc += y;
        }
        const long long r = rank[w];
        long long before = (long long)(inc - loc);
        if (before <= r && r < (long long)inc) {            // exactly one lane holds the rank
          int d = lane * 8;
          while (before + (long long)hist[w][d] <= r) before += hist[w][d++];
          sel[w] |= (unsigned long long)d << shift;
          rank[w] = r - before;
        }
      }
      __syncthreads();
    }
  }
  // true peak from the item's tiles
  const long long tiles = (n + MP_TILE - 1) / MP_TILE;
  double tp = 0.0, unused_max = -INFINITY;
  for (long long t = threadIdx.x; t < tiles; t += MR_THREADS) tp = fmax(tp, (double)tile_max[(size_t)k * max_tiles + t]);
  meter_max(tp, unused_max, red);
  if (threadIdx.x == 0) {
    double lra = NAN;
    if (kept > 0) lra = meter_loudness(__longlong_as_double((long long)sel[1])) - meter_loudness(__longlong_as_double((long long)sel[0]));
    results[1 * n_items + k] = (float)lra;
    results[2 * n_items + k] = (float)max_m;
    results[3 * n_items + k] = (float)max_s;
    results[4 * n_items + k] = tp > 0.0 ? (float)(20.0 * log10(tp)) : -INFINITY;
  }
}

static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

static long long meter_tiles(long long max_n) { return (max_n + MP_TILE - 1) / MP_TILE; }

// energy (f64) | sub-block peaks (f32) | short-term keys (f64) | tile maxima (f32) | gains of the gate kernel (f32)
static size_t meter_ws_bytes(int n_items, long long max_n, int sample_rate) {
  const size_t cells = (size_t)n_items * (size_t)loud_max_sub(max_n, sample_rate);
  return align256(cells * sizeof(double)) + align256(cells * sizeof(float)) + align256(cells * sizeof(double)) +
         align256((size_t)n_items * (size_t)meter_tiles(max_n) * sizeof(float)) + align256((size_t)n_items * sizeof(float));
}

static bool meter_rate_ok(int sample_rate) { return sample_rate % 10 == 0 && sample_rate >= MT_MIN_RATE && sample_rate <= MT_MAX_RATE; }

static bool meter_size_ok(long long max_n) { return max_n >= 1 && meter_tiles(max_n) <= 0x7fffffffll; }

}  // namespace ev

using namespace ev;

extern "C" {

size_t ev_meter_workspace_bytes(int n_items, long long max_n, int sample_rate) {
  if (max_n == 0) max_n = 1;
  return n_items >= 1 && n_items <= 65535 && meter_rate_ok(sample_rate) && meter_size_ok(max_n) ? meter_ws_bytes(n_items, max_n, sample_rate)
                                                                                                   : 0;
}

int ev_meter(const float* wav, const int64_t* start, const int64_t* n, const int64_t* n_host, int n_items, int sample_rate,
             const double* kcoef, const float* bank, int phases, int taps, float* results, float* momentary, float* short_term,
             long long series_stride, void* ws, size_t ws_bytes, void* stream) {
  EV_CHECK_ARG(wav && start && n && n_host && kcoef && results && ws, "ev_meter: null argument");
  EV_CHECK_ARG(n_items >= 1 && n_items <= 65535, "ev_meter: n_items=%d must lie in [1, 65535]", n_items);
  EV_CHECK_ARG(meter_rate_ok(sample_rate), "ev_meter: sample_rate=%d must be a multiple of 10 in [%d, %d] (100 ms sub-blocks)",
               sample_rate, MT_MIN_RATE, MT_MAX_RATE);
  long long max_n = 1;
  for (int k = 0; k < n_items; ++k) {
    EV_CHECK_ARG(n_host[k] >= 0, "ev_meter: item %d has %lld samples", k, (long long)n_host[k]);
    max_n = n_host[k] > max_n ? n_host[k] : max_n;
  }
  EV_CHECK_ARG(meter_size_ok(max_n) && loud_grid_ok(max_n, sample_rate), "ev_meter: an item of %lld samples is too long", max_n);
  for (int i = 0; i < 10; ++i) EV_CHECK_ARG(isfinite(kcoef[i]), "ev_meter: kcoef[%d] is not finite", i);
  const int W = restart_warmup(kcoef);
  EV_CHECK_ARG(W > 0, "ev_meter: the K-weighting cascade kcoef is unstable or its poles are too close to the unit circle");
  EV_CHECK_ARG(phases >= 0 && phases <= MT_MAX_PHASES && taps >= 1 && taps <= MT_MAX_TAPS && taps % 2 == 1 &&
               phases * taps <= MT_MAX_BANK && (bank || phases == 0),
               "ev_meter: a bank of %d phases of %d taps (odd taps, at most %d phases, %d taps, %d in all; NULL only without phases)",
               phases, taps, MT_MAX_PHASES, MT_MAX_TAPS, MT_MAX_BANK);
  const int S = sample_rate / 10;
  EV_CHECK_ARG(!(momentary || short_term) || series_stride >= max_n / S,
               "ev_meter: series_stride=%lld must be at least %lld (the longest item's full sub-blocks)", series_stride, max_n / S);
  const size_t need = meter_ws_bytes(n_items, max_n, sample_rate);
  EV_CHECK_ARG(ws_bytes >= need, "ev_meter: workspace of %zu bytes, %zu needed", ws_bytes, need);
  EV_TRY(use_device_of(wav));
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long long max_sub = loud_max_sub(max_n, sample_rate), max_tiles = meter_tiles(max_n);
  const size_t cells = (size_t)n_items * (size_t)max_sub;
  char* w = static_cast<char*>(ws);
  double* energy = reinterpret_cast<double*>(w);
  w += align256(cells * sizeof(double));
  float* sub_peak = reinterpret_cast<float*>(w);
  w += align256(cells * sizeof(float));
  double* keys = reinterpret_cast<double*>(w);
  w += align256(cells * sizeof(double));
  float* tile_max = reinterpret_cast<float*>(w);
  w += align256((size_t)n_items * (size_t)max_tiles * sizeof(float));
  float* gain = reinterpret_cast<float*>(w);
  const int c = (taps - 1) / 2;
  const size_t smem = (size_t)(phases * taps + MP_TILE + 2 * c) * sizeof(float);
  static std::atomic<uint64_t> attr_devs{0};
  if (first_use_on_device(attr_devs))
    cudaFuncSetAttribute(meter_peak_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
  EV_TRY(launch_loud_subblock(wav, max_n, start, n, nullptr, n_items, sample_rate, kcoef, W, energy, sub_peak, st));
  EV_TRY(launch_loud_gate(max_n, n, nullptr, n_items, sample_rate, energy, sub_peak, -23.0, results, results + 5 * (size_t)n_items, gain,
                          st));
  EV_TRY(launch("meter_peak_kernel", meter_peak_kernel, dim3((unsigned)max_tiles, n_items), MP_THREADS, smem, st, wav, start, n, max_n,
                bank, phases, taps, max_tiles, tile_max));
  return launch("meter_range_kernel", meter_range_kernel, dim3(n_items), MR_THREADS, 0, st, n, max_n, S, max_sub, (const double*)energy,
                keys, max_tiles, (const float*)tile_max, results, n_items, momentary, short_term, series_stride);
}

}  // extern "C"
