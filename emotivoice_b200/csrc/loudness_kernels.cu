// Integrated loudness of output waveforms (ITU-R BS.1770-4, one channel) and the gain that brings each output to a target
// (ev_loudness; the gain is applied by audio_out_kernel).
//
// Two launches.  loud_subblock_kernel: one thread per (listed item, 100 ms sub-block of S = sr / 10 samples).  The thread runs
// the K-weighting cascade (high shelf, then high pass; fp32 direct form I) from zero state over the W samples before its
// sub-block (read as zero before the item's start, which is the same as starting there) and then over the sub-block, and
// writes the sub-block's sum of squares (fp64) and its |x| maximum.  W is chosen on the host so that the restart's transient,
// which decays as the largest pole radius r of the cascade, is below W * r^W <= 1e-10; no state is carried between sub-blocks,
// so a sub-block's result depends only on its item's samples and the rate.  The 32 sub-blocks of a warp are consecutive: the
// warp stages 32 samples of each lane's span at a time in shared memory with coalesced loads.  Samples at or past n_in[b] are
// never read; a last, partial sub-block only gives its peak.  Item b starts at wav + b * item_stride, or at wav + start[b]
// when ev_meter passes the items' start offsets (item_stride is then the longest item's length, which bounds n_in).
// loud_gate_kernel: one CTA per listed item.  Gating blocks are four consecutive sub-blocks (400 ms, 75 % overlap); block
// loudness l = -0.691 + 10 log10(mean square), the absolute gate keeps l > -70, the relative gate l > (loudness of those) - 10,
// and L is the loudness of the blocks that pass both.  Sums are fp64 in a fixed order (thread t takes blocks t, t + T, ...,
// then a fixed tree), so L does not depend on the batch.  Gain g = min(10^((T - L) / 20), 10^(-1/20) / peak) in fp64, 1 where
// L = -inf (shorter than one block, or no block passes the gates).
#include <math.h>

#include "ev_common.cuh"

namespace ev {

constexpr int LD_THREADS = 128, LD_WARPS = LD_THREADS / 32;
constexpr int LG_THREADS = 256;
constexpr double LD_TRANSIENT = 1e-10;      // W * r^W bound of the restart
constexpr int LD_MAX_WARMUP = 1 << 20;
constexpr int LD_MIN_RATE = 4000, LD_MAX_RATE = 192000;

struct KCoef {
  float s0, s1, s2, sa1, sa2;   // shelf b0, b1, b2, a1, a2
  float h0, h1, h2, ha1, ha2;   // high pass
};

__global__ void __launch_bounds__(LD_THREADS) loud_subblock_kernel(const float* __restrict__ wav, long long item_stride,
                                                                   const int64_t* __restrict__ start,
                                                                   const int64_t* __restrict__ n_in, const int64_t* __restrict__ items,
                                                                   int S, int W, long long max_sub, KCoef c,
                                                                   double* __restrict__ energy, float* __restrict__ peak) {
  pdl_entry();
  __shared__ float stage[LD_WARPS][32][33];
  const int k = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long b = items ? items[k] : k;
  const long long n = min((long long)n_in[b], item_stride);
  const long long n_sub = (n + S - 1) / S;                    // sub-blocks holding samples: the last one may be partial
  const long long j0 = ((long long)blockIdx.x * LD_WARPS + warp) * 32;
  if (j0 >= n_sub) return;                                    // whole warps only
  const long long j = j0 + lane;
  const float* x = wav + (start ? start[b] : b * item_stride);
  float (*buf)[33] = stage[warp];
  float sx1 = 0.f, sx2 = 0.f, sy1 = 0.f, sy2 = 0.f, hy1 = 0.f, hy2 = 0.f;
  double acc = 0.0;
  float pk = 0.f;
  const int span = W + S;
  for (int p0 = 0; p0 < span; p0 += 32) {
    for (int t = 0; t < 32; ++t) {                            // lane l loads sample p0 + l of lane t's span
      const long long s = (j0 + t) * S - W + p0 + lane;
      buf[t][lane] = (s >= 0 && s < n) ? x[s] : 0.f;
    }
    __syncwarp();
    for (int i = 0; i < 32; ++i) {
      const int p = p0 + i;
      const float xv = buf[lane][i];
      const float sy = fmaf(-c.sa1, sy1, fmaf(-c.sa2, sy2, fmaf(c.s2, sx2, fmaf(c.s1, sx1, c.s0 * xv))));
      sx2 = sx1; sx1 = xv;
      const float hy = fmaf(-c.ha1, hy1, fmaf(-c.ha2, hy2, fmaf(c.h2, sy2, fmaf(c.h1, sy1, c.h0 * sy))));
      sy2 = sy1; sy1 = sy;
      hy2 = hy1; hy1 = hy;
      if (p >= W && p < span && j * S + (p - W) < n) {
        acc = fma((double)hy, (double)hy, acc);
        pk = fmaxf(pk, fabsf(xv));
      }
    }
    __syncwarp();
  }
  if (j < n_sub) {
    energy[k * max_sub + j] = acc;
    peak[k * max_sub + j] = pk;
  }
}

__device__ __forceinline__ double block_loudness(double ms) { return -0.691 + 10.0 * log10(ms); }

// fixed-order CTA sums of (count, sum) pairs: thread partials, then a tree over the threads
__device__ __forceinline__ void cta_sum(double& s, double& cnt, double* red) {
  red[threadIdx.x] = s;
  red[LG_THREADS + threadIdx.x] = cnt;
  __syncthreads();
  for (int h = LG_THREADS / 2; h > 0; h >>= 1) {
    if ((int)threadIdx.x < h) {
      red[threadIdx.x] += red[threadIdx.x + h];
      red[LG_THREADS + threadIdx.x] += red[LG_THREADS + threadIdx.x + h];
    }
    __syncthreads();
  }
  s = red[0];
  cnt = red[LG_THREADS];
  __syncthreads();
}

__global__ void __launch_bounds__(LG_THREADS) loud_gate_kernel(long long item_stride, const int64_t* __restrict__ n_in,
                                                               const int64_t* __restrict__ items, int S, long long max_sub,
                                                               const double* __restrict__ energy, const float* __restrict__ peak,
                                                               double target, float* __restrict__ lufs, float* __restrict__ peak_out,
                                                               float* __restrict__ gain) {
  pdl_entry();
  __shared__ double red[2 * LG_THREADS];
  __shared__ float pred[LG_THREADS];
  const int k = blockIdx.x;
  const long long b = items ? items[k] : k;
  const long long n = min((long long)n_in[b], item_stride);
  const long long n_full = n / S, n_sub = (n + S - 1) / S, n_blk = n_full - 3;
  const double* e = energy + k * max_sub;
  const double inv = 1.0 / (4.0 * S);
  float pk = 0.f;
  for (long long j = threadIdx.x; j < n_sub; j += LG_THREADS) pk = fmaxf(pk, peak[k * max_sub + j]);
  pred[threadIdx.x] = pk;
  __syncthreads();
  for (int h = LG_THREADS / 2; h > 0; h >>= 1) {
    if ((int)threadIdx.x < h) pred[threadIdx.x] = fmaxf(pred[threadIdx.x], pred[threadIdx.x + h]);
    __syncthreads();
  }
  pk = pred[0];
  // absolute gate
  double s1 = 0.0, c1 = 0.0;
  for (long long j = threadIdx.x; j < n_blk; j += LG_THREADS) {
    const double z = (((e[j] + e[j + 1]) + e[j + 2]) + e[j + 3]) * inv;
    if (block_loudness(z) > -70.0) { s1 += z; c1 += 1.0; }
  }
  cta_sum(s1, c1, red);
  double L = -INFINITY;
  if (c1 > 0.0) {
    const double rel = block_loudness(s1 / c1) - 10.0;
    double s2 = 0.0, c2 = 0.0;
    for (long long j = threadIdx.x; j < n_blk; j += LG_THREADS) {
      const double z = (((e[j] + e[j + 1]) + e[j + 2]) + e[j + 3]) * inv;
      const double l = block_loudness(z);
      if (l > -70.0 && l > rel) { s2 += z; c2 += 1.0; }
    }
    cta_sum(s2, c2, red);
    if (c2 > 0.0) L = block_loudness(s2 / c2);
  }
  if (threadIdx.x == 0) {
    double g = 1.0;
    if (L > -INFINITY) g = fmin(pow(10.0, (target - L) / 20.0), pow(10.0, -1.0 / 20.0) / (double)pk);
    lufs[k] = (float)L;
    peak_out[k] = pk;
    gain[k] = (float)g;
  }
}

// largest |pole| of z^2 + a1 z + a2
static double pole_radius(double a1, double a2) {
  const double d = a1 * a1 - 4.0 * a2;
  if (d < 0.0) return sqrt(a2);
  const double s = sqrt(d);
  return fmax(fabs((-a1 + s) / 2.0), fabs((-a1 - s) / 2.0));
}

// W: the smallest multiple of 32 with W * r^W <= LD_TRANSIENT, or -1 (unstable cascade, or W above LD_MAX_WARMUP)
int restart_warmup(const double* kc) {
  const double r = fmax(pole_radius(kc[3], kc[4]), pole_radius(kc[8], kc[9]));
  if (!(r < 1.0)) return -1;
  if (r == 0.0) return 32;
  for (int W = 32; W <= LD_MAX_WARMUP; W += 32)
    if (log((double)W) + W * log(r) <= log(LD_TRANSIENT)) return W;
  return -1;
}

long long loud_max_sub(long long max_n, int sample_rate) { return (max_n + sample_rate / 10 - 1) / (sample_rate / 10); }

bool loud_grid_ok(long long max_n, int sample_rate) { return (loud_max_sub(max_n, sample_rate) + LD_THREADS - 1) / LD_THREADS <= 0x7fffffffll; }

int launch_loud_subblock(const float* wav, long long item_stride, const int64_t* start, const int64_t* n_in, const int64_t* items,
                         int n_items, int sample_rate, const double* kcoef, int W, double* energy, float* peak, cudaStream_t st) {
  const long long max_sub = loud_max_sub(item_stride, sample_rate);
  KCoef c;
  c.s0 = (float)kcoef[0]; c.s1 = (float)kcoef[1]; c.s2 = (float)kcoef[2]; c.sa1 = (float)kcoef[3]; c.sa2 = (float)kcoef[4];
  c.h0 = (float)kcoef[5]; c.h1 = (float)kcoef[6]; c.h2 = (float)kcoef[7]; c.ha1 = (float)kcoef[8]; c.ha2 = (float)kcoef[9];
  const long long gx = (max_sub + LD_THREADS - 1) / LD_THREADS;
  return launch("loud_subblock_kernel", loud_subblock_kernel, dim3((unsigned)gx, n_items), LD_THREADS, 0, st, wav, item_stride, start,
                n_in, items, sample_rate / 10, W, max_sub, c, energy, peak);
}

int launch_loud_gate(long long item_stride, const int64_t* n_in, const int64_t* items, int n_items, int sample_rate,
                     const double* energy, const float* peak, double target, float* lufs, float* peak_out, float* gain, cudaStream_t st) {
  return launch("loud_gate_kernel", loud_gate_kernel, dim3(n_items), LG_THREADS, 0, st, item_stride, n_in, items, sample_rate / 10,
                loud_max_sub(item_stride, sample_rate), energy, peak, target, lufs, peak_out, gain);
}

static size_t loud_ws_bytes(int n_items, long long max_n, int sample_rate) {
  const size_t cells = (size_t)n_items * (size_t)loud_max_sub(max_n, sample_rate);
  return cells * sizeof(double) + ((cells * sizeof(float) + 255) & ~(size_t)255);
}

static bool loud_args_ok(int n_items, long long max_n, int sample_rate) {
  return n_items >= 1 && n_items <= 65535 && max_n >= 1 && sample_rate >= LD_MIN_RATE &&
         sample_rate <= LD_MAX_RATE && sample_rate % 10 == 0;
}

}  // namespace ev

using namespace ev;

extern "C" {

size_t ev_loudness_workspace_bytes(int n_items, long long max_n, int sample_rate) {
  return loud_args_ok(n_items, max_n, sample_rate) ? loud_ws_bytes(n_items, max_n, sample_rate) : 0;
}

int ev_loudness(const float* wav, long long item_stride, const int64_t* n_in, const int64_t* items, int n_items, int sample_rate,
                const double* kcoef, float target_lufs, float* lufs, float* peak, float* gain, void* ws, size_t ws_bytes, void* stream) {
  EV_CHECK_ARG(wav && n_in && kcoef && lufs && peak && gain && ws, "ev_loudness: null argument");
  EV_CHECK_ARG(n_items >= 1 && n_items <= 65535, "ev_loudness: n_items=%d must lie in [1, 65535]", n_items);
  EV_CHECK_ARG(item_stride >= 1, "ev_loudness: item_stride=%lld must be at least 1", item_stride);
  EV_CHECK_ARG(sample_rate % 10 == 0 && sample_rate >= LD_MIN_RATE && sample_rate <= LD_MAX_RATE,
               "ev_loudness: sample_rate=%d must be a multiple of 10 in [%d, %d] (100 ms sub-blocks)", sample_rate,
               LD_MIN_RATE, LD_MAX_RATE);
  EV_CHECK_ARG(target_lufs >= -70.f && target_lufs <= 0.f, "ev_loudness: target_lufs=%g must lie in [-70, 0]", (double)target_lufs);
  for (int i = 0; i < 10; ++i) EV_CHECK_ARG(isfinite(kcoef[i]), "ev_loudness: kcoef[%d] is not finite", i);
  const int W = restart_warmup(kcoef);
  EV_CHECK_ARG(W > 0, "ev_loudness: the K-weighting cascade kcoef is unstable or its poles are too close to the unit circle");
  const size_t need = loud_ws_bytes(n_items, item_stride, sample_rate);
  EV_CHECK_ARG(ws_bytes >= need, "ev_loudness: workspace of %zu bytes, %zu needed", ws_bytes, need);
  EV_TRY(use_device_of(wav));
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long long max_sub = loud_max_sub(item_stride, sample_rate);
  EV_CHECK_ARG(loud_grid_ok(item_stride, sample_rate), "ev_loudness: item_stride=%lld is too long", item_stride);
  double* energy = static_cast<double*>(ws);
  float* pks = reinterpret_cast<float*>(energy + (size_t)n_items * max_sub);
  EV_TRY(launch_loud_subblock(wav, item_stride, nullptr, n_in, items, n_items, sample_rate, kcoef, W, energy, pks, st));
  return launch_loud_gate(item_stride, n_in, items, n_items, sample_rate, energy, pks, (double)target_lufs, lufs, peak, gain, st);
}

}  // extern "C"
