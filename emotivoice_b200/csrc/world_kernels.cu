// Spectral envelopes of recordings: WORLD's CheapTrick at pyworld's defaults (q1 = -0.15, f0_floor 71, fft_size from the
// rate), and pysptk's sp2mc (SPTK freqt over the real cepstrum) as one fp64 matrix per (fft_size, order, alpha) applied to
// the log envelope.  oracle/world_oracle.py is the fp64 restatement these kernels follow step by step; its docstring lists
// where WORLD's and SPTK's behaviour was assumed (W1-W11) and the same choices are made here.
//
//   world_envelope_kernel  one CTA per (frame, item): the F0-adaptive window (W3), a radix-2 fp64 FFT in shared memory (W4),
//                          the DC correction (W5), the linear smoothing as a local sum of the mirrored spectrum (W6),
//                          the eps floor (W7), the log spectrum's cepstrum, the two lifters and the inverse (W8); then the
//                          envelope and / or table @ log envelope (the mel-cepstrum), written straight from shared memory
//   world_sp2mc_kernel     one CTA per frame: table @ log(sp) of caller envelopes
// fp64 throughout.  The window sums and the table products are block reductions in a fixed order, so results are
// not the oracle's bits but are the same bits for an item in any batch, order or padding.  No allocation, no sync.
#include <math.h>

#include "ev_common.cuh"

namespace ev {

constexpr int kWThreads = 256;
constexpr int kWMaxFft = 2048;
constexpr int kWMaxOut = 256;
constexpr double kWPi = 3.1415926535897932384;
constexpr double kWQ1 = -0.15, kWDefaultF0 = 500.0, kWEps = 2.220446049250313e-16, kWFloor = 71.0;

struct WorldParams {
  const double* x;
  long long item_stride;
  const int64_t* n_samples;
  int fs, F, n_fft, log_n, min_len;
  double frame_period;
  const double* f0;      // (B, F)
  double* sp;            // (B, F, n_fft / 2 + 1) or null
  const double* table;   // (n_out, n_fft / 2 + 1) or null
  int n_out;
  double* mc;            // (B, F, n_out) or null
  int32_t* status;
};

static int world_fft_size(int fs) { return 1 << (1 + (int)(log(3.0 * fs / kWFloor + 1.0) / log(2.0))); }
static int world_round(double x) { return x < 0 ? (int)(x - 0.5) : (int)(x + 0.5); }

__device__ __forceinline__ int wround(double x) { return x < 0 ? (int)(x - 0.5) : (int)(x + 0.5); }

// a deterministic block sum of two values (fixed warp order); every thread gets the totals
__device__ __forceinline__ double2 block_sum2(double a, double b, double2* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) red[w] = make_double2(a, b);
  __syncthreads();
  double2 s = make_double2(0.0, 0.0);
  for (int i = 0; i < kWThreads / 32; ++i) {
    s.x += red[i].x;
    s.y += red[i].y;
  }
  __syncthreads();
  return s;
}

// in place, forward sign, natural order in and out; tw[m] = exp(-2 pi i m / n), m < n / 2
__device__ void fft_inplace(double2* a, const double2* tw, int n, int log_n) {
  for (int i = threadIdx.x; i < n; i += kWThreads) {
    const int j = (int)(__brev((unsigned)i) >> (32 - log_n));
    if (i < j) {
      const double2 t = a[i];
      a[i] = a[j];
      a[j] = t;
    }
  }
  __syncthreads();
  for (int s = 1; s <= log_n; ++s) {
    const int h = 1 << (s - 1), step = n >> s;
    for (int j = threadIdx.x; j < n / 2; j += kWThreads) {
      const int k = j & (h - 1), i0 = ((j >> (s - 1)) << s) + k, i1 = i0 + h;
      const double2 w = tw[k * step], u = a[i0], v = a[i1];
      const double2 t = make_double2(v.x * w.x - v.y * w.y, v.x * w.y + v.y * w.x);
      a[i0] = make_double2(u.x + t.x, u.y + t.y);
      a[i1] = make_double2(u.x - t.x, u.y - t.y);
    }
    __syncthreads();
  }
}

// WORLD's interp1Q at one point: y sampled at x0 + k dx (k < len), read at xi
__device__ __forceinline__ double interp1q(double x0, double dx, const double* y, int len, double xi) {
  const double q = (xi - x0) / dx;
  const int base = (int)q;
  const double dy = base + 1 < len ? y[base + 1] - y[base] : 0.0;
  return y[base] + dy * (q - base);
}

// out[k] = sum_n table[k, n] lg[n], k < n_out: one warp per output, lanes over n, a fixed shuffle tree
__device__ __forceinline__ void table_products(const double* lg, const double* __restrict__ table, int bins, int n_out, double* out) {
  const int lane = threadIdx.x & 31;
  for (int k = threadIdx.x >> 5; k < n_out; k += kWThreads / 32) {
    const double* t = table + (size_t)k * bins;
    double acc = 0.0;
    for (int n = lane; n < bins; n += 32) acc = fma(t[n], lg[n], acc);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) out[k] = acc;
  }
}

__device__ __forceinline__ long long w_item_len(const WorldParams& p, int b) {
  return p.n_samples ? (long long)p.n_samples[b] : p.item_stride;
}

// shared memory: data (n_fft double2) | twiddles (n_fft / 2 double2) | pw (n_fft / 2 + 1 doubles) | block-sum scratch
__global__ void __launch_bounds__(kWThreads) world_envelope_kernel(const WorldParams p) {
  pdl_entry();
  extern __shared__ __align__(16) double2 wsm[];
  __shared__ double2 red[kWThreads / 32];
  const int f = blockIdx.x, b = blockIdx.y;
  const int N = p.n_fft, half = N / 2, bins = half + 1;
  const long long n = w_item_len(p, b);
  const bool ok = n >= p.min_len && n <= p.item_stride;
  int Fb = 0;
  if (ok) {
    Fb = (int)(1000.0 * (double)n / (double)p.fs / p.frame_period) + 1;
    Fb = Fb < p.F ? Fb : p.F;
  }
  const size_t row = (size_t)b * p.F + f;
  if (p.status) {
    if (!ok && f == 0 && threadIdx.x == 0) atomicOr(p.status, 2);
    if (f < Fb) {                                            // frame f checks its share of the item's samples
      const double* x = p.x + (size_t)b * p.item_stride;
      int bad = 0;
      for (long long i = n * f / Fb + threadIdx.x; i < n * (f + 1) / Fb; i += kWThreads) bad |= !isfinite(x[i]);
      if (__syncthreads_or(bad) && threadIdx.x == 0) atomicOr(p.status, 1);
    }
  }
  if (f >= Fb) {
    if (p.sp)
      for (int i = threadIdx.x; i < bins; i += kWThreads) p.sp[row * bins + i] = 0.0;
    if (p.mc)
      for (int i = threadIdx.x; i < p.n_out; i += kWThreads) p.mc[row * p.n_out + i] = 0.0;
    return;
  }
  double2* data = wsm;
  double2* tw = wsm + N;
  double* pw = reinterpret_cast<double*>(tw + half);
  const double fs = (double)p.fs;
  double f0 = p.f0[row];
  if (!(f0 > 3.0 * fs / (N - 3.0) && f0 <= fs / 4.0)) f0 = kWDefaultF0;     // W2
  for (int m = threadIdx.x; m < half; m += kWThreads) {
    double s, c;
    sincospi(2.0 * (double)m / (double)N, &s, &c);
    tw[m] = make_double2(c, -s);
  }
  // W3: window, normalised; weighted mean removed
  const double t = __ddiv_rn(__dmul_rn((double)f, p.frame_period), 1000.0);
  const int h = wround(1.5 * fs / f0), len = 2 * h + 1;
  const long long origin = wround(__dadd_rn(__dmul_rn(t, fs), 0.001));
  const double* x = p.x + (size_t)b * p.item_stride;
  double e = 0.0;
  for (int i = threadIdx.x; i < len; i += kWThreads) {
    const double w = 0.5 * cos(kWPi * ((double)(i - h) / 1.5 / fs) * f0) + 0.5;
    data[i].y = w;
    e += w * w;
  }
  const double norm = sqrt(block_sum2(e, 0.0, red).x);
  double sxw = 0.0, sw = 0.0;
  for (int i = threadIdx.x; i < len; i += kWThreads) {
    long long at = origin + i - h;
    at = at < 0 ? 0 : (at > n - 1 ? n - 1 : at);
    const double w = data[i].y / norm, xw = x[at] * w;
    data[i] = make_double2(xw, w);
    sxw += xw;
    sw += w;
  }
  const double2 s = block_sum2(sxw, sw, red);
  const double coef = s.x / s.y;
  for (int i = threadIdx.x; i < N; i += kWThreads)
    data[i] = i < len ? make_double2(data[i].x - data[i].y * coef, 0.0) : make_double2(0.0, 0.0);
  __syncthreads();
  // W4: power spectrum
  fft_inplace(data, tw, N, p.log_n);
  for (int k = threadIdx.x; k < bins; k += kWThreads) pw[k] = data[k].x * data[k].x + data[k].y * data[k].y;
  __syncthreads();
  // W5: DC correction, the replica gathered into scratch first
  double* tmp = reinterpret_cast<double*>(data);
  const int u = 2 + (int)(f0 * N / fs);
  const double df = fs / N;
  for (int i = threadIdx.x; i < u - 1; i += kWThreads) tmp[i] = interp1q(f0, -df, pw, u + 1, (double)i * fs / N);
  __syncthreads();
  for (int i = threadIdx.x; i < u - 1; i += kWThreads) pw[i] += tmp[i];
  __syncthreads();
  // W6: linear smoothing.  WORLD differences two interp1Q reads of the running sum S of the mirrored spectrum m; in exact
  // arithmetic hi - lo = m[bl+1] (1 - fl) + m[bl+2] + ... + m[bh] + m[bh+1] fh, which is summed here instead: every term is
  // >= 0, so the result is too, and no bin loses its digits to the cancellation of two sums of the whole spectrum.
  const double width = f0 * 2.0 / 3.0;
  const int bb = (int)(width * N / fs) + 1, ml = half + 2 * bb + 1;
  double* seg = tmp;
  for (int j = threadIdx.x; j < ml; j += kWThreads) {
    const int k = j < bb ? bb - j : (j < half + bb ? j - bb : half - (j - half - bb));
    seg[j] = pw[k] * fs / N;
  }
  __syncthreads();
  const double origin_f = -(bb - 0.5) * fs / N;
  for (int i = threadIdx.x; i < bins; i += kWThreads) {
    const double ax = __dsub_rn(__dmul_rn((double)i / N, fs), width / 2.0);
    const double ql = (ax - origin_f) / df, qh = (ax + width - origin_f) / df;
    const int bl = (int)ql, bh = (int)qh;
    const double fl = ql - bl, fh = qh - bh;
    double acc;
    if (bh == bl) {
      acc = (bl + 1 < ml ? seg[bl + 1] : 0.0) * (fh - fl);
    } else {
      acc = seg[bl + 1] * (1.0 - fl);
      for (int j = bl + 2; j <= bh; ++j) acc += seg[j];
      if (bh + 1 < ml) acc += seg[bh + 1] * fh;
    }
    pw[i] = acc / width + kWEps;                                           // W7
  }
  __syncthreads();
  // W8: cepstrum of the log spectrum, lifters, back
  for (int k = threadIdx.x; k < bins; k += kWThreads) pw[k] = log(pw[k]);
  __syncthreads();
  for (int k = threadIdx.x; k < N; k += kWThreads) data[k] = make_double2(pw[k <= half ? k : N - k], 0.0);
  __syncthreads();
  fft_inplace(data, tw, N, p.log_n);
  for (int k = threadIdx.x; k < bins; k += kWThreads) {
    const double q = (double)k / fs;
    const double sm = k == 0 ? 1.0 : sin(kWPi * f0 * q) / (kWPi * f0 * q);
    const double cp = (1.0 - 2.0 * kWQ1) + 2.0 * kWQ1 * cos(2.0 * kWPi * q * f0);
    pw[k] = data[k].x * sm * cp / N;
  }
  __syncthreads();
  for (int k = threadIdx.x; k < N; k += kWThreads) data[k] = make_double2(pw[k <= half ? k : N - k], 0.0);
  __syncthreads();
  fft_inplace(data, tw, N, p.log_n);
  for (int k = threadIdx.x; k < bins; k += kWThreads) {
    pw[k] = data[k].x;                                                     // the log envelope
    if (p.sp) p.sp[row * bins + k] = exp(data[k].x);
  }
  if (p.mc) {
    __syncthreads();
    table_products(pw, p.table, bins, p.n_out, p.mc + row * p.n_out);
  }
}

__global__ void __launch_bounds__(kWThreads) world_sp2mc_kernel(const double* __restrict__ sp, int bins, const double* __restrict__ table,
                                                                int n_out, double* __restrict__ mc) {
  pdl_entry();
  __shared__ double lg[kWMaxFft / 2 + 1];
  const size_t row = blockIdx.x;
  for (int k = threadIdx.x; k < bins; k += kWThreads) lg[k] = log(sp[row * bins + k]);
  __syncthreads();
  table_products(lg, table, bins, n_out, mc + row * n_out);
}

static size_t world_smem(int n_fft) {
  return (size_t)n_fft * sizeof(double2) + (size_t)(n_fft / 2) * sizeof(double2) + (size_t)(n_fft / 2 + 1) * sizeof(double);
}

static bool world_bins_ok(int bins) {
  const int n = 2 * (bins - 1);
  return bins >= 3 && n <= kWMaxFft && (n & (n - 1)) == 0;
}

}  // namespace ev

using namespace ev;

extern "C" {

int ev_world_envelope(const double* x, long long item_stride, const int64_t* n_samples, int B, int fs, double frame_period, int F,
                      const double* f0, double* sp, const double* mc_table, int n_out, double* mc, int32_t* status, void* stream) {
  EV_CHECK_ARG(x && f0 && (sp || mc), "ev_world_envelope: null argument (x, f0 and one of sp, mc are needed)");
  EV_CHECK_ARG(fs >= 8000 && fs <= 48000, "ev_world_envelope: fs %d is not in [8000, 48000]", fs);
  EV_CHECK_ARG(frame_period >= 0.25 && frame_period <= 1000.0, "ev_world_envelope: frame_period %g ms is not in [0.25, 1000]",
               frame_period);
  EV_CHECK_ARG(B > 0 && B <= 65535 && item_stride > 0 && F == (int)(1000.0 * (double)item_stride / (double)fs / frame_period) + 1,
               "ev_world_envelope: B=%d item_stride=%lld F=%d (F must be the row's frame count)", B, item_stride, F);
  EV_CHECK_ARG(!mc || (mc_table && n_out >= 1 && n_out <= kWMaxOut), "ev_world_envelope: mc needs a table of 1 to %d rows, got %d",
               kWMaxOut, n_out);
  const int min_len = 2 * world_round(fs / 50.0) + 1;
  EV_CHECK_ARG(n_samples || item_stride >= min_len, "ev_world_envelope: items of %lld samples are shorter than %d", item_stride, min_len);
  EV_TRY(use_device_of(x));
  WorldParams p;
  p.x = x;
  p.item_stride = item_stride;
  p.n_samples = n_samples;
  p.fs = fs;
  p.F = F;
  p.n_fft = world_fft_size(fs);
  p.log_n = 0;
  while ((1 << p.log_n) < p.n_fft) ++p.log_n;
  p.min_len = min_len;
  p.frame_period = frame_period;
  p.f0 = f0;
  p.sp = sp;
  p.table = mc ? mc_table : nullptr;
  p.n_out = mc ? n_out : 0;
  p.mc = mc;
  p.status = status;
  static std::atomic<uint64_t> attr_devs{0};
  if (first_use_on_device(attr_devs))
    cudaFuncSetAttribute(world_envelope_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)world_smem(kWMaxFft));
  return launch("world_envelope_kernel", world_envelope_kernel, dim3(F, B), kWThreads, world_smem(p.n_fft),
                reinterpret_cast<cudaStream_t>(stream), p);
}

int ev_sp2mc(const double* sp, long long n_frames, int bins, const double* table, int n_out, double* mc, void* stream) {
  EV_CHECK_ARG(sp && table && mc, "ev_sp2mc: null argument");
  EV_CHECK_ARG(world_bins_ok(bins), "ev_sp2mc: bins=%d must be fft_size / 2 + 1 with fft_size a power of two in [4, %d]", bins,
               kWMaxFft);
  EV_CHECK_ARG(n_out >= 1 && n_out <= kWMaxOut, "ev_sp2mc: n_out=%d must lie in [1, %d]", n_out, kWMaxOut);
  EV_CHECK_ARG(n_frames >= 0 && n_frames <= 0x7fffffffll, "ev_sp2mc: n_frames=%lld must lie in [0, 2^31)", n_frames);
  if (n_frames == 0) return EV_OK;
  EV_TRY(use_device_of(sp));
  return launch("world_sp2mc_kernel", world_sp2mc_kernel, dim3((unsigned)n_frames), kWThreads, 0, reinterpret_cast<cudaStream_t>(stream),
                sp, bins, table, n_out, mc);
}

}  // extern "C"
