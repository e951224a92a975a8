// Pitch of recordings: pyworld.dio + pyworld.stonemask at pyworld's defaults (f0_floor 71, f0_ceil 800, 2 channels per octave,
// speed 1, allowed_range 0.1), the two calls of the reference's feats.Pitch (models/prompt_tts_modified/feats.py:114-131), and
// its continuous interpolation and log.  oracle/pitch_oracle.py is the fp64 restatement these kernels follow step by step; its
// docstring lists where WORLD's behaviour was assumed (D1-D9, S1-S4) and the same choices are made here.
//
// fp64 throughout: the result is a chain of discrete decisions (zero-crossing signs, the argmin over band scores, the
// allowed_range tests), and the GPU agrees with the oracle on them only when its values carry the oracle's precision.
//
//   pitch_taps_kernel       the low-cut and the 7 Nuttall low-passes (D3, D4), reversed so each FIR sums in ascending order
//   pitch_mean_kernel       one CTA per item: the mean over the N + 1 analysed samples (D2)
//   pitch_lowcut_kernel     direct FIR of the mean-removed item with the low-cut, over the span the bands read
//   pitch_band_kernel       direct FIR of that with each band's low-pass, delay-compensated (D4); shared-memory tile + halo
//   pitch_events_kernel     one CTA per (item, band, kind): events compacted by a block scan (D5)
//   pitch_cand_kernel       one thread per frame: interpolated intervals, candidates, scores, the best band (D6-D8)
//   pitch_contour_kernel    one CTA per item: FixF0Contour steps 1-2 per frame, the sequential steps 3-4 by one thread (D9)
//   pitch_stonemask_kernel  one warp per frame, unvoiced frames skipped: the harmonic bins as direct DFT sums (S1-S4)
//   pitch_output_kernel     one CTA per item: continuous interpolation and log, 0 past the item's own frames
// Products and sums whose rounding the oracle fixes use __dmul_rn / __dadd_rn, so no multiply-add is contracted.  Every
// output is computed from its own item in a fixed order: a batch is bitwise its items' single calls.  No allocation, no sync.
#include <math.h>
#include "ev_common.cuh"

namespace ev {

constexpr int kBands = 7;
constexpr int kKinds = 4;
constexpr int kMaxHalf = 2048;            // >= round(2 fs / b_0) at fs <= 48000
constexpr double kMaxValue = 100000.0;
constexpr double kGuard = 1e-12;
constexpr double kFloor = 71.0, kCeil = 800.0, kAllowed = 0.1, kFloorStone = 40.0;
constexpr double kPi = 3.1415926535897932384;
constexpr double kLog2 = 0.69314718055994529;
constexpr int kFirTile = 256;
constexpr int kStoneWarps = 4;

struct PitchLayout {
  int c, halves[kBands], l0, r;
  double bound[kBands];
  long long M, S1, cap;
  size_t off_taps, off_mean, off_ylc, off_band, off_ev, off_cnt, off_cand, off_best, off_f0, off_s, off_ref, off_nb, total;
  long long tap_off[kBands + 1];  // band taps start after the low-cut's 2c + 1
};

struct PitchParams {
  const double* x;
  long long item_stride;
  const int64_t* n_samples;
  int fs, F, flags;
  double frame_period;
  PitchLayout lay;
  double* ws;
  double* raw_f0;   // (B, F): DIO's output
  double* pitch;    // (B, F)
  int32_t* status;
};

static int host_round(double x) { return x < 0 ? (int)(x - 0.5) : (int)(x + 0.5); }

static PitchLayout pitch_layout(int B, long long item_stride, int fs, int F, double frame_period) {
  PitchLayout L;
  L.c = host_round(fs / 50.0);
  L.l0 = 0;
  for (int i = 0; i < kBands; ++i) {
    L.bound[i] = kFloor * pow(2.0, (i + 1) / 2.0);
    L.halves[i] = host_round(fs / L.bound[i] * 2.0);
    L.l0 = L.halves[i] > L.l0 ? L.halves[i] : L.l0;
  }
  L.r = frame_period > 0 ? (int)(0.5 + 1000.0 / frame_period / kFloor) * 2 + 1 : 0;
  L.M = item_stride + 1;
  L.S1 = L.M + 2ll * L.l0;
  L.cap = L.M / 2 + 2;
  long long taps = 2ll * L.c + 1;
  for (int i = 0; i < kBands; ++i) {
    L.tap_off[i] = taps;
    taps += 2ll * L.halves[i] + 1;
  }
  L.tap_off[kBands] = taps;
  size_t o = 0;
  auto take = [&](size_t n) { size_t at = o; o += (n + 1) & ~(size_t)1; return at; };   // 16-byte aligned regions (in doubles)
  L.off_taps = take(taps);
  L.off_mean = take(B);
  L.off_ylc = take((size_t)B * L.S1);
  L.off_band = take((size_t)B * kBands * L.M);
  L.off_ev = take((size_t)B * kBands * kKinds * L.cap);
  L.off_cnt = take((size_t)B * kBands * kKinds);                 // counts as int64 in double slots
  L.off_cand = take((size_t)B * kBands * F);
  L.off_best = take((size_t)B * F);
  L.off_f0 = take((size_t)B * F);
  L.off_s = take((size_t)B * F * 2);
  L.off_ref = take((size_t)B * F);
  L.off_nb = take((size_t)B * F * 2);                            // nearest voiced frames, int64
  L.total = o * sizeof(double);
  return L;
}

__device__ __forceinline__ long long item_len(const PitchParams& p, int b) {
  return p.n_samples ? (long long)p.n_samples[b] : p.item_stride;
}
__device__ __forceinline__ bool item_ok(const PitchParams& p, long long n) { return n >= 2ll * p.lay.c + 1 && n <= p.item_stride; }
__device__ __forceinline__ int item_frames(const PitchParams& p, long long n) {
  if (!item_ok(p, n)) return 0;
  const int f = (int)(1000.0 * (double)n / (double)p.fs / p.frame_period) + 1;
  return f < p.F ? f : p.F;
}
__device__ __forceinline__ int mround(double x) { return x < 0 ? (int)(x - 0.5) : (int)(x + 0.5); }

__device__ __forceinline__ double hann_tap(int i, int n) { return __dsub_rn(0.5, __dmul_rn(0.5, cos(i * 2.0 * kPi / (n + 1)))); }

// ---- filters -------------------------------------------------------------------------------------------------------------
__global__ void pitch_taps_kernel(const PitchParams p) {
  pdl_entry();
  double* taps = p.ws + p.lay.off_taps;
  const int c = p.lay.c, n = 2 * c + 1;
  __shared__ double ssum;
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int i = 1; i <= n; ++i) s = __dadd_rn(s, hann_tap(i, n));
    ssum = s;
  }
  __syncthreads();
  for (int j = threadIdx.x; j < n; j += blockDim.x) {   // reversed: taps[j] = g[2c - j]
    const int i = n - j;                                  // window index i (1-based) of g[2c - j]
    double g = -hann_tap(i, n) / ssum;
    if (j == c) g += 1.0;
    taps[j] = g;
  }
  for (int bd = 0; bd < kBands; ++bd) {
    const int m = 2 * p.lay.halves[bd] + 1;
    double* w = taps + p.lay.tap_off[bd];
    for (int j = threadIdx.x; j < m; j += blockDim.x) {
      const double tmp = (m - 1 - j) / (m - 1.0);
      w[j] = __dsub_rn(__dadd_rn(__dsub_rn(0.355768, __dmul_rn(0.487396, cos(2.0 * kPi * tmp))), __dmul_rn(0.144232, cos(4.0 * kPi * tmp))),
                       __dmul_rn(0.012604, cos(6.0 * kPi * tmp)));
    }
  }
}

__global__ void __launch_bounds__(512) pitch_mean_kernel(const PitchParams p) {
  pdl_entry();
  const int b = blockIdx.x;
  const long long n = item_len(p, b);
  __shared__ double part[512];
  __shared__ int bad;
  if (threadIdx.x == 0) bad = 0;
  __syncthreads();
  double s = 0.0;
  int nf = 0;
  if (item_ok(p, n)) {
    const double* x = p.x + (long long)b * p.item_stride;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) {
      const double v = x[i];
      nf |= !isfinite(v);
      s += v;
    }
  }
  if (nf) bad = 1;
  part[threadIdx.x] = s;
  __syncthreads();
  for (int h = blockDim.x / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) part[threadIdx.x] += part[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    p.ws[p.lay.off_mean + b] = part[0] / (double)(n + 1);
    if (p.status && bad) atomicOr(p.status, 1);
    if (p.status && !item_ok(p, n)) atomicOr(p.status, 2);
  }
}

// ylc_ext[t] = sum_j taps[j] y[t + 1 - l0 - c + j], y = the N samples minus the mean, then -mean at N, zero elsewhere.
__global__ void __launch_bounds__(kFirTile) pitch_lowcut_kernel(const PitchParams p) {
  pdl_entry();
  extern __shared__ double fsm[];
  const int b = blockIdx.y, c = p.lay.c, nt = 2 * c + 1;
  const long long n = item_len(p, b);
  if (!item_ok(p, n)) return;
  const long long t0 = (long long)blockIdx.x * kFirTile;
  const long long cnt = n + 1 + 2ll * p.lay.l0;
  if (t0 >= cnt) return;
  double* taps = fsm;
  double* span = fsm + nt;
  const double mean = p.ws[p.lay.off_mean + b];
  const double* x = p.x + (long long)b * p.item_stride;
  for (int j = threadIdx.x; j < nt; j += blockDim.x) taps[j] = p.ws[p.lay.off_taps + j];
  const long long u0 = t0 + 1 - p.lay.l0 - c;
  for (int i = threadIdx.x; i < kFirTile + nt - 1; i += blockDim.x) {
    const long long u = u0 + i;
    span[i] = (u < 0 || u > n) ? 0.0 : (u == n ? -mean : x[u] - mean);
  }
  __syncthreads();
  const long long t = t0 + threadIdx.x;
  if (t >= cnt) return;
  double acc = 0.0;
  for (int j = 0; j < nt; ++j) acc = __dadd_rn(acc, __dmul_rn(taps[j], span[threadIdx.x + j]));
  p.ws[p.lay.off_ylc + (long long)b * p.lay.S1 + t] = acc;
}

// band[i] = sum_k taps_b[k] ylc_ext[(l0 - L) + i + k], i < N + 1
__global__ void __launch_bounds__(kFirTile) pitch_band_kernel(const PitchParams p) {
  pdl_entry();
  extern __shared__ double fsm[];
  const int b = blockIdx.z, bd = blockIdx.y;
  const long long n = item_len(p, b);
  if (!item_ok(p, n)) return;
  const long long i0 = (long long)blockIdx.x * kFirTile;
  const long long m = n + 1;
  if (i0 >= m) return;
  const int L = p.lay.halves[bd], nt = 2 * L + 1;
  double* taps = fsm;
  double* span = fsm + nt;
  const double* tg = p.ws + p.lay.off_taps + p.lay.tap_off[bd];
  for (int j = threadIdx.x; j < nt; j += blockDim.x) taps[j] = tg[j];
  const double* ylc = p.ws + p.lay.off_ylc + (long long)b * p.lay.S1 + (p.lay.l0 - L) + i0;
  const long long avail = n + 1 + 2ll * p.lay.l0 - (p.lay.l0 - L) - i0;
  for (int i = threadIdx.x; i < kFirTile + nt - 1; i += blockDim.x) span[i] = i < avail ? ylc[i] : 0.0;
  __syncthreads();
  const long long i = i0 + threadIdx.x;
  if (i >= m) return;
  double acc = 0.0;
  for (int k = 0; k < nt; ++k) acc = __dadd_rn(acc, __dmul_rn(taps[k], span[threadIdx.x + k]));
  p.ws[p.lay.off_band + ((long long)b * kBands + bd) * p.lay.M + i] = acc;
}

// ---- events --------------------------------------------------------------------------------------------------------------
// kind 0: v; 1: -v; 2: d = (-v[i]) - (-v[i + 1]); 3: -d.  Negative-going zero crossings of the kind's sequence.
__device__ __forceinline__ double kind_val(const double* v, int kind, long long i) {
  if (kind == 0) return v[i];
  if (kind == 1) return -v[i];
  const double d = __dsub_rn(-v[i], -v[i + 1]);
  return kind == 2 ? d : -d;
}

__global__ void __launch_bounds__(1024) pitch_events_kernel(const PitchParams p) {
  pdl_entry();
  const int b = blockIdx.y, bd = blockIdx.x / kKinds, kind = blockIdx.x % kKinds;
  const long long n = item_len(p, b);
  const long long slot = ((long long)b * kBands + bd) * kKinds + kind;
  long long* cnt = reinterpret_cast<long long*>(p.ws + p.lay.off_cnt);
  if (!item_ok(p, n)) {
    if (threadIdx.x == 0) cnt[slot] = 0;
    return;
  }
  const double* v = p.ws + p.lay.off_band + ((long long)b * kBands + bd) * p.lay.M;
  double* ev = p.ws + p.lay.off_ev + slot * p.lay.cap;
  const long long len = (kind < 2 ? n + 1 : n);   // the sequence's length
  __shared__ int wsum[32];
  __shared__ long long base;
  if (threadIdx.x == 0) base = 0;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long long i0 = 0; i0 < len - 1; i0 += blockDim.x) {
    const long long i = i0 + threadIdx.x;
    bool hit = false;
    double a = 0.0, c = 0.0;
    if (i < len - 1) {
      a = kind_val(v, kind, i);
      c = kind_val(v, kind, i + 1);
      hit = a > 0.0 && c <= 0.0;
    }
    const unsigned bal = __ballot_sync(0xffffffffu, hit);
    __syncthreads();   // base and wsum of the previous round are consumed
    if (lane == 0) wsum[warp] = __popc(bal);
    __syncthreads();
    int before = 0, total = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) {
      before += w < warp ? wsum[w] : 0;
      total += wsum[w];
    }
    if (hit) {
      const long long at = base + before + __popc(bal & ((1u << lane) - 1u));
      const double e = (double)(i + 1);
      ev[at] = __dsub_rn(e, __ddiv_rn(a, __dsub_rn(c, a)));
    }
    __syncthreads();
    if (threadIdx.x == 0) base += total;
  }
  __syncthreads();
  if (threadIdx.x == 0) cnt[slot] = base;
}

// ---- candidates ----------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) pitch_cand_kernel(const PitchParams p) {
  pdl_entry();
  const int b = blockIdx.y, f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= p.F) return;
  const long long n = item_len(p, b);
  const int Fb = item_frames(p, n);
  double* cand = p.ws + p.lay.off_cand + (long long)b * kBands * p.F;
  double* best = p.ws + p.lay.off_best + (long long)b * p.F;
  const long long* cnt = reinterpret_cast<const long long*>(p.ws + p.lay.off_cnt) + (long long)b * kBands * kKinds;
  const double fs = (double)p.fs;
  const double t = __ddiv_rn(__dmul_rn((double)f, p.frame_period), 1000.0);
  double tmp = 0.0, bf = 0.0;
  for (int bd = 0; bd < kBands; ++bd) {
    double cd = 0.0, sc = kMaxValue;
    if (f < Fb) {
      bool ok = true;
      for (int k = 0; k < kKinds; ++k) ok = ok && (cnt[bd * kKinds + k] - 1 - 2 > 0);
      if (ok) {
        double vals[kKinds];
        for (int k = 0; k < kKinds; ++k) {
          const double* e = p.ws + p.lay.off_ev + (((long long)b * kBands + bd) * kKinds + k) * p.lay.cap;
          const long long ni = cnt[bd * kKinds + k] - 1;    // intervals
          // interval j: location (e[j] + e[j+1]) / 2 / fs, value fs / (e[j+1] - e[j]); k = clamp(upper_bound(loc, t), 1, ni - 1)
          long long lo = 0, hi = ni;
          while (lo < hi) {
            const long long mid = (lo + hi) >> 1;
            const double loc = __ddiv_rn(__ddiv_rn(__dadd_rn(e[mid], e[mid + 1]), 2.0), fs);
            if (loc <= t) lo = mid + 1; else hi = mid;
          }
          const long long kk = lo < 1 ? 1 : (lo > ni - 1 ? ni - 1 : lo);
          const double x0 = __ddiv_rn(__ddiv_rn(__dadd_rn(e[kk - 1], e[kk]), 2.0), fs);
          const double x1 = __ddiv_rn(__ddiv_rn(__dadd_rn(e[kk], e[kk + 1]), 2.0), fs);
          const double y0 = __ddiv_rn(fs, __dsub_rn(e[kk], e[kk - 1]));
          const double y1 = __ddiv_rn(fs, __dsub_rn(e[kk + 1], e[kk]));
          const double s = __ddiv_rn(__dsub_rn(t, x0), __dsub_rn(x1, x0));
          vals[k] = __dadd_rn(y0, __dmul_rn(s, __dsub_rn(y1, y0)));
        }
        cd = __ddiv_rn(__dadd_rn(__dadd_rn(__dadd_rn(vals[0], vals[1]), vals[2]), vals[3]), 4.0);
        double q = 0.0;
        for (int k = 0; k < kKinds; ++k) {
          const double dv = __dsub_rn(vals[k], cd);
          q = __dadd_rn(q, __dmul_rn(dv, dv));
        }
        sc = __dsqrt_rn(__ddiv_rn(q, 3.0));
        const double bo = p.lay.bound[bd];
        if (cd > bo || cd < bo / 2.0 || cd > kCeil || cd < kFloor) {
          cd = 0.0;
          sc = kMaxValue;
        }
      }
    }
    sc = __ddiv_rn(sc, __dadd_rn(cd, kGuard));
    cand[(long long)bd * p.F + f] = cd;
    if (bd == 0 || tmp > sc) {
      tmp = sc;
      bf = cd;
    }
  }
  best[f] = f < Fb ? bf : 0.0;
}

// ---- FixF0Contour --------------------------------------------------------------------------------------------------------
__device__ double select_best(double ref, const double* cand, long long F, int j) {
  double best_f0 = 0.0, best_err = kAllowed;
  for (int i = 0; i < kBands; ++i) {
    const double c = cand[(long long)i * F + j];
    const double tmp = __ddiv_rn(fabs(__dsub_rn(ref, c)), ref);
    if (tmp > best_err) continue;
    best_f0 = c;
    best_err = tmp;
  }
  return best_f0;
}

__global__ void __launch_bounds__(256) pitch_contour_kernel(const PitchParams p) {
  pdl_entry();
  const int b = blockIdx.x, F = p.F, r = p.lay.r;
  const int Fb = item_frames(p, item_len(p, b));
  const double* best = p.ws + p.lay.off_best + (long long)b * F;
  const double* cand = p.ws + p.lay.off_cand + (long long)b * kBands * F;
  double* s1 = p.ws + p.lay.off_s + (long long)b * F * 2;
  double* s2 = s1 + F;
  double* f0 = p.raw_f0 ? p.raw_f0 + (long long)b * F : p.ws + p.lay.off_f0 + (long long)b * F;
  if (Fb <= r) {
    for (int i = threadIdx.x; i < F; i += blockDim.x) f0[i] = 0.0;
    return;
  }
  // step 1 on f0_base (first and last r frames zero)
  for (int i = threadIdx.x; i < Fb; i += blockDim.x) {
    double v = 0.0;
    if (i >= r) {
      const double cur = i < Fb - r ? best[i] : 0.0;
      const double prev = (i - 1 >= r && i - 1 < Fb - r) ? best[i - 1] : 0.0;
      v = fabs(__ddiv_rn(__dsub_rn(cur, prev), __dadd_rn(kGuard, cur))) < kAllowed ? cur : 0.0;
    }
    s1[i] = v;
  }
  __syncthreads();
  const int ctr = (r - 1) / 2;
  for (int i = threadIdx.x; i < Fb; i += blockDim.x) {
    double v = s1[i];
    if (i >= ctr && i < Fb - ctr)
      for (int j = -ctr; j <= ctr; ++j)
        if (s1[i + j] == 0) { v = 0.0; break; }
    s2[i] = v;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < F; i += blockDim.x) f0[i] = i < Fb ? s2[i] : 0.0;
  __syncthreads();
  if (threadIdx.x != 0) return;
  // steps 3 and 4: sequential, sections from step 2's contour (s2), written into f0
  int prev_neg = -1;
  for (int i = 1; i < Fb; ++i) {                // negative indices in order; each section walks up to the next one
    if (!(s2[i] == 0 && s2[i - 1] != 0)) continue;
    if (prev_neg >= 0) {
      for (int j = prev_neg; j < i - 1; ++j) {
        f0[j + 1] = select_best(f0[j], cand, F, j + 1);
        if (f0[j + 1] == 0) break;
      }
    }
    prev_neg = i - 1;
  }
  if (prev_neg >= 0) {
    for (int j = prev_neg; j < Fb - 1; ++j) {
      f0[j + 1] = select_best(f0[j], cand, F, j + 1);
      if (f0[j + 1] == 0) break;
    }
  }
  int next_pos = -1;
  for (int i = Fb - 1; i >= 1; --i) {           // positive indices from the last; each walks down to the previous one
    if (!(s2[i - 1] == 0 && s2[i] != 0)) continue;
    if (next_pos >= 0) {
      for (int j = next_pos; j > i; --j) {
        f0[j - 1] = select_best(f0[j], cand, F, j - 1);
        if (f0[j - 1] == 0) break;
      }
    }
    next_pos = i;
  }
  if (next_pos >= 0) {
    for (int j = next_pos; j > 1; --j) {
      f0[j - 1] = select_best(f0[j], cand, F, j - 1);
      if (f0[j - 1] == 0) break;
    }
  }
}

// ---- StoneMask -----------------------------------------------------------------------------------------------------------
struct StoneFrame {
  const double* x;
  long long n;
  int fs, btl, fft, basic;
  const double* win;   // shared, btl
};

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// bin k of the main and difference spectra: (mr, mi, dr, di), forward sign
__device__ void stone_bin(const StoneFrame& s, int k, int lane, double* out4) {
  double mr = 0.0, mi = 0.0, dr = 0.0, di = 0.0;
  for (int i = lane; i < s.btl; i += 32) {
    long long idx = (long long)s.basic + i - 1;
    idx = idx < 0 ? 0 : (idx > s.n - 1 ? s.n - 1 : idx);
    const double seg = s.x[idx];
    const double w = s.win[i];
    const double dw = i == 0 ? -s.win[1] / 2.0 : (i == s.btl - 1 ? s.win[s.btl - 2] / 2.0 : -(s.win[i + 1] - s.win[i - 1]) / 2.0);
    const double ms = __dmul_rn(seg, w), ds = __dmul_rn(seg, dw);
    const long long m = ((long long)k * i) % s.fft;
    double sn, cs;
    sincospi(2.0 * (double)m / (double)s.fft, &sn, &cs);
    mr += ms * cs;
    mi -= ms * sn;
    dr += ds * cs;
    di -= ds * sn;
  }
  out4[0] = warp_sum(mr);
  out4[1] = warp_sum(mi);
  out4[2] = warp_sum(dr);
  out4[3] = warp_sum(di);
}

__device__ double fix_f0(const StoneFrame& s, double f0, int nh, int lane) {
  double num = 0.0, den = 0.0;
  const double fs = (double)s.fs, fft = (double)s.fft;
  for (int i = 0; i < nh; ++i) {
    const int index = mround(__dmul_rn(__ddiv_rn(__dmul_rn(f0, fft), fs), (double)(i + 1)));
    double v[4];
    stone_bin(s, index, lane, v);
    const double numi = __dsub_rn(__dmul_rn(v[0], v[3]), __dmul_rn(v[1], v[2]));
    const double pw = __dadd_rn(__dmul_rn(v[0], v[0]), __dmul_rn(v[1], v[1]));
    const double inst = pw == 0.0 ? 0.0
                                  : __dadd_rn(__ddiv_rn(__dmul_rn((double)index, fs), fft),
                                              __ddiv_rn(__ddiv_rn(__dmul_rn(__ddiv_rn(numi, pw), fs), 2.0), kPi));
    const double amp = __dsqrt_rn(pw);
    num = __dadd_rn(num, __dmul_rn(amp, inst));
    den = __dadd_rn(den, __dmul_rn(amp, (double)(i + 1)));
  }
  return __ddiv_rn(num, __dadd_rn(den, kGuard));
}

__global__ void __launch_bounds__(kStoneWarps * 32) pitch_stonemask_kernel(const PitchParams p, int win_cap) {
  pdl_entry();
  extern __shared__ double ssm[];
  const int b = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int f = blockIdx.x * kStoneWarps + warp;
  if (f >= p.F) return;
  const long long n = item_len(p, b);
  const int Fb = item_frames(p, n);
  const double* f0s = p.raw_f0 ? p.raw_f0 + (long long)b * p.F : p.ws + p.lay.off_f0 + (long long)b * p.F;
  double* ref = p.ws + p.lay.off_ref + (long long)b * p.F;
  const double f0 = f < Fb ? f0s[f] : 0.0;
  const double fs = (double)p.fs;
  if (f >= Fb || f0 <= kFloorStone || f0 > fs / 12.0) {
    if (lane == 0) ref[f] = 0.0;
    return;
  }
  const double t = __ddiv_rn(__dmul_rn((double)f, p.frame_period), 1000.0);
  const double hw = 1.5 / f0;
  const double wl = __dadd_rn(2.0 * hw, 1.0 / fs);
  const int h = mround(__dmul_rn(hw, fs));
  StoneFrame s;
  s.x = p.x + (long long)b * p.item_stride;
  s.n = n;
  s.fs = p.fs;
  s.btl = 2 * h + 1;
  // 2^(2 + int(log(hw fs + 1) / log 2)) as a shift: the device pow need not return a power of two exactly
  s.fft = 1 << (2 + (int)(log(__dadd_rn(__dmul_rn(hw, fs), 1.0)) / kLog2));
  const double base0 = (double)(-h) / fs;
  s.basic = mround(__dadd_rn(__dmul_rn(__dadd_rn(t, base0), fs), 0.001));
  double* win = ssm + (long long)warp * win_cap;
  for (int i = lane; i < s.btl; i += 32) {
    const double u = __dsub_rn(((double)(s.basic + i) - 1.0) / fs, t);
    win[i] = __dadd_rn(__dadd_rn(0.42, __dmul_rn(0.5, cos(2.0 * kPi * u / wl))), __dmul_rn(0.08, cos(4.0 * kPi * u / wl)));
  }
  __syncwarp();
  s.win = win;
  const double tent = fix_f0(s, f0, 2, lane);
  double mean_f0 = 0.0;
  if (!(tent <= 0.0 || tent > f0 * 2)) mean_f0 = fix_f0(s, tent, 6, lane);
  if (fabs(mean_f0 - f0) > f0 * 0.2) mean_f0 = f0;
  if (lane == 0) ref[f] = mean_f0;
}

// ---- output --------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) pitch_output_kernel(const PitchParams p) {
  pdl_entry();
  const int b = blockIdx.x, F = p.F;
  const int Fb = item_frames(p, item_len(p, b));
  const double* ref = p.ws + p.lay.off_ref + (long long)b * F;
  long long* prv = reinterpret_cast<long long*>(p.ws + p.lay.off_nb) + (long long)b * F * 2;
  long long* nxt = prv + F;
  double* out = p.pitch + (long long)b * F;
  const bool cont = p.flags & 1, lg = p.flags & 2;
  if (cont) {
    if (threadIdx.x == 0) {
      long long last = -1;
      for (int i = 0; i < Fb; ++i) { if (ref[i] != 0) last = i; prv[i] = last; }
    } else if (threadIdx.x == 32) {
      long long next = -1;
      for (int i = Fb - 1; i >= 0; --i) { if (ref[i] != 0) next = i; nxt[i] = next; }
    }
    __syncthreads();
  }
  for (int i = threadIdx.x; i < F; i += blockDim.x) {
    double v = 0.0;
    if (i < Fb) {
      v = ref[i];
      if (cont && v == 0) {
        const long long a = prv[i], c = nxt[i];
        if (a < 0 && c >= 0) v = ref[c];                 // before the first voiced frame: held
        else if (a >= 0 && c < 0) v = ref[a];            // after the last: held
        else if (a >= 0 && c >= 0) {                      // np.interp between the nearest voiced frames
          const double slope = __ddiv_rn(__dsub_rn(ref[c], ref[a]), (double)(c - a));
          v = __dadd_rn(__dmul_rn(slope, (double)(i - a)), ref[a]);
        }
      }
      if (lg && v != 0) v = log(v);
    }
    out[i] = v;
  }
}

static int fir_smem(int taps) { return (int)((2 * (size_t)taps + kFirTile - 1) * sizeof(double)); }

int launch_pitch(const PitchParams& p, int B, cudaStream_t st) {
  static std::atomic<uint64_t> attr_devs{0};
  if (first_use_on_device(attr_devs)) {
    cudaFuncSetAttribute(pitch_lowcut_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(pitch_band_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(pitch_stonemask_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  }
  const PitchLayout& L = p.lay;
  EV_TRY(launch("pitch_taps_kernel", pitch_taps_kernel, 1, 256, 0, st, p));
  EV_TRY(launch("pitch_mean_kernel", pitch_mean_kernel, B, 512, 0, st, p));
  EV_TRY(launch("pitch_lowcut_kernel", pitch_lowcut_kernel, dim3((unsigned)((L.S1 + kFirTile - 1) / kFirTile), B), kFirTile,
                fir_smem(2 * L.c + 1), st, p));
  EV_TRY(launch("pitch_band_kernel", pitch_band_kernel, dim3((unsigned)((L.M + kFirTile - 1) / kFirTile), kBands, B), kFirTile,
                fir_smem(2 * L.l0 + 1), st, p));
  EV_TRY(launch("pitch_events_kernel", pitch_events_kernel, dim3(kBands * kKinds, B), 1024, 0, st, p));
  EV_TRY(launch("pitch_cand_kernel", pitch_cand_kernel, dim3((p.F + 127) / 128, B), 128, 0, st, p));
  EV_TRY(launch("pitch_contour_kernel", pitch_contour_kernel, B, 256, 0, st, p));
  const int win_cap = 2 * host_round(1.5 * p.fs / kFloorStone) + 2;
  EV_TRY(launch("pitch_stonemask_kernel", pitch_stonemask_kernel, dim3((p.F + kStoneWarps - 1) / kStoneWarps, B), kStoneWarps * 32,
                (size_t)kStoneWarps * win_cap * sizeof(double), st, p, win_cap));
  return launch("pitch_output_kernel", pitch_output_kernel, B, 256, 0, st, p);
}

static bool pitch_args_ok(int B, long long item_stride, int fs, double frame_period, int F) {
  return B > 0 && B <= 65535 && fs >= 8000 && fs <= 48000 && frame_period >= 0.25 && frame_period <= 1000.0 && item_stride > 0 &&
         F == (int)(1000.0 * (double)item_stride / (double)fs / frame_period) + 1;
}

}  // namespace ev

using namespace ev;

extern "C" {

size_t ev_pitch_workspace_bytes(int B, long long item_stride, int fs, double frame_period, int F) {
  if (!pitch_args_ok(B, item_stride, fs, frame_period, F)) return 0;
  return pitch_layout(B, item_stride, fs, F, frame_period).total;
}

int ev_pitch(const double* x, long long item_stride, const int64_t* n_samples, int B, int fs, double frame_period, int F, int flags,
             double* raw_f0, double* pitch, int32_t* status, void* workspace, size_t workspace_bytes, void* stream) {
  EV_CHECK_ARG(x && pitch && workspace, "ev_pitch: null argument");
  EV_CHECK_ARG(fs >= 8000 && fs <= 48000, "ev_pitch: fs %d is not in [8000, 48000]", fs);
  EV_CHECK_ARG(frame_period >= 0.25 && frame_period <= 1000.0, "ev_pitch: frame_period %g ms is not in [0.25, 1000]", frame_period);
  EV_CHECK_ARG(pitch_args_ok(B, item_stride, fs, frame_period, F), "ev_pitch: B=%d item_stride=%lld F=%d (F must be the row's frame count)",
               B, item_stride, F);
  EV_CHECK_ARG((flags & ~3) == 0, "ev_pitch: unknown flags %d", flags);
  const PitchLayout lay = pitch_layout(B, item_stride, fs, F, frame_period);
  EV_CHECK_ARG(n_samples || item_stride >= 2ll * lay.c + 1, "ev_pitch: items of %lld samples are shorter than the low-cut filter (%d)",
               item_stride, 2 * lay.c + 1);
  EV_CHECK_ARG(lay.l0 <= kMaxHalf, "ev_pitch: filter half length %d", lay.l0);
  EV_CHECK_ARG(workspace_bytes >= lay.total, "ev_pitch: workspace %zu < %zu bytes", workspace_bytes, lay.total);
  EV_TRY(use_device_of(x));
  PitchParams p;
  p.x = x;
  p.item_stride = item_stride;
  p.n_samples = n_samples;
  p.fs = fs;
  p.F = F;
  p.flags = flags;
  p.frame_period = frame_period;
  p.lay = lay;
  p.ws = reinterpret_cast<double*>(workspace);
  p.raw_f0 = raw_f0;
  p.pitch = pitch;
  p.status = status;
  return launch_pitch(p, B, reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
