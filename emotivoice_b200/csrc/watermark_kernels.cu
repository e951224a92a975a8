// Keyed zero-bit watermark of output waveforms at 16 kHz (ev_watermark_embed) and its detector (ev_watermark_detect).  The
// definitions are in emotivoice_b200/audio.py and oracle/watermark_oracle.py; in short, with frames of N = 1024 samples, hop
// H = 512 and the sine window w[n] = sin(pi (n + 1/2) / N):
//   MCLT   C[j,k] - i S[j,k] = post[k] * FFT_1024(w[n] pre[n] x[(j - 1) H + tau + n])[k], pre[n] = e^{-i pi n / N},
//          post[k] = e^{-i 2 pi n0 (k + 1/2) / N}, n0 = 1/2 + H / 2 (unscaled: only ratios and the synthesis below use it).
//   embed  dC[j,k] = alpha M[j,k] s(key, j mod P, k) on bins 19..217, M = |C - i S|; the IMDCT of dC, overlap-added, is
//          d[n] = (2 / H) w[n] Re(pre[n] G[n]) per frame with G = FFT_1024(dC[k] post[k]) (zero outside the band); y = x + d.
//   detect u = C / M on the band (skipped where M = 0), b[tau, r, k] = sum of u over the frames j = r mod P of grid tau,
//          z(tau, m0) = sum_{r,k} s(key, (r + m0) mod P, k) b[r,k] / sqrt(sum b^2).
// s(key, r, k) = -1 when the top bit of mix64(key ^ mix64((r << 10) | k)) is set, else +1 (SplitMix64's output function).
//
// wm_embed_kernel: one CTA per (tile of WM_HOPS hops, listed item).  Its warps compute the WM_HOPS + 1 frames that cover those
// hops (one halo frame), one frame per warp: the analysis FFT, the modulation in registers, the synthesis FFT into the warp's
// buffer; then the CTA writes y = x + (d of frame h + d of frame h + 1) for its own samples only.
// wm_detect_kernel: one CTA per (grid tau, item).  Warp w takes frames j = w mod WM_DWARPS in order, so the rows r = j mod P of
// b it adds to are its own and every cell is summed in frame order: no atomics, the same bits in any batch.  Then the CTA
// correlates b with the pattern at every m0 and keeps the largest z (the first m0 on ties).  wm_pick_kernel: per item, the
// largest z over tau (the first tau on ties).
#include <math.h>

#include "ev_common.cuh"
#include "stockham.cuh"

namespace ev {

constexpr int WM_N = 1024, WM_H = 512, WM_P = 64, WM_KLO = 19, WM_KHI = 218, WM_NB = WM_KHI - WM_KLO;
constexpr int WM_BUF = WM_N + WM_N / 8;         // one warp's padded FFT buffer (float2)
constexpr int WM_EWARPS = 8, WM_HOPS = WM_EWARPS - 1;
constexpr int WM_DWARPS = 16;                    // divides P: warp w owns the rows r = w mod WM_DWARPS of b
constexpr int WM_SR = 16000;
constexpr double WM_ALPHA = 0.070710678118654752440;  // 10^(-20/20) / sqrt(2)
constexpr int WM_TABLES = 2 * WM_N + 200;        // tw, w * pre, post (float2)
static_assert(WM_P % WM_DWARPS == 0, "a row of b must belong to one warp");

__device__ __forceinline__ uint64_t wm_mix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

__device__ __forceinline__ bool wm_negative(uint64_t key, int r, int k) {
  return (wm_mix64(key ^ wm_mix64(((uint64_t)r << 10) | (uint64_t)k)) >> 63) != 0;
}

// tw[m] = W_1024^m, wp[n] = w[n] pre[n], post[k - 19]; fp64 angles with exact argument reduction, rounded once to fp32
__device__ void wm_tables(float2* tw, float2* wp, float2* post) {
  for (int m = threadIdx.x; m < WM_N; m += blockDim.x) {
    double s, c;
    sincospi(2.0 * m / WM_N, &s, &c);
    tw[m] = make_float2((float)c, (float)-s);
    sincospi((double)m / WM_N, &s, &c);
    const double w = sinpi((m + 0.5) / WM_N);
    wp[m] = make_float2((float)(w * c), (float)(-w * s));
  }
  for (int k = WM_KLO + threadIdx.x; k < WM_KHI; k += blockDim.x) {
    double s, c;
    sincospi((0.5 + WM_H / 2) * (2 * k + 1) / WM_N, &s, &c);
    post[k - WM_KLO] = make_float2((float)c, (float)-s);
  }
}

// the windowed, pre-twiddled frame starting at sample t0 of x (zero outside [0, n)) into a warp's FFT, transformed
__device__ __forceinline__ void wm_analyse(float2* buf, const float2* tw, const float2* wp, const float* __restrict__ x, long long n,
                                           long long t0, int lane) {
  const float* xf = x + t0;
  const bool inside = t0 >= 0 && t0 + WM_N <= n;
  fft1024(buf, tw, lane, [&](int m) {
    const float v = (inside || (t0 + m >= 0 && t0 + m < n)) ? __ldg(xf + m) : 0.f;
    const float2 p = wp[m];
    return make_float2(v * p.x, v * p.y);
  });
}

__global__ void __launch_bounds__(WM_EWARPS * 32) wm_embed_kernel(const float* __restrict__ wav, long long item_stride,
                                                                  const int64_t* __restrict__ n_in, const int64_t* __restrict__ items,
                                                                  uint64_t key, float* __restrict__ out, long long out_stride) {
  pdl_entry();
  extern __shared__ __align__(16) unsigned char wm_smem[];
  float2* tw = reinterpret_cast<float2*>(wm_smem);
  float2* wp = tw + WM_N;
  float2* post = wp + WM_N;
  float2* bufs = tw + WM_TABLES;
  const int k = blockIdx.y;
  const long long b = items ? items[k] : k;
  const long long n = max(0ll, min((long long)n_in[b], item_stride));
  const long long a = (long long)blockIdx.x * WM_HOPS;      // hops [a, a + WM_HOPS); hop h holds samples [h H, h H + H)
  const long long J = (n + WM_H - 1) / WM_H;                 // frames 0 .. J cover the item
  if (a >= J) return;
  wm_tables(tw, wp, post);
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* x = wav + b * item_stride;
  const long long j = a + warp;
  float2* buf = bufs + warp * WM_BUF;
  if (j <= J) {
    wm_analyse(buf, tw, wp, x, n, (j - 1) * WM_H, lane);
    // dC post[k] of the band bins into registers (the spectrum is in fft1024_at order), then the synthesis input in natural order
    const int r = (int)(j % WM_P);
    const float scale = (float)(2.0 * WM_ALPHA / WM_H);
    constexpr int kPer = (WM_NB + 31) / 32;
    float2 c[kPer];
#pragma unroll
    for (int i = 0; i < kPer; ++i) {
      const int m = WM_KLO + lane + 32 * i;
      c[i] = make_float2(0.f, 0.f);
      if (m < WM_KHI) {
        const float2 ps = post[m - WM_KLO];
        const float2 X = cmul(buf[fft1024_at(m)], ps);
        float g = scale * sqrtf(X.x * X.x + X.y * X.y);
        if (wm_negative(key, r, m)) g = -g;
        c[i] = make_float2(g * ps.x, g * ps.y);
      }
    }
    __syncwarp();
    for (int m = lane; m < WM_N; m += 32) buf[bpad(m)] = make_float2(0.f, 0.f);
    __syncwarp();
#pragma unroll
    for (int i = 0; i < kPer; ++i) {
      const int m = WM_KLO + lane + 32 * i;
      if (m < WM_KHI) buf[bpad(m)] = c[i];
    }
    __syncwarp();
    fft1024(buf, tw, lane, [&](int m) { return buf[bpad(m)]; });
    float* d = reinterpret_cast<float*>(buf);
    for (int m = lane; m < WM_N; m += 32) {
      const float2 G = buf[fft1024_at(m)], p = wp[m];
      d[2 * fft1024_at(m)] = p.x * G.x - p.y * G.y;          // the slot this lane just read
    }
  }
  __syncthreads();
  const long long s0 = a * WM_H, s1 = min(n, (a + WM_HOPS) * WM_H);
  float* y = out + (long long)k * out_stride;
  for (long long s = s0 + threadIdx.x; s < s1; s += blockDim.x) {
    const int h = (int)(s / WM_H - a), i = (int)(s % WM_H);
    const float dA = reinterpret_cast<const float*>(bufs + h * WM_BUF)[2 * fft1024_at(i + WM_H)];
    const float dB = reinterpret_cast<const float*>(bufs + (h + 1) * WM_BUF)[2 * fft1024_at(i)];
    y[s] = x[s] + (dA + dB);
  }
}

__global__ void __launch_bounds__(WM_DWARPS * 32) wm_detect_kernel(const float* __restrict__ wav, long long item_stride,
                                                                   const int64_t* __restrict__ n_in, uint64_t key,
                                                                   float* __restrict__ zt, int32_t* __restrict__ mt) {
  pdl_entry();
  extern __shared__ __align__(16) unsigned char wm_smem[];
  float2* tw = reinterpret_cast<float2*>(wm_smem);
  float2* wp = tw + WM_N;
  float2* post = wp + WM_N;
  float2* bufs = tw + WM_TABLES;
  float* bsum = reinterpret_cast<float*>(bufs + WM_DWARPS * WM_BUF);   // (P, NB)
  __shared__ double dred[WM_DWARPS];
  __shared__ float part[8][WM_P];
  __shared__ float zm[WM_P];
  const int tau = blockIdx.x, k = blockIdx.y;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long n = max(0ll, min((long long)n_in[k], item_stride));
  const long long F = max(0ll, (n - tau + 2 * WM_H - 1) / WM_H);     // frames j >= 0 that start before n
  for (int i = threadIdx.x; i < WM_P * WM_NB; i += blockDim.x) bsum[i] = 0.f;
  wm_tables(tw, wp, post);
  __syncthreads();
  const float* x = wav + (long long)k * item_stride;
  float2* buf = bufs + warp * WM_BUF;
  for (long long j = warp; j < F; j += WM_DWARPS) {
    wm_analyse(buf, tw, wp, x, n, (j - 1) * WM_H + tau, lane);
    float* row = bsum + (int)(j % WM_P) * WM_NB;
    for (int q = lane; q < WM_NB; q += 32) {
      const float2 X = cmul(buf[fft1024_at(q + WM_KLO)], post[q]);
      const float M = sqrtf(X.x * X.x + X.y * X.y);
      if (M > 0.f) row[q] += X.x / M;
    }
    __syncwarp();
  }
  __syncthreads();
  float* sp = reinterpret_cast<float*>(bufs);                          // the pattern (P, NB) as +-1
  double e = 0.0;
  for (int i = threadIdx.x; i < WM_P * WM_NB; i += blockDim.x) {
    sp[i] = wm_negative(key, i / WM_NB, WM_KLO + i % WM_NB) ? -1.f : 1.f;
    e += (double)bsum[i] * (double)bsum[i];
  }
  for (int o = 16; o > 0; o >>= 1) e += __shfl_xor_sync(0xffffffffu, e, o);
  if (lane == 0) dred[warp] = e;
  __syncthreads();
  {
    const int m0 = threadIdx.x & (WM_P - 1), p = threadIdx.x / WM_P;   // 8 parts of 8 rows each
    float acc = 0.f;
    for (int r = 8 * p; r < 8 * p + 8; ++r) {
      const float* br = bsum + r * WM_NB;
      const float* sr = sp + ((r + m0) & (WM_P - 1)) * WM_NB;
      for (int q = 0; q < WM_NB; ++q) acc = fmaf(sr[q], br[q], acc);
    }
    part[p][m0] = acc;
  }
  __syncthreads();
  if (threadIdx.x < WM_P) {
    double den = 0.0;
    for (int w = 0; w < WM_DWARPS; ++w) den += dred[w];
    float num = 0.f;
    for (int p = 0; p < 8; ++p) num += part[p][threadIdx.x];
    zm[threadIdx.x] = den > 0.0 ? (float)((double)num / sqrt(den)) : 0.f;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int best = 0;
    for (int m = 1; m < WM_P; ++m)
      if (zm[m] > zm[best]) best = m;
    zt[(long long)k * WM_H + tau] = zm[best];
    mt[(long long)k * WM_H + tau] = best;
  }
}

__global__ void __launch_bounds__(32) wm_pick_kernel(const float* __restrict__ zt, const int32_t* __restrict__ mt, float* __restrict__ z,
                                                     int32_t* __restrict__ offset, int32_t* __restrict__ phase) {
  pdl_entry();
  const int k = blockIdx.x, lane = threadIdx.x;
  const float* zk = zt + (long long)k * WM_H;
  int bt = lane;
  for (int t = lane + 32; t < WM_H; t += 32)
    if (zk[t] > zk[bt]) bt = t;
  float bz = zk[bt];
  for (int o = 16; o > 0; o >>= 1) {
    const float oz = __shfl_xor_sync(0xffffffffu, bz, o);
    const int ot = __shfl_xor_sync(0xffffffffu, bt, o);
    if (oz > bz || (oz == bz && ot < bt)) {
      bz = oz;
      bt = ot;
    }
  }
  if (lane == 0) {
    z[k] = bz;
    offset[k] = bt;
    phase[k] = mt[(long long)k * WM_H + bt];
  }
}

constexpr size_t WM_EMBED_SMEM = (size_t)(WM_TABLES + WM_EWARPS * WM_BUF) * sizeof(float2);
constexpr size_t WM_DETECT_SMEM = (size_t)(WM_TABLES + WM_DWARPS * WM_BUF) * sizeof(float2) + (size_t)WM_P * WM_NB * sizeof(float);
static_assert(WM_DETECT_SMEM + 8 * WM_P * 4 + WM_P * 4 + WM_DWARPS * 8 <= 227 * 1024, "detect: shared memory");
static_assert((size_t)WM_P * WM_NB * sizeof(float) <= (size_t)WM_DWARPS * WM_BUF * sizeof(float2), "the pattern fits the FFT buffers");

static bool wm_key_ok(uint64_t key) { return key >= 1 && key <= 0x7fffffffffffffffull; }

}  // namespace ev

using namespace ev;

extern "C" {

int ev_watermark_embed(const float* wav, long long item_stride, const int64_t* n_in, const int64_t* items, int n_items, int sample_rate,
                       uint64_t key, float* out, long long out_stride, void* stream) {
  EV_CHECK_ARG(wav && n_in && out, "ev_watermark_embed: null argument");
  EV_CHECK_ARG(n_items >= 1 && n_items <= 65535, "ev_watermark_embed: n_items=%d must lie in [1, 65535]", n_items);
  EV_CHECK_ARG(item_stride >= 1 && out_stride >= item_stride, "ev_watermark_embed: item_stride=%lld must be at least 1 and out_stride=%lld "
               "at least item_stride", item_stride, out_stride);
  EV_CHECK_ARG(sample_rate == WM_SR, "ev_watermark_embed: sample_rate=%d; the mark is defined at %d Hz", sample_rate, WM_SR);
  EV_CHECK_ARG(wm_key_ok(key), "ev_watermark_embed: key=%llu must lie in [1, 2^63 - 1]", (unsigned long long)key);
  const long long tiles = ((item_stride + WM_H - 1) / WM_H + WM_HOPS - 1) / WM_HOPS;
  EV_CHECK_ARG(tiles <= 0x7fffffffll, "ev_watermark_embed: item_stride=%lld is too long", item_stride);
  EV_TRY(use_device_of(wav));
  static std::atomic<uint64_t> attr_devs{0};
  if (first_use_on_device(attr_devs)) cudaFuncSetAttribute(wm_embed_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WM_EMBED_SMEM);
  return launch("wm_embed_kernel", wm_embed_kernel, dim3((unsigned)tiles, n_items), WM_EWARPS * 32, WM_EMBED_SMEM,
                reinterpret_cast<cudaStream_t>(stream), wav, item_stride, n_in, items, key, out, out_stride);
}

size_t ev_watermark_detect_workspace_bytes(int n_items) {
  return n_items >= 1 && n_items <= 65535 ? (size_t)n_items * WM_H * (sizeof(float) + sizeof(int32_t)) : 0;
}

int ev_watermark_detect(const float* wav, long long item_stride, const int64_t* n, int n_items, uint64_t key, float* z, int32_t* offset,
                        int32_t* phase, void* ws, size_t ws_bytes, void* stream) {
  EV_CHECK_ARG(wav && n && z && offset && phase && ws, "ev_watermark_detect: null argument");
  EV_CHECK_ARG(n_items >= 1 && n_items <= 65535, "ev_watermark_detect: n_items=%d must lie in [1, 65535]", n_items);
  EV_CHECK_ARG(item_stride >= 1, "ev_watermark_detect: item_stride=%lld must be at least 1", item_stride);
  EV_CHECK_ARG(wm_key_ok(key), "ev_watermark_detect: key=%llu must lie in [1, 2^63 - 1]", (unsigned long long)key);
  const size_t need = ev_watermark_detect_workspace_bytes(n_items);
  EV_CHECK_ARG(ws_bytes >= need, "ev_watermark_detect: workspace of %zu bytes, %zu needed", ws_bytes, need);
  EV_TRY(use_device_of(wav));
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  static std::atomic<uint64_t> attr_devs{0};
  if (first_use_on_device(attr_devs))
    cudaFuncSetAttribute(wm_detect_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WM_DETECT_SMEM);
  float* zt = static_cast<float*>(ws);
  int32_t* mt = reinterpret_cast<int32_t*>(zt + (size_t)n_items * WM_H);
  EV_TRY(launch("wm_detect_kernel", wm_detect_kernel, dim3(WM_H, n_items), WM_DWARPS * 32, WM_DETECT_SMEM, st, wav, item_stride, n, key,
                zt, mt));
  return launch("wm_pick_kernel", wm_pick_kernel, dim3(n_items), 32, 0, st, (const float*)zt, (const int32_t*)mt, z, offset, phase);
}

}  // extern "C"
