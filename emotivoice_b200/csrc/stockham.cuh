// One warp's complex FFT in shared memory (forward, e^{-i}), fp32 FFMA: three radix-8 Stockham stages make a 512-point
// transform (stft_feats_kernel), and a radix-2 stage in front of two of them a 1024-point one (the watermark kernels).  The
// buffer has one padding slot per 8 complex values (bpad), so the stage stores hit distinct banks.  tw is the table
// W_1024^m = (cos, -sin)(2 pi m / 1024), m in [0, 1024).
#pragma once
#include <cuda_runtime.h>

namespace ev {

__device__ __forceinline__ int bpad(int i) { return i + (i >> 3); }

__device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }

__device__ __forceinline__ void bfly(float2& a, float2& b) {
  const float2 t = a;
  a = make_float2(t.x + b.x, t.y + b.y);
  b = make_float2(t.x - b.x, t.y - b.y);
}

// In-register 8-point DFT (forward, e^{-i}), radix-2 decimation in frequency: bin k ends in v[bitrev3(k)].
__device__ __forceinline__ void fft8(float2 (&v)[8]) {
  constexpr float s = 0.70710678118654752440f;
  bfly(v[0], v[4]); bfly(v[1], v[5]); bfly(v[2], v[6]); bfly(v[3], v[7]);
  v[5] = make_float2((v[5].x + v[5].y) * s, (v[5].y - v[5].x) * s);      // * W8^1
  v[6] = make_float2(v[6].y, -v[6].x);                                  // * W8^2 = -i
  v[7] = make_float2((v[7].y - v[7].x) * s, -(v[7].x + v[7].y) * s);     // * W8^3
  bfly(v[0], v[2]); bfly(v[1], v[3]); bfly(v[4], v[6]); bfly(v[5], v[7]);
  v[3] = make_float2(v[3].y, -v[3].x);
  v[7] = make_float2(v[7].y, -v[7].x);
  bfly(v[0], v[1]); bfly(v[2], v[3]); bfly(v[4], v[5]); bfly(v[6], v[7]);
}

__device__ __forceinline__ int brev3(int k) { return ((k & 1) << 2) | (k & 2) | ((k >> 2) & 1); }

// Stockham radix-8 stage of the 512-point FFT, NS = 8^stage: butterfly j reads v[r] = in[j + 64 r] * W_{8 NS}^{r (j % NS)} and
// writes bin r of its 8-point DFT to out[(j / NS) * 8 NS + j % NS + r NS].  Every lane holds its two butterflies in registers
// between the reads and the writes, so in and out may be the same buffer.
template <int NS>
__device__ __forceinline__ void stockham_store(float2 (&v)[2][8], float2* buf, int lane) {
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    const int j = lane + 32 * q;
    const int d = (j / NS) * NS * 8 + j % NS;
#pragma unroll
    for (int r = 0; r < 8; ++r) buf[bpad(d + r * NS)] = v[q][brev3(r)];
  }
}

template <int NS>
__device__ __forceinline__ void stockham_stage(float2* buf, const float2* tw, int lane) {
  float2 v[2][8];
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    const int j = lane + 32 * q;
    const int k = j % NS;
#pragma unroll
    for (int r = 0; r < 8; ++r) v[q][r] = buf[bpad(j + 64 * r)];
#pragma unroll
    for (int r = 1; r < 8; ++r) v[q][r] = cmul(v[q][r], tw[2 * r * k * (512 / (8 * NS))]);   // W_512^m = W_1024^2m
    fft8(v[q]);
  }
  __syncwarp();
  stockham_store<NS>(v, buf, lane);
  __syncwarp();
}

constexpr int kFft1024Half = 512 + 512 / 8;   // where the second 512-point half starts in a padded 1024-point buffer

// Where bin m of fft1024's result lies in the buffer: even bins in the first half, odd bins in the second.
__device__ __forceinline__ int fft1024_at(int m) { return (m & 1) * kFft1024Half + bpad(m >> 1); }

// 1024-point FFT in place, one radix-2 stage of decimation in frequency and two 512-point transforms: with a = load(j),
// b = load(j + 512), the halves are a + b (the even bins) and (a - b) W_1024^j (the odd bins), at bpad(j) and bpad(j + 512).  A
// lane stores only where it loaded from, so load may read buf at bpad(m).  The result is in the order of fft1024_at.
template <class Load>
__device__ __forceinline__ void fft1024(float2* buf, const float2* tw, int lane, Load load) {
#pragma unroll 4
  for (int j = lane; j < 512; j += 32) {
    const float2 a = load(j), b = load(j + 512);
    buf[bpad(j)] = make_float2(a.x + b.x, a.y + b.y);
    buf[kFft1024Half + bpad(j)] = cmul(make_float2(a.x - b.x, a.y - b.y), tw[j]);
  }
  __syncwarp();
#pragma unroll 1
  for (int h = 0; h < 2; ++h) {
    float2* hb = buf + h * kFft1024Half;
    stockham_stage<1>(hb, tw, lane);
    stockham_stage<8>(hb, tw, lane);
    stockham_stage<64>(hb, tw, lane);
  }
}

}  // namespace ev
