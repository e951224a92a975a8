// The true-peak detector shared by ev_limit (limiter_kernels.cu) and ev_meter (meter_kernels.cu).
#pragma once

namespace ev {

// p[s] = max(|x[s]|, |sum_j h[ph][j] * x[s + c - j]| over the phases ph), c = (taps - 1) / 2: the largest magnitude of the
// oversampled waveform around sample s.  xs points at the staged sample x[s - c] (so xs[c] = x[s]), hs at the (phases, taps)
// bank in shared memory.  fp32, one chain per phase in tap order.  phases may be 0 (p[s] = |x[s]|).
__device__ __forceinline__ float tp_detect(const float* xs, const float* hs, int phases, int taps) {
  const int c = (taps - 1) / 2;
  const float* xc = xs + 2 * c;                               // xc[-j] = x[s + c - j]
  float p = fabsf(xs[c]);
  for (int ph = 0; ph < phases; ++ph) {
    const float* h = hs + ph * taps;
    float acc = 0.f;
    for (int j = 0; j < taps; ++j) acc = fmaf(h[j], xc[-j], acc);
    p = fmaxf(p, fabsf(acc));
  }
  return p;
}

}  // namespace ev
