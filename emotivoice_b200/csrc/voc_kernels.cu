// HiFi-GAN generator kernels that are not implicit GEMMs (sm_90a, fp32): the layout change at
// the Generator.forward boundary, the final conv_post + tanh, the joined mel of long text, the callers' PCM16 conversion and
// the output formatting (resampling + PCM16 / G.711 encoding).
#include "ev_common.cuh"

namespace ev {

// (B, C, L) channels-first (the reference's Generator.forward input, hifigan/models.py:115)
// -> (B, L, C) time-major (the engine's internal layout).  32x32 smem tile transpose.
__global__ void transpose_cf_to_tm_kernel(const float* __restrict__ in, float* __restrict__ out, int C, int L) {
  pdl_entry();
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int l0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const float* ib = in + (size_t)b * C * L;
  float* ob = out + (size_t)b * C * L;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, l = l0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C && l < L) ? ib[(size_t)c * L + l] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int l = l0 + i, c = c0 + threadIdx.x;
    if (l < L && c < C) ob[(size_t)l * C + c] = tile[threadIdx.x][i];
  }
}
int launch_transpose_cf_to_tm(const float* in, float* out, int B, int C, int L, cudaStream_t st) {
  EV_CHECK_ARG(B > 0 && C > 0 && L > 0 && B <= 65535, "transpose: bad shape");
  dim3 grid((L + 31) / 32, (C + 31) / 32, B), block(32, 8);
  return launch("transpose_cf_to_tm_kernel", transpose_cf_to_tm_kernel, grid, block, 0, st, in, out, C, L);
}

// wav[b,t] = tanh( bias + sum_j sum_c w[j][c] * lrelu(x[b, t+j-(K-1)/2, c]) )
// (hifigan/models.py:127-129: F.leaky_relu default slope 0.01, Conv1d(C,1,7,pad 3), tanh).
// HBM-bound: each CTA stages (256 + K - 1) rows once; rows >= len read as zero padding.
constexpr int CP_BT = 256;
__global__ void __launch_bounds__(CP_BT) conv_post_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                          const float* __restrict__ bias, const int32_t* __restrict__ lens,
                                                          int lens_mul, int L, int C, int K, float slope,
                                                          float* __restrict__ wav) {
  pdl_entry();
  extern __shared__ __align__(16) float cp_smem[];
  const int ld = C + 1;
  float* xs = cp_smem;                          // [(CP_BT + K - 1)][C + 1]
  float* ws = cp_smem + (CP_BT + K - 1) * ld;   // [K][C]
  const int b = blockIdx.y, t0 = blockIdx.x * CP_BT;
  const int len = lens ? min(L, lens[b] * lens_mul) : L;
  const int halo = (K - 1) / 2;
  const float* xb = x + (size_t)b * L * C;
  const int rows = CP_BT + K - 1;
  const int c4n = C / 4;
  for (int i = threadIdx.x; i < rows * c4n; i += CP_BT) {
    const int r = i / c4n, c4 = i % c4n;
    const int row = t0 - halo + r;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (row >= 0 && row < len) v = __ldg(reinterpret_cast<const float4*>(xb + (size_t)row * C + c4 * 4));
    float* d = xs + r * ld + c4 * 4;
    d[0] = v.x > 0.f ? v.x : v.x * slope;
    d[1] = v.y > 0.f ? v.y : v.y * slope;
    d[2] = v.z > 0.f ? v.z : v.z * slope;
    d[3] = v.w > 0.f ? v.w : v.w * slope;
  }
  for (int i = threadIdx.x; i < K * C; i += CP_BT) ws[i] = w[i];
  __syncthreads();
  const int t = t0 + threadIdx.x;
  if (t >= L) return;
  float acc = 0.f;
  for (int c = 0; c < C; ++c) {       // channel-major reduction order, shared with the granule-planar conv_post kernels (conv1d_gp.cu)
    const float* xr = xs + threadIdx.x * ld + c;
    for (int j = 0; j < K; ++j) acc = fmaf(xr[j * ld], ws[j * C + c], acc);
  }
  wav[(size_t)b * L + t] = t < len ? tanhf(acc + bias[0]) : 0.f;
}
int launch_conv_post(const float* x, const float* w, const float* bias, const int32_t* lens, int lens_mul, int B,
                     int L, int C, int K, float slope, float* wav, cudaStream_t st) {
  EV_CHECK_ARG(C > 0 && C % 4 == 0 && C <= 128 && K >= 1 && K <= 15 && (K & 1), "conv_post: C=%d K=%d", C, K);
  EV_CHECK_ARG(B > 0 && B <= 65535 && L > 0, "conv_post: bad shape");
  const size_t smem = (size_t)((CP_BT + K - 1) * (C + 1) + K * C) * sizeof(float);
  static std::atomic<uint64_t> attr_devs{0};
  if (first_use_on_device(attr_devs))
    cudaFuncSetAttribute(conv_post_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
  dim3 grid((L + CP_BT - 1) / CP_BT, B);
  return launch("conv_post_kernel", conv_post_kernel, grid, CP_BT, smem, st, x, w, bias, lens, lens_mul, L, C, K, slope, wav);
}

// Joined mel of long-text synthesis: the valid rows mel[b, :mel_lens[b]] of consecutive items with one group id, concatenated in
// item order, -> joined (G, Fg, C) time-major, rows past a group's length zero; group_lens[g] = min(frames of group g, Fg).
// Every CTA scans the B lengths into item offsets in shared memory (B <= JM_MAX_ITEMS), then copies JM_ROWS output rows, each
// from the item a binary search over the offsets finds.  `group` must be non-decreasing from 0 in steps of 0 or 1 up to G - 1;
// other ids give an unspecified result but no out-of-bounds access.
constexpr int JM_THREADS = 256, JM_ROWS = 64, JM_MAX_ITEMS = 4096;
__global__ void __launch_bounds__(JM_THREADS) join_mel_kernel(const float* __restrict__ mel, const int32_t* __restrict__ mel_lens,
                                                              const int32_t* __restrict__ group, int B, int F, int C, int G, int Fg,
                                                              float* __restrict__ joined, int32_t* __restrict__ group_lens) {
  pdl_entry();
  extern __shared__ int jm_smem[];
  int* off = jm_smem;              // [B + 1]: first joined row of item b, counted over all items
  int* first = off + B + 1;        // [G + 1]: first item of group g; first[G] = B
  __shared__ int part[JM_THREADS];
  const int per = (B + JM_THREADS - 1) / JM_THREADS;
  const int b0 = min(B, (int)threadIdx.x * per), b1 = min(B, b0 + per);
  int s = 0;
  for (int b = b0; b < b1; ++b) s += min(max(mel_lens[b], 0), F);
  part[threadIdx.x] = s;
  for (int g = threadIdx.x; g <= G; g += JM_THREADS) first[g] = B;
  __syncthreads();
  for (int d = 1; d < JM_THREADS; d <<= 1) {       // inclusive scan of the per-thread sums
    const int v = (int)threadIdx.x >= d ? part[threadIdx.x - d] : 0;
    __syncthreads();
    part[threadIdx.x] += v;
    __syncthreads();
  }
  int o = threadIdx.x ? part[threadIdx.x - 1] : 0;
  for (int b = b0; b < b1; ++b) {
    off[b] = o;
    o += min(max(mel_lens[b], 0), F);
  }
  if (threadIdx.x == JM_THREADS - 1) off[B] = part[JM_THREADS - 1];
  for (int b = threadIdx.x; b < B; b += JM_THREADS) {
    const int g = group[b];
    if (g >= 0 && g < G && (b == 0 || group[b - 1] != g)) first[g] = b;
  }
  __syncthreads();
  if (blockIdx.x == 0)
    for (int g = threadIdx.x; g < G; g += JM_THREADS) group_lens[g] = min(max(off[max(first[g + 1], first[g])] - off[first[g]], 0), Fg);
  const int c4n = C / 4;
  const long long rows = (long long)G * Fg;
  for (int i = threadIdx.x; i < JM_ROWS * c4n; i += JM_THREADS) {
    const long long r = (long long)blockIdx.x * JM_ROWS + i / c4n;
    if (r >= rows) break;
    const int g = (int)(r / Fg), f = (int)(r % Fg), c4 = i % c4n;
    const int s0 = first[g], e = max(first[g + 1], s0);
    const int pos = off[s0] + f;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (s0 < e && pos < off[e]) {
      int lo = s0, hi = e - 1;                       // the last item of the group whose offset is <= pos
      while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (off[mid] <= pos) lo = mid; else hi = mid - 1;
      }
      v = __ldg(reinterpret_cast<const float4*>(mel + ((size_t)lo * F + (pos - off[lo])) * C) + c4);
    }
    reinterpret_cast<float4*>(joined + (size_t)r * C)[c4] = v;
  }
}
int launch_join_mel(const float* mel, const int32_t* mel_lens, const int32_t* group, int B, int F, int C, int G, int Fg, float* joined,
                    int32_t* group_lens, cudaStream_t st) {
  EV_CHECK_ARG(B > 0 && B <= JM_MAX_ITEMS, "join_mel: B=%d must lie in [1, %d]", B, JM_MAX_ITEMS);
  EV_CHECK_ARG(G > 0 && G <= B && F > 0 && Fg > 0 && C > 0 && C % 4 == 0, "join_mel: B=%d G=%d F=%d Fg=%d n_mels=%d", B, G, F, Fg, C);
  EV_CHECK_ARG((long long)B * F < (1ll << 31) && (long long)G * Fg < (1ll << 31), "join_mel: B*F or G*Fg reaches 2^31");
  const long long blocks = ((long long)G * Fg + JM_ROWS - 1) / JM_ROWS;
  const size_t smem = (size_t)(B + 1 + G + 1) * sizeof(int);
  return launch("join_mel_kernel", join_mel_kernel, (unsigned)blocks, JM_THREADS, smem, st, mel, mel_lens, group, B, F, C, G, Fg, joined,
                group_lens);
}
// pcm = (int16) trunc(wav * 32768): numpy astype('int16') of a float array is a C cast
// (inference_am_vocoder_joint.py:130-131).  Values are inside (-1, 1) after tanh; outside it they saturate.
__device__ __forceinline__ int16_t pcm16_of(float v) {
  v = truncf(v * 32768.0f);
  v = fminf(fmaxf(v, -32768.f), 32767.f);
  return (int16_t)(int)v;
}
__global__ void pcm16_kernel(const float* __restrict__ wav, int16_t* __restrict__ pcm, size_t n) {
  pdl_entry();
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) pcm[i] = pcm16_of(wav[i]);
}
int launch_pcm16(const float* wav, int16_t* pcm, size_t n, cudaStream_t st) {
  if (n == 0) return EV_OK;
  return launch("pcm16_kernel", pcm16_kernel, (unsigned)((n + 255) / 256), 256, 0, st, wav, pcm, n);
}

// G.711 of a 16-bit sample, the segment encoders of ITU-T G.711 as Python's audioop.lin2ulaw / lin2alaw apply them to 16-bit
// input: mu-law codes the top 14 bits (bias 33, magnitude clipped at 8159, all bits inverted), A-law the top 13 bits (even bits
// inverted).  tests/golden/g711.npz holds both functions over all 65,536 inputs.
__device__ __forceinline__ uint8_t mulaw_of(int16_t s) {
  int v = s >> 2;
  int mask = 0xFF;
  if (v < 0) {
    v = -v;
    mask = 0x7F;
  }
  v = min(v, 8159) + 33;
  int seg = 0;
  while (seg < 8 && v > (0x40 << seg) - 1) ++seg;
  if (seg >= 8) return (uint8_t)(0x7F ^ mask);
  return (uint8_t)(((seg << 4) | ((v >> (seg + 1)) & 0xF)) ^ mask);
}
__device__ __forceinline__ uint8_t alaw_of(int16_t s) {
  int v = s >> 3;
  int mask = 0xD5;
  if (v < 0) {
    v = -v - 1;
    mask = 0x55;
  }
  int seg = 0;
  while (seg < 8 && v > (0x20 << seg) - 1) ++seg;      // |v| <= 4095: seg <= 7
  const int q = (seg < 2 ? v >> 1 : v >> seg) & 0xF;
  return (uint8_t)(((seg << 4) | q) ^ mask);
}
__device__ __forceinline__ void store_sample(void* out, int encoding, long long i, float v) {
  switch (encoding) {
    case EV_AUDIO_FLOAT32: static_cast<float*>(out)[i] = v; break;
    case EV_AUDIO_PCM16: static_cast<int16_t*>(out)[i] = pcm16_of(v); break;
    case EV_AUDIO_MULAW: static_cast<uint8_t*>(out)[i] = mulaw_of(pcm16_of(v)); break;
    default: static_cast<uint8_t*>(out)[i] = alaw_of(pcm16_of(v)); break;
  }
}

// Output formatting: listed item k = items[k] (k when items is null) of the waveform batch, n = n_in[b] valid samples, resampled
// by up/down and encoded into out[out_off[k] ...] as ceil(n * up / down) samples.  Resampling is scipy.signal.resample_poly with
// its default filter: output o is  sum_j bank[ph][j] * x[q / up - j]  with q = o * down + half_len, ph = q % up, where bank is the
// phase-major split bank[ph][j] = h[ph + j * up] of the (2 * half_len + 1)-tap filter h (zero past its end) and x reads as zero
// outside [0, n).  Each output is one fp32 chain over the taps in order j = 0, 1, ..., so an item's samples do not depend on the
// batch, the item list, the tile or the CTA that computes them.  bank == null: up == down == 1, the samples are copied.
// A CTA takes tiles of AO_TILE consecutive outputs of one item (grid-stride over the item's tiles); it stages the bank once and,
// per tile, the input window the tile reads, with zeros outside [0, n): no sample at or past n_in[b] is ever read.
// gain (one per listed item, or null): each output is encoded as fp32(acc * gain[k]); it is read after pdl_entry() because the
// launch just before this one (ev_loudness's gate kernel) writes it.
constexpr int AO_THREADS = 256, AO_TILE = AO_THREADS, AO_CTAS_PER_SM = 8;
__global__ void __launch_bounds__(AO_THREADS) audio_out_kernel(const float* __restrict__ wav, long long item_stride,
                                                               const int64_t* __restrict__ n_in, const int64_t* __restrict__ items,
                                                               const int64_t* __restrict__ out_off, const float* __restrict__ bank,
                                                               int up, int down, int taps, int half_len, int window, int encoding,
                                                               const float* __restrict__ gain, void* __restrict__ out) {
  pdl_entry();
  extern __shared__ __align__(16) float ao_smem[];
  const int k = blockIdx.y;
  const long long b = items ? items[k] : k;
  const long long n = n_in[b];
  const long long n_out = (n * up + down - 1) / down;
  const long long tiles = (n_out + AO_TILE - 1) / AO_TILE;
  if ((long long)blockIdx.x >= tiles) return;
  const float* x = wav + b * item_stride;
  const long long o_base = out_off[k];
  if (!bank) {
    for (long long t = blockIdx.x; t < tiles; t += gridDim.x) {
      const long long o = t * AO_TILE + threadIdx.x;
      if (o < n_out) store_sample(out, encoding, o_base + o, gain ? x[o] * gain[k] : x[o]);
    }
    return;
  }
  float* hs = ao_smem;                 // [up][taps]
  float* xs = ao_smem + up * taps;     // [window]: inputs i0 .. i0 + window - 1 of the current tile
  for (int i = threadIdx.x; i < up * taps; i += AO_THREADS) hs[i] = bank[i];
  for (long long t = blockIdx.x; t < tiles; t += gridDim.x) {
    const long long o0 = t * AO_TILE;
    const long long i0 = (o0 * down + half_len) / up - (taps - 1);
    __syncthreads();                   // the previous tile's reads of xs are done
    for (int i = threadIdx.x; i < window; i += AO_THREADS) {
      const long long s = i0 + i;
      xs[i] = (s >= 0 && s < n) ? x[s] : 0.f;
    }
    __syncthreads();
    const long long o = o0 + threadIdx.x;
    if (o < n_out) {
      const long long q = o * down + half_len;
      const float* h = hs + (int)(q % up) * taps;
      const float* xr = xs + (int)(q / up - i0);
      float acc = 0.f;
      for (int j = 0; j < taps; ++j) acc = fmaf(h[j], xr[-j], acc);
      if (gain) acc *= gain[k];
      store_sample(out, encoding, o_base + o, acc);
    }
  }
}
int launch_audio_out(const float* wav, long long item_stride, const int64_t* n_in, const int64_t* items, int n_items,
                     const int64_t* out_off, const float* bank, int up, int down, int taps, int encoding, const float* gain, void* out,
                     cudaStream_t st) {
  EV_CHECK_ARG(n_items >= 1 && n_items <= 65535 && item_stride >= 0, "format_audio: n_items=%d must lie in [1, 65535], item_stride=%lld",
               n_items, item_stride);
  EV_CHECK_ARG(encoding >= EV_AUDIO_FLOAT32 && encoding <= EV_AUDIO_ALAW, "format_audio: unknown encoding %d", encoding);
  EV_CHECK_ARG(up >= 1 && down >= 1 && up <= AO_MAX_FACTOR && down <= AO_MAX_FACTOR, "format_audio: up=%d down=%d must lie in [1, %d]", up,
               down, AO_MAX_FACTOR);
  int a = up, c = down;
  while (c) { const int r = a % c; a = c; c = r; }
  EV_CHECK_ARG(a == 1, "format_audio: up=%d and down=%d must be coprime", up, down);
  EV_CHECK_ARG((bank == nullptr) == (up == 1 && down == 1), "format_audio: a filter bank is needed exactly when up/down != 1");
  const int half_len = 10 * (up > down ? up : down);
  int window = 0;
  size_t smem = 0;
  if (bank) {
    const int want = (2 * half_len + 1 + up - 1) / up;
    EV_CHECK_ARG(taps == want, "format_audio: taps_per_phase=%d, the %d-tap filter of up=%d down=%d has %d", taps, 2 * half_len + 1, up,
                 down, want);
    window = ((AO_TILE - 1) * down + up - 1) / up + taps;
    smem = (size_t)(up * taps + window) * sizeof(float);
    static std::atomic<uint64_t> attr_devs{0};
    if (first_use_on_device(attr_devs))
      cudaFuncSetAttribute(audio_out_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
  }
  const int per_item = (AO_CTAS_PER_SM * sm_count() + n_items - 1) / n_items;
  dim3 grid(per_item, n_items);
  return launch("audio_out_kernel", audio_out_kernel, grid, AO_THREADS, smem, st, wav, item_stride, n_in, items, out_off, bank, up, down,
                taps, half_len, window, encoding, gain, out);
}

void preload_voc_kernels() {      // see preload_conv1d_gp
  cudaFuncAttributes fa;
  cudaFuncGetAttributes(&fa, join_mel_kernel);
  cudaFuncGetAttributes(&fa, audio_out_kernel);
  cudaGetLastError();
}

}  // namespace ev
