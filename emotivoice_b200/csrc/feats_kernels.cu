// Log-mel spectrograms and frame energy of recordings (the reference computes them on the CPU with librosa / conv1d):
//   * TacotronSTFT.mel_spectrogram   (tacotron_stft.py:71-80, stft.py:132-160)  reflect pad 512, |X|, mel, log(clamp 1e-5)
//   * mel_spectrogram_torch          (mel_process.py:77-110)                    reflect pad (1024-hop)/2, sqrt(|X|^2 + 1e-6), mel, log
//   * Energy._calculate_energy       (feats.py:188-196)                         reflect pad 512, sqrt(max(sum_k |X_k|^2, 1e-10))
// They share one kernel: the caller passes the padding, the window (each variant's own fp32 rounding of the periodic Hann
// window), the magnitude's epsilon and the band table of the mel basis.  The FFT size is fixed at 1024.
//
// One CTA per (item, tile of kTile frames).  The tile's input span is staged in shared memory once, with the reflect padding
// applied in the index map; nothing at or past n_samples[b] is read.  Each warp transforms one frame at a time: the 1024 real
// samples are taken as 512 complex pairs z[n] = w[2n] x[2n] + i w[2n+1] x[2n+1], transformed by three radix-8 Stockham stages
// in shared memory (stockham.cuh: fp32 FFMA, twiddles from a host table built in fp64), and split into bins 0..512 of the
// real transform:
//   X[k] = E[k] + W_1024^k O[k],  E = (Z[k] + conj Z[512-k]) / 2,  O = (Z[k] - conj Z[512-k]) / 2i.
// The epilogue (magnitude, energy, mel bands, log) runs in the same warp; results leave through a per-tile buffer so the
// channels-first mel rows are stored along time.  Every output is computed from its own item's samples in a fixed order, so a
// batch is bitwise its items' single-item calls.
#include "ev_common.cuh"
#include "stockham.cuh"

namespace ev {

constexpr int kNfft = 1024;
constexpr int kHalf = kNfft / 2;           // points of the complex FFT
constexpr int kBins = kHalf + 1;           // one-sided bins 0..512
constexpr int kTile = 32;                  // frames per CTA
constexpr int kWarps = 8;
constexpr int kBufLd = kHalf + kHalf / 8;  // one padding slot per 8 complex values: the stage stores hit distinct banks
constexpr int kMagLd = 516;
constexpr int kMaxMels = 128;
constexpr size_t kSmemMax = 227 * 1024;

struct FeatsParams {
  const float* wav;
  long long item_stride;
  const int64_t* n_samples;  // (B) or null: every item has item_stride samples
  int pad, hop, F, n_mels;
  const float* window;       // (1024)
  const float2* twiddle;     // (1024): (cos, -sin)(2 pi k / 1024)
  float mag_eps;
  const int32_t* bands;      // (n_mels, 3): first bin, bin count, offset into band_w
  const float* band_w;
  float* mel;                // (B, n_mels, F) or null
  float* energy;             // (B, F) or null
  int32_t* status;           // or null
};

__global__ void __launch_bounds__(kWarps * 32) stft_feats_kernel(const FeatsParams p) {
  pdl_entry();
  extern __shared__ __align__(16) unsigned char feats_smem[];
  float2* tw = reinterpret_cast<float2*>(feats_smem);                  // kNfft
  float* win = reinterpret_cast<float*>(tw + kNfft);                   // kNfft
  float2* bufs = reinterpret_cast<float2*>(win + kNfft);               // kWarps x kBufLd
  float* mags = reinterpret_cast<float*>(bufs + kWarps * kBufLd);      // kWarps x kMagLd
  float* otile = mags + kWarps * kMagLd;                               // (n_mels + 1) x kTile: mel rows, then energy
  float* span = otile + (p.n_mels + 1) * kTile;                        // hop * (kTile - 1) + kNfft samples

  const int b = blockIdx.y, f0 = blockIdx.x * kTile;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long n = p.n_samples ? (long long)p.n_samples[b] : p.item_stride;
  // an item must be longer than the padding (F.pad(reflect)) and fill at least one frame; otherwise it has no frames
  const long long padded = n + 2ll * p.pad;
  const bool valid = n > p.pad && n <= p.item_stride && padded >= kNfft;
  const int Fb = valid ? (int)min((long long)p.F, (padded - kNfft) / p.hop + 1) : 0;
  const int nf = max(0, min(kTile, Fb - f0));
  int bad = 0;
  if (nf > 0) {
    const float* x = p.wav + (long long)b * p.item_stride;
    for (int i = tid; i < kNfft; i += blockDim.x) {
      tw[i] = p.twiddle[i];
      win[i] = p.window[i];
    }
    const int len = p.hop * (nf - 1) + kNfft;
    const long long s0 = (long long)f0 * p.hop - p.pad;
    for (int i = tid; i < len; i += blockDim.x) {
      long long s = s0 + i;
      s = s < 0 ? -s : (s >= n ? 2 * (n - 1) - s : s);                  // reflect: the edge sample is not repeated
      const float v = x[s];
      bad |= !(fabsf(v) <= 1.f);
      span[i] = v;
    }
    if (f0 + nf == Fb) {                                                  // samples past the last frame: the range check only
      for (long long s = max(0ll, s0 + len) + tid; s < n; s += blockDim.x) bad |= !(fabsf(x[s]) <= 1.f);
    }
  }
  if (__syncthreads_or(bad) && tid == 0 && p.status) atomicOr(p.status, 1);
  if (tid == 0 && p.status && !valid && blockIdx.x == 0) atomicOr(p.status, 2);

  float2* buf = bufs + warp * kBufLd;
  float* mag = mags + warp * kMagLd;
  for (int fl = warp; fl < nf; fl += kWarps) {
    const float* fr = span + fl * p.hop;
    {
      // stage 1 (NS = 1, no twiddles) straight from the windowed samples
      float2 v[2][8];
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int j = lane + 32 * q;
#pragma unroll
        for (int r = 0; r < 8; ++r) {
          const int m = 2 * (j + 64 * r);
          v[q][r] = make_float2(win[m] * fr[m], win[m + 1] * fr[m + 1]);
        }
        fft8(v[q]);
      }
      stockham_store<1>(v, buf, lane);
      __syncwarp();
    }
    stockham_stage<8>(buf, tw, lane);
    stockham_stage<64>(buf, tw, lane);
    // bins of the real transform, magnitudes and the energy sum (each lane over its bins in ascending order, then a fixed tree)
    float esum = 0.f;
    for (int k = lane; k < kBins; k += 32) {
      const float2 zk = buf[bpad(k & (kHalf - 1))], zm = buf[bpad((kHalf - k) & (kHalf - 1))];
      const float er = 0.5f * (zk.x + zm.x), ei = 0.5f * (zk.y - zm.y);
      const float orr = 0.5f * (zk.y + zm.y), oi = -0.5f * (zk.x - zm.x);
      const float2 w = tw[k];
      const float xr = er + (orr * w.x - oi * w.y);
      const float xi = ei + (orr * w.y + oi * w.x);
      const float pw = xr * xr + xi * xi;
      esum += pw;
      mag[k] = sqrtf(pw + p.mag_eps);
    }
    __syncwarp();
    if (p.energy) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) esum += __shfl_xor_sync(0xffffffffu, esum, o);
      if (lane == 0) otile[p.n_mels * kTile + fl] = sqrtf(fmaxf(esum, 1e-10f));
    }
    if (p.mel) {
      for (int j = lane; j < p.n_mels; j += 32) {
        const int first = __ldg(p.bands + 3 * j), cnt = __ldg(p.bands + 3 * j + 1), off = __ldg(p.bands + 3 * j + 2);
        float acc = 0.f;
        for (int t = 0; t < cnt; ++t) acc = fmaf(__ldg(p.band_w + off + t), mag[first + t], acc);
        otile[j * kTile + fl] = logf(fmaxf(acc, 1e-5f));
      }
    }
    __syncwarp();
  }
  __syncthreads();
  // frames f0 .. f0 + kTile - 1 that exist in the output; those past the item's own frame count are stored as 0
  const int nout = min(kTile, p.F - f0);
  if (p.mel) {
    for (int i = tid; i < p.n_mels * kTile; i += blockDim.x) {
      const int j = i / kTile, fl = i % kTile;
      if (fl < nout) p.mel[((long long)b * p.n_mels + j) * p.F + f0 + fl] = fl < nf ? otile[j * kTile + fl] : 0.f;
    }
  }
  if (p.energy) {
    for (int fl = tid; fl < nout; fl += blockDim.x) p.energy[(long long)b * p.F + f0 + fl] = fl < nf ? otile[p.n_mels * kTile + fl] : 0.f;
  }
}

static size_t feats_smem_bytes(int hop, int n_mels) {
  return (size_t)kNfft * sizeof(float2) + kNfft * sizeof(float) + (size_t)kWarps * kBufLd * sizeof(float2) +
         (size_t)kWarps * kMagLd * sizeof(float) + (size_t)(n_mels + 1) * kTile * sizeof(float) +
         ((size_t)hop * (kTile - 1) + kNfft) * sizeof(float);
}

int launch_stft_features(const FeatsParams& p, int B, cudaStream_t st) {
  const size_t smem = feats_smem_bytes(p.hop, p.n_mels);
  EV_CHECK_ARG(smem <= kSmemMax, "stft_features: %zu bytes of shared memory", smem);
  static std::atomic<uint64_t> attr_devs{0};
  if (first_use_on_device(attr_devs)) cudaFuncSetAttribute(stft_feats_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemMax);
  dim3 grid((p.F + kTile - 1) / kTile, B);
  return launch("stft_feats_kernel", stft_feats_kernel, grid, kWarps * 32, smem, st, p);
}

}  // namespace ev

using namespace ev;

extern "C" {

int ev_stft_features(const float* wav, long long item_stride, const int64_t* n_samples, int B, int pad, int hop, int F,
                     const float* window, const float* twiddle, float mag_eps, const int32_t* bands, const float* band_w, int n_mels,
                     float* mel, float* energy, int32_t* status, void* stream) {
  EV_CHECK_ARG(wav && window && twiddle, "ev_stft_features: null argument");
  EV_CHECK_ARG(mel || energy, "ev_stft_features: neither mel nor energy requested");
  EV_CHECK_ARG(B > 0 && B <= 65535 && F > 0 && item_stride > 0, "ev_stft_features: B=%d F=%d item_stride=%lld", B, F, item_stride);
  EV_CHECK_ARG(hop >= 1 && hop <= kNfft && pad >= 0 && pad < kNfft, "ev_stft_features: hop %d must be in [1, 1024], pad %d in [0, 1024)", hop,
               pad);
  EV_CHECK_ARG(!mel || (bands && band_w && n_mels >= 1 && n_mels <= kMaxMels), "ev_stft_features: mel needs band tables and 1 <= n_mels <= %d (%d)",
               kMaxMels, n_mels);
  EV_CHECK_ARG(mag_eps >= 0.f, "ev_stft_features: mag_eps %g < 0", (double)mag_eps);
  EV_CHECK_ARG(n_samples || item_stride > pad, "ev_stft_features: items of %lld samples are not longer than the padding %d", item_stride, pad);
  EV_TRY(use_device_of(wav));
  FeatsParams p;
  p.wav = wav;
  p.item_stride = item_stride;
  p.n_samples = n_samples;
  p.pad = pad;
  p.hop = hop;
  p.F = F;
  p.n_mels = mel ? n_mels : 0;
  p.window = window;
  p.twiddle = reinterpret_cast<const float2*>(twiddle);
  p.mag_eps = mag_eps;
  p.bands = bands;
  p.band_w = band_w;
  p.mel = mel;
  p.energy = energy;
  p.status = status;
  return launch_stft_features(p, B, reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
