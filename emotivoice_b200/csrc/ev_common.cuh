// Shared declarations of the sm_90a engine (internal; the public ABI is include/emotivoice_b200.h).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>
#include <string>
#include "../../include/emotivoice_b200.h"

namespace ev {

// thread-local error string behind ev_last_error()
void set_error(const char* fmt, ...);
void count_launch(int n = 1);

// Per-device one-time set-up.  cudaFuncSetAttribute and the SM count are per device and an engine may live on any GPU of the
// process, so "done once" is tracked per device (bit d of `mask`); a benign race sets an attribute twice.
inline bool first_use_on_device(std::atomic<uint64_t>& mask) {
  int d = 0;
  cudaGetDevice(&d);
  const uint64_t bit = 1ull << (d & 63);
  if (mask.load(std::memory_order_relaxed) & bit) return false;
  mask.fetch_or(bit, std::memory_order_relaxed);
  return true;
}
int sm_count();                          // SMs of the CURRENT device (cached per device)
// eager loading of the big tensor-core kernels' code on the current device (ev_create calls them once per device)
void preload_conv1d_gp();
void preload_resblock_gp();
void preload_attention_tc();
void preload_conv1d_tc();
int use_device_of(const void* dev_ptr);  // cudaSetDevice(the device that owns dev_ptr); EV_OK / EV_ECUDA

#define EV_CHECK_ARG(cond, ...)                      \
  do {                                               \
    if (!(cond)) {                                   \
      ev::set_error(__VA_ARGS__);                    \
      return EV_EINVAL;                              \
    }                                                \
  } while (0)

#define EV_TRY(expr)                 \
  do {                               \
    int rc__ = (expr);               \
    if (rc__ != EV_OK) return rc__;  \
  } while (0)

// ---------------------------------------------------------------------------------
// Programmatic dependent launch (measured 9 % on the batch-1 step, bitwise-identical results).  Every kernel of the engine
// starts with griddepcontrol.launch_dependents (the next launch in the stream may be scheduled as soon as every CTA of this
// grid has started) followed by griddepcontrol.wait (returns once the preceding grid has completed and its writes are
// visible) -- before its first memory access, so stream order semantics are unchanged; what is gained is the launch
// latency and, for the convolutions, the set-up (barriers, first weight stages) that runs before the wait.  Launched
// without the attribute (EV_PDL=0), both instructions are no-ops.
// Transitivity: every kernel has at least one thread that waits unconditionally, so "grid N complete" implies "grid N-1 complete".
// ---------------------------------------------------------------------------------
__device__ __forceinline__ void pdl_entry() {
  asm volatile("griddepcontrol.launch_dependents;\n\tgriddepcontrol.wait;" ::: "memory");
}
bool pdl_enabled();  // false iff EV_PDL=0 (read once)

// The engine's one way to launch a kernel: with programmatic stream serialization unless EV_PDL=0.  Reports the launch's own
// error, or else the one cudaGetLastError() holds (and clears it), as "what: <error>"; counts the launch on success.
template <typename... KArgs, typename... Args>
inline int launch(const char* what, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cfg.attrs = at;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, args...);
  const cudaError_t last = cudaGetLastError();
  if (e == cudaSuccess) e = last;
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    return EV_ECUDA;
  }
  count_launch();
  return EV_OK;
}

// ---------------------------------------------------------------------------------
// generic time-major conv (conv1d_tm.cu)
// ---------------------------------------------------------------------------------
struct ConvParams {
  const float* x;      // (B, L, Cin)
  const float* w;      // (K, Cin, Cout)
  const float* bias;   // (Cout) or per item (bias_bs floats apart); may be null
  const float* res;    // (B, L, Cout) or null
  float* out;          // (B, L, Cout)
  long long bias_bs;
  int B, L, Cin, Cout, K, dil;
  const int32_t* lens; // valid rows per item = lens[b]*lens_mul (null: L)
  int lens_mul;
  int in_act;          // EV_ACT_NONE / EV_ACT_LRELU
  float in_slope;
  int out_act;         // EV_ACT_*
  int acc;             // EV_ACC_*
  float div;
  // optional scratch for deterministic split-K on the tensor-core path (conv1d_tc.cu); floats
  float* splitk_ws = nullptr;
  size_t splitk_cap = 0;
  int ksplit = 0;      // requested K-split factor (fixed per LAYER by the engine, never by batch size: keeps the
                       // summation order, hence every output bit, independent of how utterances are batched)
};
int launch_conv1d(const ConvParams& p, cudaStream_t st);
// host-only: the plan launch_conv1d would use, {TXN, NV, TM, BM, BN, rows_a, a_ld, smem bytes, grid.x, grid.y}
int debug_conv1d_plan(const ConvParams& p, int* v10);
// tensor-core variant (conv1d_tc.cu); p.w in the tensor-core layout [plane hi|lo][Cout/BNp][K][Cin/4][BNp][4], BNp = min(Cout,128);
// mode 0: one tf32 MMA per K step; 1: 3xTF32 fp32 emulation (three MMAs per K step); 2: bf16 operands
// (p.w then in the bf16 layout [Cout/BNp][K][Cin/8][BNp][8 bf16]).
int launch_conv1d_tc(const ConvParams& p, int mode, cudaStream_t st);
int debug_tc_plan(const ConvParams& p, int mode, int* v11);   // host-only: the plan launch_conv1d_tc would use
int tc_shape_kbg(const ConvParams& p, int mode);               // K granules per stage: a function of the layer shape only

// ---------------------------------------------------------------------------------
// HiFi-GAN convolutions on granule-planar activations (conv1d_gp.cu): [b][C/cpg][L][cpg], 16-byte granules of 4 fp32 or
// 8 bf16 channels; the A operand is bulk-copied, the epilogue stores straight from the accumulator registers.
// ---------------------------------------------------------------------------------
struct GpConvParams {
  const void* x;       // GP (B, Cin/cpg, L, cpg)
  const float* w;      // tensor-core weight layout of conv1d_tc (mode 0/1: two tf32 planes; mode 2: bf16)
  const float* bias;   // (Cout) fp32 or null
  const void* res;     // GP, shape of the output, or null (rate == 1 only)
  void* out;           // GP (B, (Cout/rate)/cpg, L*rate, cpg)
  int B, L, Cin, Cout, K, dil;
  int rate;            // polyphase ConvTranspose1d: the Cout GEMM columns are `rate` output phases of Cout/rate channels
  const int32_t* lens; // valid input rows per item = lens[b]*lens_mul (null: L); rows >= len are neither read nor written
  int lens_mul;
  int in_act;          // EV_ACT_NONE / EV_ACT_LRELU
  float in_slope;
  int acc;             // EV_ACC_*
  float div;
};
// What differs between the (up to three) convolutions of one grouped launch; the kernel's view of every launch (a single
// convolution is a group of one, filled from the scalar fields above).
struct GpGroup {
  const void* x;
  const float* w;
  const float* bias;
  const void* res;
  void* out;
  int K, dil;
};
struct GpGroups {
  int ng;
  GpGroup g[3];
};
int launch_conv1d_gp(const GpConvParams& p, int mode, cudaStream_t st);    // mode 0: tf32, 1: 3xTF32 (fp32 activations); 2: bf16 activations
// n <= 3 convolutions that share B, L, Cin, Cout, lens, the input activation and rate == 1, acc == STORE, as ONE launch (the three
// parallel ResBlocks of a HiFi-GAN stage at small batch, where a single convolution has too few tiles for the machine).  Every tile is
// computed exactly as in the convolution's own launch: bitwise equal.  EV_EINVAL (nothing launched) if the shapes cannot share a launch.
int launch_conv1d_gp_group(const GpConvParams* ps, int n, int mode, cudaStream_t st);
bool gp_group_supported(const GpConvParams* ps, int n, int mode);
int debug_gp_group_plan(const GpConvParams* ps, int n, int mode, int* v11);
int gp_solo_tiles(const GpConvParams& p, int mode);       // tiles of the convolution's own launch (0 if it cannot be planned)
int debug_gp_plan(const GpConvParams& p, int mode, int* v11);
int gp_shape_kbg(const GpConvParams& p, int mode);     // K granules per stage: a function of the layer shape, it fixes the reduction order
// fp32 in[b*sb + t*st + c*sc] -> GP (fp32, or bf16 when bf16 != 0)
int launch_to_gp(const float* in, long long sb, long long st_, long long sc, void* out, int B, int L, int C, int bf16, cudaStream_t st);
// One ResBlock1 layer  out = [acc]( x + c2(lrelu(c1(lrelu(x), dil)), 1) )  as one kernel on granule-planar activations
// (resblock_gp.cu); bitwise equal to the two launch_conv1d_gp calls it replaces.  C in {32, 64, 128}.
struct GpPairParams {
  const void* x;       // GP (B, C/cpg, L, cpg): the layer input, also the residual
  const float* w1;     // c1 weights (k taps, dilation dil), tensor-core layout of the mode
  const float* b1;
  const float* w2;     // c2 weights (k taps, dilation 1)
  const float* b2;
  void* out;           // GP, same shape; must not alias x
  int B, L, C, K, dil;
  const int32_t* lens; // valid rows per item = lens[b]*lens_mul (null: L)
  int lens_mul;
  float slope;         // LeakyReLU slope of both prologues (0.1)
  int acc;             // EV_ACC_*
  float div;
};
// The kernel's view: up to three layers of one shape in a launch (a single layer is a group of one).
struct GpPairGroup {
  const void* x;
  const float *w1, *b1, *w2, *b2;
  void* out;
  int K, dil;
  int R, tiles_m, tile0;   // output rows per tile (128*MT - (K-1)), row tiles per item, first tile index of the member
};
struct GpPairGroups {
  int ng;
  GpPairGroup g[3];
};
bool gp_pair_supported(const GpPairParams& p, int mode);
int launch_gp_pair(const GpPairParams& p, int mode, cudaStream_t st);      // mode as launch_conv1d_gp
// n <= 3 layers sharing B, L, C, lens, slope and acc == STORE as ONE launch (the same-index layers of HiFi-GAN's parallel ResBlocks
// at small batch); every tile is computed as in the member's own launch: bitwise equal.
bool gp_pair_group_supported(const GpPairParams* ps, int n, int mode);
int launch_gp_pair_group(const GpPairParams* ps, int n, int mode, cudaStream_t st);
int gp_pair_solo_tiles(const GpPairParams& p, int mode);
int debug_gp_pair_group_plan(const GpPairParams* ps, int n, int mode, int* v16);
int debug_gp_pair_plan(const GpPairParams& p, int mode, int* v11);
// out = ((b + a) [+ c]) / div on whole fp32 tensors (c may be null): the stage-level `xs / n` after a grouped last layer
int launch_gp_sum_div(const float* a, const float* b, const float* c, float* out, size_t n_floats, float div, cudaStream_t st);
int launch_conv_post_gp(const void* x, int bf16, const float* w, const float* bias, const int32_t* lens, int lens_mul, int B, int L, int C, int K,
                        float slope, float* wav, cudaStream_t st);

// ---------------------------------------------------------------------------------
// acoustic-model kernels (am_kernels.cu)
// ---------------------------------------------------------------------------------
// y = LN(x) over C; optional prologue x = emb[ids] + alpha*pe[t] (written to x_out).
int launch_layernorm(const float* x, const int64_t* ids, const float* emb, const float* pe, const float* alpha,
                     float* x_out, const float* w, const float* b, float* y, int rows, int L, int C,
                     cudaStream_t st, int n_emb = 0);
int launch_attention(const float* qkv, const int32_t* key_lens, float* ctx, int B, int L, int H, int heads,
                     cudaStream_t st);
// tensor-core variant (attention_tc.cu), d_k = 48 only; tc_mode 1: 3xTF32 fp32 emulation, 0: one tf32 MMA per K step
int launch_attention_tc(const float* qkv, const int32_t* key_lens, float* ctx, int B, int L, int H, int heads, int tc_mode, cudaStream_t st);
int launch_cond_gather(const int64_t* spk, const float* spk_emb, const float* style, const float* content,
                       float* out, int B, int H, int bert, int n_spk, cudaStream_t st);
int launch_cond_gemv(const float* c, const float* w, const float* bias, float* out, int B, int K, int N, cudaStream_t st);
// y[row] = dot(x[row,:], w) + b ; masked rows (t >= lens[b]) -> 0.  mode 0: float out; mode 1: duration int64
int launch_rowdot(const float* x, const float* w, const float* b, const int32_t* lens, int B, int T, int C,
                  int mode, float* out_f, int64_t* out_i, cudaStream_t st);
// lens -> int32 clamped to [0, T] + range checks of token / speaker ids and lengths into *status (bits 1 / 2 / 4); ling, spk, status may be null
int launch_validate_inputs(const int64_t* ling, const int64_t* lens, const int64_t* spk, int32_t* lens_out, int32_t* status, int B,
                           int T, int n_vocab, int n_spk, cudaStream_t st);
// zero rows t >= lens[b] of x (B,T,C) into y (masked_fill of the predictors' input)
int launch_mask_rows(const float* x, const int32_t* lens, float* y, int B, int T, int C, cudaStream_t st);
// prosody {alpha, p_scale, p_shift, e_scale, e_shift} rows or null (neutral): (B,5), or (B,T,5) when per_token (rows of pad
// tokens t >= lens[b] act as neutral); lens: item lengths or null; window: with prosody the window ends at lens[b];
// zero_pads: track entries at t >= lens[b] read as 0 (caller-given tracks)
int launch_var_embed_add(float* x, const float* pitch, const float* energy, const float* wp, const float* bp,
                         const float* we, const float* be, const float* prosody, int per_token, const int32_t* lens, int window,
                         int zero_pads, int B, int T, int C, int K, cudaStream_t st);
// alpha[b * alpha_stride + t * alpha_tstride] scales duration (b,t) (null: 1); caller: dur holds caller durations (pads
// t >= lens[b] ignored, negatives clamped to 0); status (may be null) |= 8 when an output has no frames, |= 16 when a caller
// duration is negative or an item's frame count (before or after scaling) exceeds max_frames
int launch_duration_scan(const int64_t* dur, int caller, const int32_t* lens, const float* alpha, int alpha_stride, int alpha_tstride,
                         int invariant, int B, int T, float* centers, float* ds_f, int32_t* mel_lens, int32_t* status, int max_frames,
                         cudaStream_t st);
int launch_gauss_upsample(const float* hs, const float* centers, const int32_t* lens, const int32_t* mel_lens,
                          int B, int T, int H, int F, int invariant, const float* pe, const float* alpha,
                          float* out, cudaStream_t st);

// ---------------------------------------------------------------------------------
// vocoder kernels (voc_kernels.cu)
// ---------------------------------------------------------------------------------
int launch_transpose_cf_to_tm(const float* in, float* out, int B, int C, int L, cudaStream_t st);
// wav[b,t] = tanh(bias + sum_j sum_c w[j][c] * lrelu_slope(x[b,t+j-K/2,c])); rows >= len -> 0
int launch_conv_post(const float* x, const float* w, const float* bias, const int32_t* lens, int lens_mul, int B,
                     int L, int C, int K, float slope, float* wav, cudaStream_t st);
int launch_pcm16(const float* wav, int16_t* pcm, size_t n, cudaStream_t st);
// resample by up/down (scipy.signal.resample_poly, default filter) + scale by an optional per-item gain + encode the valid samples
// of listed waveform items, packed (ev_format_audio)
constexpr int AO_MAX_FACTOR = 1024;
int launch_audio_out(const float* wav, long long item_stride, const int64_t* n_in, const int64_t* items, int n_items,
                     const int64_t* out_off, const float* bank, int up, int down, int taps, int encoding, const float* gain, void* out,
                     cudaStream_t st);
// valid rows of mel (B,F,C) of consecutive items with one group id, concatenated -> joined (G,Fg,C), zero past each group's
// length; group_lens[g] = min(group frames, Fg).  B <= 4096.
int launch_join_mel(const float* mel, const int32_t* mel_lens, const int32_t* group, int B, int F, int C, int G, int Fg, float* joined,
                    int32_t* group_lens, cudaStream_t st);
void preload_voc_kernels();

// ---------------------------------------------------------------------------------
// loudness stages of ev_loudness (loudness_kernels.cu), which ev_meter runs too
// ---------------------------------------------------------------------------------
long long loud_max_sub(long long max_n, int sample_rate);      // 100 ms sub-blocks of an item of max_n samples (the last partial)
bool loud_grid_ok(long long max_n, int sample_rate);           // the sub-block grid of max_n fits a launch
int restart_warmup(const double* kcoef);                       // W of the K-weighting restart, or -1 (unstable / too slow)
// energy / peak (n_items, loud_max_sub(item_stride)) of every sub-block; item b at wav + start[b] (start NULL: b * item_stride),
// n_in[b] valid samples clamped to item_stride
int launch_loud_subblock(const float* wav, long long item_stride, const int64_t* start, const int64_t* n_in, const int64_t* items,
                         int n_items, int sample_rate, const double* kcoef, int W, double* energy, float* peak, cudaStream_t st);
// gated integrated loudness, sample peak and normalisation gain of each item from those sub-blocks
int launch_loud_gate(long long item_stride, const int64_t* n_in, const int64_t* items, int n_items, int sample_rate,
                     const double* energy, const float* peak, double target, float* lufs, float* peak_out, float* gain, cudaStream_t st);

__device__ __forceinline__ float act_apply(float v, int act, float slope) {
  switch (act) {
    case EV_ACT_LRELU: return v > 0.f ? v : v * slope;
    case EV_ACT_RELU: return v > 0.f ? v : 0.f;
    case EV_ACT_GELU: return 0.5f * v * (1.0f + erff(v * 0.70710678118654752440f));
    case EV_ACT_TANH: return tanhf(v);
    default: return v;
  }
}

}  // namespace ev
