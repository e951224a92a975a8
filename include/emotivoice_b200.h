/*
 * emotivoice_b200.h -- C ABI of libemotivoice_b200.so (sm_90a, H100).
 *
 * The reference (netease-youdao/EmotiVoice) has no FFI / plugin registry: its
 * boundary for this path is the Python torch.nn.Module API of
 *   JETSGenerator.forward      models/prompt_tts_modified/jets.py:50-71
 *   PromptTTS.forward          models/prompt_tts_modified/model_open_source.py:102-163
 *   Generator.forward          models/hifigan/models.py:115-131
 * The host-side mirror of those classes lives in emotivoice_b200/modules.py and
 * binds the entry points below with ctypes (see INTEGRATION.md for the stub a
 * reference maintainer would add).  Everything here is plain C: device pointers,
 * sizes, a CUDA stream handle passed as void*.  No torch types.
 *
 * Conventions
 *   - every function returns 0 on success or a negative EV_E* code; nothing throws
 *     or aborts across the ABI; ev_last_error() gives the message (thread local).
 *   - all work is enqueued asynchronously on the caller's stream; the library never
 *     synchronises and never allocates device memory: the caller (PyTorch's caching
 *     allocator) owns weights, workspace, inputs and outputs.
 *   - activations are fp32, TIME-MAJOR ("channels last"): a tensor of L steps and C
 *     channels of batch item b lives at base + b*L*C, element (t, c) at t*C + c.
 *   - `lens` arrays are int32 on the device; NULL means "every item is L long"
 *     (the reference's literal padded-batch semantics).  With `lens` given, item b
 *     is treated exactly as the reference treats a B=1 call of that length: rows
 *     >= lens[b] read as zero padding and are written as zeros.
 *   - an ev_ctx is immutable after ev_bind_*; concurrent calls are safe as long as
 *     each call has its own workspace (reference callers are multi-threaded:
 *     openaiapi.py:162-163).
 */
#ifndef EMOTIVOICE_B200_H_
#define EMOTIVOICE_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EV_API __attribute__((visibility("default")))
#define EV_ABI_VERSION 1

enum {
  EV_OK = 0,
  EV_EINVAL = -1,      /* bad argument / unsupported shape */
  EV_ENOWEIGHT = -2,   /* a required tensor is missing from the bound blob */
  EV_ECUDA = -3,       /* CUDA runtime error (message has the cudaError string) */
  EV_EWORKSPACE = -4,  /* workspace too small */
  EV_EPELEN = -5,      /* positional table shorter than the sequence: rebind a longer one */
  EV_EARCH = -6        /* device is not sm_90 */
};

/* activation / epilogue selectors of ev_op_conv1d */
enum { EV_ACT_NONE = 0, EV_ACT_LRELU = 1, EV_ACT_RELU = 2, EV_ACT_GELU = 3, EV_ACT_TANH = 4 };
enum { EV_ACC_STORE = 0, EV_ACC_ADD = 1, EV_ACC_ADD_DIV = 2 };

typedef struct ev_ctx ev_ctx;

/* The integers of config/joint/config.yaml:36-94 (+ n_vocab / n_speaker patched in by
 * every reference caller, inference_am_vocoder_joint.py:57-58). */
typedef struct ev_config {
  int32_t n_vocab, n_speaker;
  int32_t hidden;            /* encoder_n_hidden == decoder_n_hidden == variance_n_hidden (384) */
  int32_t n_heads;           /* 8 */
  int32_t enc_layers, dec_layers;
  int32_t ffn_kernel;        /* *_kernel_size_conv_mod (3) */
  int32_t bert_dim;          /* bert_embedding (768) */
  int32_t dur_layers, pitch_layers, energy_layers;
  int32_t pred_kernel;       /* duration/variance kernel size (3) */
  int32_t embed_kernel;      /* variance_embed_kernel_size (9) */
  int32_t n_mels;            /* 80 */
  int32_t voc_c0;            /* upsample_initial_channel (512) */
  int32_t n_ups;             /* len(upsample_rates) (4) */
  int32_t up_rates[8];
  int32_t up_kernels[8];
  int32_t n_resk;            /* len(resblock_kernel_sizes) (3) */
  int32_t res_kernels[4];
  int32_t n_dil;             /* dilations per ResBlock1 (3) */
  int32_t res_dils[4][4];
} ev_config;

/* One tensor of the packed weight blob (built by emotivoice_b200/packing.py). */
typedef struct ev_weight_entry {
  char name[56];
  uint64_t offset;   /* in floats from the blob base */
  uint64_t numel;
} ev_weight_entry;

EV_API int ev_abi_version(void);
EV_API const char* ev_last_error(void);

/* Replaces: JETSGenerator.__init__ (jets.py:27-47). */
EV_API int ev_create(ev_ctx** out, int device, const ev_config* cfg);
EV_API void ev_destroy(ev_ctx* ctx);

/* Replaces: module.load_state_dict + the per-forward weight_norm recomputation
 * (hifigan/models.py:31-46,96-111).  The blob holds folded / re-laid-out fp32 weights;
 * the engine borrows it (caller keeps it alive). */
EV_API int ev_bind_weights(ev_ctx* ctx, const float* blob, size_t n_floats,
                           const ev_weight_entry* index, int n_entries);
/* Replaces: PositionalEncoding.extend_pe (encoder.py:206-237).  pe is (pe_len, hidden)
 * fp32 on the device, built by the host with the reference's formula. */
EV_API int ev_bind_pe(ev_ctx* ctx, const float* pe, int pe_len);

/* Arithmetic of the GEMM-shaped layers (linear / conv / transposed conv):
 *   EV_PREC_FP32 (default): fp32-accurate on the tensor cores: the duration-critical prefix (encoder, conditioning,
 *     predictors) by 3xTF32 splitting (x = hi + lo, three tf32 MMAs per K step), decoder + vocoder by bf16x3 splitting
 *     (two bf16 planes, three bf16 MMAs per K step); fp32 accumulation, error ~1e-6 / ~1e-5 relative.
 *   EV_PREC_TF32: decoder + vocoder with ONE tf32 MMA per K step (operands rounded to nearest tf32) -- the
 *     arithmetic the reference's eager PyTorch uses for convolutions on a GPU (cudnn.allow_tf32 default);
 *     the duration-critical prefix (encoder, conditioning, predictors) stays 3xTF32.
 *   EV_PREC_BF16: decoder + vocoder with bf16 operands (wgmma bf16, fp32 accumulation; activations stay fp32
 *     in HBM and are rounded by the staging warps); prefix 3xTF32 like EV_PREC_TF32.  BASELINE.json configs[2].
 *   EV_PREC_FP32_FFMA: plain fp32 FFMA kernels everywhere (no tensor cores; the round-1 baseline path).
 * Attention, LayerNorm, softmax, upsampling and the heads are fp32 in every mode.
 * Each mode reads one weight copy per layer ('.tc', '.tc16' or '.tc16x2'; packing.add_tc_weights writes all of them):
 * ev_bind_weights checks the blob against the context's mode and ev_set_precision a bound blob against the new mode: a missing
 * copy returns EV_ENOWEIGHT, leaving the context unbound / in its previous mode. */
enum { EV_PREC_FP32 = 0, EV_PREC_TF32 = 1, EV_PREC_FP32_FFMA = 2, EV_PREC_BF16 = 3 };
EV_API int ev_set_precision(ev_ctx* ctx, int precision);

/* Workspace sizes (bytes).  Phase 1 (encoder .. durations) is sized by (B, T); phase 2
 * (length regulator, decoder, to_mel) and the vocoder share one buffer sized by (B, F) --
 * F is only known after the host has read mel_lens_out[B] back. */
EV_API size_t ev_phase1_workspace_bytes(const ev_ctx* ctx, int B, int T);
EV_API size_t ev_phase2_workspace_bytes(const ev_ctx* ctx, int B, int F);

/* Replaces: PromptTTS.forward up to the duration prediction
 * (model_open_source.py:102-134; encoder.py:316-324; variance.py:36-56,101-124) plus
 * the cumsum / length bookkeeping of GaussianUpsampling (alignment.py:183-199).
 *   ling (B,T) i64; lens (B) i64 true phoneme counts (as the reference passes them); spk (B) i64;
 *   style, content (B,bert) f32
 *   dur_out (B,T) i64; pitch_out / energy_out (B,T) f32;
 *   lens32_out (B) i32: lens clamped to [0,T] (input of the later phases);
 *   mel_lens_out (B+2) i32: per-item frame counts, max over items in slot B, and in slot B+1 an input
 *     status word the host checks at the same read-back (the reference raises IndexError from nn.Embedding
 *     for these; the kernels clamp so nothing is read out of bounds): bit 0 = a token id outside
 *     [0, n_vocab), bit 1 = a speaker id outside [0, n_speaker), bit 2 = a length outside [1, T],
 *     bit 3 = an output with no frames (set only by ev_am_phase1_prosody with duration scales below 1:
 *     under the batch-invariant contract any item, otherwise the whole batch; the reference's decoder raises
 *     RuntimeError on a zero-length input), bit 4 = invalid caller durations or an item with more frames than
 *     the vocoder can index (see ev_am_phase1_controls).  Do not run phase 2 when bit 3 or 4 is set.
 *   invariant != 0: batch-invariant contract (each item == the reference's B=1 call);
 *   invariant == 0: literal padded-batch forward of the reference. */
EV_API int ev_am_phase1(ev_ctx* ctx, const int64_t* ling, const int64_t* lens, const int64_t* spk,
                        const float* style, const float* content, int B, int T, int invariant,
                        int64_t* dur_out, float* pitch_out, float* energy_out, int32_t* lens32_out,
                        int32_t* mel_lens_out, void* workspace, size_t workspace_bytes, void* stream);

/* ev_am_phase1 with per-item prosody controls.  prosody (B,5) f32 on the device, or NULL (== ev_am_phase1):
 * row b = {alpha, p_scale, p_shift, e_scale, e_shift}.
 *   alpha scales the predicted durations before the length regulator, ds = fl32(d * alpha), exactly the
 *     alpha of GaussianUpsampling.forward (alignment.py:180-183); the all-zero guard then writes 1, not alpha.
 *     The cumsum runs in fp64 (exact for these inputs) and rounds to fp32 like ATen's CPU cumsum;
 *     mel_lens[b] = trunc(fl32(exact sum)).  The reference's fp32 cascade sum can differ by one frame when the
 *     exact sum lies within a few fp32 ulps of an integer.
 *   pitch / energy enter pitch_embed / energy_embed (model_open_source.py:131-134) as p*p_scale + p_shift and
 *     e*e_scale + e_shift (two fp32 roundings each; 1 and 0 give the unscaled track back bit for bit).
 *   dur_out, pitch_out and energy_out stay the model's raw predictions.
 * Equivalent to ev_am_phase1_controls(..., prosody, 0, NULL, NULL, NULL, ...). */
EV_API int ev_am_phase1_prosody(ev_ctx* ctx, const int64_t* ling, const int64_t* lens, const int64_t* spk,
                                const float* style, const float* content, int B, int T, int invariant,
                                const float* prosody, int64_t* dur_out, float* pitch_out, float* energy_out,
                                int32_t* lens32_out, int32_t* mel_lens_out, void* workspace, size_t workspace_bytes,
                                void* stream);

/* ev_am_phase1_prosody with phoneme-level controls; it launches the same kernels.
 *   prosody: NULL, (B,5) f32 per item (prosody_per_token == 0, as ev_am_phase1_prosody), or (B,T,5) f32 per token
 *     (prosody_per_token != 0): row (b,t) = {alpha, p_scale, p_shift, e_scale, e_shift} of token t, acting exactly where
 *     the per-item row acts (token t's duration is fl32(fl32(d_t) * alpha_t); token t's pitch enters pitch_embed as
 *     p_t * p_scale_t + p_shift_t, each tap of the k-wide window with its own token's row).  Rows of tokens
 *     t >= lens[b] are ignored (neutral).  Per-token alphas must lie in [1/16, 16] (the exactness of the scan rests on it;
 *     the library does not check it); per-item alphas only need to be > 0.
 *   durations: NULL, or (B,T) i64 caller durations that replace the predictions in the length regulator; entries at
 *     t >= lens[b] are ignored.  The all-zero guard applies to them as to predicted ones.  They are checked on the device:
 *     a negative entry, or an item whose frame count before or after scaling reaches 2^31 / prod(upsample_rates)
 *     (the vocoder indexes samples with int32; at most 2^24 - 1 frames in any case), sets bit 4 (value 16) of the status
 *     word.  That bit can also be set by predicted durations scaled past the limit.  Do not run phase 2 when it is set.
 *   pitch_in / energy_in: NULL, or (B,T) f32 caller tracks that replace the predictions where they enter
 *     pitch_embed / energy_embed (entries at t >= lens[b] are ignored, i.e. read as the 0 the predictors write there);
 *     the prosody rows apply on top.  Not checked, as in the reference.
 *   dur_out, pitch_out and energy_out stay the model's raw predictions; mel_lens_out counts the frames actually used.
 *   All caller arrays are device memory, read in stream order. */
EV_API int ev_am_phase1_controls(ev_ctx* ctx, const int64_t* ling, const int64_t* lens, const int64_t* spk,
                                 const float* style, const float* content, int B, int T, int invariant,
                                 const float* prosody, int prosody_per_token, const int64_t* durations,
                                 const float* pitch_in, const float* energy_in, int64_t* dur_out, float* pitch_out,
                                 float* energy_out, int32_t* lens32_out, int32_t* mel_lens_out, void* workspace,
                                 size_t workspace_bytes, void* stream);

/* Replaces: GaussianUpsampling.forward matmul (alignment.py:201-211), the decoder
 * (model_open_source.py:146) and to_mel (:147).  Must follow ev_am_phase1 on the same stream;
 * phase1_workspace is the (still live) buffer phase 1 ran on.  F = mel_lens_out[B] read back
 * by the host (the path's one sync).
 *   mel_out (B,F,n_mels) f32 time-major == outputs["dec_outputs"]. */
EV_API int ev_am_phase2(ev_ctx* ctx, const void* phase1_workspace, const int32_t* lens32, const int32_t* mel_lens,
                        int B, int T, int F, int invariant, float* mel_out, void* workspace,
                        size_t workspace_bytes, void* stream);

/* Replaces: Generator.forward (hifigan/models.py:115-131).
 *   mel (B,F,n_mels) time-major if mel_time_major else (B,n_mels,F) (the reference layout);
 *   mel_lens (B) i32 or NULL (literal padded semantics); wav_out (B, F*prod(up_rates)) f32.
 *   mel_lens must be COMPLETE when this is called (not pending in a kernel still running on the stream): the vocoder's kernels start
 *   under their predecessors' tails (programmatic dependent launch) and read the lengths before they wait.  The engine's own flow
 *   satisfies this by construction -- the host reads mel_lens_out back to learn F before it can call ev_am_phase2 / ev_vocoder.  The
 *   same holds for the `lens` argument of the ev_op_*_gp entry points below. */
EV_API int ev_vocoder(ev_ctx* ctx, const float* mel, int mel_time_major, const int32_t* mel_lens, int B, int F,
                      float* wav_out, void* workspace, size_t workspace_bytes, void* stream);

/* Long text: the mel of several items (the segments of one text, synthesised as one batch) joined into one vocoder input, so that
 * ev_vocoder runs over each text's seams and returns one continuous waveform per text.
 *   mel (B,F,n_mels) f32 time-major (ev_am_phase2's mel_out); mel_lens (B) i32 (its frame counts); group (B) i32: the output each
 *   item belongs to, 0 for the first item, each next id equal to the previous one or one more, G - 1 for the last (1 <= B <= 4096).
 *   joined (G,Fg,n_mels) f32 time-major: group g's rows are the valid rows mel[b, :mel_lens[b]] of its items in item order, zeros past
 *   its length; group_lens (G) i32: min(that length, Fg).  Fg is at least the longest group (the host knows every length from the
 *   mel_lens it read back).  No allocation, no sync.
 *   group_lens is written by a kernel, so like any kernel output it is still pending when this returns: do not pass it as the
 *   mel_lens of an ev_vocoder enqueued behind it (see ev_vocoder); give that call lengths that were complete before, e.g. copied from
 *   the host. */
EV_API int ev_join_mel(const float* mel, const int32_t* mel_lens, const int32_t* group, int B, int F, int n_mels, int G, int Fg,
                       float* joined, int32_t* group_lens, void* stream);

/* Replaces the callers' post-processing (inference_am_vocoder_joint.py:130-131):
 * pcm[i] = (int16) trunc(wav[i] * 32768), n elements. */
EV_API int ev_wav_to_pcm16(const float* wav, int16_t* pcm, size_t n, void* stream);

/* Output formats of ev_format_audio: fp32 samples; int16 as ev_wav_to_pcm16 computes them (saturated); one byte of G.711
 * mu-law or A-law of that int16 value (ITU-T G.711 as Python's audioop.lin2ulaw / lin2alaw apply it to 16-bit samples). */
enum { EV_AUDIO_FLOAT32 = 0, EV_AUDIO_PCM16 = 1, EV_AUDIO_MULAW = 2, EV_AUDIO_ALAW = 3 };

/* Replaces the server-side conversion after synthesis (resampling to the client's rate, int16 / G.711 encoding, trimming each
 * item to its length): the valid samples of several waveform items, resampled and encoded, packed back to back in one buffer.
 *   wav: fp32 items item_stride floats apart (wav_out of ev_vocoder: item_stride = F * prod(up_rates)); n_in (B) i64: the valid
 *   samples of item b (mel_lens[b] * prod(up_rates)), at most item_stride; samples at or past n_in[b] are never read.
 *   items (n_items) i64: the items to format, in output order, or NULL for items 0 .. n_items - 1; 1 <= n_items <= 65535.
 *   out_off (n_items) i64: where listed item k starts in out, in samples; it writes ceil(n_in[b] * up / down) samples there.
 *   up / down: coprime, each in [1, 1024]; the rate changes by up / down.  bank: NULL when up == down == 1 (the samples are
 *   copied), else the (up, taps_per_phase) f32 phase-major split of scipy.signal.resample_poly's default filter
 *   h = firwin(20 * max(up, down) + 1, 1 / max(up, down), window=('kaiser', 5.0)) * up: bank[p][j] = h[p + j * up], zero past
 *   the end of h, taps_per_phase = ceil(len(h) / up).  Output o is sum_j bank[q % up][j] * x[q / up - j], q = o * down +
 *   10 * max(up, down), with x zero outside [0, n_in[b]): scipy.signal.resample_poly(x[:n_in[b]], up, down) to fp32 accuracy,
 *   one fp32 chain per output in tap order, so an item's output does not depend on the other items of the call.
 *   encoding: EV_AUDIO_*; out holds 4, 2, 1 or 1 byte(s) per sample.
 *   gain: NULL, or (n_items) f32 per-item gains: listed item k's outputs are then encoded from fp32(y * gain[k]), y the
 *   resampled sample (at up == down == 1 the sample itself).  gain may be written by the launch just before (ev_loudness).
 *   All arrays are device memory read in stream order (the kernel reads them after the work before it on the stream has
 *   completed); out_off and n_in must describe disjoint output ranges.  No allocation, no sync. */
EV_API int ev_format_audio(const float* wav, long long item_stride, const int64_t* n_in, const int64_t* items, int n_items,
                           const int64_t* out_off, const float* bank, int up, int down, int taps_per_phase, int encoding, void* out,
                           const float* gain, void* stream);

/* Integrated loudness (ITU-R BS.1770-4, one channel) of listed waveform items and the gain that brings each to a target: the
 * server-side loudness normalisation of responses (EBU R128 at -23 LUFS, podcasts at -16), before ev_format_audio applies
 * the gain and encodes them.  Arguments as ev_format_audio: wav items item_stride floats apart, n_in (B) i64 valid samples (at
 * most item_stride; samples at or past n_in[b] are never read), items (n_items) i64 or NULL for 0 .. n_items - 1,
 * 1 <= n_items <= 65535.
 *   sample_rate: the items' rate, a multiple of 10 in [4000, 192000] (100 ms sub-blocks of sample_rate / 10 samples).
 *   kcoef: HOST array of 10 doubles, the K-weighting cascade (b0, b1, b2, a1, a2) of the high shelf, then of the high pass, with
 *   a0 = 1 (emotivoice_b200.audio.k_weighting(sample_rate)).  The cascade runs in fp32 (direct form I) on each 100 ms
 *   sub-block, restarted from zero state W samples before it (W the smallest multiple of 32 with W * r^W <= 1e-10, r the
 *   cascade's largest pole radius; 2048 at 16 kHz), so every sub-block is computed on its own.
 *   Gating blocks are 400 ms with 75 % overlap, only those entirely inside the item; block loudness l = -0.691 +
 *   10 log10(mean square); the absolute gate keeps l > -70, the relative gate l > (loudness of the blocks kept) - 10; fp64 sums
 *   in a fixed order, so an item's results do not depend on the other items of the call.
 *   lufs (n_items) f32: integrated loudness L, -inf for an item shorter than 400 ms or with no block passing the gates.
 *   peak (n_items) f32: max |x| over the item's valid samples.
 *   gain (n_items) f32: fp32 of min(10^((target_lufs - L) / 20), 10^(-1/20) / peak) computed in fp64 (a -1 dBFS sample-peak
 *   ceiling); 1 where L = -inf.  target_lufs in [-70, 0].
 *   ws / ws_bytes: device workspace of at least ev_loudness_workspace_bytes(n_items, item_stride, sample_rate) bytes.
 * Two launches; device arrays are read in stream order.  No allocation, no sync. */
EV_API size_t ev_loudness_workspace_bytes(int n_items, long long max_n, int sample_rate);  /* 0 for arguments out of range */
EV_API int ev_loudness(const float* wav, long long item_stride, const int64_t* n_in, const int64_t* items, int n_items, int sample_rate,
                       const double* kcoef, float target_lufs, float* lufs, float* peak, float* gain, void* ws, size_t ws_bytes,
                       void* stream);

/* True-peak limiter of listed waveform items: holds each item, scaled by its loudness pre-gain, at or below ceiling_dbtp in
 * true peak, before ev_format_audio resamples and encodes it.  wav / item_stride / n_in / items / n_items as ev_loudness.
 *   Pre-gain g = 10^((target_lufs - lufs0[k]) / 20) * 10^((target_lufs - lufs1[k]) / 20) in fp64, a factor 1 where its array is
 *   NULL or its loudness is -inf (lufs0 / lufs1: (n_items) f32 device arrays, ev_loudness's lufs; lufs1 needs lufs0;
 *   target_lufs in [-70, 0] when lufs0 is given).  ceiling_dbtp in [-20, 0].
 *   Detector: p[s] = max(|x[s]|, |sum_j bank[ph][j] * x[s + c - j]| over the phases ph), c = (taps - 1) / 2, x zero outside
 *   [0, n): bank (phases, taps) f32 device array, taps odd (emotivoice_b200.audio.limit_bank).  Required gain r[s] = min(0,
 *   ceiling - 20 log10(g p[s])) in fp64, at least -1000 dB, rounded down to a multiple of 2^-32 dB.
 *   Envelope: m[s] = min r over [s - hold, s + lookahead + hold] (r = 0 outside the item), for s from -lookahead; release
 *   G1[s] = min(m[s], G1[s - 1] + release_db_per_sample) from G1 = 0, computed as an exact fp64 prefix minimum
 *   (release_db_per_sample in (0, 1], a multiple of 2^-32); attack G[s] = mean of G1 over [s - lookahead, s], so G[s] <= r[s].
 *   hold >= (taps - 1) / 2, lookahead in [0, 1024].
 *   out[k * out_stride + s] = fp32(x[s] * g * 10^(G[s] / 20)) for s < n (out_stride >= item_stride); nothing else is written.
 *   ws: ev_limit_workspace_bytes(n_items, item_stride, lookahead) bytes.  Three launches; an item's output is bitwise the same
 *   in any batch or order.  No allocation, no sync. */
EV_API size_t ev_limit_workspace_bytes(int n_items, long long max_n, int lookahead);   /* 0 for arguments out of range */
EV_API int ev_limit(const float* wav, long long item_stride, const int64_t* n_in, const int64_t* items, int n_items, int sample_rate,
                    const float* lufs0, const float* lufs1, float target_lufs, float ceiling_dbtp, const float* bank, int phases,
                    int taps, int lookahead, int hold, double release_db_per_sample, float* out, long long out_stride, void* ws,
                    size_t ws_bytes, void* stream);

/* Loudness meter (EBU R128: ITU-R BS.1770-4 and EBU Tech 3342, one channel) of waveform items, for checking what a server
 * delivers and measuring recordings: item k is the n[k] samples at wav + start[k] (start, n: (n_items) i64 DEVICE arrays, so a
 * (B, L) batch and ev_format_audio's packed EV_AUDIO_FLOAT32 outputs are both read in place), n_host (n_items) i64 HOST array
 * of the same counts (>= 0; it sizes the grid, the workspace and the series; a device count is clamped to the largest of them).
 * 1 <= n_items <= 65535.  sample_rate: a multiple of 10 in [4000, 192000]; kcoef: as ev_loudness (HOST, 10 doubles).
 *   Sub-blocks: ev_loudness's, 100 ms of S = sample_rate / 10 samples, K-weighted, sum of squares e[j]; only the n / S full
 *   ones count.  Loudness of a mean square z: -0.691 + 10 log10(z).
 *   momentary M[j] of (((e[j] + e[j+1]) + e[j+2]) + e[j+3]) / (4 S), j < n / S - 3: ev_loudness's gating blocks, ungated (10 Hz).
 *   short-term S[j] of (e[j] + ... + e[j+29], left to right) / (30 S), j < n / S - 29 (3 s windows, 10 Hz).
 *   LRA (EBU Tech 3342): the short-term values S > -70; of those the values S > 10 log10(mean of 10^(S/10)) - 20 (the mean
 *   taken over the mean squares in fp64, in a fixed order); of the m left, sorted ascending, v[round(0.95 (m - 1))] -
 *   v[round(0.10 (m - 1))], round half away from zero, each v the exact element (a radix select); NaN when m = 0.
 *   True peak: 20 log10 of max p[s] over the item, p ev_limit's detector (max of |x[s]| and |sum_j bank[ph][j] x[s + c - j]|,
 *   c = (taps - 1) / 2, x zero outside [0, n)) with bank (phases, taps) f32 device array, taps odd: emotivoice_b200.audio.
 *   true_peak_bank(sample_rate), all R = ceil(192000 / sample_rate) phases of the limiter's interpolator, so p reads exactly
 *   scipy.signal.resample_poly(x, R, 1) and |x|; phases may be 0 (bank NULL; 192 kHz).
 *   results (6, n_items) f32 device, row r for item k at results[r * n_items + k]: 0 integrated loudness I (bitwise
 *   ev_loudness's lufs), 1 LRA (LU), 2 max M, 3 max S (-inf for an empty or silent series), 4 true peak (dBTP, -inf for
 *   silence), 5 sample peak max |x| (linear, ev_loudness's peak).
 *   momentary / short_term: NULL, or (n_items, series_stride) f32 device arrays, series_stride >= (max n_host) / S: row k holds
 *   M (S) of item k, then NaN to the end of the row.
 *   ws: ev_meter_workspace_bytes(n_items, max n_host, sample_rate) bytes.  Four launches; each item's results are bitwise the
 *   same in any batch or order.  No allocation, no sync. */
EV_API size_t ev_meter_workspace_bytes(int n_items, long long max_n, int sample_rate);   /* 0 for arguments out of range */
EV_API int ev_meter(const float* wav, const int64_t* start, const int64_t* n, const int64_t* n_host, int n_items, int sample_rate,
                    const double* kcoef, const float* bank, int phases, int taps, float* results, float* momentary, float* short_term,
                    long long series_stride, void* ws, size_t ws_bytes, void* stream);

/* FLAC (RFC 9639) file images of int16 items, the lossless compressed response of a TTS server: item k is pcm[pcm_off[k] ..
 * pcm_off[k + 1]) (pcm_off (n_items + 1) i64 DEVICE array, items packed back to back as ev_format_audio writes EV_AUDIO_PCM16),
 * n_samples (n_items) i64 HOST array of the same counts (each in [1, 2^36]; it sizes the grid and the checks below).
 *   Each image: fLaC, STREAMINFO (last-metadata flag; block sizes 4096 / 4096, the real min / max frame size, sample_rate, one
 *   channel, 16 bits, the sample count, MD5 all zero = unknown), then frames of 4096 samples (the last one shorter): sync
 *   0xFFF8, the standard sample rate code where one exists, else 8-bit kHz, 16-bit Hz or 16-bit tens of Hz, else 0000 (from
 *   STREAMINFO), CRC-8 and CRC-16.  Each subframe is the smallest exact bit count of CONSTANT, FIXED 0-4, LPC 1-12 (integer
 *   Welch window, fp64 Levinson-Durbin without contraction) and VERBATIM, with Rice partitions of 4-bit parameters; the stream
 *   is byte for byte the one oracle/flac_oracle.py defines.  It is in FLAC's streamable subset except at rates above 65535 Hz
 *   that are not a multiple of 10, whose frame headers need code 0000.
 *   out (out_bytes >= sum of ev_flac_bound_bytes(n_samples[k])): the images back to back; out_off (n_items + 1) i64 device:
 *   image k is out[out_off[k] .. out_off[k + 1]).  sample_rate in [4000, 192000].  ws: ev_flac_workspace_bytes(n_items,
 *   max n_samples) bytes of device workspace.  Four launches; each image depends only on its own item.  If pcm_off disagrees
 *   with n_samples the images are wrong, but nothing outside the items or out is touched.  No allocation, no sync. */
EV_API size_t ev_flac_bound_bytes(long long n_samples);                        /* worst-case image (VERBATIM frames); 0 out of range */
EV_API size_t ev_flac_workspace_bytes(int n_items, long long max_n);          /* 0 for arguments out of range */
EV_API int ev_flac_encode(const int16_t* pcm, const int64_t* pcm_off, int n_items, const int64_t* n_samples, int sample_rate,
                          uint8_t* out, size_t out_bytes, int64_t* out_off, void* ws, size_t ws_bytes, void* stream);

/* Keyed zero-bit watermark of listed 16 kHz waveform items, a machine-readable mark that the output is synthetic
 * (emotivoice_b200.audio holds the definition; oracle/watermark_oracle.py restates it in fp64).  The MCLT of frames of 1024
 * samples, hop 512, sine window, frame j over samples [(j - 1) 512, (j + 1) 512) for j = 0 .. ceil(n / 512), zero outside the
 * item: each MDCT coefficient C of bins 19..217 (300-3400 Hz) gets alpha * M * s(key, j mod 64, k), M = sqrt(C^2 + S^2) the
 * MCLT magnitude, alpha = 10^(-20/20) / sqrt(2), s = +-1 from SplitMix64's output function; y = x + the overlap-added IMDCT
 * of that change.  Silent stretches stay silent and nothing is added outside the band.
 *   wav / item_stride / n_in / items / n_items as ev_loudness.  sample_rate must be 16000.  key in [1, 2^63 - 1].
 *   out[k * out_stride + s] = y[s] for s < n (out_stride >= item_stride; out must not overlap wav); nothing else is written.
 * One launch; each output is bitwise the same in any batch or order.  No allocation, no sync. */
EV_API int ev_watermark_embed(const float* wav, long long item_stride, const int64_t* n_in, const int64_t* items, int n_items,
                              int sample_rate, uint64_t key, float* out, long long out_stride, void* stream);

/* The detector of ev_watermark_embed's mark in 16 kHz items: item k is wav[k * item_stride ..], n (n_items) i64 device array
 * of its valid samples (clamped to [0, item_stride]).  For each grid offset tau in [0, 512) and frame phase m0 in [0, 64): the
 * MCLT on frames shifted by tau samples, u = C / M in the band (cells with M = 0 skipped), b[r, k] = sum of u over frames
 * j = r mod 64, z = sum_{r,k} s(key, (r + m0) mod 64, k) b[r, k] / sqrt(sum b^2) (0 when b is all zero).
 *   z (n_items) f32, offset / phase (n_items) i32: the largest z of each item and its (tau, m0), the first in (tau, m0) order on
 *   ties.  ws: ev_watermark_detect_workspace_bytes(n_items) bytes; afterwards it holds each item's best z per tau ((n_items, 512)
 *   f32) and that z's m0 ((n_items, 512) i32).  Two launches; each result depends only on its own item.
 *   No allocation, no sync. */
EV_API size_t ev_watermark_detect_workspace_bytes(int n_items);                  /* 0 for arguments out of range */
EV_API int ev_watermark_detect(const float* wav, long long item_stride, const int64_t* n, int n_items, uint64_t key, float* z,
                               int32_t* offset, int32_t* phase, void* ws, size_t ws_bytes, void* stream);

/* Objective comparison of syntheses with recordings: cepstral distance after dynamic time warping (DTW), F0 error and voicing
 * error along the warping path.  Pair k compares N = n_syn[k] syn frames with M = n_ref[k] ref frames (n_syn, n_ref: (n_items)
 * i32 DEVICE arrays, clamped to [1, max_n] and [1, max_m]; max_n, max_m in [1, 4096] are HOST maxima, they size the grid and
 * the workspace).  1 <= n_items <= 65535.
 *   mel_syn (n_items, 80, syn_frames) f32 log-mels (ln of the mel magnitude), f0_syn (n_items, syn_frames) f64 F0 in Hz, 0 or
 *   less for unvoiced; syn_frames >= max_n; likewise mel_ref, f0_ref, ref_frames >= max_m.  Frames past a pair's N and M are
 *   never read.  table (24, 80) f64 DEVICE: row k - 1 holds cos(pi k (m + 1/2) / 80), m = 0..79.
 *   c_k[f] = (sum_m fp64(L[m, f]) * table[k - 1][m], ascending m) / 80, k = 1..24; d(i, j) = sqrt(sum_k (c_k[i] - c'_k[j])^2),
 *   ascending k; every product, sum, difference, quotient and square root rounded on its own (no FMA).
 *   D(0,0) = d(0,0), D(i,j) = d(i,j) + min(D(i-1,j-1), D(i-1,j), D(i,j-1)) over the predecessors that exist, ties to the
 *   first in that order; the path: the backtrack from (N-1, M-1) to (0,0), P pairs, max(N, M) <= P <= N + M - 1.
 *   stats (3, n_items) f64 DEVICE, row r for pair k at stats[r * n_items + k]: 0 mcd = (10 sqrt(2) / ln 10) (D(N-1, M-1) / P)
 *   in dB (D(N-1, M-1) is the sum of d along the path in path order); 1 f0_rmse = sqrt(E / V) in cents, E the sum in path
 *   order of (1200 log2(f_syn / f_ref))^2 over the V pairs voiced on both sides (NaN when V = 0); 2 vuv_error = (pairs whose
 *   voicing differs) / P.  counts (2, n_items) i32 DEVICE: 0 V, 1 P.
 *   path: NULL, or (n_items, path_stride, 2) i32 DEVICE, path_stride >= max_n + max_m - 1: row k holds the P pairs (syn frame,
 *   ref frame) from (0,0), then -1 to the end of the row.
 *   ws: ev_eval_workspace_bytes(n_items, max_n, max_m) bytes (9 max_n max_m bytes per pair, plus the cepstra).  Three launches;
 *   each pair's results are bitwise the same in any batch or order.  No allocation, no sync. */
EV_API size_t ev_eval_workspace_bytes(int n_items, int max_n, int max_m);            /* 0 for arguments out of range */
EV_API int ev_eval_compare(const float* mel_syn, const double* f0_syn, long long syn_frames, const int32_t* n_syn, int max_n,
                           const float* mel_ref, const double* f0_ref, long long ref_frames, const int32_t* n_ref, int max_m,
                           int n_items, const double* table, double* stats, int32_t* counts, int32_t* path, long long path_stride,
                           void* ws, size_t ws_bytes, void* stream);
/* The cost and DTW launches of ev_eval_compare from caller cepstra: cep_syn (n_items, syn_frames, 24) f64 DEVICE, row (k, f)
 * holding c_1..c_24 of pair k's syn frame f; cep_ref likewise with ref_frames.  d, the DTW, the path and the statistics are
 * ev_eval_compare's, with every other argument as there.  ws: ev_eval_workspace_bytes(n_items, max_n, max_m) bytes.  Two
 * launches; each pair's results are bitwise the same in any batch or order.  No allocation, no sync. */
EV_API int ev_eval_align(const double* cep_syn, const double* f0_syn, long long syn_frames, const int32_t* n_syn, int max_n,
                         const double* cep_ref, const double* f0_ref, long long ref_frames, const int32_t* n_ref, int max_m,
                         int n_items, double* stats, int32_t* counts, int32_t* path, long long path_stride, void* ws,
                         size_t ws_bytes, void* stream);

/* Number of kernel launches this library has enqueued in this process (bench.py's
 * `gpu_launches`). */
EV_API uint64_t ev_launch_count(void);

/* ---- single operators (used by the per-kernel parity tests) ------------------- */

/* Generic time-major 1-D convolution / linear layer (implicit GEMM):
 *   out[b,t,co] = epi( bias[co] + sum_{j<K} sum_{ci} w[j][ci][co] * act_in(x[b, t+(j-(K-1)/2)*dil, ci]) )
 * x rows outside [0, len_b) read as zero.  w is (K, Cin, Cout).  bias_bstride: floats between
 * per-item biases (0 = shared).  res (same layout as out) is added after out_act.
 * acc: EV_ACC_STORE out=v; EV_ACC_ADD out+=v; EV_ACC_ADD_DIV out=(out+v)/div.
 * Covers nn.Linear (K=1), the conv-FFN (encoder.py:50-52), predictor convs (variance.py:17-31),
 * conv_pre / ResBlock1 convs (hifigan/models.py:50-57,116) and, with polyphase-packed
 * weights, ConvTranspose1d (hifigan/models.py:100-103). */
EV_API int ev_op_conv1d(const float* x, const float* w, const float* bias, size_t bias_bstride,
                        const float* res, float* out, int B, int L, int Cin, int Cout, int K, int dil,
                        const int32_t* lens, int lens_mul, int in_act, float in_slope, int out_act,
                        int acc, float div, void* stream);
/* Host-only introspection (no GPU needed; without a device it assumes 132 SMs): the plan ev_op_conv1d would use for a shape.
 * out10 = {TXN, NV, TM, BM, BN, rows_a, a_ld, smem bytes, grid.x, grid.y}: the kernel variant <TXN, NV, TM>, its BM x BN tile, the
 * rows (BM + (K-1)*dil) and leading dimension of its shared A tile.  EV_EINVAL for a shape ev_op_conv1d rejects. */
EV_API int ev_debug_conv1d_plan(int B, int L, int Cin, int Cout, int K, int dil, int* out10);
/* Same contract on the tensor cores (wgmma tf32 / bf16, fp32 accumulators in registers); w_tc is in the
 * tensor-core layout (2 planes hi|lo, Cout/BNp N tiles, K, Cin/4, BNp = min(Cout,128), 4; packing.to_tc_layout);
 * split3 = 0: 1xTF32, 1: 3xTF32 fp32 emulation, 2: bf16 operands (w_tc then in the bf16 layout of
 * packing.to_tc16_layout; Cin % 16 == 0), 3: bf16x3 fp32 emulation (w_tc then holds the two bf16 planes of
 * packing.to_tc16x2_layout; Cin % 16 == 0).  Requires Cin % 8 == 0, Cout % 16 == 0 and Cout <= 128 or Cout % 128 == 0.
 * splitk_ws (optional, splitk_floats floats of scratch) lets a launch with few output tiles and a long reduction be split
 * along K into 4 slices (deterministic two-pass). */
EV_API int ev_op_conv1d_tc(const float* x, const float* w_tc, int split3, const float* bias, size_t bias_bstride,
                           const float* res, float* out, int B, int L, int Cin, int Cout, int K, int dil,
                           const int32_t* lens, int lens_mul, int in_act, float in_slope, int out_act,
                           int acc, float div, float* splitk_ws, size_t splitk_floats, void* stream);
/* ev_op_conv1d_tc with an explicit K-split factor: ksplit <= 1 runs one pass; ksplit = S > 1 (needs splitk_ws) shares each
 * output tile's reduction among S CTAs -- clamped to the number of C_in blocks, exactly as the engine's layers request it --
 * and sums the slices in a second, fixed-order pass.  ev_op_conv1d_tc is this call with ksplit = 4 (0 without scratch). */
EV_API int ev_op_conv1d_tc_ks(const float* x, const float* w_tc, int split3, const float* bias, size_t bias_bstride,
                              const float* res, float* out, int B, int L, int Cin, int Cout, int K, int dil,
                              const int32_t* lens, int lens_mul, int in_act, float in_slope, int out_act,
                              int acc, float div, int ksplit, float* splitk_ws, size_t splitk_floats, void* stream);
/* Host-only introspection (no GPU needed): the tile / pipeline plan ev_op_conv1d_tc would use for a shape.
 * out11 = {BN, MT, KBG, a_stages, b_stages, producer groups, ksplit, accumulator columns (MT x BN), smem bytes, tiles, rows_pad}.
 * The CPU tests check the invariants the kernel relies on (ring depth >= producer groups, register/smem limits,
 * summation-order parameters independent of batch and length). */
EV_API int ev_debug_tc_plan(int B, int L, int Cin, int Cout, int K, int dil, int split3, int ksplit, int* out11);
/* HiFi-GAN convolution on GRANULE-PLANAR activations (csrc/conv1d_gp.cu; what ev_vocoder runs in every tensor-core mode).
 * Layout: a (B, L, C) tensor is stored [b][C/cpg][l][cpg] in 16-byte granules, cpg = 4 fp32 (mode 0 tf32, 1 3xTF32) or 8 bf16
 * (mode 2); mode 3 = "bf16x3": fp32 activations, every operand split into bf16 hi + lo, three bf16 MMAs per K step (fp32-class
 * result at half the cost of 3xTF32; w then holds two bf16 planes).  w: the ev_op_conv1d_tc weight layout of that mode.  rate > 1: polyphase ConvTranspose1d, the Cout GEMM columns
 * are `rate` phases of Cout/rate channels, out is (B, (Cout/rate)/cpg, L*rate, cpg).  res (rate == 1): same shape as out.
 * Rows >= lens[b]*lens_mul are neither read (they count as zero padding) nor written.  Replaces hifigan/models.py:50-57,
 * :116, :118-119. */
EV_API int ev_op_conv1d_gp(const void* x, const float* w, int mode, const float* bias, const void* res, void* out, int B, int L,
                           int Cin, int Cout, int K, int dil, int rate, const int32_t* lens, int lens_mul, int in_act,
                           float in_slope, int acc, float div, void* stream);
/* n <= 3 convolutions of ONE shape (B, L, Cin -> Cout, rate 1, plain store) but different taps / dilations / weights / tensors as ONE
 * launch: the same-index convolutions of the three parallel ResBlocks of a HiFi-GAN stage (hifigan/models.py:120-126), which at small
 * batch have too few tiles each to fill the machine.  Tables of n entries; bias / res may be null (or hold nulls).  Every tile is
 * computed as in the member's own ev_op_conv1d_gp launch: bitwise equal.  EV_EINVAL if the members cannot share a launch. */
EV_API int ev_op_conv1d_gp_group(int n, const void* const* x, const float* const* w, int mode, const float* const* bias,
                                 const void* const* res, void* const* out, const int* K, const int* dil, int B, int L, int Cin,
                                 int Cout, const int32_t* lens, int lens_mul, int in_act, float in_slope, void* stream);
/* out = ((b + a) [+ c]) / div elementwise over n_floats fp32 values (c may be null): the pass that forms a HiFi-GAN stage's
 * `xs / n` after its ResBlocks' last layers ran as one grouped launch (fp32 storage modes); bitwise equal to the ACC_ADD /
 * ACC_ADD_DIV epilogues it replaces.  n_floats % 4 == 0. */
EV_API int ev_op_gp_sum_div(const float* a, const float* b, const float* c, float* out, size_t n_floats, float div, void* stream);
/* Host-only: the plan of a grouped launch, out11 as ev_debug_gp_plan (tiles = all members'). */
EV_API int ev_debug_gp_group_plan(int n, const int* K, const int* dil, int B, int L, int Cin, int Cout, int mode, int* out11);
/* One ResBlock1 layer (hifigan/models.py:50-57) as ONE kernel on granule-planar activations (csrc/resblock_gp.cu):
 * out = [acc]( x + c2(lrelu(c1(lrelu(x), dil)), 1) ), C -> C channels (C in {32, 64, 128}), slope 0.1, both weights in the layout of
 * `mode` (as ev_op_conv1d_gp).  Bitwise equal to the two ev_op_conv1d_gp launches it replaces; EV_EINVAL for shapes it does not take
 * (the engine then runs the pair unfused). */
EV_API int ev_op_resblock_gp(const void* x, const float* w1, const float* b1, const float* w2, const float* b2, int mode, void* out, int B,
                             int L, int C, int K, int dil, const int32_t* lens, int lens_mul, int acc, float div, void* stream);
/* n <= 3 such layers of ONE shape (B, L, C; plain store) with their own taps / dilations / weights / tensors as ONE launch: the
 * same-index layers of HiFi-GAN's three parallel ResBlocks at small batch.  Bitwise equal to the members' own launches; EV_EINVAL if
 * they cannot share a launch (each member must itself be a shape ev_op_resblock_gp takes with at least two accumulators per tile). */
EV_API int ev_op_resblock_gp_group(int n, const void* const* x, const float* const* w1, const float* const* b1, const float* const* w2,
                                   const float* const* b2, int mode, void* const* out, int B, int L, int C, const int* K, const int* dil,
                                   const int32_t* lens, int lens_mul, void* stream);
/* Host-only: the plan of a grouped fused launch: out16 = {MT, KBG, tiles (all members), rows1_pad, rows2_pad, smem bytes, tmem columns,
 * then per member in launch order (heaviest first) {K, row tiles per item, first tile index}}. */
EV_API int ev_debug_resblock_gp_group_plan(int n, const int* K, const int* dil, int B, int L, int C, int mode, int* out16);
/* Host-only: out11 = {MT, KBG, x stages, weight stages, transform warps, tmem columns, smem bytes, tiles, rows per tile, rows1_pad, rows2_pad}. */
EV_API int ev_debug_resblock_gp_plan(int B, int L, int C, int K, int dil, int mode, int* out11);
/* Host-only: out11 = {BN, MT, KBG, a_stages, b_stages, transform warps, planes, tmem columns, smem bytes, tiles, rows_pad}. */
EV_API int ev_debug_gp_plan(int B, int L, int Cin, int Cout, int K, int dil, int rate, int mode, int* out11);
/* fp32 in[b*stride_b + t*stride_t + c*stride_c] -> granule-planar (fp32, or bf16 when bf16 != 0): the vocoder's input boundary
 * (hifigan/models.py:115 takes (B, n_mels, F); jets.py:62 hands over dec_outputs (B, F, n_mels) transposed). */
EV_API int ev_op_to_gp(const float* in, long long stride_b, long long stride_t, long long stride_c, void* out, int B, int L, int C,
                       int bf16, void* stream);
/* wav[b,t] = tanh(bias + conv_post(leaky_relu(x, slope))) on a granule-planar input (hifigan/models.py:127-129). */
EV_API int ev_op_conv_post_gp(const void* x, int bf16, const float* w, const float* bias, const int32_t* lens, int lens_mul, int B,
                              int L, int C, int K, float slope, float* wav, void* stream);
/* The same on a time-major (B, L, C) fp32 input: what ev_vocoder runs in EV_PREC_FP32_FFMA.  C % 4 == 0, C <= 128, K odd <= 15;
 * same channel-major summation order as ev_op_conv_post_gp.  Samples >= lens[b]*lens_mul (null: L) are written as zeros. */
EV_API int ev_op_conv_post(const float* x, const float* w, const float* bias, const int32_t* lens, int lens_mul, int B, int L, int C,
                           int K, float slope, float* wav, void* stream);
/* LayerNorm over the last dim, eps 1e-12 (encoder.py:112-127). rows x C. */
EV_API int ev_op_layernorm(const float* x, const float* w, const float* b, float* y, int rows, int C, void* stream);
/* Multi-head self-attention core (encoder.py:84-109) on a packed (B,L,3H) q|k|v buffer. */
EV_API int ev_op_attention(const float* qkv, const int32_t* key_lens, float* ctx_out, int B, int L, int H,
                           int n_heads, void* stream);
/* The same attention on the tensor cores (csrc/attention_tc.cu): QK^T and PV as wgmma with the softmax on the register
 * accumulators; d_k = 48 only.  tc_mode 1 = 3xTF32 fp32 emulation (what the engine uses wherever a layer runs fp32-accurate),
 * 0 = one tf32 MMA per K step. */
EV_API int ev_op_attention_tc(const float* qkv, const int32_t* key_lens, float* ctx_out, int B, int L, int H, int n_heads,
                              int tc_mode, void* stream);
/* Gaussian upsampling (alignment.py:180-211) incl. cumsum; out (B,F,H); adds alpha*pe[f] when pe != NULL.
 * centers_tmp: 2*B*T floats of scratch; mel_lens_tmp: B+1 int32 (frame counts, max in slot B). */
/* The duration bookkeeping of ev_am_phase1_prosody alone: dur (B,T) i64; lens (B) i32 or NULL; alpha (B) f32 or
 * NULL (1); centers, ds (B,T) f32 = cumsum(ds) - ds/2 and ds = fl32(d * alpha) after the all-zero guard;
 * mel_lens (B+1) i32: trunc(fl32(sum ds)) per item, max in slot B. */
EV_API int ev_op_duration_scan(const int64_t* dur, const int32_t* lens, const float* alpha, int invariant, int B, int T,
                               float* centers, float* ds, int32_t* mel_lens, void* stream);
/* The duration bookkeeping of ev_am_phase1_controls alone: as ev_op_duration_scan, with alpha[b * alpha_stride +
 * t * alpha_tstride] (alpha_tstride 0: per item); caller != 0: dur holds caller durations (entries t >= lens[b] ignored,
 * negative ones clamped to 0); status (may be NULL) |= 8 when an output has no frames, |= 16 when a caller duration is
 * negative or an item's frame count before or after scaling exceeds max_frames (in [1, 2^24 - 1]). */
EV_API int ev_op_duration_scan_controls(const int64_t* dur, int caller, const int32_t* lens, const float* alpha, int alpha_stride,
                                        int alpha_tstride, int invariant, int B, int T, int max_frames, float* centers, float* ds,
                                        int32_t* mel_lens, int32_t* status, void* stream);
EV_API int ev_op_gauss_upsample(const float* hs, const int64_t* dur, const int32_t* lens, int B, int T, int H,
                                int F, int invariant, const float* pe, const float* alpha, float* centers_tmp,
                                int32_t* mel_lens_tmp, float* out, void* stream);
/* The Gaussian upsampling launch of ev_am_phase2 alone, on given centres (B,T) f32 and frame counts mel_lens (B) i32 (the
 * outputs of ev_op_duration_scan): out (B,F,H); frames >= mel_lens[b] are zeros when invariant != 0; adds alpha*pe[f] when
 * pe != NULL. */
EV_API int ev_op_gauss_upsample_centers(const float* hs, const float* centers, const int32_t* lens, const int32_t* mel_lens, int B,
                                        int T, int H, int F, int invariant, const float* pe, const float* alpha, float* out,
                                        void* stream);
/* The encoder's first LayerNorm with its embedding prologue, as ev_am_phase1 launches it:
 * x_out[r] = emb[clamp(ids[r], 0, n_emb - 1)] + alpha[0] * pe[r % L] (product and sum rounded separately),
 * y[r] = LayerNorm(x_out[r]) * w + b, eps 1e-12.  rows x C. */
EV_API int ev_op_layernorm_embed(const int64_t* ids, const float* emb, int n_emb, const float* pe, const float* alpha, int L,
                                 float* x_out, const float* w, const float* b, float* y, int rows, int C, void* stream);
/* The per-utterance conditioning bias of ev_am_phase1 (model_open_source.py:109-111):
 * cond_in (B, H + 2*bert) = [spk_emb[clamp(spk[b], 0, n_spk - 1)] | style[b] | content[b]], out (B,H) = cond_in w + bias with
 * w (H + 2*bert, H) row-major. */
EV_API int ev_op_cond_bias(const int64_t* spk, const float* spk_emb, int n_spk, const float* style, const float* content, int B, int H,
                           int bert, const float* w, const float* bias, float* cond_in, float* out, void* stream);
/* Predictor head (variance.py:46-56): s = x[b,t,:] . w + b[0]; mode 0: out_f[b,t] = s; mode 1: out_i[b,t] =
 * clamp(rint(exp(s) - 1), 0) (the durations).  Rows t >= lens[b] give 0 (lens may be NULL).  x (B,T,C). */
EV_API int ev_op_rowdot(const float* x, const float* w, const float* b, const int32_t* lens, int B, int T, int C, int mode,
                        float* out_f, int64_t* out_i, void* stream);
/* y = x with rows t >= lens[b] set to zero (variance.py:38-39).  (B,T,C). */
EV_API int ev_op_mask_rows(const float* x, const int32_t* lens, float* y, int B, int T, int C, void* stream);
/* x (B,T,C) += Conv1d(1->C, K)(p') + bp + Conv1d(1->C, K)(e') + be (model_open_source.py:131-134), wp / we tap-major (K,C),
 * p' = pitch * prosody[b,1] + prosody[b,2] and e' = energy * prosody[b,3] + prosody[b,4] (prosody (B,5) or NULL: p' = pitch).
 * With prosody and lens both given the window ends at lens[b]; otherwise at T. */
EV_API int ev_op_var_embed_add(float* x, const float* pitch, const float* energy, const float* wp, const float* bp, const float* we,
                               const float* be, const float* prosody, const int32_t* lens, int B, int T, int C, int K, void* stream);

/* ---- style encoder (the callers' prompt / content embedding: simbert.py:33-72 -> transformers BertModel) ---------------
 * Next-row widening (SURVEY.md s8f rank 1): the reference runs this BERT-base on the CPU twice per utterance
 * (inference_am_vocoder_joint.py:25-38,106-107).  Separate context: it is a separate model with its own checkpoint. */
typedef struct ev_style_ctx ev_style_ctx;

/* The integers of the checkpoint's BertConfig + the width of the packed classification heads. */
typedef struct ev_style_config {
  int32_t vocab_size, max_position, type_vocab;
  int32_t hidden;            /* 768; multiple of 128, <= 768 */
  int32_t n_heads;           /* 12; hidden / n_heads in {32, 48, 64} */
  int32_t n_layers;          /* 12 */
  int32_t intermediate;      /* 3072; multiple of 128 */
  int32_t n_head_out;        /* columns of the packed [pitch|speed|energy|emotion] classifier (multiple of 8), 0 = none */
} ev_style_config;

/* StyleEncoder.__init__ (simbert.py:34-44). */
EV_API int ev_style_create(ev_style_ctx** out, int device, const ev_style_config* cfg);
EV_API void ev_style_destroy(ev_style_ctx* ctx);
/* load_state_dict (inference_am_vocoder_joint.py:60-65): same blob + index convention as ev_bind_weights; names are
 * the ones emotivoice_b200.packing.pack_style_state_dict emits ("sty.*"). */
EV_API int ev_style_bind_weights(ev_style_ctx* ctx, const float* blob, size_t blob_floats, const ev_weight_entry* index,
                                 int n_entries);
/* EV_PREC_FP32 (3xTF32 on the tensor cores, default) or EV_PREC_TF32. */
EV_API int ev_style_set_precision(ev_style_ctx* ctx, int precision);
EV_API size_t ev_style_workspace_bytes(const ev_style_ctx* ctx, int B, int N);
/* StyleEncoder.forward (simbert.py:48-72): ids / type_ids (B,N) int64, lens (B,) int64 = number of leading tokens with
 * attention_mask == 1 (tokenizer padding is a suffix).  pooled (B, hidden) = BertModel's pooler_output;
 * heads (B, n_head_out) = the four classification heads side by side, or NULL to skip them. */
EV_API int ev_style_forward(ev_style_ctx* ctx, const int64_t* ids, const int64_t* type_ids, const int64_t* lens, int B, int N,
                            float* pooled, float* heads, void* workspace, size_t workspace_bytes, void* stream);
/* The style encoder's two own kernels alone (single-operator tests).  BertEmbeddings: y[r] = LayerNorm((word[ids[r]] +
 * type[type_ids[r]]) + pos[r % N]) * w + b, eps 1e-12, rows x C; ids must be in range (ev_style_forward does not check them
 * either).  Row GEMV: out[b,n] = act(x[b*x_stride : +K] . w[:,n] + bias[n]), w (K,N) row-major, act EV_ACT_NONE or EV_ACT_TANH. */
EV_API int ev_op_bert_embed_ln(const int64_t* ids, const int64_t* type_ids, const float* word, const float* type, const float* pos,
                               const float* w, const float* b, float* y, int rows, int N, int C, void* stream);
EV_API int ev_op_row_gemv(const float* x, size_t x_stride, const float* w, const float* bias, float* out, int B, int K, int N, int act,
                          void* stream);

/* ---- training-mode alignment helpers (SURVEY.md s8f rank 4; not used by any inference path) --------------------------------
 * viterbi_decode (alignment.py:124-142): monotonic alignment search per item on log_p_attn (B, T_mel, T_inp) float32 restricted
 * to [:feats_lens[b], :text_lens[b]].  path (B, T_mel) int32 (token per frame, -1 past the item), durations (B, T_inp) float32
 * = bincount(path), bin_loss (B) = -mean_j log_p[j, path[j]] per item (the reference averages them over B).
 * Bit-exact paths / durations vs the reference's numba loop (float64 scores, float32 row-0 sums, ties -> smaller index).
 * workspace: B*T_mel*T_inp bytes. */
EV_API int ev_op_mas(const float* log_p_attn, const int64_t* text_lens, const int64_t* feats_lens, int B, int T_mel, int T_inp,
                     int32_t* path, float* durations, float* bin_loss, uint8_t* workspace, size_t workspace_bytes, void* stream);
/* average_by_duration (alignment.py:145-177): out (B, T_inp) = per-token mean of xs (B, T_mel) over the token's frames. */
EV_API int ev_op_average_by_duration(const float* durations, const float* xs, const int64_t* text_lens, const int64_t* feats_lens,
                                     int B, int T_mel, int T_inp, float* out, void* stream);
/* AlignmentModule.forward after its convolutions (alignment.py:39-56): log_p_attn[b,f,t] = log_softmax_t( -||feats_feat[b,f,:] -
 * text_feat[b,t,:]||_2 ) with tokens t >= text_lens[b] masked to -inf, + prior (B,T_mel,T_inp; may be NULL).  text_feat (B,T_inp,A),
 * feats_feat (B,T_mel,A) time-major fp32, A a multiple of 128.  Training only. */
EV_API int ev_op_align_logp(const float* text_feat, const float* feats_feat, const int64_t* text_lens, const float* prior, int B, int T_mel,
                            int T_inp, int A, float* log_p_attn, void* stream);
/* get_segments (models/hifigan/get_random_segments.py:19-27; jets.py:55-60): out[b,c,i] = x[b,c,start_idxs[b]+i], zero past T.
 * x (B,C,T) channels-first, out (B,C,segment_size). */
EV_API int ev_op_get_segments(const float* x, const int64_t* start_idxs, int B, int C, int T, int segment_size, float* out, void* stream);

/* ---- features of recordings (not used by any inference path) -------------------------------------------------------------
 * Log-mel spectrogram and frame energy of fp32 waveforms, 1024-point STFT, one launch:
 *   TacotronSTFT.mel_spectrogram (tacotron_stft.py:71-80, stft.py:132-160, audio_processing.py:50-51): pad 512, mag_eps 0;
 *   mel_spectrogram_torch (mel_process.py:77-110): pad (1024 - hop) / 2, mag_eps 1e-6;
 *   Energy.get_energy (feats.py:178-196, librosa.stft center=True): pad 512, energy only.
 * Item b is wav[b * item_stride + t], t < n_samples[b] (n_samples (B) i64, or NULL: item_stride samples each), reflect-padded
 * by pad samples at both of its own ends (edge sample not repeated); samples at or past n_samples[b] are never read.  Frame f
 * of an item is padded samples [f * hop, f * hop + 1024) times window (1024 f32, the caller's rounding of the periodic Hann
 * window); its item has F_b = (n_samples[b] + 2 pad - 1024) / hop + 1 frames (clamped to F).  X = rfft of the frame (fp32,
 * twiddle (1024, 2) f32 = (cos, -sin)(2 pi k / 1024) rounded from fp64), |X_k| = sqrt(re^2 + im^2 + mag_eps), k = 0..512.
 *   mel (B, n_mels, F) or NULL: log(max(sum_k M[j,k] |X_k|, 1e-5)), the sum over band j's bins in ascending order: bands
 *   (n_mels, 3) i32 = {first bin, bin count, offset into band_w}, band_w f32 = the basis entries M[j, first .. first+count).
 *   n_mels <= 128.
 *   energy (B, F) or NULL: sqrt(max(sum_{k=0..512} |X_k|^2, 1e-10)) (|X_k|^2 without mag_eps).
 *   Frames f >= F_b are stored as 0.  status (i32, may be NULL) |= 1 when a sample in [0, n_samples[b]) is outside [-1, 1] or
 *   NaN (the reference's assert), |= 2 when an item is not longer than pad, is longer than item_stride or fills no frame (its
 *   outputs are all 0).  hop in [1, 1024], pad in [0, 1024).  Each output depends only on its own item: a batch is bitwise its
 *   items' single calls.  No allocation, no sync. */
EV_API int ev_stft_features(const float* wav, long long item_stride, const int64_t* n_samples, int B, int pad, int hop, int F,
                            const float* window, const float* twiddle, float mag_eps, const int32_t* bands, const float* band_w,
                            int n_mels, float* mel, float* energy, int32_t* status, void* stream);

/* Pitch of fp64 recordings: pyworld.dio then pyworld.stonemask at pyworld's defaults (f0_floor 71, f0_ceil 800, 2 channels per
 * octave, speed 1, allowed_range 0.1), as feats.Pitch._calculate_pitch (feats.py:114-131) calls them, restated from the published
 * algorithms (oracle/pitch_oracle.py lists every assumed detail; not checked against pyworld).  Item b is x[b * item_stride + t],
 * t < n_samples[b] (n_samples (B) i64, or NULL: item_stride samples each); nothing at or past n_samples[b] is read.  fs in
 * [8000, 48000] Hz, frame_period in [0.25, 1000] ms, F = int(1000 item_stride / fs / frame_period) + 1 (the row's frame
 * count); item b has F_b = int(1000 n_samples[b] / fs / frame_period) + 1 frames at times f * frame_period / 1000 s.
 *   raw_f0 (B, F) f64 or NULL: DIO's contour.
 *   pitch (B, F) f64: StoneMask's refined contour; with flags & 1 the reference's continuous interpolation (ends held, linear
 *   between voiced frames, as feats.py:92-112), then with flags & 2 the log of every nonzero frame.
 * Frames f >= F_b are stored as 0; an item of at most int(0.5 + 1000 / frame_period / 71) * 2 + 1 frames is all 0 (WORLD's
 * FixF0Contour).  status (i32, may be NULL) |= 1 when a sample is not finite, |= 2 when an item is shorter than the low-cut
 * filter (2 round(fs / 50) + 1 samples) or longer than item_stride (its outputs are all 0).  workspace: at least
 * ev_pitch_workspace_bytes(B, item_stride, fs, frame_period, F) bytes, 16-byte aligned (0 for arguments ev_pitch rejects).
 * fp64 throughout.  Each output depends only on its own item: a batch is bitwise its items' single calls.  No allocation, no
 * sync. */
EV_API size_t ev_pitch_workspace_bytes(int B, long long item_stride, int fs, double frame_period, int F);
EV_API int ev_pitch(const double* x, long long item_stride, const int64_t* n_samples, int B, int fs, double frame_period, int F,
                    int flags, double* raw_f0, double* pitch, int32_t* status, void* workspace, size_t workspace_bytes, void* stream);

/* Spectral envelopes of fp64 recordings: WORLD's CheapTrick at pyworld's defaults (q1 = -0.15, f0_floor 71), restated from the
 * published algorithm (oracle/world_oracle.py lists every assumed detail, W1-W11; not checked against pyworld).  x, item_stride,
 * n_samples, B, fs, frame_period, F and the frames F_b of each item are ev_pitch's.  f0 (B, F) f64 DEVICE: the F0 of each frame
 * in Hz; a frame whose F0 is at or below 3 fs / (fft_size - 3), above fs / 4 or not finite is analysed at 500 Hz.  fft_size =
 * 2^(1 + int(log(3 fs / 71 + 1) / log 2)): 512 at 8 kHz, 1024 at 16 to 24 kHz, 2048 at 44.1 and 48 kHz; bins = fft_size / 2 + 1.
 * WORLD's random noise is replaced by a floor of 2^-52 on every smoothed power bin, so every frame depends on its own samples
 * and digital silence gives finite output; the linear smoothing is summed over the bins it spans (what WORLD's difference of
 * two running sums equals in exact arithmetic), so no smoothed bin is negative and every output is finite for finite input.
 *   sp (B, F, bins) f64 or NULL: the power envelope (pyworld.cheaptrick's output).
 *   mc (B, F, n_out) f64 or NULL: mc_table (n_out, bins) f64 DEVICE, 1 <= n_out <= 256, times the log envelope of the frame
 *   (the log before the final exp): with the table of sp2mc (emotivoice_b200.feats.sp2mc_table) the mel-cepstrum.
 * One of sp, mc is needed.  Frames f >= F_b are stored as 0.  status (i32, may be NULL): ev_pitch's bits (|= 1 a sample is not
 * finite, |= 2 an item is shorter than 2 round(fs / 50) + 1 samples or longer than item_stride: its outputs are all 0).  fp64
 * throughout; one launch.  Each output depends only on its own item: a batch is bitwise its items' single calls.  No
 * workspace, no allocation, no sync. */
EV_API int ev_world_envelope(const double* x, long long item_stride, const int64_t* n_samples, int B, int fs, double frame_period,
                             int F, const double* f0, double* sp, const double* mc_table, int n_out, double* mc, int32_t* status,
                             void* stream);
/* Mel-cepstra of power envelopes (pysptk.sp2mc through a table): mc[r, k] = sum_j table[k, j] log(sp[r, j]), rows r < n_frames
 * of sp (n_frames, bins) f64 DEVICE, bins = fft_size / 2 + 1 with fft_size a power of two in [4, 2048], sp > 0; table
 * (n_out, bins) f64 DEVICE, 1 <= n_out <= 256; mc (n_frames, n_out) f64.  One launch (none for n_frames = 0); each row depends
 * only on its own. */
EV_API int ev_sp2mc(const double* sp, long long n_frames, int bins, const double* table, int n_out, double* mc, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* EMOTIVOICE_B200_H_ */
