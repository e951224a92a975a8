// Training-mode alignment helpers on the GPU (SURVEY.md s8f rank 4), replacing the per-sample numba loops the reference runs on
// the CPU in the middle of every training step (models/prompt_tts_modified/modules/alignment.py:90-177):
//   * mas_kernel            monotonic alignment search + durations + bin loss (_monotonic_alignment_search, viterbi_decode)
//   * avg_by_duration_kernel  per-token mean of a frame-level track (average_by_duration)
// Integer outputs (path, durations) are bit-exact with the reference: the dynamic programme is restated with its arithmetic --
// float32 inputs, float64 scores, row 0 = float32 running sums widened to float64, ties prefer the smaller token index.
// Not launched by any inference path.
#include "ev_common.cuh"

namespace ev {

// One CTA per batch item; threads over token index i, frames j sequentially (column j needs column j-1).
// dec[j][i] (bytes, frames x tokens of this item's slice of the workspace) = 1 iff Q[i-1, j-1] >= Q[i, j-1]: the predecessor
// of cell (i, j) on the best path is token i-1 (alignment.py:109-119 compares exactly these two scores, ties -> i-1).
__global__ void __launch_bounds__(256) mas_kernel(const float* __restrict__ log_p, const int64_t* __restrict__ text_lens,
                                                  const int64_t* __restrict__ feats_lens, int T_mel, int T_inp,
                                                  int32_t* __restrict__ path, float* __restrict__ durations,
                                                  float* __restrict__ bin_loss, uint8_t* __restrict__ dec_ws) {
  pdl_entry();
  extern __shared__ __align__(16) unsigned char mas_smem[];
  double* q0 = reinterpret_cast<double*>(mas_smem);
  double* q1 = q0 + T_inp;
  int* cnt = reinterpret_cast<int*>(q1 + T_inp);
  const int b = blockIdx.x, tid = threadIdx.x;
  const int T = (int)min((long long)T_inp, max(0ll, (long long)text_lens[b]));
  const int F = (int)min((long long)T_mel, max(0ll, (long long)feats_lens[b]));
  const float* lp = log_p + (size_t)b * T_mel * T_inp;       // (frame j, token i) at j*T_inp + i
  uint8_t* dec = dec_ws + (size_t)b * T_mel * T_inp;
  int32_t* pb = path + (size_t)b * T_mel;
  float* db = durations + (size_t)b * T_inp;
  for (int i = tid; i < T_inp; i += blockDim.x) { db[i] = 0.f; cnt[i] = 0; }
  for (int j = tid; j < T_mel; j += blockDim.x) pb[j] = -1;
  if (T <= 0 || F <= 0) {
    if (tid == 0) bin_loss[b] = 0.f;
    return;
  }
  const double NEG_INF = -INFINITY;
  float run = 0.f;                                            // thread 0: float32 running sum of row 0 (numba sums the slice in float32)
  double* prev = q0;
  double* cur = q1;
  // column 0
  for (int i = tid; i < T; i += blockDim.x) cur[i] = (i == 0) ? (double)lp[0] : NEG_INF;
  if (tid == 0) run = lp[0];
  __syncthreads();
  for (int j = 1; j < F; ++j) {
    double* t = prev; prev = cur; cur = t;
    const float* row = lp + (size_t)j * T_inp;
    uint8_t* drow = dec + (size_t)j * T_inp;
    for (int i = tid; i < T; i += blockDim.x) {
      if (i == 0) {
        run = __fadd_rn(run, row[0]);
        cur[0] = (double)run;
      } else {
        const double a = prev[i - 1], c = prev[i];
        const bool take_a = a >= c;
        drow[i] = take_a ? 1 : 0;
        cur[i] = (i <= j) ? __dadd_rn(take_a ? a : c, (double)row[i]) : NEG_INF;
      }
    }
    __syncthreads();
  }
  // backtrack (alignment.py:107-120), durations = bincount(path), bin loss = -mean_j log_p[j, path[j]]
  if (tid == 0) {
    int i = T - 1;
    double acc = 0.0;
    for (int j = F - 1; j >= 0; --j) {
      pb[j] = i;
      cnt[i] += 1;
      acc += (double)lp[(size_t)j * T_inp + i];
      if (j > 0 && i > 0 && dec[(size_t)j * T_inp + i]) i -= 1;
    }
    bin_loss[b] = (float)(-acc / (double)F);
  }
  __syncthreads();
  for (int i = tid; i < T; i += blockDim.x) db[i] = (float)cnt[i];
}

int launch_mas(const float* log_p, const int64_t* text_lens, const int64_t* feats_lens, int B, int T_mel, int T_inp, int32_t* path,
               float* durations, float* bin_loss, uint8_t* dec_ws, cudaStream_t st) {
  EV_CHECK_ARG(B > 0 && T_mel > 0 && T_inp > 0, "mas: B=%d T_mel=%d T_inp=%d", B, T_mel, T_inp);
  const size_t smem = (size_t)T_inp * (2 * sizeof(double) + sizeof(int));
  EV_CHECK_ARG(smem <= 200 * 1024, "mas: %d tokens exceed the shared-memory budget", T_inp);
  static std::atomic<uint64_t> attr_devs{0};
  if (first_use_on_device(attr_devs)) cudaFuncSetAttribute(mas_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  return launch("mas_kernel", mas_kernel, B, 256, smem, st, log_p, text_lens, feats_lens, T_mel, T_inp, path, durations, bin_loss, dec_ws);
}

// out[b, n] = mean(xs[b, start_n : start_n + d_n]) (0 when the slice is empty), start = exclusive cumsum of the durations; tokens
// past text_lens[b] stay 0 (alignment.py:145-165).  One CTA per item; thread 0 builds the prefix, then threads over tokens.
// Each slice bound is normalised like a numpy slice of the length-F row: a negative bound counts from the end (+ F), then both
// are clipped to [0, F].  So negative durations give the reference's answer, and no index outside the item's [0, F) is formed.
__device__ __forceinline__ int abd_slice_bound(int v, int F) { return min(max(v < 0 ? v + F : v, 0), F); }

__global__ void __launch_bounds__(256) avg_by_duration_kernel(const float* __restrict__ durations, const float* __restrict__ xs,
                                                              const int64_t* __restrict__ text_lens, const int64_t* __restrict__ feats_lens,
                                                              int T_mel, int T_inp, float* __restrict__ out) {
  pdl_entry();
  extern __shared__ int abd_start[];     // T_inp + 1
  const int b = blockIdx.x, tid = threadIdx.x;
  const int T = (int)min((long long)T_inp, max(0ll, (long long)text_lens[b]));
  const int F = (int)min((long long)T_mel, max(0ll, (long long)feats_lens[b]));
  const float* d = durations + (size_t)b * T_inp;
  const float* x = xs + (size_t)b * T_mel;
  float* o = out + (size_t)b * T_inp;
  if (tid == 0) {
    int s = 0;
    for (int n = 0; n < T; ++n) { abd_start[n] = s; s += (int)d[n]; }
    abd_start[T] = s;
  }
  __syncthreads();
  for (int n = tid; n < T_inp; n += blockDim.x) {
    float v = 0.f;
    if (n < T) {
      const int s = abd_slice_bound(abd_start[n], F), e = abd_slice_bound(abd_start[n + 1], F);     // x[start:end] of the length-F row
      if (e > s) {
        double acc = 0.0;
        for (int j = s; j < e; ++j) acc += (double)x[j];
        v = (float)(acc / (double)(e - s));
      }
    }
    o[n] = v;
  }
}

int launch_avg_by_duration(const float* durations, const float* xs, const int64_t* text_lens, const int64_t* feats_lens, int B,
                           int T_mel, int T_inp, float* out, cudaStream_t st) {
  EV_CHECK_ARG(B > 0 && T_mel > 0 && T_inp > 0, "average_by_duration: B=%d T_mel=%d T_inp=%d", B, T_mel, T_inp);
  const size_t smem = (size_t)(T_inp + 1) * sizeof(int);
  EV_CHECK_ARG(smem <= 48 * 1024, "average_by_duration: %d tokens exceed the shared-memory budget", T_inp);
  return launch("avg_by_duration_kernel", avg_by_duration_kernel, B, 256, smem, st, durations, xs, text_lens, feats_lens, T_mel, T_inp, out);
}


// ---------------------------------------------------------------------------------------------
// AlignmentModule.forward after its convolutions (alignment.py:39-56): score[b,f,t] = -|| feats[b,f,:] - text[b,t,:] ||_2,
// tokens t >= text_lens[b] masked to -inf (x_masks), log_softmax over t, + the beta-binomial prior (built on the host like
// the reference builds it, -inf outside each item's (T_feats, T_text) rectangle).  One warp per frame: the frame's feature row
// lives in registers (A = NC*128 channels), the text rows stream through L1/L2, the T scores of the frame sit in shared memory
// for the two softmax passes.  Training only.
// ---------------------------------------------------------------------------------------------
template <int NC>
__global__ void __launch_bounds__(128) align_logp_kernel(const float* __restrict__ text, const float* __restrict__ feats,
                                                         const int64_t* __restrict__ text_lens, const float* __restrict__ prior, int F, int T,
                                                         float* __restrict__ out) {
  pdl_entry();
  constexpr int A = NC * 128;
  extern __shared__ float alp_sc[];            // [4 warps][T]
  const int b = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int f = blockIdx.x * 4 + warp;
  if (f >= F) return;
  const int tl = text_lens ? (int)min((long long)T, max(0ll, (long long)text_lens[b])) : T;
  float* sc = alp_sc + (size_t)warp * T;
  const float* fr = feats + ((size_t)b * F + f) * A;
  float4 fv[NC];
#pragma unroll
  for (int j = 0; j < NC; ++j) fv[j] = *reinterpret_cast<const float4*>(fr + (lane + 32 * j) * 4);
  float mx = -INFINITY;
  for (int t = 0; t < tl; ++t) {
    const float* tr = text + ((size_t)b * T + t) * A;
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < NC; ++j) {
      const float4 tv = __ldg(reinterpret_cast<const float4*>(tr + (lane + 32 * j) * 4));
      const float dx = fv[j].x - tv.x, dy = fv[j].y - tv.y, dz = fv[j].z - tv.z, dw = fv[j].w - tv.w;
      s += (dx * dx + dy * dy) + (dz * dz + dw * dw);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float score = -sqrtf(s);
    mx = fmaxf(mx, score);
    if (lane == 0) sc[t] = score;
  }
  __syncwarp();
  float sum = 0.f;
  for (int t = lane; t < tl; t += 32) sum += expf(sc[t] - mx);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float lse = mx + logf(sum);
  const size_t ob = ((size_t)b * F + f) * T;
  for (int t = lane; t < T; t += 32) {
    const float lp = t < tl ? sc[t] - lse : -INFINITY;
    out[ob + t] = lp + (prior ? prior[ob + t] : 0.f);
  }
}

int launch_align_logp(const float* text, const float* feats, const int64_t* text_lens, const float* prior, int B, int F, int T, int A,
                      float* out, cudaStream_t st) {
  EV_CHECK_ARG(B > 0 && B <= 65535 && F > 0 && T > 0 && T <= 3072, "align_logp: B=%d F=%d T=%d (T <= 3072 tokens)", B, F, T);
  EV_CHECK_ARG(A % 128 == 0 && A <= 512, "align_logp: feature width %d must be a multiple of 128, <= 512", A);
  dim3 grid((F + 3) / 4, B);
  const size_t smem = (size_t)4 * T * sizeof(float);
  auto k = align_logp_kernel<4>;
  switch (A / 128) {
    case 1: k = align_logp_kernel<1>; break;
    case 2: k = align_logp_kernel<2>; break;
    case 3: k = align_logp_kernel<3>; break;
  }
  return launch("align_logp_kernel", k, grid, 128, smem, st, text, feats, text_lens, prior, F, T, out);
}

// get_segments (models/hifigan/get_random_segments.py:19-27): out[b, c, i] = x[b, c, start[b] + i] while start[b] + i < T, else 0.
// x is (B, C, T) channels-first like the reference's z = dec_outputs.transpose(1, 2) (jets.py:55-60).
__global__ void __launch_bounds__(256) segments_kernel(const float* __restrict__ x, const int64_t* __restrict__ start, int C, int T, int seg,
                                                       float* __restrict__ out, size_t n) {
  pdl_entry();
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int k = (int)(i % seg);
  const size_t bc = i / seg;
  const int b = (int)(bc / C);
  const long long t = (long long)start[b] + k;
  out[i] = (t >= 0 && t < T) ? x[bc * T + t] : 0.f;
}

int launch_segments(const float* x, const int64_t* start, int B, int C, int T, int seg, float* out, cudaStream_t st) {
  EV_CHECK_ARG(B > 0 && C > 0 && T > 0 && seg > 0, "get_segments: B=%d C=%d T=%d segment=%d", B, C, T, seg);
  const size_t n = (size_t)B * C * seg;
  return launch("segments_kernel", segments_kernel, (unsigned)((n + 255) / 256), 256, 0, st, x, start, C, T, seg, out, n);
}

}  // namespace ev

using namespace ev;

extern "C" {

int ev_op_mas(const float* log_p_attn, const int64_t* text_lens, const int64_t* feats_lens, int B, int T_mel, int T_inp,
              int32_t* path, float* durations, float* bin_loss, uint8_t* workspace, size_t workspace_bytes, void* stream) {
  EV_CHECK_ARG(log_p_attn && text_lens && feats_lens && path && durations && bin_loss && workspace, "ev_op_mas: null argument");
  EV_CHECK_ARG(workspace_bytes >= (size_t)B * T_mel * T_inp, "ev_op_mas: workspace %zu < %zu bytes", workspace_bytes, (size_t)B * T_mel * T_inp);
  EV_TRY(use_device_of(log_p_attn));
  return launch_mas(log_p_attn, text_lens, feats_lens, B, T_mel, T_inp, path, durations, bin_loss, workspace, reinterpret_cast<cudaStream_t>(stream));
}

int ev_op_average_by_duration(const float* durations, const float* xs, const int64_t* text_lens, const int64_t* feats_lens, int B,
                              int T_mel, int T_inp, float* out, void* stream) {
  EV_CHECK_ARG(durations && xs && text_lens && feats_lens && out, "ev_op_average_by_duration: null argument");
  EV_TRY(use_device_of(durations));
  return launch_avg_by_duration(durations, xs, text_lens, feats_lens, B, T_mel, T_inp, out, reinterpret_cast<cudaStream_t>(stream));
}

int ev_op_align_logp(const float* text_feat, const float* feats_feat, const int64_t* text_lens, const float* prior, int B, int T_mel, int T_inp,
                     int A, float* log_p_attn, void* stream) {
  EV_CHECK_ARG(text_feat && feats_feat && log_p_attn, "ev_op_align_logp: null argument");
  EV_TRY(use_device_of(text_feat));
  return launch_align_logp(text_feat, feats_feat, text_lens, prior, B, T_mel, T_inp, A, log_p_attn, reinterpret_cast<cudaStream_t>(stream));
}

int ev_op_get_segments(const float* x, const int64_t* start_idxs, int B, int C, int T, int segment_size, float* out, void* stream) {
  EV_CHECK_ARG(x && start_idxs && out, "ev_op_get_segments: null argument");
  EV_TRY(use_device_of(x));
  return launch_segments(x, start_idxs, B, C, T, segment_size, out, reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
