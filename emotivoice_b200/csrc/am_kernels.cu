// Acoustic-model kernels of the PromptTTS path (fp32, sm_90a): LayerNorm (+embedding/PE
// prologue), fused multi-head attention, conditioning gather, predictor heads, pitch/energy
// embedding, duration scan and Gaussian upsampling.  Reference semantics are cited per kernel.
#include "ev_common.cuh"

namespace ev {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---------------------------------------------------------------------------------------------
// LayerNorm over the last dim, eps = 1e-12, biased variance (encoder.py:112-127).  One warp per
// row, the row lives in registers (C <= 768, C % 128 == 0; 768 = the style encoder's BERT width).  Optional prologue for the first
// layer of the encoder: x = word_emb[id] + alpha * pe[t]  (model_open_source.py:107,
// encoder.py:257-261), which is also written back as the residual stream.
// ---------------------------------------------------------------------------------------------
template <int NV>  // float4 per lane
__global__ void __launch_bounds__(256) layernorm_kernel(const float* __restrict__ x, const int64_t* __restrict__ ids,
                                                        const float* __restrict__ emb, const float* __restrict__ pe,
                                                        const float* __restrict__ alpha, float* __restrict__ x_out,
                                                        const float* __restrict__ w, const float* __restrict__ b,
                                                        float* __restrict__ y, int rows, int L, int n_emb) {
  pdl_entry();
  constexpr int C = NV * 128;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  float4 v[NV];
  if (ids) {
    const int t = row % L;
    const float a = *alpha;
    // out-of-range ids are reported by validate_inputs_kernel (the host raises); clamped here so the read stays in bounds
    const long long id = ids[row];
    const float* e = emb + (size_t)(id < 0 ? 0 : (id >= n_emb ? n_emb - 1 : id)) * C;
    const float* pr = pe + (size_t)t * C;
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const float4 ev4 = *reinterpret_cast<const float4*>(e + (lane + 32 * j) * 4);
      const float4 p4 = *reinterpret_cast<const float4*>(pr + (lane + 32 * j) * 4);
      // mul and add rounded separately, like the reference's `x + alpha * pe` (no FMA contraction)
      v[j] = make_float4(__fadd_rn(ev4.x, __fmul_rn(a, p4.x)), __fadd_rn(ev4.y, __fmul_rn(a, p4.y)),
                         __fadd_rn(ev4.z, __fmul_rn(a, p4.z)), __fadd_rn(ev4.w, __fmul_rn(a, p4.w)));
      *reinterpret_cast<float4*>(x_out + (size_t)row * C + (lane + 32 * j) * 4) = v[j];
    }
  } else {
#pragma unroll
    for (int j = 0; j < NV; ++j) v[j] = *reinterpret_cast<const float4*>(x + (size_t)row * C + (lane + 32 * j) * 4);
  }
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < NV; ++j) s += (v[j].x + v[j].y) + (v[j].z + v[j].w);
  const float mean = warp_sum(s) / (float)C;
  float q = 0.f;
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    const float dx = v[j].x - mean, dy = v[j].y - mean, dz = v[j].z - mean, dw = v[j].w - mean;
    q += (dx * dx + dy * dy) + (dz * dz + dw * dw);
  }
  const float var = warp_sum(q) / (float)C;
  const float rstd = 1.0f / sqrtf(var + 1e-12f);
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    const int c = (lane + 32 * j) * 4;
    const float4 w4 = *reinterpret_cast<const float4*>(w + c);
    const float4 b4 = *reinterpret_cast<const float4*>(b + c);
    float4 o;
    o.x = (v[j].x - mean) * rstd * w4.x + b4.x;
    o.y = (v[j].y - mean) * rstd * w4.y + b4.y;
    o.z = (v[j].z - mean) * rstd * w4.z + b4.z;
    o.w = (v[j].w - mean) * rstd * w4.w + b4.w;
    *reinterpret_cast<float4*>(y + (size_t)row * C + c) = o;
  }
}

int launch_layernorm(const float* x, const int64_t* ids, const float* emb, const float* pe, const float* alpha,
                     float* x_out, const float* w, const float* b, float* y, int rows, int L, int C,
                     cudaStream_t st, int n_emb) {
  EV_CHECK_ARG(rows > 0, "layernorm: rows=%d", rows);
  EV_CHECK_ARG(!ids || n_emb > 0, "layernorm: embedding prologue without a table size");
  EV_CHECK_ARG(C % 128 == 0 && C <= 768, "layernorm: C=%d must be a multiple of 128 and <= 768", C);
  const int wpb = 8;
  dim3 grid((rows + wpb - 1) / wpb);
  auto k = layernorm_kernel<6>;
  switch (C / 128) {
    case 1: k = layernorm_kernel<1>; break;
    case 2: k = layernorm_kernel<2>; break;
    case 3: k = layernorm_kernel<3>; break;
    case 4: k = layernorm_kernel<4>; break;
    case 5: k = layernorm_kernel<5>; break;
  }
  return launch("layernorm_kernel", k, grid, 256, 0, st, x, ids, emb, pe, alpha, x_out, w, b, y, rows, L, n_emb);
}

// ---------------------------------------------------------------------------------------------
// Fused multi-head self-attention (encoder.py:84-109): scores = q k^T / sqrt(d_k), key-padding
// mask, softmax, P v -- never materialising the (L x L) score matrix (flash-style online
// softmax, fp32).  One CTA = 64 queries of one (batch item, head); d_k = DK (48 for EmotiVoice).
// qkv is the packed (B, L, 3H) output of the fused q|k|v projection; head h owns columns
// [h*DK, (h+1)*DK) of each third (encoder.py:72-82).  Query rows >= key_len are computed like
// the reference computes them (they attend to the valid keys).
// ---------------------------------------------------------------------------------------------
template <int DK, int BQ>
__global__ void __launch_bounds__(128) attention_kernel(const float* __restrict__ qkv, const int32_t* __restrict__ key_lens,
                                                        float* __restrict__ ctx, int L, int H) {
  pdl_entry();
  constexpr int BK = 64, LDQ = BQ + 1, LDT = BK + 1;
  constexpr int RQ = BQ / 16;   // query rows per thread
  constexpr int OC = DK / 8;    // output columns per thread
  constexpr int D4 = DK / 4;    // float4 per head row
  extern __shared__ __align__(16) float att_smem[];
  float (*Qt)[LDQ] = reinterpret_cast<float (*)[LDQ]>(att_smem);                        // [DK][LDQ] transposed: [d][query]
  float (*Kt)[LDT] = reinterpret_cast<float (*)[LDT]>(att_smem + DK * LDQ);             // [DK][LDT] transposed: [d][key]
  float (*Vs)[DK] = reinterpret_cast<float (*)[DK]>(att_smem + DK * LDQ + DK * LDT);    // [BK][DK]
  float (*Ps)[LDT] = reinterpret_cast<float (*)[LDT]>(att_smem + DK * LDQ + DK * LDT + BK * DK);   // [BQ][LDT]

  const int tid = threadIdx.x;
  const int tx = tid & 7, ty = tid >> 3;   // 8 x 16
  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * BQ;
  const int klen = key_lens ? min(L, key_lens[b]) : L;
  const size_t ld = (size_t)3 * H;
  const float* base = qkv + (size_t)b * L * ld;
  const float sqrt_dk = sqrtf((float)DK);

  // load the Q tile (transposed), 16-byte global loads
  for (int idx = tid; idx < BQ * D4; idx += 128) {
    const int r = idx / D4, d4 = idx % D4;
    const int row = q0 + r;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (row < L) v = *reinterpret_cast<const float4*>(base + (size_t)row * ld + h * DK + d4 * 4);
    Qt[d4 * 4 + 0][r] = v.x; Qt[d4 * 4 + 1][r] = v.y; Qt[d4 * 4 + 2][r] = v.z; Qt[d4 * 4 + 3][r] = v.w;
  }

  float m_i[RQ], l_i[RQ], o[RQ][OC];
#pragma unroll
  for (int i = 0; i < RQ; ++i) {
    m_i[i] = -INFINITY;
    l_i[i] = 0.f;
#pragma unroll
    for (int c = 0; c < OC; ++c) o[i][c] = 0.f;
  }

  for (int k0 = 0; k0 < klen; k0 += BK) {
    __syncthreads();   // previous tile fully consumed (also orders the Q tile on the first pass)
    for (int idx = tid; idx < BK * D4; idx += 128) {
      const int r = idx / D4, d4 = idx % D4;
      const int row = k0 + r;
      float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
      if (row < klen) {
        kv = *reinterpret_cast<const float4*>(base + (size_t)row * ld + H + h * DK + d4 * 4);
        vv = *reinterpret_cast<const float4*>(base + (size_t)row * ld + 2 * H + h * DK + d4 * 4);
      }
      Kt[d4 * 4 + 0][r] = kv.x; Kt[d4 * 4 + 1][r] = kv.y; Kt[d4 * 4 + 2][r] = kv.z; Kt[d4 * 4 + 3][r] = kv.w;
      *reinterpret_cast<float4*>(&Vs[r][d4 * 4]) = vv;
    }
    __syncthreads();

    // S = Q K^T : thread owns rows ty*RQ..+RQ-1, cols tx + 8j
    float s[RQ][8];
#pragma unroll
    for (int i = 0; i < RQ; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) s[i][j] = 0.f;
#pragma unroll 4
    for (int d = 0; d < DK; ++d) {
      float qv[RQ], kv[8];
#pragma unroll
      for (int i = 0; i < RQ; ++i) qv[i] = Qt[d][ty * RQ + i];
#pragma unroll
      for (int j = 0; j < 8; ++j) kv[j] = Kt[d][tx + 8 * j];
#pragma unroll
      for (int i = 0; i < RQ; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) s[i][j] = fmaf(qv[i], kv[j], s[i][j]);
    }
    // scale, mask, online softmax
#pragma unroll
    for (int i = 0; i < RQ; ++i) {
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int col = k0 + tx + 8 * j;
        s[i][j] = col < klen ? s[i][j] / sqrt_dk : -INFINITY;
        mx = fmaxf(mx, s[i][j]);
      }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 4));
      const float m_new = fmaxf(m_i[i], mx);      // finite: every key tile has >= 1 valid key
      const float scale = expf(m_i[i] - m_new);   // exp(-inf) = 0 on the first tile
      float rs = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float pv = expf(s[i][j] - m_new);
        rs += pv;
        Ps[ty * RQ + i][tx + 8 * j] = pv;
      }
      rs += __shfl_xor_sync(0xffffffffu, rs, 1);
      rs += __shfl_xor_sync(0xffffffffu, rs, 2);
      rs += __shfl_xor_sync(0xffffffffu, rs, 4);
      l_i[i] = l_i[i] * scale + rs;
      m_i[i] = m_new;
#pragma unroll
      for (int c = 0; c < OC; ++c) o[i][c] *= scale;
    }
    __syncwarp();   // Ps rows ty*RQ.. are written and read by the same 8 lanes (one warp)
    // O += P V : thread owns rows ty*RQ..+RQ-1, cols tx + 8c
#pragma unroll 4
    for (int k = 0; k < BK; ++k) {
      float pv[RQ], vv[OC];
#pragma unroll
      for (int i = 0; i < RQ; ++i) pv[i] = Ps[ty * RQ + i][k];
#pragma unroll
      for (int c = 0; c < OC; ++c) vv[c] = Vs[k][tx + 8 * c];
#pragma unroll
      for (int i = 0; i < RQ; ++i)
#pragma unroll
        for (int c = 0; c < OC; ++c) o[i][c] = fmaf(pv[i], vv[c], o[i][c]);
    }
  }

  float* ob = ctx + (size_t)b * L * H;
#pragma unroll
  for (int i = 0; i < RQ; ++i) {
    const int row = q0 + ty * RQ + i;
    if (row >= L) continue;
    const float inv = 1.0f / l_i[i];
#pragma unroll
    for (int c = 0; c < OC; ++c) ob[(size_t)row * H + h * DK + tx + 8 * c] = o[i][c] * inv;
  }
}

template <int DK, int BQ>
static int launch_attention_dk(const float* qkv, const int32_t* key_lens, float* ctx, int B, int L, int H, int heads,
                               cudaStream_t st) {
  const size_t smem = (size_t)(DK * (BQ + 1) + DK * 65 + 64 * DK + BQ * 65) * sizeof(float);
  static std::atomic<uint64_t> attr_devs{0};
  if (first_use_on_device(attr_devs))
    cudaFuncSetAttribute(attention_kernel<DK, BQ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  dim3 grid((L + BQ - 1) / BQ, heads, B);
  return launch("attention_kernel", attention_kernel<DK, BQ>, grid, 128, smem, st, qkv, key_lens, ctx, L, H);
}

int launch_attention(const float* qkv, const int32_t* key_lens, float* ctx, int B, int L, int H, int heads,
                     cudaStream_t st) {
  EV_CHECK_ARG(B > 0 && L > 0 && heads > 0 && H % heads == 0, "attention: bad shape B=%d L=%d H=%d heads=%d", B, L, H, heads);
  EV_CHECK_ARG(B <= 65535 && heads <= 65535, "attention: grid too large");
  const int dk = H / heads;
  // 32-query tiles while 64-query tiles would leave SMs idle (batch 1), 64-query tiles otherwise
  const bool small = (long long)((L + 63) / 64) * heads * B < 2 * sm_count();
  if (dk == 48) return small ? launch_attention_dk<48, 32>(qkv, key_lens, ctx, B, L, H, heads, st)
                             : launch_attention_dk<48, 64>(qkv, key_lens, ctx, B, L, H, heads, st);
  if (dk == 64) return small ? launch_attention_dk<64, 32>(qkv, key_lens, ctx, B, L, H, heads, st)
                             : launch_attention_dk<64, 64>(qkv, key_lens, ctx, B, L, H, heads, st);
  if (dk == 32) return small ? launch_attention_dk<32, 32>(qkv, key_lens, ctx, B, L, H, heads, st)
                             : launch_attention_dk<32, 64>(qkv, key_lens, ctx, B, L, H, heads, st);
  set_error("attention: unsupported head dim %d (32/48/64)", dk);
  return EV_EINVAL;
}

// ---------------------------------------------------------------------------------------------
// Conditioning gather: c[b] = [ spk_emb[spk[b]] | style[b] | content[b] ]   (model_open_source.py:109-110).
// The 2304->384 projection (:111) is split: W_x x_t + (W_c c_b + bias); the second term is a
// per-utterance bias computed once per item by the generic GEMM on this gathered vector.
// ---------------------------------------------------------------------------------------------
__global__ void cond_gather_kernel(const int64_t* __restrict__ spk, const float* __restrict__ spk_emb,
                                   const float* __restrict__ style, const float* __restrict__ content,
                                   float* __restrict__ out, int H, int bert, int n_spk) {
  pdl_entry();
  const int b = blockIdx.x;
  const int W = H + 2 * bert;
  const long long sid_raw = spk[b];      // range errors are reported by validate_inputs_kernel; clamp keeps the read in bounds
  const size_t sid = (size_t)(sid_raw < 0 ? 0 : (sid_raw >= n_spk ? n_spk - 1 : sid_raw));
  for (int i = threadIdx.x; i < W; i += blockDim.x) {
    float v;
    if (i < H) v = spk_emb[sid * H + i];
    else if (i < H + bert) v = style[(size_t)b * bert + (i - H)];
    else v = content[(size_t)b * bert + (i - H - bert)];
    out[(size_t)b * W + i] = v;
  }
}
int launch_cond_gather(const int64_t* spk, const float* spk_emb, const float* style, const float* content,
                       float* out, int B, int H, int bert, int n_spk, cudaStream_t st) {
  return launch("cond_gather_kernel", cond_gather_kernel, B, 256, 0, st, spk, spk_emb, style, content, out, H, bert, n_spk);
}

// ---------------------------------------------------------------------------------------------
// Per-utterance conditioning bias  u[b] = W_c^T c[b] + bias  (the utterance-constant 5/6 of
// embed_projection1, model_open_source.py:110-111).  A skinny GEMV (M = B rows, K = 1920): one CTA
// per (8 output columns, batch item); the K axis is split over the CTA's threads and reduced in a
// fixed order (deterministic).  w is (K, N) row-major.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) cond_gemv_kernel(const float* __restrict__ c, const float* __restrict__ w,
                                                        const float* __restrict__ bias, float* __restrict__ out, int K,
                                                        int N) {
  pdl_entry();
  __shared__ float red[8][8][33];
  const int b = blockIdx.y, n0 = blockIdx.x * 8;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  const float* cb = c + (size_t)b * K;
  for (int k = tid; k < K; k += 256) {
    const float cv = cb[k];
    const float4 w0 = *reinterpret_cast<const float4*>(w + (size_t)k * N + n0);
    const float4 w1 = *reinterpret_cast<const float4*>(w + (size_t)k * N + n0 + 4);
    acc[0] = fmaf(cv, w0.x, acc[0]); acc[1] = fmaf(cv, w0.y, acc[1]); acc[2] = fmaf(cv, w0.z, acc[2]); acc[3] = fmaf(cv, w0.w, acc[3]);
    acc[4] = fmaf(cv, w1.x, acc[4]); acc[5] = fmaf(cv, w1.y, acc[5]); acc[6] = fmaf(cv, w1.z, acc[6]); acc[7] = fmaf(cv, w1.w, acc[7]);
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[wid][j][lane] = acc[j];
  __syncthreads();
  if (tid < 64) {
    const int j = tid >> 3, w8 = tid & 7;      // 8 threads per column, each sums one warp's 32 partials
    float s = 0.f;
    for (int l = 0; l < 32; ++l) s += red[w8][j][l];
    s += __shfl_down_sync(0xffffffffu, s, 4, 8);
    s += __shfl_down_sync(0xffffffffu, s, 2, 8);
    s += __shfl_down_sync(0xffffffffu, s, 1, 8);
    if (w8 == 0) out[(size_t)b * N + n0 + j] = s + bias[n0 + j];
  }
}
int launch_cond_gemv(const float* c, const float* w, const float* bias, float* out, int B, int K, int N, cudaStream_t st) {
  EV_CHECK_ARG(N % 8 == 0 && B > 0 && B <= 65535, "cond_gemv: N=%d B=%d", N, B);
  dim3 grid(N / 8, B);
  return launch("cond_gemv_kernel", cond_gemv_kernel, grid, 256, 0, st, c, w, bias, out, K, N);
}

// ---------------------------------------------------------------------------------------------
// Predictor head: Linear(C -> 1) + output mask (variance.py:46-56, :119-124).
// mode 0: float (pitch / energy);  mode 1: duration = clamp(rint(exp(y) - 1), 0) as int64.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) rowdot_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                     const float* __restrict__ bias, const int32_t* __restrict__ lens,
                                                     int rows, int T, int C, int mode, float* __restrict__ out_f,
                                                     int64_t* __restrict__ out_i) {
  pdl_entry();
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const int b = row / T, t = row % T;
  const bool pad = lens && t >= lens[b];
  float s = 0.f;
  for (int c = lane * 4; c < C; c += 128) {
    const float4 xv = *reinterpret_cast<const float4*>(x + (size_t)row * C + c);
    const float4 wv = *reinterpret_cast<const float4*>(w + c);
    s = fmaf(xv.x, wv.x, s); s = fmaf(xv.y, wv.y, s); s = fmaf(xv.z, wv.z, s); s = fmaf(xv.w, wv.w, s);
  }
  s = warp_sum(s) + bias[0];
  if (lane == 0) {
    if (mode == 0) {
      out_f[row] = pad ? 0.f : s;
    } else {
      const float d = fmaxf(rintf(expf(s) - 1.0f), 0.f);   // torch.round == round-half-even == rintf
      out_i[row] = pad ? 0 : (int64_t)d;
    }
  }
}
int launch_rowdot(const float* x, const float* w, const float* b, const int32_t* lens, int B, int T, int C,
                  int mode, float* out_f, int64_t* out_i, cudaStream_t st) {
  EV_CHECK_ARG(C % 4 == 0, "rowdot: C=%d", C);
  const int rows = B * T;
  return launch("rowdot_kernel", rowdot_kernel, (rows + 7) / 8, 256, 0, st, x, w, b, lens, rows, T, C, mode, out_f, out_i);
}

// Input validation + length conversion, ONE CTA (B*T is a few thousand elements at most).  The reference raises
// IndexError from nn.Embedding for a bad token / speaker id and a shape error for a bad length; here the kernels index
// raw device memory, so this kernel reports range errors in a status word that the host reads with the mel lengths at
// the path's single sync (no extra round trip), and every consumer clamps so nothing is read out of bounds meanwhile.
// status bits: 1 = token id outside [0, n_vocab), 2 = speaker id outside [0, n_speaker), 4 = length outside [1, T].
// lens arrive as int64 (inference_am_vocoder_joint.py:114); the kernels take int32 clamped to [0, T].
__global__ void __launch_bounds__(1024) validate_inputs_kernel(const int64_t* __restrict__ ling, const int64_t* __restrict__ lens,
                                                               const int64_t* __restrict__ spk, int32_t* __restrict__ lens_out,
                                                               int32_t* __restrict__ status, int B, int T, int n_vocab, int n_spk) {
  pdl_entry();
  __shared__ int s_flags;
  if (threadIdx.x == 0) s_flags = 0;
  __syncthreads();
  int flags = 0;
  for (int i = threadIdx.x; i < B; i += blockDim.x) {
    const long long v = lens[i];
    if (v < 1 || v > T) flags |= 4;
    lens_out[i] = (int32_t)(v < 0 ? 0 : (v > T ? T : v));
    if (spk) { const long long sp = spk[i]; if (sp < 0 || sp >= n_spk) flags |= 2; }
  }
  if (ling)
    for (int i = threadIdx.x; i < B * T; i += blockDim.x) {
      const long long id = ling[i];
      if (id < 0 || id >= n_vocab) flags |= 1;
    }
  flags = __reduce_or_sync(0xffffffffu, flags);
  if ((threadIdx.x & 31) == 0 && flags) atomicOr(&s_flags, flags);
  __syncthreads();
  if (threadIdx.x == 0 && status) *status = s_flags;
}
int launch_validate_inputs(const int64_t* ling, const int64_t* lens, const int64_t* spk, int32_t* lens_out, int32_t* status, int B,
                           int T, int n_vocab, int n_spk, cudaStream_t st) {
  return launch("validate_inputs_kernel", validate_inputs_kernel, 1, 1024, 0, st, ling, lens, spk, lens_out, status, B, T, n_vocab, n_spk);
}

// masked_fill(x_masks, 0) on the predictors' input (variance.py:38-39, :109-110)
__global__ void mask_rows_kernel(const float4* __restrict__ x, const int32_t* __restrict__ lens, float4* __restrict__ y,
                                 int T, int C4, size_t n4) {
  pdl_entry();
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const size_t row = i / C4;
  const int b = (int)(row / T), t = (int)(row % T);
  y[i] = (lens && t >= lens[b]) ? make_float4(0.f, 0.f, 0.f, 0.f) : x[i];
}
int launch_mask_rows(const float* x, const int32_t* lens, float* y, int B, int T, int C, cudaStream_t st) {
  EV_CHECK_ARG(C % 4 == 0, "mask_rows: C=%d", C);
  const size_t n4 = (size_t)B * T * C / 4;
  return launch("mask_rows_kernel", mask_rows_kernel, (unsigned)((n4 + 255) / 256), 256, 0, st, (const float4*)x, lens, (float4*)y, T, C / 4, n4);
}

// ---------------------------------------------------------------------------------------------
// x += pitch_embed(p) + energy_embed(e): two Conv1d(1 -> C, k=K, pad=(K-1)/2) on the predicted
// scalar tracks (model_open_source.py:131-134).  wp/we are tap-major (K, C).
// prosody or null: {alpha, p_scale, p_shift, e_scale, e_shift} rows, one per item (B,5) or, with
// per_token, one per token (B,T,5); the tracks enter the convolutions as p*p_scale + p_shift and
// e*e_scale + e_shift (unfused, so 1 and 0 give p back), each tap with its own token's row.  With
// prosody and window (batch-invariant contract) the window ends at lens[b] like the item's own B=1
// call, where the conv's zero padding follows the last token; the shifted pads would otherwise leak
// in.  Per-token rows of pad tokens (t >= lens[b]) act as neutral.  zero_pads: the tracks are the
// caller's, and their pad entries read as 0, what the predictors write there.
// ---------------------------------------------------------------------------------------------
__global__ void var_embed_add_kernel(float* __restrict__ x, const float* __restrict__ pitch,
                                     const float* __restrict__ energy, const float* __restrict__ wp,
                                     const float* __restrict__ bp, const float* __restrict__ we,
                                     const float* __restrict__ be, const float* __restrict__ prosody, int per_token,
                                     const int32_t* __restrict__ lens, int window, int zero_pads, int T, int C, int K) {
  pdl_entry();
  const int row = blockIdx.x;   // b*T + t
  const int b = row / T, t = row % T;
  __shared__ float ps[16], es[16];
  if (threadIdx.x < K) {
    const int len = lens ? min(T, lens[b]) : T;
    const int tl = (prosody && window) ? len : T;
    const int tt = t + threadIdx.x - (K - 1) / 2;
    const bool ok = tt >= 0 && tt < tl;
    const bool rd = ok && !(zero_pads && tt >= len);
    float p = rd ? pitch[(size_t)b * T + tt] : 0.f;
    float e = rd ? energy[(size_t)b * T + tt] : 0.f;
    if (prosody && ok && !(per_token && tt >= len)) {
      const float* pr = prosody + (per_token ? (size_t)b * T + tt : (size_t)b) * 5;
      p = __fadd_rn(__fmul_rn(p, pr[1]), pr[2]);
      e = __fadd_rn(__fmul_rn(e, pr[3]), pr[4]);
    }
    ps[threadIdx.x] = p;
    es[threadIdx.x] = e;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float pe_ = 0.f, ee_ = 0.f;
    for (int j = 0; j < K; ++j) {
      pe_ = fmaf(wp[j * C + c], ps[j], pe_);
      ee_ = fmaf(we[j * C + c], es[j], ee_);
    }
    const size_t i = (size_t)row * C + c;
    x[i] = (x[i] + (pe_ + bp[c])) + (ee_ + be[c]);
  }
}
int launch_var_embed_add(float* x, const float* pitch, const float* energy, const float* wp, const float* bp,
                         const float* we, const float* be, const float* prosody, int per_token, const int32_t* lens, int window,
                         int zero_pads, int B, int T, int C, int K, cudaStream_t st) {
  EV_CHECK_ARG(K <= 16, "var_embed: K=%d > 16", K);
  EV_CHECK_ARG(lens || !(per_token || zero_pads), "var_embed: per-token rows and caller tracks need lens");
  return launch("var_embed_add_kernel", var_embed_add_kernel, B * T, 128, 0, st, x, pitch, energy, wp, bp, we, be, prosody, per_token,
                lens, window, zero_pads, T, C, K);
}

// ---------------------------------------------------------------------------------------------
// Duration bookkeeping of GaussianUpsampling.forward (alignment.py:183-199): ds = float(d) * alpha
// (alpha[b * alpha_stride + t * alpha_tstride]: per item when alpha_tstride is 0, per token
// otherwise; 1 when alpha is null); the "all durations are zero" guard (:187-191, applied after the
// scaling and over the WHOLE batch, pads included; it writes 1, not alpha); c = cumsum(ds) - ds/2;
// mel_lens[b] = trunc(fl32(sum_t ds)); mel_lens[B] = max_b.
// The scan runs in fp64 and rounds each output to fp32, which is what ATen's CPU cumsum does.  Every
// fp64 partial sum is exact, so the order of the parallel scan cannot change a bit:
//  * one alpha per item: each nonzero ds = fl32(d * alpha) >= alpha is a multiple of ulp(alpha), and
//    an item's sum stays below 2 * alpha * D with D = sum_t d <= max_frames < 2^24, so the sum has
//    fewer than 49 significant bits;
//  * alphas per token: the host keeps them in [1/16, 16]; every fp32 value >= 1/16 is a multiple of
//    2^-27, and a sum that passes the frame check is below 2^24, so it has fewer than 52 bits.
// (d itself converts exactly: it is at most max_frames < 2^24.)  The frame count rounds the exact sum
// once; the reference's cascade fp32 sum can land one frame off when the exact sum lies within a few
// fp32 ulps of an integer.
// caller != 0: dur holds caller durations: entries at t >= lens[b] are ignored (read as 0), negative
// ones are clamped to 0 and entries above max_frames to max_frames + 1 before anything is summed, so the
// u64 sums cannot overflow and both passes over the durations see the same values.
// status (may be null) gets bit 8 when an output would have no frames: any item under the
// batch-invariant contract (its own B=1 call fails in the decoder), or the whole batch otherwise; and
// bit 16 when a caller duration is negative or an item's frame count, before or after scaling,
// exceeds max_frames (the vocoder indexes samples with int32: F * prod(upsample_rates) < 2^31).
// One CTA (B*T is tiny).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ long long scan_dur(const int64_t* __restrict__ dur, int caller, const int32_t* __restrict__ lens,
                                              int b, int t, int T, int max_frames, int& bad) {
  const long long v = dur[(size_t)b * T + t];
  if (!caller) return v;
  if (lens && t >= lens[b]) return 0;
  if (v < 0) { bad = 1; return 0; }
  if (v > max_frames) { bad = 1; return (long long)max_frames + 1; }
  return v;
}

__global__ void __launch_bounds__(1024) duration_scan_kernel(const int64_t* __restrict__ dur, int caller,
                                                             const int32_t* __restrict__ lens,
                                                             const float* __restrict__ alpha, int alpha_stride,
                                                             int alpha_tstride, int invariant, int B, int T,
                                                             float* __restrict__ centers, float* __restrict__ ds_f,
                                                             int32_t* __restrict__ mel_lens, int32_t* __restrict__ status,
                                                             int max_frames) {
  pdl_entry();
  __shared__ unsigned long long s_total;
  __shared__ int s_max, s_min, s_bad;
  const int tid = threadIdx.x, nw = blockDim.x >> 5, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) { s_total = 0ull; s_max = 0; s_min = 0x7fffffff; s_bad = 0; }
  __syncthreads();
  unsigned long long part = 0;
  int bad = 0;
  for (int i = tid; i < B * T; i += blockDim.x) part += (unsigned long long)scan_dur(dur, caller, lens, i / T, i % T, T, max_frames, bad);
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  if (lane == 0 && part) atomicAdd(&s_total, part);
  if (bad) s_bad = 1;
  __syncthreads();
  const bool batch_all_zero = (s_total == 0ull);
  // one warp per batch item: chunked inclusive scan
  for (int b = wid; b < B; b += nw) {
    // literal batch: the guard looks at the whole batch and rewrites whole rows (pads included);
    // batch-invariant contract: each item is its own B=1 call of length lens[b].
    const int tl = invariant ? (lens ? min(T, lens[b]) : T) : T;
    unsigned long long own = 0;
    for (int t = lane; t < tl; t += 32) own += (unsigned long long)scan_dur(dur, caller, lens, b, t, T, max_frames, bad);
    for (int o = 16; o > 0; o >>= 1) own += __shfl_xor_sync(0xffffffffu, own, o);
    const bool all_zero = invariant ? (own == 0ull) : batch_all_zero;
    if (own > (unsigned long long)max_frames) bad = 1;
    double run = 0.0;
    for (int t0 = 0; t0 < T; t0 += 32) {
      const int t = t0 + lane;
      float d = 0.f;
      if (t < T) {
        const float a = alpha ? alpha[(size_t)b * alpha_stride + (size_t)t * alpha_tstride] : 1.0f;
        d = all_zero ? (t < tl ? 1.0f : 0.f) : __fmul_rn((float)scan_dur(dur, caller, lens, b, t, T, max_frames, bad), a);
      }
      double incl = d;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const double n = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += n;
      }
      if (t < T) {
        centers[(size_t)b * T + t] = __fsub_rn(__double2float_rn(run + incl), d * 0.5f);
        ds_f[(size_t)b * T + t] = d;
      }
      run += __shfl_sync(0xffffffffu, incl, 31);
    }
    if (lane == 0) {
      const int n = (int)__double2float_rn(run);       // the conversion saturates: an oversized sum cannot wrap
      if (n > max_frames) bad = 1;
      mel_lens[b] = n;
      atomicMax(&s_max, n);
      atomicMin(&s_min, n);
    }
  }
  if (bad) s_bad = 1;
  __syncthreads();
  if (tid == 0) {
    mel_lens[B] = s_max;
    if (status && (invariant ? s_min == 0 : s_max == 0)) atomicOr(status, 8);
    if (status && s_bad) atomicOr(status, 16);
  }
}
int launch_duration_scan(const int64_t* dur, int caller, const int32_t* lens, const float* alpha, int alpha_stride, int alpha_tstride,
                         int invariant, int B, int T, float* centers, float* ds_f, int32_t* mel_lens, int32_t* status, int max_frames,
                         cudaStream_t st) {
  EV_CHECK_ARG(max_frames > 0 && max_frames < (1 << 24), "duration_scan: max_frames=%d", max_frames);
  return launch("duration_scan_kernel", duration_scan_kernel, 1, 1024, 0, st, dur, caller, lens, alpha, alpha_stride, alpha_tstride,
                invariant, B, T, centers, ds_f, mel_lens, status, max_frames);
}

// ---------------------------------------------------------------------------------------------
// Gaussian upsampling (alignment.py:198-211): w[f,t] = softmax_t(-0.1 (f - c_t)^2) over the valid
// tokens, out[f] = sum_t w[f,t] hs[t].  One CTA = FT frames of one item; the token axis is
// streamed through shared memory; softmax statistics first (max, sum), then the weighted
// gather.  Optional epilogue out += alpha * pe[f]: the decoder's ScaledPositionalEncoding
// (encoder.py:257-261), fused here so the upsampled tensor is written once.
// invariant != 0: frames >= mel_lens[b] are written as zeros (B=1 semantics per item);
// otherwise all F frames are computed like the reference's padded batch does.
// ---------------------------------------------------------------------------------------------
constexpr int GU_TT = 16;   // tokens per smem chunk
// GU_FT frames per CTA (16, or 8 when the launch would otherwise leave most SMs idle: batch 1; the per-output token order, hence every
// bit, does not depend on it)
template <int NC, int GU_FT>           // channels per thread: H = NC * 128
__global__ void __launch_bounds__(128) gauss_upsample_kernel(const float* __restrict__ hs, const float* __restrict__ centers,
                                                             const int32_t* __restrict__ lens,
                                                             const int32_t* __restrict__ mel_lens, int T, int F,
                                                             int invariant, const float* __restrict__ pe,
                                                             const float* __restrict__ alpha, float* __restrict__ out) {
  pdl_entry();
  constexpr int H = NC * 128;
  __shared__ float s_w[GU_FT][GU_TT];
  __shared__ float s_max[GU_FT], s_inv[GU_FT];
  __shared__ __align__(16) float s_h[GU_TT][H];
  const int b = blockIdx.y, f0 = blockIdx.x * GU_FT;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int tlen = lens ? min(T, lens[b]) : T;
  const int flen = invariant ? min(F, mel_lens[b]) : F;
  float* ob = out + (size_t)b * F * H;
  if (f0 >= flen) {
    for (int i = tid; i < GU_FT * H; i += 128) {
      const int f = f0 + i / H;
      if (f < F) ob[(size_t)f * H + i % H] = 0.f;
    }
    return;
  }
  const float* cb = centers + (size_t)b * T;
  const float* hb = hs + (size_t)b * T * H;
  // pass 1: per-frame max and sum of exp (4 warps x 4 frames)
  for (int fi = wid; fi < GU_FT; fi += 4) {
    const float f = (float)(f0 + fi);
    float mx = -INFINITY;
    for (int t = lane; t < tlen; t += 32) {
      const float d = f - cb[t];
      mx = fmaxf(mx, -0.1f * (d * d));
    }
    mx = warp_max(mx);
    float sm = 0.f;
    for (int t = lane; t < tlen; t += 32) {
      const float d = f - cb[t];
      sm += expf(-0.1f * (d * d) - mx);
    }
    sm = warp_sum(sm);
    if (lane == 0) { s_max[fi] = mx; s_inv[fi] = 1.0f / sm; }
  }
  float acc[GU_FT][NC];
#pragma unroll
  for (int i = 0; i < GU_FT; ++i)
#pragma unroll
    for (int c = 0; c < NC; ++c) acc[i][c] = 0.f;
  __syncthreads();
  for (int tt = 0; tt < tlen; tt += GU_TT) {
    // weights of this token chunk
    for (int i = tid; i < GU_FT * GU_TT; i += 128) {
      const int fi = i / GU_TT, tj = i % GU_TT;
      const int t = tt + tj;
      float wv = 0.f;
      if (t < tlen) {
        const float d = (float)(f0 + fi) - cb[t];
        wv = expf(-0.1f * (d * d) - s_max[fi]) * s_inv[fi];
      }
      s_w[fi][tj] = wv;
    }
    for (int i = tid; i < GU_TT * H / 4; i += 128) {
      const int tj = i / (H / 4), c4 = i % (H / 4);
      const int t = tt + tj;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (t < tlen) v = *reinterpret_cast<const float4*>(hb + (size_t)t * H + c4 * 4);
      *reinterpret_cast<float4*>(&s_h[tj][c4 * 4]) = v;
    }
    __syncthreads();
#pragma unroll 4
    for (int tj = 0; tj < GU_TT; ++tj) {
      float hv[NC];
#pragma unroll
      for (int c = 0; c < NC; ++c) hv[c] = s_h[tj][tid + 128 * c];
#pragma unroll
      for (int i = 0; i < GU_FT; ++i) {
        const float wv = s_w[i][tj];
#pragma unroll
        for (int c = 0; c < NC; ++c) acc[i][c] = fmaf(wv, hv[c], acc[i][c]);
      }
    }
    __syncthreads();
  }
  const float a = (pe && alpha) ? *alpha : 0.f;
#pragma unroll
  for (int i = 0; i < GU_FT; ++i) {
    const int f = f0 + i;
    if (f >= F) continue;
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      const int ch = tid + 128 * c;
      float v = 0.f;
      if (f < flen) {
        v = acc[i][c];
        if (pe) v = __fadd_rn(v, __fmul_rn(a, pe[(size_t)f * H + ch]));
      }
      ob[(size_t)f * H + ch] = v;
    }
  }
}
int launch_gauss_upsample(const float* hs, const float* centers, const int32_t* lens, const int32_t* mel_lens,
                          int B, int T, int H, int F, int invariant, const float* pe, const float* alpha,
                          float* out, cudaStream_t st) {
  EV_CHECK_ARG(H % 128 == 0 && H <= 512, "gauss_upsample: H=%d", H);
  EV_CHECK_ARG(F > 0 && T > 0, "gauss_upsample: F=%d T=%d", F, T);
  EV_CHECK_ARG(B <= 65535, "gauss_upsample: B too large");
  const bool small = (long long)B * ((F + 15) / 16) < 2 * sm_count();
  const int ft = small ? 8 : 16;
  dim3 grid((F + ft - 1) / ft, B);
  auto k = small ? gauss_upsample_kernel<4, 8> : gauss_upsample_kernel<4, 16>;
  switch (H / 128) {
    case 1: k = small ? gauss_upsample_kernel<1, 8> : gauss_upsample_kernel<1, 16>; break;
    case 2: k = small ? gauss_upsample_kernel<2, 8> : gauss_upsample_kernel<2, 16>; break;
    case 3: k = small ? gauss_upsample_kernel<3, 8> : gauss_upsample_kernel<3, 16>; break;
  }
  return launch("gauss_upsample_kernel", k, grid, 128, 0, st, hs, centers, lens, mel_lens, T, F, invariant, pe, alpha, out);
}

}  // namespace ev
