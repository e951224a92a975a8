// Style encoder on the GPU (SURVEY.md s8f rank 1): the reference's StyleEncoder (simbert.py:33-72) is transformers'
// BertModel + pooler, run on the CPU twice per utterance by every caller (inference_am_vocoder_joint.py:25-38,106-107).
// This file holds its two small kernels (embedding sum + LayerNorm, the [CLS] GEMV with tanh), the context, weight
// resolution, launch sequencing and the ev_style_* C ABI.  The GEMMs run in conv1d_tc.cu (K = 1 convolutions, 3xTF32 on
// tensor cores by default), attention / LayerNorm in am_kernels.cu -- the kernels the acoustic model already uses.
//
// BertModel.forward restated (post-LN blocks; cited from the published architecture, the library is not vendored):
//   x = LN(word[id] + type[tt] + pos[t])
//   per layer:  a = x + Wo·Attn(x Wqkv + b) ;  x = LN(a) ;  f = x + W2·gelu_erf(W1 x + b1) + b2 ;  x = LN(f)
//   pooled = tanh(Wp x[0] + bp)             heads = Wc pooled + bc   (simbert.py:58-62)
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

#include "ev_common.cuh"

namespace ev {

__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---------------------------------------------------------------------------------------------
// BertEmbeddings: y[b,t,:] = LayerNorm( (word[ids[b,t]] + type[tt[b,t]]) + pos[t] ), eps 1e-12.
// One warp per token, the row lives in registers (C = NV*128 <= 768).
// ---------------------------------------------------------------------------------------------
template <int NV>
__global__ void __launch_bounds__(256) bert_embed_ln_kernel(const int64_t* __restrict__ ids, const int64_t* __restrict__ tts,
                                                             const float* __restrict__ word, const float* __restrict__ type,
                                                             const float* __restrict__ pos, const float* __restrict__ w,
                                                             const float* __restrict__ b, float* __restrict__ y, int rows, int N) {
  pdl_entry();
  constexpr int C = NV * 128;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const int t = row % N;
  const float* we = word + (size_t)ids[row] * C;
  const float* te = type + (size_t)tts[row] * C;
  const float* pe = pos + (size_t)t * C;
  float4 v[NV];
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    const int c = (lane + 32 * j) * 4;
    const float4 a = *reinterpret_cast<const float4*>(we + c);
    const float4 d = *reinterpret_cast<const float4*>(te + c);
    const float4 p = *reinterpret_cast<const float4*>(pe + c);
    v[j] = make_float4((a.x + d.x) + p.x, (a.y + d.y) + p.y, (a.z + d.z) + p.z, (a.w + d.w) + p.w);
  }
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < NV; ++j) s += (v[j].x + v[j].y) + (v[j].z + v[j].w);
  const float mean = warp_sum_f(s) / (float)C;
  float q = 0.f;
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    const float dx = v[j].x - mean, dy = v[j].y - mean, dz = v[j].z - mean, dw = v[j].w - mean;
    q += (dx * dx + dy * dy) + (dz * dz + dw * dw);
  }
  const float rstd = 1.0f / sqrtf(warp_sum_f(q) / (float)C + 1e-12f);
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

static int launch_bert_embed_ln(const int64_t* ids, const int64_t* tts, const float* word, const float* type, const float* pos,
                                const float* w, const float* b, float* y, int rows, int N, int C, cudaStream_t st) {
  EV_CHECK_ARG(rows > 0 && C % 128 == 0 && C <= 768, "bert_embed_ln: rows=%d C=%d (C must be a multiple of 128, <= 768)", rows, C);
  dim3 grid((rows + 7) / 8);
  auto k = bert_embed_ln_kernel<6>;
  switch (C / 128) {
    case 1: k = bert_embed_ln_kernel<1>; break;
    case 2: k = bert_embed_ln_kernel<2>; break;
    case 3: k = bert_embed_ln_kernel<3>; break;
    case 4: k = bert_embed_ln_kernel<4>; break;
    case 5: k = bert_embed_ln_kernel<5>; break;
  }
  return launch("bert_embed_ln_kernel", k, grid, 256, 0, st, ids, tts, word, type, pos, w, b, y, rows, N);
}

// ---------------------------------------------------------------------------------------------
// Skinny GEMV with an activation: out[b, n] = act( sum_k x[b*x_stride + k] * w[k*N + n] + bias[n] ).
// BertPooler (x = the [CLS] row of each item: stride N_tokens*H, tanh) and the classification heads (stride H, none).
// One CTA per (8 output columns, batch item); K is split over the CTA's threads and reduced in a fixed order.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) row_gemv_kernel(const float* __restrict__ x, size_t x_stride, const float* __restrict__ w,
                                                       const float* __restrict__ bias, float* __restrict__ out, int K, int N,
                                                       int act) {
  pdl_entry();
  __shared__ float red[8][8][33];
  const int b = blockIdx.y, n0 = blockIdx.x * 8;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  const float* xb = x + (size_t)b * x_stride;
  for (int k = tid; k < K; k += 256) {
    const float xv = xb[k];
    const float4 w0 = *reinterpret_cast<const float4*>(w + (size_t)k * N + n0);
    const float4 w1 = *reinterpret_cast<const float4*>(w + (size_t)k * N + n0 + 4);
    acc[0] = fmaf(xv, w0.x, acc[0]); acc[1] = fmaf(xv, w0.y, acc[1]); acc[2] = fmaf(xv, w0.z, acc[2]); acc[3] = fmaf(xv, w0.w, acc[3]);
    acc[4] = fmaf(xv, w1.x, acc[4]); acc[5] = fmaf(xv, w1.y, acc[5]); acc[6] = fmaf(xv, w1.z, acc[6]); acc[7] = fmaf(xv, w1.w, acc[7]);
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
    if (w8 == 0) out[(size_t)b * N + n0 + j] = act_apply(s + bias[n0 + j], act, 0.f);
  }
}

static int launch_row_gemv(const float* x, size_t x_stride, const float* w, const float* bias, float* out, int B, int K, int N,
                           int act, cudaStream_t st) {
  EV_CHECK_ARG(N % 8 == 0 && N > 0 && B > 0 && B <= 65535, "row_gemv: N=%d B=%d", N, B);
  dim3 grid(N / 8, B);
  return launch("row_gemv_kernel", row_gemv_kernel, grid, 256, 0, st, x, x_stride, w, bias, out, K, N, act);
}

struct StyleLayerW {
  const float *wqkv, *bqkv, *wo, *bo, *ln1w, *ln1b, *w1, *b1, *w2, *b2, *ln2w, *ln2b;   // w*: tensor-core layout, 2 planes
};

}  // namespace ev

struct ev_style_ctx {
  ev_style_config cfg;
  int device = 0;
  bool bound = false;
  int precision = EV_PREC_FP32;
  std::unordered_map<std::string, std::pair<const float*, uint64_t>> tensors;
  const float *word = nullptr, *pos = nullptr, *type = nullptr, *elnw = nullptr, *elnb = nullptr;
  std::vector<ev::StyleLayerW> layers;
  const float *pool_w = nullptr, *pool_b = nullptr, *heads_w = nullptr, *heads_b = nullptr;
};

namespace ev {

static int sfind(ev_style_ctx* c, const std::string& name, uint64_t expect, const float** out) {
  auto it = c->tensors.find(name);
  if (it == c->tensors.end()) { set_error("style weight '%s' missing from the bound blob", name.c_str()); return EV_ENOWEIGHT; }
  if (it->second.second != expect) {
    set_error("style weight '%s' has %llu elements, expected %llu", name.c_str(), (unsigned long long)it->second.second,
              (unsigned long long)expect);
    return EV_EINVAL;
  }
  *out = it->second.first;
  return EV_OK;
}

static inline size_t salign(size_t v) { return (v + 255) / 256 * 256; }

struct StyleBufs {
  float *x, *y, *qkv, *ctx, *h, *part, *pooled_tmp;
  int32_t* lens32;
  size_t part_cap, total;
};

// 256-byte aligned carve of the caller's workspace; base == nullptr only computes the size
static void carve_style(const ev_style_config& g, int B, int N, char* base, StyleBufs* o) {
  const size_t n = (size_t)B * N, H = g.hidden, I = g.intermediate;
  size_t off = 0;
  auto take = [&](size_t floats) {
    float* r = base ? reinterpret_cast<float*>(base + off) : nullptr;
    off += salign(floats * sizeof(float));
    return r;
  };
  o->x = take(n * H);
  o->y = take(n * H);
  o->qkv = take(n * 3 * H);
  o->ctx = take(n * H);
  o->h = take(n * I);
  const size_t widest = (2 * I > 4 * H ? 2 * I : 4 * H);      // split-K partials: 2 slices of the widest output (I) or 4 of H
  o->part_cap = n * (widest > 2 * 3 * H ? widest : 2 * 3 * H);
  o->part = take(o->part_cap);
  o->pooled_tmp = take((size_t)B * H);
  o->lens32 = reinterpret_cast<int32_t*>(take((size_t)B));
  o->total = off;
}

static int style_gemm(const ev_style_ctx* c, const float* x, const float* w_tc, const float* bias, const float* res, float* out,
                      int B, int N, int Cin, int Cout, int out_act, int ksplit, const int32_t* lens, const StyleBufs& bf,
                      cudaStream_t st) {
  ConvParams p;
  p.x = x; p.w = w_tc; p.bias = bias; p.res = res; p.out = out; p.bias_bs = 0;
  p.B = B; p.L = N; p.Cin = Cin; p.Cout = Cout; p.K = 1; p.dil = 1;
  p.lens = lens; p.lens_mul = 1; p.in_act = EV_ACT_NONE; p.in_slope = 0.f;
  p.out_act = out_act; p.acc = EV_ACC_STORE; p.div = 1.f;
  p.splitk_ws = bf.part; p.splitk_cap = bf.part_cap; p.ksplit = ksplit;      // fixed per layer: batch-invariant summation order
  return launch_conv1d_tc(p, c->precision == EV_PREC_TF32 ? 0 : 1, st);
}

}  // namespace ev

using namespace ev;

extern "C" {

int ev_style_create(ev_style_ctx** out, int device, const ev_style_config* cfg) {
  EV_CHECK_ARG(out && cfg, "ev_style_create: null argument");
  *out = nullptr;
  cudaDeviceProp prop;
  cudaError_t e = cudaGetDeviceProperties(&prop, device);
  if (e != cudaSuccess) { set_error("ev_style_create: cudaGetDeviceProperties(%d): %s", device, cudaGetErrorString(e)); return EV_ECUDA; }
  if (prop.major != 9) {
    set_error("ev_style_create: device %d is sm_%d%d; this library is built for sm_90a only", device, prop.major, prop.minor);
    return EV_EARCH;
  }
  const ev_style_config& g = *cfg;
  EV_CHECK_ARG(g.hidden > 0 && g.hidden % 128 == 0 && g.hidden <= 768, "style: hidden=%d must be a multiple of 128, <= 768", g.hidden);
  EV_CHECK_ARG(g.n_heads > 0 && g.hidden % g.n_heads == 0, "style: hidden=%d not divisible by n_heads=%d", g.hidden, g.n_heads);
  const int dk = g.hidden / g.n_heads;
  EV_CHECK_ARG(dk == 32 || dk == 48 || dk == 64, "style: head dim %d unsupported (32/48/64)", dk);
  EV_CHECK_ARG(g.intermediate > 0 && g.intermediate % 128 == 0, "style: intermediate=%d must be a multiple of 128", g.intermediate);
  EV_CHECK_ARG(g.n_layers > 0 && g.vocab_size > 0 && g.max_position > 0 && g.type_vocab > 0, "style: bad config");
  EV_CHECK_ARG(g.n_head_out >= 0 && g.n_head_out % 8 == 0, "style: n_head_out=%d must be a multiple of 8", g.n_head_out);
  ev_style_ctx* c = new ev_style_ctx();
  c->cfg = g;
  c->device = device;
  *out = c;
  return EV_OK;
}

void ev_style_destroy(ev_style_ctx* ctx) { delete ctx; }

int ev_style_bind_weights(ev_style_ctx* c, const float* blob, size_t blob_floats, const ev_weight_entry* index, int n_entries) {
  EV_CHECK_ARG(c && blob && index && n_entries > 0, "ev_style_bind_weights: null argument");
  c->bound = false;
  c->tensors.clear();
  for (int i = 0; i < n_entries; ++i) {
    const ev_weight_entry& e = index[i];
    EV_CHECK_ARG(e.offset + e.numel <= blob_floats, "ev_style_bind_weights: entry %d exceeds the blob", i);
    char name[57];
    memcpy(name, e.name, 56);
    name[56] = 0;
    c->tensors[name] = std::make_pair(blob + e.offset, e.numel);
  }
  const ev_style_config& g = c->cfg;
  const uint64_t H = g.hidden, I = g.intermediate;
  EV_TRY(sfind(c, "sty.emb.word", (uint64_t)g.vocab_size * H, &c->word));
  EV_TRY(sfind(c, "sty.emb.pos", (uint64_t)g.max_position * H, &c->pos));
  EV_TRY(sfind(c, "sty.emb.type", (uint64_t)g.type_vocab * H, &c->type));
  EV_TRY(sfind(c, "sty.emb.ln.w", H, &c->elnw));
  EV_TRY(sfind(c, "sty.emb.ln.b", H, &c->elnb));
  c->layers.resize(g.n_layers);
  for (int i = 0; i < g.n_layers; ++i) {
    const std::string q = "sty." + std::to_string(i);
    StyleLayerW& l = c->layers[i];
    EV_TRY(sfind(c, q + ".wqkv.tc", 2 * H * 3 * H, &l.wqkv));
    EV_TRY(sfind(c, q + ".bqkv", 3 * H, &l.bqkv));
    EV_TRY(sfind(c, q + ".wo.tc", 2 * H * H, &l.wo));
    EV_TRY(sfind(c, q + ".bo", H, &l.bo));
    EV_TRY(sfind(c, q + ".ln1.w", H, &l.ln1w));
    EV_TRY(sfind(c, q + ".ln1.b", H, &l.ln1b));
    EV_TRY(sfind(c, q + ".w1.tc", 2 * H * I, &l.w1));
    EV_TRY(sfind(c, q + ".b1", I, &l.b1));
    EV_TRY(sfind(c, q + ".w2.tc", 2 * I * H, &l.w2));
    EV_TRY(sfind(c, q + ".b2", H, &l.b2));
    EV_TRY(sfind(c, q + ".ln2.w", H, &l.ln2w));
    EV_TRY(sfind(c, q + ".ln2.b", H, &l.ln2b));
  }
  EV_TRY(sfind(c, "sty.pool.w", H * H, &c->pool_w));
  EV_TRY(sfind(c, "sty.pool.b", H, &c->pool_b));
  if (g.n_head_out > 0) {
    EV_TRY(sfind(c, "sty.heads.w", H * (uint64_t)g.n_head_out, &c->heads_w));
    EV_TRY(sfind(c, "sty.heads.b", (uint64_t)g.n_head_out, &c->heads_b));
  }
  c->bound = true;
  return EV_OK;
}

int ev_style_set_precision(ev_style_ctx* c, int precision) {
  EV_CHECK_ARG(c, "ev_style_set_precision: null context");
  EV_CHECK_ARG(precision == EV_PREC_FP32 || precision == EV_PREC_TF32, "ev_style_set_precision: %d (EV_PREC_FP32 or EV_PREC_TF32)", precision);
  c->precision = precision;
  return EV_OK;
}

size_t ev_style_workspace_bytes(const ev_style_ctx* c, int B, int N) {
  if (!c || B <= 0 || N <= 0) return 0;
  StyleBufs bf;
  carve_style(c->cfg, B, N, nullptr, &bf);
  return bf.total;
}

int ev_style_forward(ev_style_ctx* c, const int64_t* ids, const int64_t* type_ids, const int64_t* lens, int B, int N,
                     float* pooled, float* heads, void* workspace, size_t workspace_bytes, void* stream) {
  EV_CHECK_ARG(c && c->bound, "ev_style_forward: weights are not bound");
  EV_CHECK_ARG(ids && type_ids && lens && pooled && workspace, "ev_style_forward: null argument");
  EV_CHECK_ARG(B > 0 && N > 0, "ev_style_forward: B=%d N=%d", B, N);
  const ev_style_config& g = c->cfg;
  EV_CHECK_ARG(N <= g.max_position, "ev_style_forward: %d tokens exceed max_position_embeddings=%d", N, g.max_position);
  EV_CHECK_ARG(heads == nullptr || g.n_head_out > 0, "ev_style_forward: heads requested but the context has none");
  EV_CHECK_ARG(((uintptr_t)workspace & 255) == 0, "ev_style_forward: workspace must be 256-byte aligned");
  StyleBufs bf;
  carve_style(g, B, N, reinterpret_cast<char*>(workspace), &bf);
  if (bf.total > workspace_bytes) { set_error("ev_style_forward: workspace %zu < %zu bytes", workspace_bytes, bf.total); return EV_EWORKSPACE; }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int H = g.hidden, I = g.intermediate, rows = B * N;
  {   // kernels and function attributes belong to the context's device, whatever device is current for the calling thread
    int cur = -1;
    cudaError_t e = cudaGetDevice(&cur);
    if (e == cudaSuccess && cur != c->device) e = cudaSetDevice(c->device);
    if (e != cudaSuccess) { set_error("ev_style_forward: cudaSetDevice(%d): %s", c->device, cudaGetErrorString(e)); return EV_ECUDA; }
  }
  EV_TRY(launch_validate_inputs(nullptr, lens, nullptr, bf.lens32, nullptr, B, N, 0, 0, st));
  EV_TRY(launch_bert_embed_ln(ids, type_ids, c->word, c->type, c->pos, c->elnw, c->elnb, bf.x, rows, N, H, st));
  for (int i = 0; i < g.n_layers; ++i) {
    const StyleLayerW& l = c->layers[i];
    EV_TRY(style_gemm(c, bf.x, l.wqkv, l.bqkv, nullptr, bf.qkv, B, N, H, 3 * H, EV_ACT_NONE, 2, bf.lens32, bf, st));
    EV_TRY(launch_attention(bf.qkv, bf.lens32, bf.ctx, B, N, H, g.n_heads, st));
    EV_TRY(style_gemm(c, bf.ctx, l.wo, l.bo, bf.x, bf.y, B, N, H, H, EV_ACT_NONE, 2, bf.lens32, bf, st));        // + residual
    EV_TRY(launch_layernorm(bf.y, nullptr, nullptr, nullptr, nullptr, nullptr, l.ln1w, l.ln1b, bf.x, rows, N, H, st));
    EV_TRY(style_gemm(c, bf.x, l.w1, l.b1, nullptr, bf.h, B, N, H, I, EV_ACT_GELU, 2, bf.lens32, bf, st));
    EV_TRY(style_gemm(c, bf.h, l.w2, l.b2, bf.x, bf.y, B, N, I, H, EV_ACT_NONE, 4, bf.lens32, bf, st));          // + residual
    EV_TRY(launch_layernorm(bf.y, nullptr, nullptr, nullptr, nullptr, nullptr, l.ln2w, l.ln2b, bf.x, rows, N, H, st));
  }
  EV_TRY(launch_row_gemv(bf.x, (size_t)N * H, c->pool_w, c->pool_b, pooled, B, H, H, EV_ACT_TANH, st));           // BertPooler on [CLS]
  if (heads) EV_TRY(launch_row_gemv(pooled, (size_t)H, c->heads_w, c->heads_b, heads, B, H, g.n_head_out, EV_ACT_NONE, st));
  return EV_OK;
}

int ev_op_bert_embed_ln(const int64_t* ids, const int64_t* type_ids, const float* word, const float* type, const float* pos, const float* w,
                        const float* b, float* y, int rows, int N, int C, void* stream) {
  EV_CHECK_ARG(ids && type_ids && word && type && pos && w && b && y, "ev_op_bert_embed_ln: null argument");
  EV_CHECK_ARG(N > 0, "ev_op_bert_embed_ln: N=%d", N);
  EV_TRY(use_device_of(word));
  return launch_bert_embed_ln(ids, type_ids, word, type, pos, w, b, y, rows, N, C, reinterpret_cast<cudaStream_t>(stream));
}

int ev_op_row_gemv(const float* x, size_t x_stride, const float* w, const float* bias, float* out, int B, int K, int N, int act,
                   void* stream) {
  EV_CHECK_ARG(x && w && bias && out, "ev_op_row_gemv: null argument");
  EV_CHECK_ARG(K > 0 && (act == EV_ACT_NONE || act == EV_ACT_TANH), "ev_op_row_gemv: K=%d act=%d", K, act);
  EV_TRY(use_device_of(x));
  return launch_row_gemv(x, x_stride, w, bias, out, B, K, N, act, reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
