// libemotivoice_b200.so -- context, weight binding, layer orchestration and the C ABI
// (include/emotivoice_b200.h).  All math runs in the hand-written sm_90a kernels of
// conv1d_tm.cu / am_kernels.cu / voc_kernels.cu; this file only sequences launches on the
// caller's stream and carves the caller-provided workspace.
#include <atomic>
#include <cstdarg>
#include <cstdlib>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

#include <nvtx3/nvToolsExt.h>

#include "ev_common.cuh"

namespace ev {

// NVTX range per stage of the path (SURVEY.md s5: the reference has no tracing at all).  Costs nothing without a tool attached;
// with one, `ncu --nvtx --nvtx-include "voc:stage1/"` selects the kernels of a stage.  Popped on every return path.
struct Range {
  explicit Range(const char* name) { nvtxRangePushA(name); }
  ~Range() { nvtxRangePop(); }
  Range(const Range&) = delete;
  Range& operator=(const Range&) = delete;
};

static thread_local std::string g_err;
static std::atomic<uint64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
}
void count_launch(int n) { g_launches.fetch_add((uint64_t)n, std::memory_order_relaxed); }
int sm_count() {
  static std::atomic<int> cache[64];
  int dev = 0;
  cudaGetDevice(&dev);
  int n = cache[dev & 63].load(std::memory_order_relaxed);
  if (n == 0) {
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
    cache[dev & 63].store(n, std::memory_order_relaxed);
  }
  return n;
}
int use_device_of(const void* dev_ptr) {
  cudaPointerAttributes at;
  cudaError_t e = cudaPointerGetAttributes(&at, dev_ptr);
  if (e == cudaSuccess && at.type != cudaMemoryTypeDevice && at.type != cudaMemoryTypeManaged) {
    set_error("pointer %p is not device memory (there is no CPU path in this library)", dev_ptr);
    return EV_EINVAL;
  }
  int cur = -1;
  if (e == cudaSuccess) e = cudaGetDevice(&cur);
  if (e == cudaSuccess && cur != at.device) e = cudaSetDevice(at.device);
  if (e != cudaSuccess) { set_error("selecting the device of %p: %s", dev_ptr, cudaGetErrorString(e)); cudaGetLastError(); return EV_ECUDA; }
  return EV_OK;
}
bool pdl_enabled() {
  static const bool v = [] { const char* e = getenv("EV_PDL"); return !(e && strcmp(e, "0") == 0); }();
  return v;
}

struct Tensor {
  const float* p = nullptr;
  uint64_t numel = 0;
};

// The weights of one GEMM-shaped layer: the plain fp32 copy (K, C_in, C_out) the FFMA kernels read, and the tensor-core copies
// packing.add_tc_weights adds: '.tc' (two tf32 planes), '.tc16' (bf16), '.tc16x2' (two bf16 planes).  A copy the blob lacks is null.
struct GemmW {
  const float *w = nullptr, *tc = nullptr, *tc16 = nullptr, *tc16x2 = nullptr;
};
struct EncLayerW {
  const float *ln1w, *ln1b, *bqkv, *bo, *ln2w, *ln2b, *b1, *b2;
  GemmW wqkv, wo, w1, w2;
};
struct StackW {
  const float* alpha;
  std::vector<EncLayerW> layers;
  const float *lnfw, *lnfb;
};
struct PredW {
  std::vector<GemmW> w;
  std::vector<const float*> b, lnw, lnb;
  const float *linw, *linb;
};
struct ConvW {
  GemmW w;
  const float* b;
  int K, dil, cin, cout;
};
struct UpW {
  GemmW w;
  const float* b;
  int K, cin, cout_packed, rate, cout;
};

}  // namespace ev

struct ev_ctx {
  ev_config cfg;
  int device = 0;
  bool bound = false;
  bool has_am = false, has_voc = false;
  int precision = EV_PREC_FP32;
  std::unordered_map<std::string, ev::Tensor> tensors;
  const float* pe = nullptr;
  int pe_len = 0;
  // resolved weights
  const float *emb_word = nullptr, *emb_spk = nullptr;
  ev::StackW enc, dec;
  ev::GemmW cond_wx;
  const float *cond_wc, *cond_b;
  ev::PredW dur, pitch, energy;
  const float *pemb_w, *pemb_b, *eemb_w, *eemb_b;
  ev::GemmW mel_w;
  const float* mel_b;
  ev::ConvW pre;
  std::vector<ev::UpW> ups;
  std::vector<ev::ConvW> rb_c1, rb_c2;   // [(stage*n_resk + j)*n_dil + l]
  const float *post_w, *post_b;
  int post_k = 7;
  int total_up = 1;
  int max_stage_width = 0;   // max over stages of prod(rates so far) * channels
};

namespace ev {

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// bump allocator over the caller's workspace (counts in floats, 256-byte aligned blocks)
struct Carver {
  char* base;
  size_t off = 0;
  explicit Carver(void* p) : base(reinterpret_cast<char*>(p)) {}
  float* take(size_t n_floats) {
    float* r = reinterpret_cast<float*>(base + off);
    off += align_up(n_floats * sizeof(float), 256);
    return r;
  }
};

struct Phase1Bufs {
  float *x, *y, *qkv, *ctx, *h, *cond_in, *cond_bias, *hs, *pm, *p1[3], *p2[3], *centers, *ds_f, *part;
  size_t part_cap;
};
struct Phase2Bufs {
  float *x, *y, *qkv, *ctx, *h, *part;
  size_t part_cap;
};
struct VocBufs {
  float *X, *ACC;
  float *Tm, *R1, *R2;   // ResBlock chain scratch
  float *G0, *G1, *G2;   // small batches only: the three parallel ResBlocks of a stage advance together (grouped launches)
};

static void carve_phase1(const ev_ctx* c, Carver& cv, int B, int T, Phase1Bufs* o) {
  const size_t H = c->cfg.hidden, n = (size_t)B * T;
  o->x = cv.take(n * H);
  o->y = cv.take(n * H);
  o->qkv = cv.take(n * 3 * H);
  o->ctx = cv.take(n * H);
  o->h = cv.take(n * 4 * H);
  o->cond_in = cv.take((size_t)B * (H + 2 * c->cfg.bert_dim));
  o->cond_bias = cv.take((size_t)B * H);
  o->hs = cv.take(n * H);
  o->pm = cv.take(n * H);
  for (int i = 0; i < 3; ++i) { o->p1[i] = cv.take(n * H); o->p2[i] = cv.take(n * H); }
  o->centers = cv.take(n);
  o->ds_f = cv.take(n);
  o->part_cap = 8 * n * 4 * H;          // split-K partials: up to 8 slices of the widest GEMM output (4H)
  o->part = cv.take(o->part_cap);
}
static void carve_phase2(const ev_ctx* c, Carver& cv, int B, int F, Phase2Bufs* o) {
  const size_t H = c->cfg.hidden, n = (size_t)B * F;
  o->x = cv.take(n * H);
  o->y = cv.take(n * H);
  o->qkv = cv.take(n * 3 * H);
  o->ctx = cv.take(n * H);
  o->h = cv.take(n * 4 * H);
  o->part_cap = 8 * n * 4 * H;
  o->part = cv.take(o->part_cap);
}
// Grouped launches (one kernel for the same-index convolutions of the three parallel ResBlocks of a stage) need three more stage-sized
// buffers; they only pay while one convolution has too few tiles for the machine, i.e. up to a few thousand batch-frames.
static inline bool voc_group_frames(int B, int F) {
  static const int v = [] { const char* e = getenv("EV_VOC_GROUP"); return (e && e[0] == '0') ? 0 : 1; }();
  return v == 1 && (long long)B * F <= 2400;
}
static void carve_voc(const ev_ctx* c, Carver& cv, int B, int F, VocBufs* o) {
  const size_t n = (size_t)B * F * (size_t)c->max_stage_width;
  o->X = cv.take(n);
  o->ACC = cv.take(n);
  o->Tm = cv.take(n);
  o->R1 = cv.take(n);
  o->R2 = cv.take(n);
  o->G0 = o->G1 = o->G2 = nullptr;
  if (voc_group_frames(B, F)) { o->G0 = cv.take(n); o->G1 = cv.take(n); o->G2 = cv.take(n); }
}

static int find(ev_ctx* c, const std::string& name, uint64_t expect, const float** out) {
  auto it = c->tensors.find(name);
  if (it == c->tensors.end()) {
    set_error("weight '%s' missing from the bound blob", name.c_str());
    return EV_ENOWEIGHT;
  }
  if (expect && it->second.numel != expect) {
    set_error("weight '%s' has %llu elements, expected %llu", name.c_str(), (unsigned long long)it->second.numel,
              (unsigned long long)expect);
    return EV_EINVAL;
  }
  *out = it->second.p;
  return EV_OK;
}

static const float* find_opt(ev_ctx* c, const std::string& name, uint64_t expect) {
  auto it = c->tensors.find(name);
  if (it == c->tensors.end() || it->second.numel != expect) return nullptr;
  return it->second.p;
}

// the plain weight `name` of n elements, and whichever tensor-core copies of it the blob carries
static int find_gemm(ev_ctx* c, const std::string& name, uint64_t n, GemmW* o) {
  EV_TRY(find(c, name, n, &o->w));
  o->tc = find_opt(c, name + ".tc", 2 * n);
  o->tc16 = find_opt(c, name + ".tc16", n / 2);
  o->tc16x2 = find_opt(c, name + ".tc16x2", n);
  return EV_OK;
}

static int resolve_stack(ev_ctx* c, const char* pre, int n_layers, StackW* s) {
  const uint64_t H = c->cfg.hidden, K = c->cfg.ffn_kernel;
  std::string p(pre);
  EV_TRY(find(c, p + ".alpha", 1, &s->alpha));
  s->layers.resize(n_layers);
  for (int i = 0; i < n_layers; ++i) {
    std::string q = p + "." + std::to_string(i);
    EncLayerW& l = s->layers[i];
    EV_TRY(find(c, q + ".ln1.w", H, &l.ln1w));
    EV_TRY(find(c, q + ".ln1.b", H, &l.ln1b));
    EV_TRY(find_gemm(c, q + ".wqkv", H * 3 * H, &l.wqkv));
    EV_TRY(find(c, q + ".bqkv", 3 * H, &l.bqkv));
    EV_TRY(find_gemm(c, q + ".wo", H * H, &l.wo));
    EV_TRY(find(c, q + ".bo", H, &l.bo));
    EV_TRY(find(c, q + ".ln2.w", H, &l.ln2w));
    EV_TRY(find(c, q + ".ln2.b", H, &l.ln2b));
    EV_TRY(find_gemm(c, q + ".w1", K * H * 4 * H, &l.w1));
    EV_TRY(find(c, q + ".b1", 4 * H, &l.b1));
    EV_TRY(find_gemm(c, q + ".w2", K * 4 * H * H, &l.w2));
    EV_TRY(find(c, q + ".b2", H, &l.b2));
  }
  EV_TRY(find(c, p + ".lnf.w", H, &s->lnfw));
  EV_TRY(find(c, p + ".lnf.b", H, &s->lnfb));
  return EV_OK;
}

static int resolve_pred(ev_ctx* c, const char* pre, int n_layers, PredW* s) {
  const uint64_t H = c->cfg.hidden, K = c->cfg.pred_kernel;
  std::string p(pre);
  s->w.resize(n_layers); s->b.resize(n_layers); s->lnw.resize(n_layers); s->lnb.resize(n_layers);
  for (int i = 0; i < n_layers; ++i) {
    std::string q = p + "." + std::to_string(i);
    EV_TRY(find_gemm(c, q + ".w", K * H * H, &s->w[i]));
    EV_TRY(find(c, q + ".b", H, &s->b[i]));
    EV_TRY(find(c, q + ".ln.w", H, &s->lnw[i]));
    EV_TRY(find(c, q + ".ln.b", H, &s->lnb[i]));
  }
  EV_TRY(find(c, p + ".lin.w", H, &s->linw));
  EV_TRY(find(c, p + ".lin.b", 1, &s->linb));
  return EV_OK;
}

static int resolve_voc(ev_ctx* c);

static int resolve_all(ev_ctx* c) {
  c->has_am = c->tensors.count("emb.word") != 0;
  c->has_voc = c->tensors.count("voc.pre.w") != 0;
  if (!c->has_am && !c->has_voc) {
    set_error("ev_bind_weights: blob holds neither the acoustic model ('emb.word') nor the vocoder ('voc.pre.w')");
    return EV_ENOWEIGHT;
  }
  if (c->has_voc) EV_TRY(resolve_voc(c));
  if (!c->has_am) return EV_OK;
  const ev_config& g = c->cfg;
  const uint64_t H = g.hidden;
  EV_TRY(find(c, "emb.word", (uint64_t)g.n_vocab * H, &c->emb_word));
  EV_TRY(find(c, "emb.spk", (uint64_t)g.n_speaker * H, &c->emb_spk));
  EV_TRY(resolve_stack(c, "enc", g.enc_layers, &c->enc));
  EV_TRY(resolve_stack(c, "dec", g.dec_layers, &c->dec));
  EV_TRY(find_gemm(c, "cond.wx", H * H, &c->cond_wx));
  EV_TRY(find(c, "cond.wc", (H + 2 * (uint64_t)g.bert_dim) * H, &c->cond_wc));
  EV_TRY(find(c, "cond.b", H, &c->cond_b));
  EV_TRY(resolve_pred(c, "dur", g.dur_layers, &c->dur));
  EV_TRY(resolve_pred(c, "pitch", g.pitch_layers, &c->pitch));
  EV_TRY(resolve_pred(c, "energy", g.energy_layers, &c->energy));
  EV_TRY(find(c, "pitch_emb.w", (uint64_t)g.embed_kernel * H, &c->pemb_w));
  EV_TRY(find(c, "pitch_emb.b", H, &c->pemb_b));
  EV_TRY(find(c, "energy_emb.w", (uint64_t)g.embed_kernel * H, &c->eemb_w));
  EV_TRY(find(c, "energy_emb.b", H, &c->eemb_b));
  EV_TRY(find_gemm(c, "to_mel.w", H * g.n_mels, &c->mel_w));
  EV_TRY(find(c, "to_mel.b", g.n_mels, &c->mel_b));
  return EV_OK;
}

static int resolve_voc(ev_ctx* c) {
  const ev_config& g = c->cfg;
  c->pre.K = 7; c->pre.dil = 1; c->pre.cin = g.n_mels; c->pre.cout = g.voc_c0;
  EV_TRY(find_gemm(c, "voc.pre.w", (uint64_t)7 * g.n_mels * g.voc_c0, &c->pre.w));
  EV_TRY(find(c, "voc.pre.b", g.voc_c0, &c->pre.b));
  c->ups.resize(g.n_ups);
  c->rb_c1.clear(); c->rb_c2.clear();
  int ch = g.voc_c0, mul = 1;
  c->max_stage_width = g.voc_c0;
  for (int s = 0; s < g.n_ups; ++s) {
    UpW& u = c->ups[s];
    u.rate = g.up_rates[s]; u.cin = ch; u.cout = ch / 2; u.cout_packed = u.cout * u.rate;
    std::string q = "voc.up." + std::to_string(s);
    auto it = c->tensors.find(q + ".w");
    if (it == c->tensors.end()) { set_error("weight '%s.w' missing", q.c_str()); return EV_ENOWEIGHT; }
    const uint64_t per_tap = (uint64_t)u.cin * u.cout_packed;
    if (it->second.numel % per_tap != 0 || ((it->second.numel / per_tap) & 1) == 0) {
      set_error("weight '%s.w': %llu elements is not an odd number of (%d x %d) taps", q.c_str(),
                (unsigned long long)it->second.numel, u.cin, u.cout_packed);
      return EV_EINVAL;
    }
    u.K = (int)(it->second.numel / per_tap);
    EV_TRY(find_gemm(c, q + ".w", it->second.numel, &u.w));
    EV_TRY(find(c, q + ".b", u.cout_packed, &u.b));
    ch = u.cout; mul *= u.rate;
    if (mul * ch > c->max_stage_width) c->max_stage_width = mul * ch;
    for (int j = 0; j < g.n_resk; ++j)
      for (int l = 0; l < g.n_dil; ++l) {
        const int k = g.res_kernels[j];
        std::string r = "voc.rb." + std::to_string(s * g.n_resk + j);
        ConvW c1, c2;
        c1.K = k; c1.dil = g.res_dils[j][l]; c1.cin = ch; c1.cout = ch;
        c2.K = k; c2.dil = 1; c2.cin = ch; c2.cout = ch;
        EV_TRY(find_gemm(c, r + ".c1." + std::to_string(l) + ".w", (uint64_t)k * ch * ch, &c1.w));
        EV_TRY(find(c, r + ".c1." + std::to_string(l) + ".b", ch, &c1.b));
        EV_TRY(find_gemm(c, r + ".c2." + std::to_string(l) + ".w", (uint64_t)k * ch * ch, &c2.w));
        EV_TRY(find(c, r + ".c2." + std::to_string(l) + ".b", ch, &c2.b));
        c->rb_c1.push_back(c1); c->rb_c2.push_back(c2);
      }
  }
  c->total_up = mul;
  c->post_k = 7;
  EV_TRY(find(c, "voc.post.w", (uint64_t)7 * ch, &c->post_w));
  EV_TRY(find(c, "voc.post.b", 1, &c->post_b));
  return EV_OK;
}

static ConvParams conv_params(const float* x, const float* w, const float* bias, long long bias_bs, const float* res, float* out,
                              int B, int L, int Cin, int Cout, int K, int dil, const int32_t* lens, int lens_mul, int in_act,
                              float in_slope, int out_act, int acc, float div) {
  ConvParams p;
  p.x = x; p.w = w; p.bias = bias; p.res = res; p.out = out; p.bias_bs = bias_bs;
  p.B = B; p.L = L; p.Cin = Cin; p.Cout = Cout; p.K = K; p.dil = dil;
  p.lens = lens; p.lens_mul = lens_mul; p.in_act = in_act; p.in_slope = in_slope;
  p.out_act = out_act; p.acc = acc; p.div = div;
  return p;
}
// the fp32 FFMA kernel on time-major activations (conv1d_tm.cu)
static int conv(const float* x, const float* w, const float* bias, long long bias_bs, const float* res, float* out,
                int B, int L, int Cin, int Cout, int K, int dil, const int32_t* lens, int lens_mul, int in_act,
                float in_slope, int out_act, int acc, float div, cudaStream_t st) {
  return launch_conv1d(conv_params(x, w, bias, bias_bs, res, out, B, L, Cin, Cout, K, dil, lens, lens_mul, in_act, in_slope, out_act,
                                   acc, div), st);
}

static GpConvParams gp_params(const float* w, const void* x, const float* bias, const void* res, void* out, int B, int L, int Cin,
                              int Cout, int K, int dil, int rate, const int32_t* lens, int lens_mul, int in_act, float in_slope, int acc,
                              float div) {
  GpConvParams p;
  p.x = x; p.w = w; p.bias = bias; p.res = res; p.out = out;
  p.B = B; p.L = L; p.Cin = Cin; p.Cout = Cout; p.K = K; p.dil = dil; p.rate = rate;
  p.lens = lens; p.lens_mul = lens_mul; p.in_act = in_act; p.in_slope = in_slope; p.acc = acc; p.div = div;
  return p;
}

// Kernel MODEs of the tensor-core kernels (conv1d_tc.cu, conv1d_gp.cu, resblock_gp.cu): 0 = 1xTF32, 1 = 3xTF32, 2 = bf16 (bf16
// activations in the vocoder), 3 = bf16x3.  kFfma: the fp32 FFMA kernels on the plain weights.
enum { kFfma = -1 };
static const char* const kModeCopy[4] = {".tc", ".tc", ".tc16", ".tc16x2"};   // the weight copy each MODE reads
struct LayerRun {
  const float* w;      // null when the blob lacks the copy
  int mode;
};

// The one place a precision becomes arithmetic.  The duration-critical prefix (encoder, cond.wx, predictors) is fp32-accurate in every
// precision: 3xTF32, or FFMA in "fp32_ffma".  The decoder, to_mel and the vocoder run bf16x3 / 1xTF32 / bf16 / FFMA in "fp32" /
// "tf32" / "bf16" / "fp32_ffma".
static LayerRun layer_run(const GemmW& l, int precision, bool prefix) {
  if (precision == EV_PREC_FP32_FFMA) return {l.w, kFfma};
  if (prefix) return {l.tc, 1};
  if (precision == EV_PREC_TF32) return {l.tc, 0};
  if (precision == EV_PREC_BF16) return {l.tc16, 2};
  return {l.tc16x2, 3};
}

// EV_ENOWEIGHT unless every bound layer has the copy `precision` runs it on (blobs from packing.add_tc_weights carry all of them)
static int check_weights(const ev_ctx* c, int precision, const char* who) {
  int missing = -1;      // the MODE of the first layer without its copy
  auto need = [&](const GemmW& l, bool prefix) {
    const LayerRun r = layer_run(l, precision, prefix);
    if (!r.w && missing < 0) missing = r.mode;
  };
  if (c->has_am) {
    for (const EncLayerW& l : c->enc.layers) { need(l.wqkv, true); need(l.wo, true); need(l.w1, true); need(l.w2, true); }
    need(c->cond_wx, true);
    for (const PredW* p : {&c->dur, &c->pitch, &c->energy})
      for (const GemmW& w : p->w) need(w, true);
    for (const EncLayerW& l : c->dec.layers) { need(l.wqkv, false); need(l.wo, false); need(l.w1, false); need(l.w2, false); }
    need(c->mel_w, false);
  }
  if (c->has_voc) {
    need(c->pre.w, false);
    for (const UpW& u : c->ups) need(u.w, false);
    for (const ConvW& w : c->rb_c1) need(w.w, false);
    for (const ConvW& w : c->rb_c2) need(w.w, false);
  }
  if (missing < 0) return EV_OK;
  set_error("%s: precision %d needs the '%s' weight copies, which the bound blob lacks", who, precision, kModeCopy[missing]);
  return EV_ENOWEIGHT;
}

// split-K scratch of a phase, carved from its workspace
struct SplitWs {
  float* p;
  size_t cap;      // floats
};

// One GEMM-shaped layer of the acoustic model (a convolution over time; K = 1 is a linear layer) on the kernel layer_run picks.
// ksplit: the layer's K-split factor on the tensor cores (conv1d_tc.cu), with the phase's scratch ws.
static int conv_x(const ev_ctx* c, const GemmW& l, bool prefix, int ksplit, const SplitWs& ws, const float* x, const float* bias,
                  long long bias_bs, const float* res, float* out, int B, int L, int Cin, int Cout, int K, const int32_t* lens,
                  int out_act, cudaStream_t st) {
  const LayerRun r = layer_run(l, c->precision, prefix);
  ConvParams p = conv_params(x, r.w, bias, bias_bs, res, out, B, L, Cin, Cout, K, 1, lens, 1, EV_ACT_NONE, 0.f, out_act, EV_ACC_STORE, 1.f);
  if (r.mode == kFfma) return launch_conv1d(p, st);
  p.splitk_ws = ws.p; p.splitk_cap = ws.cap; p.ksplit = ksplit;
  return launch_conv1d_tc(p, r.mode, st);
}

// One ResBlock layer through the fused kernel (resblock_gp.cu) where it takes the shape (C <= 128); EV_FUSE_RES=0 keeps two launches.
static inline bool fuse_res_enabled() {
  static const int v = [] { const char* e = getenv("EV_FUSE_RES"); return (e && e[0] == '0') ? 0 : 1; }();
  return v == 1;
}
// Fused and unfused are bitwise equal, so the choice may depend on the batch: measured (profiles/r02_fused_vs_unfused.jsonl) the fused
// layer wins 1.1-1.8x on the HBM-bound shapes (k <= 7, or 32 channels) and wherever the launch count matters (batch 1), and loses
// ~25 % on 64 channels x 11 taps once the batch is large enough to be tensor / issue bound.
static bool fuse_layer(const GpPairParams& p, int mode) {
  if (!fuse_res_enabled() || (p.C >= 64 && p.K > 7 && (long long)p.B * p.L > 4ll * 70000)) return false;
  return gp_pair_supported(p, mode);
}

// One (block j, layer l) step of a stage's ResBlocks, xt = c1(lrelu(x)); x = c2(lrelu(xt)) + x (hifigan/models.py:50-57): one fused
// launch where the shape takes it, else two.
struct ResStep {
  bool fused;
  GpPairParams pair;     // fused
  GpConvParams c1, c2;   // unfused
  void *in, *out;        // where the step reads x and where it leaves it
};

// A stage's buffers: X, its input, which no step writes; ACC, its output xs; and two buffers A[j], I[j] per block.  A grouped stage
// gives every block its own; run one step after another, all blocks share R1 and Tm.
struct StageBufs {
  void *X, *ACC;
  void *A[4], *I[4];
};

// Step (j, l) of a stage with layer input s (X at l = 0):
//   * a fused layer writes s == A ? I : A (the fused kernel's output must not alias its input);
//   * an unfused layer runs c1 into s == I ? A : I (never its own input), then c2 into s in place -- each residual element is read by
//     the thread that overwrites it -- or into A when s is X;
//   * to_acc: the last layer writes ACC instead, in block order xs = x_0, xs += x_j, xs = (xs + x_J-1) / J (:120-126).
static ResStep res_step(const ev_ctx* ctx, const StageBufs& b, size_t rb0, int j, int l, void* s, bool to_acc, int B, int L, int C,
                        const int32_t* lens, int mul) {
  const int J = ctx->cfg.n_resk;
  const ConvW& w1 = ctx->rb_c1[rb0 + (size_t)j * ctx->cfg.n_dil + l];
  const ConvW& w2 = ctx->rb_c2[rb0 + (size_t)j * ctx->cfg.n_dil + l];
  const LayerRun r1 = layer_run(w1.w, ctx->precision, false), r2 = layer_run(w2.w, ctx->precision, false);
  const int acc = (!to_acc || j == 0) ? EV_ACC_STORE : (j == J - 1 ? EV_ACC_ADD_DIV : EV_ACC_ADD);
  void *A = b.A[j], *I = b.I[j];
  ResStep st{};
  st.in = s;
  st.pair = GpPairParams{s, r1.w, w1.b, r2.w, w2.b, to_acc ? b.ACC : (s == A ? I : A), B, L, C, w1.K, w1.dil, lens, mul, 0.1f, acc, (float)J};
  st.fused = fuse_layer(st.pair, r1.mode);
  if (st.fused) {
    st.out = st.pair.out;
    return st;
  }
  void* t = (s == I) ? A : I;
  st.out = to_acc ? b.ACC : (s == b.X ? A : s);
  st.c1 = gp_params(r1.w, s, w1.b, nullptr, t, B, L, C, C, w1.K, w1.dil, 1, lens, mul, EV_ACT_LRELU, 0.1f, EV_ACC_STORE, 1.f);
  st.c2 = gp_params(r2.w, t, w2.b, s, st.out, B, L, C, C, w2.K, 1, 1, lens, mul, EV_ACT_LRELU, 0.1f, acc, (float)J);
  return st;
}

// the members of one layer of a grouped stage, side by side as the grouped launches take them
struct LayerGroup {
  GpPairParams pair[3];
  GpConvParams c1[3], c2[3];
  LayerGroup(const ResStep* m, int J) {
    for (int j = 0; j < J; ++j) { pair[j] = m[j].pair; c1[j] = m[j].c1; c2[j] = m[j].c2; }
  }
};

// Grouping pays while one convolution has fewer than two waves of tiles (batch 1: 68 / 135 tiles on 132 SMs).  It needs the layers
// all fused or none, and every layer's members able to share a launch.
static bool groupable(ResStep (*s)[3], int J, int D, int mode) {
  int n_fused = 0;
  for (int l = 0; l < D; ++l)
    for (int j = 0; j < J; ++j) n_fused += s[l][j].fused ? 1 : 0;
  if (n_fused != 0 && n_fused != J * D) return false;
  for (int l = 0; l < D; ++l) {
    const LayerGroup m(s[l], J);
    if (n_fused ? !gp_pair_group_supported(m.pair, J, mode) : !(gp_group_supported(m.c1, J, mode) && gp_group_supported(m.c2, J, mode)))
      return false;
  }
  const ResStep& a = s[D - 1][0];
  return (n_fused ? gp_pair_solo_tiles(a.pair, mode) : gp_solo_tiles(a.c2, mode)) < 2 * sm_count();
}

// One HiFi-GAN stage's ResBlocks (hifigan/models.py:120-126): ACC = sum_j ResBlock_j(X) / J.  Where the stage buffers exist (small
// batches, carve_voc) and the stage is groupable, the J blocks advance together: the same-index convolutions of the blocks (different
// taps / dilations / weights, one shape) are ONE launch.  Every tile is computed as in the ungrouped launches: bitwise the same.
static int run_resblocks(const ev_ctx* ctx, const VocBufs& v, size_t rb0, int mode, int B, int L, int C, const int32_t* lens, int mul,
                         cudaStream_t st) {
  const int J = ctx->cfg.n_resk, D = ctx->cfg.n_dil;
  if (v.G0 && J >= 2 && J <= 3) {
    const StageBufs b = {v.X, v.ACC, {v.R1, v.R2, v.G2}, {v.Tm, v.G0, v.G1}};
    ResStep s[4][3];
    for (int l = 0; l < D; ++l)
      for (int j = 0; j < J; ++j) s[l][j] = res_step(ctx, b, rb0, j, l, l ? s[l - 1][j].out : v.X, false, B, L, C, lens, mul);
    if (groupable(s, J, D, mode)) {
      // fp32 storage: the last layer is grouped too, into the blocks' own buffers, and one elementwise pass forms ((x1 + x0) + x2) / J
      // -- the additions of the accumulate modes in their order, identical bits.  bf16 storage rounds xs after every accumulation,
      // which that pass cannot reproduce: there the last layer accumulates into ACC block by block.
      const bool sum_pass = mode != 2 && D >= 2;
      for (int l = 0; l < D; ++l) {
        const LayerGroup m(s[l], J);
        const bool fused = s[l][0].fused;
        if (l < D - 1 || sum_pass) {
          EV_TRY(fused ? launch_gp_pair_group(m.pair, J, mode, st) : launch_conv1d_gp_group(m.c1, J, mode, st));
          if (!fused) EV_TRY(launch_conv1d_gp_group(m.c2, J, mode, st));
          continue;
        }
        if (!fused) EV_TRY(launch_conv1d_gp_group(m.c1, J, mode, st));     // c1 does not depend on where the layer's output goes
        for (int j = 0; j < J; ++j) {
          const ResStep a = res_step(ctx, b, rb0, j, l, s[l][j].in, true, B, L, C, lens, mul);
          EV_TRY(fused ? launch_gp_pair(a.pair, mode, st) : launch_conv1d_gp(a.c2, mode, st));
        }
      }
      if (!sum_pass) return EV_OK;
      const ResStep* last = s[D - 1];
      return launch_gp_sum_div((const float*)last[0].out, (const float*)last[1].out, J == 3 ? (const float*)last[2].out : nullptr, v.ACC,
                               (size_t)B * L * C, (float)J, st);
    }
  }
  const StageBufs b = {v.X, v.ACC, {v.R1, v.R1, v.R1, v.R1}, {v.Tm, v.Tm, v.Tm, v.Tm}};
  for (int j = 0; j < J; ++j) {
    void* x = v.X;
    for (int l = 0; l < D; ++l) {
      const ResStep s = res_step(ctx, b, rb0, j, l, x, l == D - 1, B, L, C, lens, mul);
      if (s.fused) {
        EV_TRY(launch_gp_pair(s.pair, mode, st));
      } else {
        EV_TRY(launch_conv1d_gp(s.c1, mode, st));
        EV_TRY(launch_conv1d_gp(s.c2, mode, st));
      }
      x = s.out;
    }
  }
  return EV_OK;
}

// Encoder.forward (encoder.py:316-324) minus the positional prologue (done by the caller of this
// function): n x [ x += W_o Attn(LN1 x) ; x += Conv2(GELU(Conv1(LN2 x))) ], then after_norm -> y.
// K-split factors of a stack's four GEMM-shaped layers.  They are part of the layer's definition (they fix the order of each output
// element's reduction), never a function of batch or length.  The encoder runs on ~100 tokens per utterance -- one or two row tiles --
// so its launches have only (N tiles x S) CTAs to stream the layer's weights with: more slices.  The decoder has ~5 row tiles per
// utterance.  Measured at batch 1: 32 us -> ~12 us per encoder GEMM; at batch 32 the extra partial-sum traffic is ~1 % of the step.
struct StackSplits { int qkv, wo, ffn1, ffn2; };
static const StackSplits kEncSplits = {4, 8, 4, 16};
static const StackSplits kDecSplits = {2, 4, 4, 8};

static int run_stack(const ev_ctx* c, const StackW& s, float* x, float* y, float* qkv, float* ctxb, float* h,
                     int B, int L, const int32_t* key_lens, const int32_t* conv_lens, bool first_ln_done, bool prefix,
                     const StackSplits& sp, const SplitWs& ws, cudaStream_t st) {
  const int H = c->cfg.hidden, K = c->cfg.ffn_kernel, heads = c->cfg.n_heads;
  for (size_t i = 0; i < s.layers.size(); ++i) {
    const EncLayerW& l = s.layers[i];
    if (!(i == 0 && first_ln_done))
      EV_TRY(launch_layernorm(x, nullptr, nullptr, nullptr, nullptr, nullptr, l.ln1w, l.ln1b, y, B * L, L, H, st));
    EV_TRY(conv_x(c, l.wqkv, prefix, sp.qkv, ws, y, l.bqkv, 0, nullptr, qkv, B, L, H, 3 * H, 1, conv_lens, EV_ACT_NONE, st));
    // QK^T / softmax / PV on the tensor cores for d_k = 48: 3xTF32 beside fp32-accurate layers (MODE 1 / 3), one tf32 MMA otherwise;
    // the fp32 FFMA flash kernel in the "fp32_ffma" mode and for other head sizes
    const int mode = layer_run(l.wqkv, c->precision, prefix).mode;
    if (mode != kFfma && H / heads == 48)
      EV_TRY(launch_attention_tc(qkv, key_lens, ctxb, B, L, H, heads, (mode == 1 || mode == 3) ? 1 : 0, st));
    else
      EV_TRY(launch_attention(qkv, key_lens, ctxb, B, L, H, heads, st));
    EV_TRY(conv_x(c, l.wo, prefix, sp.wo, ws, ctxb, l.bo, 0, x, x, B, L, H, H, 1, conv_lens, EV_ACT_NONE, st));
    EV_TRY(launch_layernorm(x, nullptr, nullptr, nullptr, nullptr, nullptr, l.ln2w, l.ln2b, y, B * L, L, H, st));
    EV_TRY(conv_x(c, l.w1, prefix, sp.ffn1, ws, y, l.b1, 0, nullptr, h, B, L, H, 4 * H, K, conv_lens, EV_ACT_GELU, st));
    EV_TRY(conv_x(c, l.w2, prefix, sp.ffn2, ws, h, l.b2, 0, x, x, B, L, 4 * H, H, K, conv_lens, EV_ACT_NONE, st));
  }
  EV_TRY(launch_layernorm(x, nullptr, nullptr, nullptr, nullptr, nullptr, s.lnfw, s.lnfb, y, B * L, L, H, st));
  return EV_OK;
}

// [conv k -> ReLU -> channel LN] x n -> Linear(H -> 1) (variance.py:36-56, :101-124)
static int run_predictor(const ev_ctx* c, const PredW& p, const float* in, float* t1, float* t2, int B, int T,
                         const int32_t* lens, const int32_t* conv_lens, int mode, float* out_f, int64_t* out_i,
                         const SplitWs& ws, cudaStream_t st) {
  const int H = c->cfg.hidden, K = c->cfg.pred_kernel;
  const float* cur = in;
  for (size_t i = 0; i < p.w.size(); ++i) {
    // K = 3H on ~100 tokens and 3 N tiles: eight slices (see StackSplits)
    EV_TRY(conv_x(c, p.w[i], true, 8, ws, cur, p.b[i], 0, nullptr, t1, B, T, H, H, K, conv_lens, EV_ACT_RELU, st));
    EV_TRY(launch_layernorm(t1, nullptr, nullptr, nullptr, nullptr, nullptr, p.lnw[i], p.lnb[i], t2, B * T, T, H, st));
    cur = t2;
  }
  return launch_rowdot(cur, p.linw, p.linb, lens, B, T, H, mode, out_f, out_i, st);
}

}  // namespace ev

using namespace ev;

extern "C" {

int ev_abi_version(void) { return EV_ABI_VERSION; }
const char* ev_last_error(void) { return g_err.c_str(); }
uint64_t ev_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

int ev_create(ev_ctx** out, int device, const ev_config* cfg) {
  EV_CHECK_ARG(out && cfg, "ev_create: null argument");
  *out = nullptr;
  cudaDeviceProp prop;
  cudaError_t e = cudaGetDeviceProperties(&prop, device);
  if (e != cudaSuccess) { set_error("ev_create: cudaGetDeviceProperties(%d): %s", device, cudaGetErrorString(e)); return EV_ECUDA; }
  if (prop.major != 9) {
    set_error("ev_create: device %d is sm_%d%d; this library is built for sm_90a only", device, prop.major, prop.minor);
    return EV_EARCH;
  }
  EV_CHECK_ARG(cfg->hidden % 128 == 0 && cfg->hidden <= 512, "ev_create: hidden=%d unsupported", cfg->hidden);
  EV_CHECK_ARG(cfg->n_heads > 0 && cfg->hidden % cfg->n_heads == 0, "ev_create: heads=%d", cfg->n_heads);
  EV_CHECK_ARG((cfg->ffn_kernel & 1) && (cfg->pred_kernel & 1) && (cfg->embed_kernel & 1) && cfg->embed_kernel <= 15,
               "ev_create: kernel sizes must be odd");
  EV_CHECK_ARG(cfg->n_ups >= 1 && cfg->n_ups <= 8 && cfg->n_resk >= 1 && cfg->n_resk <= 4 && cfg->n_dil >= 1 && cfg->n_dil <= 4,
               "ev_create: vocoder shape out of range");
  EV_CHECK_ARG(cfg->n_mels % 16 == 0 && cfg->bert_dim % 8 == 0, "ev_create: n_mels must be a multiple of 16");
  ev_ctx* c = new ev_ctx();
  c->cfg = *cfg;
  c->device = device;
  {   // CUDA loads kernel code lazily at first launch; for the large tensor-core kernels that is tens of milliseconds each, which would
      // land on whichever utterance first needs a new tile shape.  Load them now, once per device.
    static std::atomic<uint64_t> loaded{0};
    int prev = -1;
    cudaGetDevice(&prev);
    if (prev != device) cudaSetDevice(device);
    if (first_use_on_device(loaded)) {
      preload_conv1d_gp(); preload_resblock_gp(); preload_attention_tc(); preload_conv1d_tc(); preload_voc_kernels();
    }
    if (prev >= 0 && prev != device) cudaSetDevice(prev);
    cudaGetLastError();
  }
  *out = c;
  return EV_OK;
}

void ev_destroy(ev_ctx* ctx) {
  delete ctx;
}

int ev_bind_weights(ev_ctx* ctx, const float* blob, size_t n_floats, const ev_weight_entry* index, int n_entries) {
  EV_CHECK_ARG(ctx && blob && index && n_entries > 0, "ev_bind_weights: null argument");
  ctx->tensors.clear();
  ctx->bound = false;
  for (int i = 0; i < n_entries; ++i) {
    const ev_weight_entry& e = index[i];
    EV_CHECK_ARG(e.offset + e.numel <= n_floats, "ev_bind_weights: entry '%.55s' exceeds the blob", e.name);
    EV_CHECK_ARG(e.offset % 4 == 0, "ev_bind_weights: entry '%.55s' is not 16-byte aligned", e.name);
    Tensor t;
    t.p = blob + e.offset;
    t.numel = e.numel;
    char nm[57];
    memcpy(nm, e.name, 56);
    nm[56] = 0;
    ctx->tensors[std::string(nm)] = t;
  }
  EV_TRY(resolve_all(ctx));
  EV_TRY(check_weights(ctx, ctx->precision, "ev_bind_weights"));
  ctx->bound = true;
  return EV_OK;
}

int ev_bind_pe(ev_ctx* ctx, const float* pe, int pe_len) {
  EV_CHECK_ARG(ctx && pe && pe_len > 0, "ev_bind_pe: bad argument");
  ctx->pe = pe;
  ctx->pe_len = pe_len;
  return EV_OK;
}

size_t ev_phase1_workspace_bytes(const ev_ctx* ctx, int B, int T) {
  if (!ctx || !ctx->bound || !ctx->has_am || B <= 0 || T <= 0) return 0;
  Carver cv(nullptr);
  Phase1Bufs p1;
  carve_phase1(ctx, cv, B, T, &p1);
  return cv.off + 256;
}

size_t ev_phase2_workspace_bytes(const ev_ctx* ctx, int B, int F) {
  if (!ctx || !ctx->bound || B <= 0 || F <= 0) return 0;
  // the vocoder runs after phase 2 on the same stream and re-carves the buffer from its start
  Carver am(nullptr), voc(nullptr);
  Phase2Bufs p2;
  VocBufs vb;
  if (ctx->has_am) carve_phase2(ctx, am, B, F, &p2);
  if (ctx->has_voc) carve_voc(ctx, voc, B, F, &vb);
  return (am.off > voc.off ? am.off : voc.off) + 256;
}

static int use_device(const ev_ctx* ctx) {
  int cur = -1;
  cudaError_t e = cudaGetDevice(&cur);
  if (e == cudaSuccess && cur != ctx->device) e = cudaSetDevice(ctx->device);
  if (e != cudaSuccess) { set_error("cudaSetDevice(%d): %s", ctx->device, cudaGetErrorString(e)); return EV_ECUDA; }
  return EV_OK;
}

int ev_am_phase1(ev_ctx* ctx, const int64_t* ling, const int64_t* lens64, const int64_t* spk, const float* style,
                 const float* content, int B, int T, int invariant, int64_t* dur_out, float* pitch_out,
                 float* energy_out, int32_t* lens32_out, int32_t* mel_lens_out, void* workspace, size_t workspace_bytes,
                 void* stream) {
  return ev_am_phase1_prosody(ctx, ling, lens64, spk, style, content, B, T, invariant, nullptr, dur_out, pitch_out, energy_out,
                              lens32_out, mel_lens_out, workspace, workspace_bytes, stream);
}

int ev_am_phase1_prosody(ev_ctx* ctx, const int64_t* ling, const int64_t* lens64, const int64_t* spk, const float* style,
                         const float* content, int B, int T, int invariant, const float* prosody, int64_t* dur_out,
                         float* pitch_out, float* energy_out, int32_t* lens32_out, int32_t* mel_lens_out, void* workspace,
                         size_t workspace_bytes, void* stream) {
  return ev_am_phase1_controls(ctx, ling, lens64, spk, style, content, B, T, invariant, prosody, 0, nullptr, nullptr, nullptr, dur_out,
                               pitch_out, energy_out, lens32_out, mel_lens_out, workspace, workspace_bytes, stream);
}

// Largest frame count an item may have: the vocoder indexes an item's samples with int32 (F * prod(upsample_rates) < 2^31),
// and the duration scan's exactness argument wants counts below 2^24.
static const int kScanMaxFrames = (1 << 24) - 1;
static int max_item_frames(const ev_config& g) {
  long long up = 1;
  for (int i = 0; i < g.n_ups; ++i) up *= g.up_rates[i] > 0 ? g.up_rates[i] : 1;
  const long long m = 2147483647LL / up;
  return (int)(m < kScanMaxFrames ? m : kScanMaxFrames);
}

int ev_am_phase1_controls(ev_ctx* ctx, const int64_t* ling, const int64_t* lens64, const int64_t* spk, const float* style,
                          const float* content, int B, int T, int invariant, const float* prosody, int prosody_per_token,
                          const int64_t* durations, const float* pitch_in, const float* energy_in, int64_t* dur_out,
                          float* pitch_out, float* energy_out, int32_t* lens32_out, int32_t* mel_lens_out, void* workspace,
                          size_t workspace_bytes, void* stream) {
  EV_CHECK_ARG(ctx && ctx->bound && ctx->has_am, "ev_am_phase1: acoustic-model weights not bound");
  EV_CHECK_ARG(ling && lens64 && spk && style && content && dur_out && pitch_out && energy_out && lens32_out &&
                   mel_lens_out && workspace,
               "ev_am_phase1: null argument");
  EV_CHECK_ARG(B > 0 && T > 0, "ev_am_phase1: B=%d T=%d", B, T);
  if (!ctx->pe || ctx->pe_len < T) { set_error("ev_am_phase1: positional table has %d rows, need %d", ctx->pe_len, T); return EV_EPELEN; }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const ev_config& g = ctx->cfg;
  const int H = g.hidden;
  Carver cv(workspace);
  Phase1Bufs b;
  carve_phase1(ctx, cv, B, T, &b);
  if (cv.off > workspace_bytes) { set_error("ev_am_phase1: workspace %zu < %zu bytes", workspace_bytes, cv.off); return EV_EWORKSPACE; }
  EV_TRY(use_device(ctx));
  const SplitWs ws{b.part, b.part_cap};
  // lengths -> int32, plus range checks of ids / speakers / lengths into the status word mel_lens_out[B + 1]
  EV_TRY(launch_validate_inputs(ling, lens64, spk, lens32_out, mel_lens_out + B + 1, B, T, g.n_vocab, g.n_speaker, st));
  const int32_t* lens = lens32_out;
  const int32_t* conv_lens = invariant ? lens : nullptr;

  Range r_phase("ev:am_phase1");
  // encoder: x = word_emb[ids] + alpha*pe (model_open_source.py:107, encoder.py:257-261), fused with LN1 of layer 0
  EV_TRY(launch_layernorm(nullptr, ling, ctx->emb_word, ctx->pe, ctx->enc.alpha, b.x, ctx->enc.layers[0].ln1w,
                          ctx->enc.layers[0].ln1b, b.y, B * T, T, H, st, g.n_vocab));
  EV_TRY(run_stack(ctx, ctx->enc, b.x, b.y, b.qkv, b.ctx, b.h, B, T, lens, conv_lens, true, true, kEncSplits, ws, st));
  // conditioning (model_open_source.py:109-111): per-utterance bias + W_x x
  EV_TRY(launch_cond_gather(spk, ctx->emb_spk, style, content, b.cond_in, B, H, g.bert_dim, g.n_speaker, st));
  EV_TRY(launch_cond_gemv(b.cond_in, ctx->cond_wc, ctx->cond_b, b.cond_bias, B, H + 2 * g.bert_dim, H, st));
  EV_TRY(conv_x(ctx, ctx->cond_wx, true, 4, ws, b.y, b.cond_bias, H, nullptr, b.hs, B, T, H, H, 1, conv_lens, EV_ACT_NONE, st));
  // predictors (model_open_source.py:120-121,130)
  const float* pin = b.hs;
  if (!invariant) {   // literal batch: masked_fill on the input only (variance.py:38-39); pads of hs are live data
    EV_TRY(launch_mask_rows(b.hs, lens, b.pm, B, T, H, st));
    pin = b.pm;
  }
  EV_TRY(run_predictor(ctx, ctx->pitch, pin, b.p1[0], b.p2[0], B, T, lens, conv_lens, 0, pitch_out, nullptr, ws, st));
  EV_TRY(run_predictor(ctx, ctx->energy, pin, b.p1[1], b.p2[1], B, T, lens, conv_lens, 0, energy_out, nullptr, ws, st));
  EV_TRY(run_predictor(ctx, ctx->dur, pin, b.p1[2], b.p2[2], B, T, lens, conv_lens, 1, nullptr, dur_out, ws, st));
  // x = x + pitch_embed + energy_embed (model_open_source.py:131-134) on the predicted tracks or the caller's, shifted / scaled
  // per item or per token when prosody is given
  EV_TRY(launch_var_embed_add(b.hs, pitch_in ? pitch_in : pitch_out, energy_in ? energy_in : energy_out, ctx->pemb_w, ctx->pemb_b,
                              ctx->eemb_w, ctx->eemb_b, prosody, prosody_per_token, lens, invariant, (pitch_in || energy_in) ? 1 : 0,
                              B, T, H, g.embed_kernel, st));
  // duration bookkeeping for the length regulator (alignment.py:183-199) on the predicted durations or the caller's, scaled by
  // alpha = prosody[(b*T + t)*5] per token or prosody[b*5] per item
  EV_TRY(launch_duration_scan(durations ? durations : dur_out, durations ? 1 : 0, lens, prosody, prosody_per_token ? 5 * T : 5,
                              prosody_per_token ? 5 : 0, invariant, B, T, b.centers, b.ds_f, mel_lens_out, mel_lens_out + B + 1,
                              max_item_frames(g), st));
  return EV_OK;
}

int ev_am_phase2(ev_ctx* ctx, const void* phase1_workspace, const int32_t* lens, const int32_t* mel_lens, int B, int T,
                 int F, int invariant, float* mel_out, void* workspace, size_t workspace_bytes, void* stream) {
  EV_CHECK_ARG(ctx && ctx->bound && ctx->has_am, "ev_am_phase2: acoustic-model weights not bound");
  EV_CHECK_ARG(phase1_workspace && lens && mel_lens && mel_out && workspace, "ev_am_phase2: null argument");
  EV_CHECK_ARG(B > 0 && T > 0 && F > 0, "ev_am_phase2: B=%d T=%d F=%d", B, T, F);
  if (!ctx->pe || ctx->pe_len < F) { set_error("ev_am_phase2: positional table has %d rows, need %d", ctx->pe_len, F); return EV_EPELEN; }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const ev_config& g = ctx->cfg;
  const int H = g.hidden;
  EV_TRY(use_device(ctx));
  Carver cv1(const_cast<void*>(phase1_workspace)), cv(workspace);
  Phase1Bufs b1;
  Phase2Bufs b;
  carve_phase1(ctx, cv1, B, T, &b1);
  carve_phase2(ctx, cv, B, F, &b);
  if (cv.off > workspace_bytes) { set_error("ev_am_phase2: workspace %zu < %zu bytes", workspace_bytes, cv.off); return EV_EWORKSPACE; }
  const int32_t* flens = invariant ? mel_lens : nullptr;
  const SplitWs ws{b.part, b.part_cap};
  Range r_phase("ev:am_phase2");
  // length regulator + the decoder's positional encoding (alignment.py:198-211, encoder.py:257-261)
  EV_TRY(launch_gauss_upsample(b1.hs, b1.centers, lens, mel_lens, B, T, H, F, invariant, ctx->pe, ctx->dec.alpha, b.x, st));
  // decoder (model_open_source.py:146: mask None in the reference; per-item lengths under the invariant contract)
  EV_TRY(run_stack(ctx, ctx->dec, b.x, b.y, b.qkv, b.ctx, b.h, B, F, flens, flens, false, false, kDecSplits, ws, st));
  // to_mel (model_open_source.py:147)
  EV_TRY(conv_x(ctx, ctx->mel_w, false, 2, ws, b.y, ctx->mel_b, 0, nullptr, mel_out, B, F, H, g.n_mels, 1, flens, EV_ACT_NONE, st));
  return EV_OK;
}

int ev_vocoder(ev_ctx* ctx, const float* mel, int mel_time_major, const int32_t* mel_lens, int B, int F, float* wav_out,
               void* workspace, size_t workspace_bytes, void* stream) {
  EV_CHECK_ARG(ctx && ctx->bound && ctx->has_voc, "ev_vocoder: vocoder weights not bound");
  EV_CHECK_ARG(mel && wav_out && workspace, "ev_vocoder: null argument");
  EV_CHECK_ARG(B > 0 && F > 0, "ev_vocoder: B=%d F=%d", B, F);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const ev_config& g = ctx->cfg;
  EV_TRY(use_device(ctx));
  Carver cv(workspace);
  VocBufs v;
  carve_voc(ctx, cv, B, F, &v);
  if (cv.off > workspace_bytes) { set_error("ev_vocoder: workspace %zu < %zu bytes", workspace_bytes, cv.off); return EV_EWORKSPACE; }
  static const char* const kStageNames[8] = {"voc:stage1", "voc:stage2", "voc:stage3", "voc:stage4", "voc:stage5", "voc:stage6",
                                             "voc:stage7", "voc:stage8"};
  int L = F, mul = 1;
  if (ctx->precision == EV_PREC_FP32_FFMA) {
    // ---- "fp32_ffma": time-major activations and the fp32 FFMA kernel ----
    const float* m = mel;
    if (!mel_time_major) {
      EV_TRY(launch_transpose_cf_to_tm(mel, v.Tm, B, g.n_mels, F, st));
      m = v.Tm;
    }
    Range r_phase("ev:vocoder");
    // conv_pre (hifigan/models.py:116)
    EV_TRY(conv(m, ctx->pre.w.w, ctx->pre.b, 0, nullptr, v.ACC, B, F, g.n_mels, g.voc_c0, ctx->pre.K, 1, mel_lens, 1, EV_ACT_NONE, 0.f,
                EV_ACT_NONE, EV_ACC_STORE, 1.f, st));
    size_t rb = 0;
    for (int s = 0; s < g.n_ups; ++s) {
      Range r_stage(kStageNames[s & 7]);
      const UpW& u = ctx->ups[s];
      // x = ups[i](leaky_relu(x, 0.1)) (:118-119): polyphase-packed transposed conv, output viewed (L, rate*Cout)
      EV_TRY(conv(v.ACC, u.w.w, u.b, 0, nullptr, v.X, B, L, u.cin, u.cout_packed, u.K, 1, mel_lens, mul, EV_ACT_LRELU, 0.1f, EV_ACT_NONE,
                  EV_ACC_STORE, 1.f, st));
      L *= u.rate; mul *= u.rate;
      const int C = u.cout;
      for (int j = 0; j < g.n_resk; ++j) {
        const float* src = v.X;
        for (int l = 0; l < g.n_dil; ++l, ++rb) {
          const ConvW& c1 = ctx->rb_c1[rb];
          const ConvW& c2 = ctx->rb_c2[rb];
          const bool last = (l == g.n_dil - 1);
          float* dst = last ? v.ACC : ((l & 1) ? v.R2 : v.R1);
          int acc = EV_ACC_STORE;
          if (last && j > 0) acc = (j == g.n_resk - 1) ? EV_ACC_ADD_DIV : EV_ACC_ADD;   // xs += ...; x = xs / n (:120-126)
          // xt = c1(lrelu(x)) ; x = c2(lrelu(xt)) + x   (:50-57)
          EV_TRY(conv(src, c1.w.w, c1.b, 0, nullptr, v.Tm, B, L, C, C, c1.K, c1.dil, mel_lens, mul, EV_ACT_LRELU, 0.1f, EV_ACT_NONE,
                      EV_ACC_STORE, 1.f, st));
          EV_TRY(conv(v.Tm, c2.w.w, c2.b, 0, src, dst, B, L, C, C, c2.K, 1, mel_lens, mul, EV_ACT_LRELU, 0.1f, EV_ACT_NONE, acc,
                      (float)g.n_resk, st));
          src = dst;
        }
      }
    }
    EV_CHECK_ARG(mul == ctx->total_up, "ev_vocoder: internal rate mismatch");
    // x = leaky_relu(x) [slope 0.01]; conv_post; tanh (:127-129)
    return launch_conv_post(v.ACC, ctx->post_w, ctx->post_b, mel_lens, mul, B, L, ctx->ups.back().cout, ctx->post_k, 0.01f, wav_out, st);
  }
  // ---- tensor cores: granule-planar [b][C/cpg][l][cpg] activations, bulk-copied A operands, direct coalesced epilogues ----
  Range r_phase("ev:vocoder");
  const LayerRun pre = layer_run(ctx->pre.w, ctx->precision, false);
  const int mode = pre.mode, bf = (mode == 2) ? 1 : 0;      // bf16: bf16 activations in HBM
  // mel (B,F,n_mels) time-major or (B,n_mels,F) channels-first -> GP
  EV_TRY(launch_to_gp(mel, (long long)F * g.n_mels, mel_time_major ? g.n_mels : 1, mel_time_major ? 1 : F, v.Tm, B, F, g.n_mels, bf, st));
  // conv_pre (hifigan/models.py:116)
  EV_TRY(launch_conv1d_gp(gp_params(pre.w, v.Tm, ctx->pre.b, nullptr, v.ACC, B, F, g.n_mels, g.voc_c0, ctx->pre.K, 1, 1, mel_lens, 1,
                                    EV_ACT_NONE, 0.f, EV_ACC_STORE, 1.f), mode, st));
  for (int s = 0; s < g.n_ups; ++s) {
    Range r_stage(kStageNames[s & 7]);
    const UpW& u = ctx->ups[s];
    // x = ups[i](leaky_relu(x, 0.1)) (:118-119): polyphase transposed conv, the `rate` output phases are GEMM column groups
    EV_TRY(launch_conv1d_gp(gp_params(layer_run(u.w, ctx->precision, false).w, v.ACC, u.b, nullptr, v.X, B, L, u.cin, u.cout_packed, u.K, 1,
                                      u.rate, mel_lens, mul, EV_ACT_LRELU, 0.1f, EV_ACC_STORE, 1.f), mode, st));
    L *= u.rate; mul *= u.rate;
    EV_TRY(run_resblocks(ctx, v, (size_t)s * g.n_resk * g.n_dil, mode, B, L, u.cout, mel_lens, mul, st));
  }
  EV_CHECK_ARG(mul == ctx->total_up, "ev_vocoder: internal rate mismatch");
  // x = leaky_relu(x) [slope 0.01]; conv_post; tanh (:127-129)
  return launch_conv_post_gp(v.ACC, bf, ctx->post_w, ctx->post_b, mel_lens, mul, B, L, ctx->ups.back().cout, ctx->post_k, 0.01f, wav_out, st);
}

int ev_join_mel(const float* mel, const int32_t* mel_lens, const int32_t* group, int B, int F, int n_mels, int G, int Fg, float* joined,
                int32_t* group_lens, void* stream) {
  EV_CHECK_ARG(mel && mel_lens && group && joined && group_lens, "ev_join_mel: null argument");
  EV_TRY(use_device_of(mel));
  return launch_join_mel(mel, mel_lens, group, B, F, n_mels, G, Fg, joined, group_lens, reinterpret_cast<cudaStream_t>(stream));
}

int ev_wav_to_pcm16(const float* wav, int16_t* pcm, size_t n, void* stream) {
  EV_CHECK_ARG(wav && pcm, "ev_wav_to_pcm16: null argument");
  EV_TRY(use_device_of(wav));
  return launch_pcm16(wav, pcm, n, reinterpret_cast<cudaStream_t>(stream));
}

int ev_format_audio(const float* wav, long long item_stride, const int64_t* n_in, const int64_t* items, int n_items,
                    const int64_t* out_off, const float* bank, int up, int down, int taps_per_phase, int encoding, void* out,
                    const float* gain, void* stream) {
  EV_CHECK_ARG(wav && n_in && out_off && out, "ev_format_audio: null argument");
  EV_TRY(use_device_of(wav));
  return launch_audio_out(wav, item_stride, n_in, items, n_items, out_off, bank, up, down, taps_per_phase, encoding, gain, out,
                          reinterpret_cast<cudaStream_t>(stream));
}

int ev_op_conv1d(const float* x, const float* w, const float* bias, size_t bias_bstride, const float* res, float* out,
                 int B, int L, int Cin, int Cout, int K, int dil, const int32_t* lens, int lens_mul, int in_act,
                 float in_slope, int out_act, int acc, float div, void* stream) {
  EV_CHECK_ARG(x && w && out, "ev_op_conv1d: null argument");
  EV_TRY(use_device_of(x));
  return conv(x, w, bias, (long long)bias_bstride, res, out, B, L, Cin, Cout, K, dil, lens, lens_mul, in_act, in_slope,
              out_act, acc, div, reinterpret_cast<cudaStream_t>(stream));
}

int ev_debug_conv1d_plan(int B, int L, int Cin, int Cout, int K, int dil, int* out10) {
  EV_CHECK_ARG(out10, "ev_debug_conv1d_plan: null output");
  ConvParams p{};
  p.B = B; p.L = L; p.Cin = Cin; p.Cout = Cout; p.K = K; p.dil = dil; p.in_act = EV_ACT_NONE;
  return debug_conv1d_plan(p, out10);
}

int ev_op_conv_post(const float* x, const float* w, const float* bias, const int32_t* lens, int lens_mul, int B, int L, int C, int K,
                    float slope, float* wav, void* stream) {
  EV_CHECK_ARG(x && w && bias && wav, "ev_op_conv_post: null argument");
  EV_TRY(use_device_of(x));
  return launch_conv_post(x, w, bias, lens, lens_mul, B, L, C, K, slope, wav, reinterpret_cast<cudaStream_t>(stream));
}

int ev_op_conv1d_tc(const float* x, const float* w_tc, int split3, const float* bias, size_t bias_bstride, const float* res,
                    float* out, int B, int L, int Cin, int Cout, int K, int dil, const int32_t* lens, int lens_mul,
                    int in_act, float in_slope, int out_act, int acc, float div, float* splitk_ws, size_t splitk_floats,
                    void* stream) {
  return ev_op_conv1d_tc_ks(x, w_tc, split3, bias, bias_bstride, res, out, B, L, Cin, Cout, K, dil, lens, lens_mul, in_act, in_slope,
                            out_act, acc, div, splitk_ws ? 4 : 0, splitk_ws, splitk_floats, stream);
}

int ev_op_conv1d_tc_ks(const float* x, const float* w_tc, int split3, const float* bias, size_t bias_bstride, const float* res,
                       float* out, int B, int L, int Cin, int Cout, int K, int dil, const int32_t* lens, int lens_mul,
                       int in_act, float in_slope, int out_act, int acc, float div, int ksplit, float* splitk_ws,
                       size_t splitk_floats, void* stream) {
  EV_CHECK_ARG(x && w_tc && out, "ev_op_conv1d_tc: null argument");
  EV_CHECK_ARG(ksplit <= 1 || splitk_ws, "ev_op_conv1d_tc: ksplit=%d needs split-K scratch", ksplit);
  EV_CHECK_ARG(split3 >= 0 && split3 <= 3, "ev_op_conv1d_tc: split3=%d is not a kernel mode (0..3)", split3);
  EV_TRY(use_device_of(x));
  EV_CHECK_ARG(Cin % 8 == 0 && Cout % 16 == 0 && (Cout <= 128 || Cout % 128 == 0),
               "ev_op_conv1d_tc: needs Cin %% 8 == 0, Cout %% 16 == 0 and Cout <= 128 or a multiple of 128 (Cin=%d Cout=%d)", Cin, Cout);
  EV_CHECK_ARG(split3 < 2 || Cin % 16 == 0, "ev_op_conv1d_tc: the bf16 / bf16x3 modes need Cin %% 16 == 0 (Cin=%d)", Cin);
  ConvParams p = conv_params(x, w_tc, bias, (long long)bias_bstride, res, out, B, L, Cin, Cout, K, dil, lens, lens_mul, in_act, in_slope,
                             out_act, acc, div);
  p.splitk_ws = splitk_ws; p.splitk_cap = splitk_ws ? splitk_floats : 0; p.ksplit = splitk_ws ? ksplit : 0;
  return launch_conv1d_tc(p, split3, reinterpret_cast<cudaStream_t>(stream));
}

int ev_debug_tc_plan(int B, int L, int Cin, int Cout, int K, int dil, int split3, int ksplit, int* out11) {
  EV_CHECK_ARG(out11, "ev_debug_tc_plan: null output");
  ConvParams p{};
  p.B = B; p.L = L; p.Cin = Cin; p.Cout = Cout; p.K = K; p.dil = dil; p.in_act = EV_ACT_NONE;
  p.ksplit = ksplit; p.splitk_ws = nullptr; p.splitk_cap = (size_t)-1;   // "scratch of any size is available"
  return debug_tc_plan(p, split3, out11);
}

int ev_op_conv1d_gp(const void* x, const float* w, int mode, const float* bias, const void* res, void* out, int B, int L, int Cin, int Cout,
                    int K, int dil, int rate, const int32_t* lens, int lens_mul, int in_act, float in_slope, int acc, float div, void* stream) {
  EV_CHECK_ARG(x && w && out, "ev_op_conv1d_gp: null argument");
  EV_TRY(use_device_of(x));
  return launch_conv1d_gp(gp_params(w, x, bias, res, out, B, L, Cin, Cout, K, dil, rate, lens, lens_mul, in_act, in_slope, acc, div), mode,
                          reinterpret_cast<cudaStream_t>(stream));
}

int ev_op_conv1d_gp_group(int n, const void* const* x, const float* const* w, int mode, const float* const* bias, const void* const* res, void* const* out,
                          const int* K, const int* dil, int B, int L, int Cin, int Cout, const int32_t* lens, int lens_mul, int in_act, float in_slope,
                          void* stream) {
  EV_CHECK_ARG(n >= 1 && n <= 3 && x && w && out && K && dil, "ev_op_conv1d_gp_group: 1..3 convolutions, non-null tables");
  GpConvParams ps[3];
  for (int i = 0; i < n; ++i) {
    GpConvParams& p = ps[i];
    EV_CHECK_ARG(x[i] && w[i] && out[i], "ev_op_conv1d_gp_group: null tensor in member %d", i);
    p.x = x[i]; p.w = w[i]; p.bias = bias ? bias[i] : nullptr; p.res = res ? res[i] : nullptr; p.out = out[i];
    p.B = B; p.L = L; p.Cin = Cin; p.Cout = Cout; p.K = K[i]; p.dil = dil[i]; p.rate = 1;
    p.lens = lens; p.lens_mul = lens_mul; p.in_act = in_act; p.in_slope = in_slope; p.acc = EV_ACC_STORE; p.div = 1.f;
  }
  EV_TRY(use_device_of(x[0]));
  return launch_conv1d_gp_group(ps, n, mode, reinterpret_cast<cudaStream_t>(stream));
}

int ev_op_gp_sum_div(const float* a, const float* b, const float* c, float* out, size_t n_floats, float div, void* stream) {
  EV_CHECK_ARG(a && b && out, "ev_op_gp_sum_div: null argument");
  EV_TRY(use_device_of(a));
  return launch_gp_sum_div(a, b, c, out, n_floats, div, reinterpret_cast<cudaStream_t>(stream));
}

int ev_debug_gp_group_plan(int n, const int* K, const int* dil, int B, int L, int Cin, int Cout, int mode, int* out11) {
  EV_CHECK_ARG(out11 && K && dil && n >= 1 && n <= 3, "ev_debug_gp_group_plan: bad arguments");
  static float dummy_in, dummy_w, dummy_out[3];
  GpConvParams ps[3];
  for (int i = 0; i < n; ++i) {
    ps[i] = GpConvParams{};
    ps[i].x = &dummy_in; ps[i].w = &dummy_w; ps[i].out = &dummy_out[i]; ps[i].B = B; ps[i].L = L; ps[i].Cin = Cin; ps[i].Cout = Cout; ps[i].K = K[i]; ps[i].dil = dil[i];
    ps[i].rate = 1; ps[i].lens_mul = 1; ps[i].in_act = EV_ACT_LRELU; ps[i].in_slope = 0.1f; ps[i].acc = EV_ACC_STORE; ps[i].div = 1.f;
  }
  return debug_gp_group_plan(ps, n, mode, out11);
}

int ev_op_resblock_gp(const void* x, const float* w1, const float* b1, const float* w2, const float* b2, int mode, void* out, int B, int L, int C, int K,
                      int dil, const int32_t* lens, int lens_mul, int acc, float div, void* stream) {
  EV_CHECK_ARG(x && w1 && b1 && w2 && b2 && out, "ev_op_resblock_gp: null argument");
  EV_TRY(use_device_of(x));
  GpPairParams p;
  p.x = x; p.w1 = w1; p.b1 = b1; p.w2 = w2; p.b2 = b2; p.out = out; p.B = B; p.L = L; p.C = C; p.K = K; p.dil = dil; p.lens = lens; p.lens_mul = lens_mul;
  p.slope = 0.1f; p.acc = acc; p.div = div;
  return launch_gp_pair(p, mode, reinterpret_cast<cudaStream_t>(stream));
}

int ev_op_resblock_gp_group(int n, const void* const* x, const float* const* w1, const float* const* b1, const float* const* w2, const float* const* b2,
                            int mode, void* const* out, int B, int L, int C, const int* K, const int* dil, const int32_t* lens, int lens_mul, void* stream) {
  EV_CHECK_ARG(n >= 1 && n <= 3 && x && w1 && b1 && w2 && b2 && out && K && dil, "ev_op_resblock_gp_group: 1..3 layers, non-null tables");
  GpPairParams ps[3];
  for (int i = 0; i < n; ++i) {
    GpPairParams& p = ps[i];
    EV_CHECK_ARG(x[i] && w1[i] && b1[i] && w2[i] && b2[i] && out[i], "ev_op_resblock_gp_group: null tensor in member %d", i);
    p.x = x[i]; p.w1 = w1[i]; p.b1 = b1[i]; p.w2 = w2[i]; p.b2 = b2[i]; p.out = out[i]; p.B = B; p.L = L; p.C = C; p.K = K[i]; p.dil = dil[i];
    p.lens = lens; p.lens_mul = lens_mul; p.slope = 0.1f; p.acc = EV_ACC_STORE; p.div = 1.f;
  }
  EV_TRY(use_device_of(x[0]));
  return launch_gp_pair_group(ps, n, mode, reinterpret_cast<cudaStream_t>(stream));
}

int ev_debug_resblock_gp_group_plan(int n, const int* K, const int* dil, int B, int L, int C, int mode, int* out16) {
  EV_CHECK_ARG(out16 && K && dil && n >= 1 && n <= 3, "ev_debug_resblock_gp_group_plan: bad arguments");
  static float dummy_in[3], dummy_out[3], dummy_w;
  GpPairParams ps[3];
  for (int i = 0; i < n; ++i) {
    ps[i] = GpPairParams{};
    ps[i].x = &dummy_in[i]; ps[i].out = &dummy_out[i]; ps[i].w1 = ps[i].w2 = ps[i].b1 = ps[i].b2 = &dummy_w;
    ps[i].B = B; ps[i].L = L; ps[i].C = C; ps[i].K = K[i]; ps[i].dil = dil[i]; ps[i].lens_mul = 1; ps[i].slope = 0.1f; ps[i].acc = EV_ACC_STORE; ps[i].div = 1.f;
  }
  return debug_gp_pair_group_plan(ps, n, mode, out16);
}

int ev_debug_resblock_gp_plan(int B, int L, int C, int K, int dil, int mode, int* out11) {
  EV_CHECK_ARG(out11, "ev_debug_resblock_gp_plan: null output");
  static float dummy_in, dummy_out;
  GpPairParams p{};
  p.x = &dummy_in; p.out = &dummy_out; p.B = B; p.L = L; p.C = C; p.K = K; p.dil = dil; p.lens_mul = 1; p.slope = 0.1f; p.acc = EV_ACC_STORE; p.div = 1.f;
  return debug_gp_pair_plan(p, mode, out11);
}

int ev_debug_gp_plan(int B, int L, int Cin, int Cout, int K, int dil, int rate, int mode, int* out11) {
  EV_CHECK_ARG(out11, "ev_debug_gp_plan: null output");
  GpConvParams p{};
  p.B = B; p.L = L; p.Cin = Cin; p.Cout = Cout; p.K = K; p.dil = dil; p.rate = rate; p.in_act = EV_ACT_NONE; p.acc = EV_ACC_STORE;
  return debug_gp_plan(p, mode, out11);
}

int ev_op_to_gp(const float* in, long long stride_b, long long stride_t, long long stride_c, void* out, int B, int L, int C, int bf16, void* stream) {
  EV_CHECK_ARG(in && out, "ev_op_to_gp: null argument");
  EV_TRY(use_device_of(in));
  return launch_to_gp(in, stride_b, stride_t, stride_c, out, B, L, C, bf16, reinterpret_cast<cudaStream_t>(stream));
}

int ev_op_conv_post_gp(const void* x, int bf16, const float* w, const float* bias, const int32_t* lens, int lens_mul, int B, int L, int C, int K,
                       float slope, float* wav, void* stream) {
  EV_CHECK_ARG(x && w && bias && wav, "ev_op_conv_post_gp: null argument");
  EV_TRY(use_device_of(x));
  return launch_conv_post_gp(x, bf16, w, bias, lens, lens_mul, B, L, C, K, slope, wav, reinterpret_cast<cudaStream_t>(stream));
}

int ev_set_precision(ev_ctx* ctx, int precision) {
  EV_CHECK_ARG(ctx, "ev_set_precision: null context");
  EV_CHECK_ARG(precision == EV_PREC_FP32 || precision == EV_PREC_TF32 || precision == EV_PREC_FP32_FFMA || precision == EV_PREC_BF16,
               "ev_set_precision: unknown precision %d", precision);
  if (ctx->bound) EV_TRY(check_weights(ctx, precision, "ev_set_precision"));
  ctx->precision = precision;
  return EV_OK;
}

int ev_op_layernorm(const float* x, const float* w, const float* b, float* y, int rows, int C, void* stream) {
  EV_CHECK_ARG(x && w && b && y, "ev_op_layernorm: null argument");
  EV_TRY(use_device_of(x));
  return launch_layernorm(x, nullptr, nullptr, nullptr, nullptr, nullptr, w, b, y, rows, rows, C,
                          reinterpret_cast<cudaStream_t>(stream));
}

int ev_op_attention(const float* qkv, const int32_t* key_lens, float* ctx_out, int B, int L, int H, int n_heads,
                    void* stream) {
  EV_CHECK_ARG(qkv && ctx_out, "ev_op_attention: null argument");
  EV_TRY(use_device_of(qkv));
  return launch_attention(qkv, key_lens, ctx_out, B, L, H, n_heads, reinterpret_cast<cudaStream_t>(stream));
}

int ev_op_attention_tc(const float* qkv, const int32_t* key_lens, float* ctx_out, int B, int L, int H, int n_heads, int tc_mode, void* stream) {
  EV_CHECK_ARG(qkv && ctx_out, "ev_op_attention_tc: null argument");
  EV_TRY(use_device_of(qkv));
  return launch_attention_tc(qkv, key_lens, ctx_out, B, L, H, n_heads, tc_mode, reinterpret_cast<cudaStream_t>(stream));
}

int ev_op_gauss_upsample(const float* hs, const int64_t* dur, const int32_t* lens, int B, int T, int H, int F,
                         int invariant, const float* pe, const float* alpha, float* centers_tmp, int32_t* mel_lens_tmp,
                         float* out, void* stream) {
  EV_CHECK_ARG(hs && dur && centers_tmp && mel_lens_tmp && out, "ev_op_gauss_upsample: null argument");
  EV_TRY(use_device_of(hs));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  // centers_tmp holds 2*B*T floats: centres then float durations
  EV_TRY(launch_duration_scan(dur, 0, lens, nullptr, 0, 0, invariant, B, T, centers_tmp, centers_tmp + (size_t)B * T, mel_lens_tmp,
                              nullptr, kScanMaxFrames, st));
  return launch_gauss_upsample(hs, centers_tmp, lens, mel_lens_tmp, B, T, H, F, invariant, pe, alpha, out, st);
}

int ev_op_gauss_upsample_centers(const float* hs, const float* centers, const int32_t* lens, const int32_t* mel_lens, int B, int T,
                                 int H, int F, int invariant, const float* pe, const float* alpha, float* out, void* stream) {
  EV_CHECK_ARG(hs && centers && out && (mel_lens || !invariant) && (alpha || !pe), "ev_op_gauss_upsample_centers: null argument");
  EV_CHECK_ARG(B > 0, "ev_op_gauss_upsample_centers: B=%d", B);
  EV_TRY(use_device_of(hs));
  return launch_gauss_upsample(hs, centers, lens, mel_lens, B, T, H, F, invariant, pe, alpha, out, reinterpret_cast<cudaStream_t>(stream));
}

int ev_op_layernorm_embed(const int64_t* ids, const float* emb, int n_emb, const float* pe, const float* alpha, int L, float* x_out,
                          const float* w, const float* b, float* y, int rows, int C, void* stream) {
  EV_CHECK_ARG(ids && emb && pe && alpha && x_out && w && b && y, "ev_op_layernorm_embed: null argument");
  EV_CHECK_ARG(L > 0, "ev_op_layernorm_embed: L=%d", L);
  EV_TRY(use_device_of(emb));
  return launch_layernorm(nullptr, ids, emb, pe, alpha, x_out, w, b, y, rows, L, C, reinterpret_cast<cudaStream_t>(stream), n_emb);
}

int ev_op_cond_bias(const int64_t* spk, const float* spk_emb, int n_spk, const float* style, const float* content, int B, int H, int bert,
                    const float* w, const float* bias, float* cond_in, float* out, void* stream) {
  EV_CHECK_ARG(spk && spk_emb && style && content && w && bias && cond_in && out, "ev_op_cond_bias: null argument");
  EV_CHECK_ARG(n_spk > 0 && H > 0 && H % 8 == 0 && bert >= 0 && B > 0 && B <= 65535, "ev_op_cond_bias: B=%d n_spk=%d H=%d bert=%d", B,
               n_spk, H, bert);
  EV_TRY(use_device_of(w));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  EV_TRY(launch_cond_gather(spk, spk_emb, style, content, cond_in, B, H, bert, n_spk, st));
  return launch_cond_gemv(cond_in, w, bias, out, B, H + 2 * bert, H, st);
}

int ev_op_rowdot(const float* x, const float* w, const float* b, const int32_t* lens, int B, int T, int C, int mode, float* out_f,
                 int64_t* out_i, void* stream) {
  EV_CHECK_ARG(x && w && b && (mode == 0 ? out_f != nullptr : (mode == 1 && out_i)), "ev_op_rowdot: null argument or mode %d", mode);
  EV_CHECK_ARG(B > 0 && T > 0, "ev_op_rowdot: B=%d T=%d", B, T);
  EV_TRY(use_device_of(x));
  return launch_rowdot(x, w, b, lens, B, T, C, mode, out_f, out_i, reinterpret_cast<cudaStream_t>(stream));
}

int ev_op_mask_rows(const float* x, const int32_t* lens, float* y, int B, int T, int C, void* stream) {
  EV_CHECK_ARG(x && y, "ev_op_mask_rows: null argument");
  EV_CHECK_ARG(B > 0 && T > 0 && C > 0, "ev_op_mask_rows: B=%d T=%d C=%d", B, T, C);
  EV_TRY(use_device_of(x));
  return launch_mask_rows(x, lens, y, B, T, C, reinterpret_cast<cudaStream_t>(stream));
}

int ev_op_var_embed_add(float* x, const float* pitch, const float* energy, const float* wp, const float* bp, const float* we, const float* be,
                        const float* prosody, const int32_t* lens, int B, int T, int C, int K, void* stream) {
  EV_CHECK_ARG(x && pitch && energy && wp && bp && we && be, "ev_op_var_embed_add: null argument");
  EV_CHECK_ARG(B > 0 && T > 0 && C > 0 && K > 0 && (K & 1), "ev_op_var_embed_add: B=%d T=%d C=%d K=%d", B, T, C, K);
  EV_TRY(use_device_of(x));
  return launch_var_embed_add(x, pitch, energy, wp, bp, we, be, prosody, 0, lens, lens ? 1 : 0, 0, B, T, C, K,
                              reinterpret_cast<cudaStream_t>(stream));
}

int ev_op_duration_scan(const int64_t* dur, const int32_t* lens, const float* alpha, int invariant, int B, int T, float* centers,
                        float* ds, int32_t* mel_lens, void* stream) {
  EV_CHECK_ARG(dur && centers && ds && mel_lens, "ev_op_duration_scan: null argument");
  EV_CHECK_ARG(B > 0 && T > 0, "ev_op_duration_scan: B=%d T=%d", B, T);
  EV_TRY(use_device_of(dur));
  return launch_duration_scan(dur, 0, lens, alpha, 1, 0, invariant, B, T, centers, ds, mel_lens, nullptr, kScanMaxFrames,
                              reinterpret_cast<cudaStream_t>(stream));
}

int ev_op_duration_scan_controls(const int64_t* dur, int caller, const int32_t* lens, const float* alpha, int alpha_stride,
                                 int alpha_tstride, int invariant, int B, int T, int max_frames, float* centers, float* ds,
                                 int32_t* mel_lens, int32_t* status, void* stream) {
  EV_CHECK_ARG(dur && centers && ds && mel_lens, "ev_op_duration_scan_controls: null argument");
  EV_CHECK_ARG(B > 0 && T > 0 && alpha_stride >= 0 && alpha_tstride >= 0, "ev_op_duration_scan_controls: B=%d T=%d strides %d %d", B,
               T, alpha_stride, alpha_tstride);
  EV_TRY(use_device_of(dur));
  return launch_duration_scan(dur, caller, lens, alpha, alpha_stride, alpha_tstride, invariant, B, T, centers, ds, mel_lens, status,
                              max_frames, reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
