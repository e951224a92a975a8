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
static thread_local cudaError_t g_parked_launch_error = cudaSuccess;
void park_launch_error(cudaError_t e) { if (e != cudaSuccess) g_parked_launch_error = e; }
cudaError_t take_launch_error() {
  const cudaError_t e = g_parked_launch_error;
  g_parked_launch_error = cudaSuccess;
  return e;
}
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
int pdl_mode() {
  static const int v = [] { const char* e = getenv("EV_PDL"); return (e && *e) ? atoi(e) : 2; }();
  return v;
}

struct Tensor {
  const float* p = nullptr;
  uint64_t numel = 0;
};

struct EncLayerW {
  const float *ln1w, *ln1b, *wqkv, *bqkv, *wo, *bo, *ln2w, *ln2b, *w1, *b1, *w2, *b2;
  const float *wqkv_tc = nullptr, *wo_tc = nullptr, *w1_tc = nullptr, *w2_tc = nullptr;   // tensor-core layout (optional)
  const float *wqkv_h = nullptr, *wo_h = nullptr, *w1_h = nullptr, *w2_h = nullptr;       // bf16 tensor-core layout (optional)
  const float *wqkv_x2 = nullptr, *wo_x2 = nullptr, *w1_x2 = nullptr, *w2_x2 = nullptr;   // two bf16 planes (bf16x3 emulation; decoder only)
};
struct StackW {
  const float* alpha;
  std::vector<EncLayerW> layers;
  const float *lnfw, *lnfb;
};
struct PredW {
  std::vector<const float*> w, b, lnw, lnb, w_tc;
  const float *linw, *linb;
};
struct ConvW {
  const float *w, *b;
  const float* w_tc = nullptr;
  const float* w_h = nullptr;
  const float* w_x2 = nullptr;     // two bf16 planes (hi, lo): the bf16x3 fp32 emulation of the granule-planar vocoder
  int K, dil, cin, cout;
};
struct UpW {
  const float *w, *b;
  const float* w_tc = nullptr;
  const float* w_h = nullptr;
  const float* w_x2 = nullptr;
  int K, cin, cout_packed, rate, cout;
};

}  // namespace ev

struct ev_ctx {
  ev_config cfg;
  int device = 0;
  bool bound = false;
  bool has_am = false, has_voc = false;
  bool has_tc = false;      // every '.tc' tensor the tf32 path needs is present
  int precision = EV_PREC_FP32;
  const float* mel_w_tc = nullptr;
  const float* mel_w_h = nullptr;
  const float* mel_w_x2 = nullptr;
  const float* cond_wx_tc = nullptr;   // a blob may carry only one half (PromptTTS / Generator used alone)
  std::unordered_map<std::string, ev::Tensor> tensors;
  const float* pe = nullptr;
  int pe_len = 0;
  // resolved weights
  const float *emb_word = nullptr, *emb_spk = nullptr;
  ev::StackW enc, dec;
  const float *cond_wx, *cond_wc, *cond_b;
  ev::PredW dur, pitch, energy;
  const float *pemb_w, *pemb_b, *eemb_w, *eemb_b;
  const float *mel_w, *mel_b;
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
  float *X, *ACC, *part;
  size_t part_cap;
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
  o->part_cap = n / 2;                  // split-K partials of the first (widest-channel) stage: 2 slices of B*r0*F*C1
  o->part = cv.take(o->part_cap);
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
    EV_TRY(find(c, q + ".wqkv", H * 3 * H, &l.wqkv));
    EV_TRY(find(c, q + ".bqkv", 3 * H, &l.bqkv));
    EV_TRY(find(c, q + ".wo", H * H, &l.wo));
    EV_TRY(find(c, q + ".bo", H, &l.bo));
    EV_TRY(find(c, q + ".ln2.w", H, &l.ln2w));
    EV_TRY(find(c, q + ".ln2.b", H, &l.ln2b));
    EV_TRY(find(c, q + ".w1", K * H * 4 * H, &l.w1));
    EV_TRY(find(c, q + ".b1", 4 * H, &l.b1));
    EV_TRY(find(c, q + ".w2", K * 4 * H * H, &l.w2));
    EV_TRY(find(c, q + ".b2", H, &l.b2));
    l.wqkv_tc = find_opt(c, q + ".wqkv.tc", 2 * H * 3 * H);
    l.wo_tc = find_opt(c, q + ".wo.tc", 2 * H * H);
    l.w1_tc = find_opt(c, q + ".w1.tc", 2 * K * H * 4 * H);
    l.w2_tc = find_opt(c, q + ".w2.tc", 2 * K * 4 * H * H);
    l.wqkv_h = find_opt(c, q + ".wqkv.tc16", H * 3 * H / 2);
    l.wo_h = find_opt(c, q + ".wo.tc16", H * H / 2);
    l.w1_h = find_opt(c, q + ".w1.tc16", K * H * 4 * H / 2);
    l.w2_h = find_opt(c, q + ".w2.tc16", K * 4 * H * H / 2);
    l.wqkv_x2 = find_opt(c, q + ".wqkv.tc16x2", H * 3 * H);
    l.wo_x2 = find_opt(c, q + ".wo.tc16x2", H * H);
    l.w1_x2 = find_opt(c, q + ".w1.tc16x2", K * H * 4 * H);
    l.w2_x2 = find_opt(c, q + ".w2.tc16x2", K * 4 * H * H);
  }
  EV_TRY(find(c, p + ".lnf.w", H, &s->lnfw));
  EV_TRY(find(c, p + ".lnf.b", H, &s->lnfb));
  return EV_OK;
}

static int resolve_pred(ev_ctx* c, const char* pre, int n_layers, PredW* s) {
  const uint64_t H = c->cfg.hidden, K = c->cfg.pred_kernel;
  std::string p(pre);
  s->w.resize(n_layers); s->b.resize(n_layers); s->lnw.resize(n_layers); s->lnb.resize(n_layers); s->w_tc.resize(n_layers);
  for (int i = 0; i < n_layers; ++i) {
    std::string q = p + "." + std::to_string(i);
    EV_TRY(find(c, q + ".w", K * H * H, &s->w[i]));
    s->w_tc[i] = find_opt(c, q + ".w.tc", 2 * K * H * H);
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
  EV_TRY(find(c, "cond.wx", H * H, &c->cond_wx));
  c->cond_wx_tc = find_opt(c, "cond.wx.tc", 2 * H * H);
  EV_TRY(find(c, "cond.wc", (H + 2 * (uint64_t)g.bert_dim) * H, &c->cond_wc));
  EV_TRY(find(c, "cond.b", H, &c->cond_b));
  EV_TRY(resolve_pred(c, "dur", g.dur_layers, &c->dur));
  EV_TRY(resolve_pred(c, "pitch", g.pitch_layers, &c->pitch));
  EV_TRY(resolve_pred(c, "energy", g.energy_layers, &c->energy));
  EV_TRY(find(c, "pitch_emb.w", (uint64_t)g.embed_kernel * H, &c->pemb_w));
  EV_TRY(find(c, "pitch_emb.b", H, &c->pemb_b));
  EV_TRY(find(c, "energy_emb.w", (uint64_t)g.embed_kernel * H, &c->eemb_w));
  EV_TRY(find(c, "energy_emb.b", H, &c->eemb_b));
  EV_TRY(find(c, "to_mel.w", H * g.n_mels, &c->mel_w));
  EV_TRY(find(c, "to_mel.b", g.n_mels, &c->mel_b));
  c->mel_w_tc = find_opt(c, "to_mel.w.tc", 2 * H * g.n_mels);
  c->mel_w_h = find_opt(c, "to_mel.w.tc16", H * g.n_mels / 2);
  c->mel_w_x2 = find_opt(c, "to_mel.w.tc16x2", H * g.n_mels);
  return EV_OK;
}

static int resolve_voc(ev_ctx* c) {
  const ev_config& g = c->cfg;
  c->pre.K = 7; c->pre.dil = 1; c->pre.cin = g.n_mels; c->pre.cout = g.voc_c0;
  EV_TRY(find(c, "voc.pre.w", (uint64_t)7 * g.n_mels * g.voc_c0, &c->pre.w));
  EV_TRY(find(c, "voc.pre.b", g.voc_c0, &c->pre.b));
  c->pre.w_tc = find_opt(c, "voc.pre.w.tc", (uint64_t)2 * 7 * g.n_mels * g.voc_c0);
  c->pre.w_h = find_opt(c, "voc.pre.w.tc16", (uint64_t)7 * g.n_mels * g.voc_c0 / 2);
  c->pre.w_x2 = find_opt(c, "voc.pre.w.tc16x2", (uint64_t)7 * g.n_mels * g.voc_c0);
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
    u.w = it->second.p;
    u.w_tc = find_opt(c, q + ".w.tc", 2 * it->second.numel);
    u.w_h = find_opt(c, q + ".w.tc16", it->second.numel / 2);
    u.w_x2 = find_opt(c, q + ".w.tc16x2", it->second.numel);
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
        EV_TRY(find(c, r + ".c1." + std::to_string(l) + ".w", (uint64_t)k * ch * ch, &c1.w));
        EV_TRY(find(c, r + ".c1." + std::to_string(l) + ".b", ch, &c1.b));
        EV_TRY(find(c, r + ".c2." + std::to_string(l) + ".w", (uint64_t)k * ch * ch, &c2.w));
        EV_TRY(find(c, r + ".c2." + std::to_string(l) + ".b", ch, &c2.b));
        c1.w_tc = find_opt(c, r + ".c1." + std::to_string(l) + ".w.tc", (uint64_t)2 * k * ch * ch);
        c2.w_tc = find_opt(c, r + ".c2." + std::to_string(l) + ".w.tc", (uint64_t)2 * k * ch * ch);
        c1.w_h = find_opt(c, r + ".c1." + std::to_string(l) + ".w.tc16", (uint64_t)k * ch * ch / 2);
        c2.w_h = find_opt(c, r + ".c2." + std::to_string(l) + ".w.tc16", (uint64_t)k * ch * ch / 2);
        c1.w_x2 = find_opt(c, r + ".c1." + std::to_string(l) + ".w.tc16x2", (uint64_t)k * ch * ch);
        c2.w_x2 = find_opt(c, r + ".c2." + std::to_string(l) + ".w.tc16x2", (uint64_t)k * ch * ch);
        c->rb_c1.push_back(c1); c->rb_c2.push_back(c2);
      }
  }
  c->total_up = mul;
  c->post_k = 7;
  EV_TRY(find(c, "voc.post.w", (uint64_t)7 * ch, &c->post_w));
  EV_TRY(find(c, "voc.post.b", 1, &c->post_b));
  return EV_OK;
}

static int conv(const float* x, const float* w, const float* bias, long long bias_bs, const float* res, float* out,
                int B, int L, int Cin, int Cout, int K, int dil, const int32_t* lens, int lens_mul, int in_act,
                float in_slope, int out_act, int acc, float div, cudaStream_t st) {
  ConvParams p;
  p.x = x; p.w = w; p.bias = bias; p.res = res; p.out = out; p.bias_bs = bias_bs;
  p.B = B; p.L = L; p.Cin = Cin; p.Cout = Cout; p.K = K; p.dil = dil;
  p.lens = lens; p.lens_mul = lens_mul; p.in_act = in_act; p.in_slope = in_slope;
  p.out_act = out_act; p.acc = acc; p.div = div;
  return launch_conv1d(p, st);
}

// mode 0: fp32 FFMA kernel; 1: tensor cores, one tf32 MMA per K step; 3: tensor cores, 3xTF32 fp32 emulation;
// 2: tensor cores, bf16 operands (needs w_h; layers without bf16 weights run 3xTF32).
// Falls back to the FFMA kernel when the layer has no tensor-core weights or an unsupported shape.
struct SplitWs {
  float* p = nullptr;
  size_t cap = 0;
  int ksplit = 0;     // K-split factor for the convs launched next (set per layer, see conv1d_tc.cu)
};
static thread_local SplitWs g_split_ws;   // set by the phase entry points for the convs they launch

static int set_split_ws(float* part, size_t cap, int ksplit) {
  g_split_ws = SplitWs{};
  g_split_ws.p = part; g_split_ws.cap = part ? cap : 0; g_split_ws.ksplit = ksplit;
  return EV_OK;
}

// bf16x3 in the decoder (fp32 mode): EV_AM_FP32=tf32x3 keeps 3xTF32 there as well
static inline bool am_bf16x3_enabled() {
  static const int v = [] { const char* e = getenv("EV_AM_FP32"); return (e && e[0] == 't') ? 0 : 1; }();
  return v == 1;
}
// w_x2: two bf16 planes; when given (decoder layers only) and the mode is the fp32-accurate one (3), the layer runs the bf16x3
// emulation instead of 3xTF32.  The duration-critical prefix never passes it.
static int conv_x(int mode, const float* w_tc, const float* w_h, const float* x, const float* w, const float* bias,
                  long long bias_bs, const float* res, float* out, int B, int L, int Cin, int Cout, int K, int dil,
                  const int32_t* lens, int lens_mul, int in_act, float in_slope, int out_act, int acc, float div,
                  cudaStream_t st, const float* w_x2 = nullptr) {
  const bool x3b = mode == 3 && w_x2 && (Cin % 16) == 0 && am_bf16x3_enabled();
  if (mode == 2 && (!w_h || (Cin % 16))) mode = 3;
  if (mode == 0 || (mode != 2 && !w_tc) || (Cin % 8) || (Cout % 16) || (Cout > 128 && Cout % 128))
    return conv(x, w, bias, bias_bs, res, out, B, L, Cin, Cout, K, dil, lens, lens_mul, in_act, in_slope, out_act, acc, div, st);
  ConvParams p;
  p.x = x; p.w = x3b ? w_x2 : ((mode == 2) ? w_h : w_tc); p.bias = bias; p.res = res; p.out = out; p.bias_bs = bias_bs;
  p.B = B; p.L = L; p.Cin = Cin; p.Cout = Cout; p.K = K; p.dil = dil;
  p.lens = lens; p.lens_mul = lens_mul; p.in_act = in_act; p.in_slope = in_slope;
  p.out_act = out_act; p.acc = acc; p.div = div;
  p.splitk_ws = g_split_ws.p; p.splitk_cap = g_split_ws.cap; p.ksplit = g_split_ws.ksplit;
  return launch_conv1d_tc(p, x3b ? 3 : (mode == 3 ? 1 : (mode == 2 ? 2 : 0)), st);
}

// HiFi-GAN convolution on granule-planar activations (conv1d_gp.cu).  mode as conv_x: 1 = tf32, 2 = bf16 (bf16 activations), 3 = 3xTF32.
// In the fp32-accurate mode (3) the vocoder runs the "bf16x3" emulation when the blob carries the two-plane bf16 weights (half the
// tensor-core and shared-memory cost of 3xTF32, ~1e-5 relative error; EV_VOC_FP32=tf32x3 keeps 3xTF32).
static inline bool voc_bf16x3_enabled() {
  static const int v = [] { const char* e = getenv("EV_VOC_FP32"); return (e && e[0] == 't') ? 0 : 1; }();
  return v == 1;
}
static int gp_params(int mode, const float* w_tc, const float* w_h, const float* w_x2, const void* x, const float* bias, const void* res, void* out,
                     int B, int L, int Cin, int Cout, int K, int dil, int rate, const int32_t* lens, int lens_mul, int in_act, float in_slope, int acc,
                     float div, GpConvParams* o) {      // returns the kernel mode
  GpConvParams& p = *o;
  const bool x3b = mode == 3 && w_x2 && voc_bf16x3_enabled();
  p.x = x; p.w = x3b ? w_x2 : ((mode == 2) ? w_h : w_tc); p.bias = bias; p.res = res; p.out = out;
  p.B = B; p.L = L; p.Cin = Cin; p.Cout = Cout; p.K = K; p.dil = dil; p.rate = rate;
  p.lens = lens; p.lens_mul = lens_mul; p.in_act = in_act; p.in_slope = in_slope; p.acc = acc; p.div = div;
  return x3b ? 3 : (mode == 3 ? 1 : (mode == 2 ? 2 : 0));
}
static int conv_gp(int mode, const float* w_tc, const float* w_h, const float* w_x2, const void* x, const float* bias, const void* res, void* out,
                   int B, int L, int Cin, int Cout, int K, int dil, int rate, const int32_t* lens, int lens_mul, int in_act, float in_slope, int acc,
                   float div, cudaStream_t st) {
  GpConvParams p;
  const int gm = gp_params(mode, w_tc, w_h, w_x2, x, bias, res, out, B, L, Cin, Cout, K, dil, rate, lens, lens_mul, in_act, in_slope, acc, div, &p);
  return launch_conv1d_gp(p, gm, st);
}

// One ResBlock layer through the fused kernel (resblock_gp.cu) where it takes the shape (C <= 128); EV_FUSE_RES=0 keeps two launches.
static inline bool fuse_res_enabled() {
  static const int v = [] { const char* e = getenv("EV_FUSE_RES"); return (e && e[0] == '0') ? 0 : 1; }();
  return v == 1;
}
static bool try_gp_pair(int mode, const ConvW& c1, const ConvW& c2, const void* src, void* dst, int B, int L, int C, const int32_t* lens, int lens_mul,
                        int acc, float div, cudaStream_t st, int* rc, bool dry_run = false, GpPairParams* p_out = nullptr, int* gm_out = nullptr) {
  if (!fuse_res_enabled() || c1.K != c2.K || c2.dil != 1) return false;
  // Fused and unfused are bitwise equal, so the choice may depend on the batch: measured (profiles/r02_fused_vs_unfused.jsonl) the fused
  // layer wins 1.1-1.8x on the HBM-bound shapes (k <= 7, or 32 channels) and wherever the launch count matters (batch 1), and loses
  // ~25 % on 64 channels x 11 taps once the batch is large enough to be tensor / issue bound.
  if (C >= 64 && c1.K > 7 && (long long)B * L > 4ll * 70000) return false;
  const bool x3b = mode == 3 && c1.w_x2 && c2.w_x2 && voc_bf16x3_enabled();
  const int gm = x3b ? 3 : (mode == 3 ? 1 : (mode == 2 ? 2 : 0));
  GpPairParams p;
  p.x = src; p.out = dst; p.b1 = c1.b; p.b2 = c2.b;
  p.w1 = x3b ? c1.w_x2 : (mode == 2 ? c1.w_h : c1.w_tc);
  p.w2 = x3b ? c2.w_x2 : (mode == 2 ? c2.w_h : c2.w_tc);
  p.B = B; p.L = L; p.C = C; p.K = c1.K; p.dil = c1.dil; p.lens = lens; p.lens_mul = lens_mul; p.slope = 0.1f; p.acc = acc; p.div = div;
  if (!p.w1 || !p.w2 || !gp_pair_supported(p, gm)) return false;
  if (p_out) *p_out = p;
  if (gm_out) *gm_out = gm;
  if (!dry_run) *rc = launch_gp_pair(p, gm, st);
  return true;
}

// One HiFi-GAN stage's ResBlocks (hifigan/models.py:120-126) with the three parallel blocks advancing together: the same-index
// convolutions of the blocks (different taps / dilations / weights, one shape) are ONE launch.  Used while a single convolution has
// fewer than two waves of tiles (batch 1: 68 / 135 tiles on 132 SMs); every tile is computed as in the ungrouped launches, so the
// result is bitwise the same.  The last c2 of each block accumulates into xs in block order (three plain launches).
// Returns false (nothing launched) when the stage does not qualify.
static bool try_grouped_stage(ev_ctx* ctx, const VocBufs& v, int mode, size_t rb0, int B, int L, int C, const int32_t* lens, int mul, cudaStream_t st, int* rc) {
  const ev_config& g = ctx->cfg;
  const int J = g.n_resk, D = g.n_dil;
  if (!v.G0 || J < 2 || J > 3 || D < 1) return false;
  void* T[3] = {v.Tm, v.G0, v.G1};
  void* Y[3] = {v.R1, v.R2, v.G2};
  int frc = EV_OK;
  // qualify: the stage's layers either all take the fused-pair kernel or none does, every step's members can share a launch, and
  // one member alone is small
  GpConvParams ps[3];
  GpPairParams pp[3];
  int gm = 0, n_pair = 0;
  for (int l = 0; l < D; ++l)
    for (int j = 0; j < J; ++j)
      n_pair += try_gp_pair(mode, ctx->rb_c1[rb0 + (size_t)j * D + l], ctx->rb_c2[rb0 + (size_t)j * D + l], v.X, Y[j], B, L, C, lens, mul, EV_ACC_STORE, 1.f, st,
                            &frc, true) ? 1 : 0;
  if (n_pair == J * D) {
    // ---- fused layers: layer l of the three blocks is one launch (x -> Y, Y -> T, T -> Y, ...); the last layer accumulates into
    // ---- xs block by block (three single launches) ----------------------------------------------------------------------------
    for (int l = 0; l < D; ++l) {
      for (int j = 0; j < J; ++j)
        try_gp_pair(mode, ctx->rb_c1[rb0 + (size_t)j * D + l], ctx->rb_c2[rb0 + (size_t)j * D + l], v.X, Y[j], B, L, C, lens, mul, EV_ACC_STORE, 1.f, st, &frc, true,
                    &pp[j], &gm);
      if (!gp_pair_group_supported(pp, J, gm)) return false;
    }
    if (gp_pair_solo_tiles(pp[0], gm) >= 2 * sm_count()) return false;
    *rc = EV_OK;
    for (int l = 0; l < D && *rc == EV_OK; ++l) {
      const bool last = (l == D - 1);
      // fp32 storage: the last layer is grouped too, into the blocks' own tensors, and one elementwise pass forms ((y1 + y0) + y2) / n
      // -- the additions of the accumulate modes in their order, identical bits.  (With bf16 storage xs is rounded after every
      // accumulation, which that pass cannot reproduce: three single launches.)
      const bool sum_pass = last && gm != 2 && D >= 2;
      for (int j = 0; j < J; ++j) {
        const void* src = l == 0 ? (const void*)v.X : ((l & 1) ? Y[j] : T[j]);
        void* dst = (last && !sum_pass) ? (void*)v.ACC : ((l & 1) ? T[j] : Y[j]);
        int acc = EV_ACC_STORE;
        if (last && !sum_pass && j > 0) acc = (j == J - 1) ? EV_ACC_ADD_DIV : EV_ACC_ADD;
        try_gp_pair(mode, ctx->rb_c1[rb0 + (size_t)j * D + l], ctx->rb_c2[rb0 + (size_t)j * D + l], src, dst, B, L, C, lens, mul, acc, (float)J, st, &frc, true,
                    &pp[j], &gm);
      }
      if (!last || sum_pass) {
        *rc = launch_gp_pair_group(pp, J, gm, st);
        if (sum_pass && *rc == EV_OK)
          *rc = launch_gp_sum_div((const float*)pp[0].out, (const float*)pp[1].out, J == 3 ? (const float*)pp[2].out : nullptr, v.ACC, (size_t)B * L * C, (float)J, st);
      } else {
        for (int j = 0; j < J && *rc == EV_OK; ++j) *rc = launch_gp_pair(pp[j], gm, st);
      }
    }
    return true;
  }
  if (n_pair != 0) return false;
  for (int l = 0; l < D; ++l) {
    for (int j = 0; j < J; ++j) {
      const ConvW& c1 = ctx->rb_c1[rb0 + (size_t)j * D + l];
      gm = gp_params(mode, c1.w_tc, c1.w_h, c1.w_x2, v.X, c1.b, nullptr, T[j], B, L, C, C, c1.K, c1.dil, 1, lens, mul, EV_ACT_LRELU, 0.1f, EV_ACC_STORE, 1.f, &ps[j]);
      if (!ps[j].w) return false;
    }
    if (!gp_group_supported(ps, J, gm)) return false;
    for (int j = 0; j < J; ++j) {
      const ConvW& c2 = ctx->rb_c2[rb0 + (size_t)j * D + l];
      gp_params(mode, c2.w_tc, c2.w_h, c2.w_x2, T[j], c2.b, v.X, Y[j], B, L, C, C, c2.K, 1, 1, lens, mul, EV_ACT_LRELU, 0.1f, EV_ACC_STORE, 1.f, &ps[j]);
      if (!ps[j].w) return false;
    }
    if (!gp_group_supported(ps, J, gm)) return false;
  }
  if (gp_solo_tiles(ps[0], gm) >= 2 * sm_count()) return false;
  *rc = EV_OK;
  for (int l = 0; l < D && *rc == EV_OK; ++l) {
    const bool last = (l == D - 1);
    const bool sum_pass = last && gm != 2 && D >= 2;      // see the fused path above
    for (int j = 0; j < J; ++j) {      // xt_j = c1_j(lrelu(x_j))
      const ConvW& c1 = ctx->rb_c1[rb0 + (size_t)j * D + l];
      gp_params(mode, c1.w_tc, c1.w_h, c1.w_x2, l == 0 ? (const void*)v.X : Y[j], c1.b, nullptr, T[j], B, L, C, C, c1.K, c1.dil, 1, lens, mul, EV_ACT_LRELU, 0.1f,
                EV_ACC_STORE, 1.f, &ps[j]);
    }
    *rc = launch_conv1d_gp_group(ps, J, gm, st);
    if (*rc != EV_OK) break;
    for (int j = 0; j < J; ++j) {      // x_j = c2_j(lrelu(xt_j)) + x_j  (in place from the second layer on: a thread reads and writes its own elements)
      const ConvW& c2 = ctx->rb_c2[rb0 + (size_t)j * D + l];
      const void* res = l == 0 ? (const void*)v.X : Y[j];
      int acc = EV_ACC_STORE;
      if (last && j > 0) acc = (j == J - 1) ? EV_ACC_ADD_DIV : EV_ACC_ADD;       // xs += ...; x = xs / n
      if (sum_pass) acc = EV_ACC_STORE;
      gp_params(mode, c2.w_tc, c2.w_h, c2.w_x2, T[j], c2.b, res, (last && !sum_pass) ? (void*)v.ACC : Y[j], B, L, C, C, c2.K, 1, 1, lens, mul, EV_ACT_LRELU, 0.1f, acc,
                (float)J, &ps[j]);
    }
    if (!last || sum_pass) {
      *rc = launch_conv1d_gp_group(ps, J, gm, st);
      if (sum_pass && *rc == EV_OK)
        *rc = launch_gp_sum_div((const float*)Y[0], (const float*)Y[1], J == 3 ? (const float*)Y[2] : nullptr, v.ACC, (size_t)B * L * C, (float)J, st);
    } else {
      for (int j = 0; j < J && *rc == EV_OK; ++j) *rc = launch_conv1d_gp(ps[j], gm, st);
    }
  }
  return true;
}

// The vocoder runs on granule-planar activations whenever it runs on the tensor cores (every mode but "fp32_ffma");
// EV_VOC_LAYOUT=tm keeps the round-1 time-major path (conv1d_tc.cu) for A/B measurements.
static inline bool voc_gp_enabled() {
  static const int v = [] { const char* e = getenv("EV_VOC_LAYOUT"); return (e && e[0] == 't') ? 0 : 1; }();
  return v == 1;
}

static inline int body_mode(const ev_ctx* c) {
  return c->precision == EV_PREC_FP32_FFMA ? 0 : (c->precision == EV_PREC_TF32 ? 1 : (c->precision == EV_PREC_BF16 ? 2 : 3));
}

static inline bool attn_tc_enabled() {
  static const int v = [] { const char* e = getenv("EV_ATTN"); return (e && e[0] == 'f') ? 0 : 1; }();
  return v == 1;
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
                     int B, int L, const int32_t* key_lens, const int32_t* conv_lens, bool first_ln_done, int mode,
                     const StackSplits& sp, cudaStream_t st) {
  const int H = c->cfg.hidden, K = c->cfg.ffn_kernel, heads = c->cfg.n_heads;
  for (size_t i = 0; i < s.layers.size(); ++i) {
    const EncLayerW& l = s.layers[i];
    if (!(i == 0 && first_ln_done))
      EV_TRY(launch_layernorm(x, nullptr, nullptr, nullptr, nullptr, nullptr, l.ln1w, l.ln1b, y, B * L, L, H, st));
    g_split_ws.ksplit = sp.qkv;
    EV_TRY(conv_x(mode, l.wqkv_tc, l.wqkv_h, y, l.wqkv, l.bqkv, 0, nullptr, qkv, B, L, H, 3 * H, 1, 1, conv_lens, 1, EV_ACT_NONE, 0.f,
                  EV_ACT_NONE, EV_ACC_STORE, 1.f, st, l.wqkv_x2));
    // QK^T / softmax / PV: tensor cores (3xTF32 where the layer runs fp32-accurate, one tf32 MMA otherwise) for d_k = 48; the fp32 FFMA
    // flash kernel in the "fp32_ffma" mode, for other head sizes, or with EV_ATTN=ffma (A/B measurements)
    if (mode != 0 && H / heads == 48 && attn_tc_enabled())
      EV_TRY(launch_attention_tc(qkv, key_lens, ctxb, B, L, H, heads, mode == 3 ? 1 : 0, st));
    else
      EV_TRY(launch_attention(qkv, key_lens, ctxb, B, L, H, heads, st));
    g_split_ws.ksplit = sp.wo;
    EV_TRY(conv_x(mode, l.wo_tc, l.wo_h, ctxb, l.wo, l.bo, 0, x, x, B, L, H, H, 1, 1, conv_lens, 1, EV_ACT_NONE, 0.f, EV_ACT_NONE,
                  EV_ACC_STORE, 1.f, st, l.wo_x2));
    EV_TRY(launch_layernorm(x, nullptr, nullptr, nullptr, nullptr, nullptr, l.ln2w, l.ln2b, y, B * L, L, H, st));
    g_split_ws.ksplit = sp.ffn1;
    EV_TRY(conv_x(mode, l.w1_tc, l.w1_h, y, l.w1, l.b1, 0, nullptr, h, B, L, H, 4 * H, K, 1, conv_lens, 1, EV_ACT_NONE, 0.f, EV_ACT_GELU,
                  EV_ACC_STORE, 1.f, st, l.w1_x2));
    g_split_ws.ksplit = sp.ffn2;
    EV_TRY(conv_x(mode, l.w2_tc, l.w2_h, h, l.w2, l.b2, 0, x, x, B, L, 4 * H, H, K, 1, conv_lens, 1, EV_ACT_NONE, 0.f, EV_ACT_NONE,
                  EV_ACC_STORE, 1.f, st, l.w2_x2));
  }
  g_split_ws.ksplit = 2;
  EV_TRY(launch_layernorm(x, nullptr, nullptr, nullptr, nullptr, nullptr, s.lnfw, s.lnfb, y, B * L, L, H, st));
  return EV_OK;
}

// [conv k -> ReLU -> channel LN] x n -> Linear(H -> 1) (variance.py:36-56, :101-124)
static int run_predictor(const ev_ctx* c, const PredW& p, const float* in, float* t1, float* t2, int B, int T,
                         const int32_t* lens, const int32_t* conv_lens, int mode, float* out_f, int64_t* out_i,
                         int cmode, cudaStream_t st) {
  const int H = c->cfg.hidden, K = c->cfg.pred_kernel;
  g_split_ws.ksplit = 8;      // K = 3H on ~100 tokens and 3 N tiles: eight slices (see StackSplits)
  const float* cur = in;
  for (size_t i = 0; i < p.w.size(); ++i) {
    EV_TRY(conv_x(cmode, p.w_tc[i], nullptr, cur, p.w[i], p.b[i], 0, nullptr, t1, B, T, H, H, K, 1, conv_lens, 1, EV_ACT_NONE, 0.f,
                  EV_ACT_RELU, EV_ACC_STORE, 1.f, st));
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
    if (first_use_on_device(loaded)) { preload_conv1d_gp(); preload_resblock_gp(); preload_attention_tc(); preload_conv1d_tc(); }
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
  EV_TRY(set_split_ws(b.part, b.part_cap, 2));
  // lengths -> int32, plus range checks of ids / speakers / lengths into the status word mel_lens_out[B + 1]
  EV_TRY(launch_validate_inputs(ling, lens64, spk, lens32_out, mel_lens_out + B + 1, B, T, g.n_vocab, g.n_speaker, st));
  const int32_t* lens = lens32_out;
  const int32_t* conv_lens = invariant ? lens : nullptr;
  // the duration-critical prefix is fp32-accurate in every mode: 3xTF32 on the tensor cores, or FFMA
  const int prefix_mode = (ctx->precision == EV_PREC_FP32_FFMA) ? 0 : 3;

  Range r_phase("ev:am_phase1");
  // encoder: x = word_emb[ids] + alpha*pe (model_open_source.py:107, encoder.py:257-261), fused with LN1 of layer 0
  EV_TRY(launch_layernorm(nullptr, ling, ctx->emb_word, ctx->pe, ctx->enc.alpha, b.x, ctx->enc.layers[0].ln1w,
                          ctx->enc.layers[0].ln1b, b.y, B * T, T, H, st, g.n_vocab));
  EV_TRY(run_stack(ctx, ctx->enc, b.x, b.y, b.qkv, b.ctx, b.h, B, T, lens, conv_lens, true, prefix_mode, kEncSplits, st));
  g_split_ws.ksplit = 4;
  // conditioning (model_open_source.py:109-111): per-utterance bias + W_x x
  EV_TRY(launch_cond_gather(spk, ctx->emb_spk, style, content, b.cond_in, B, H, g.bert_dim, g.n_speaker, st));
  EV_TRY(launch_cond_gemv(b.cond_in, ctx->cond_wc, ctx->cond_b, b.cond_bias, B, H + 2 * g.bert_dim, H, st));
  EV_TRY(conv_x(prefix_mode, ctx->cond_wx_tc, nullptr, b.y, ctx->cond_wx, b.cond_bias, H, nullptr, b.hs, B, T, H, H, 1, 1, conv_lens, 1,
                EV_ACT_NONE, 0.f, EV_ACT_NONE, EV_ACC_STORE, 1.f, st));
  // predictors (model_open_source.py:120-121,130)
  const float* pin = b.hs;
  if (!invariant) {   // literal batch: masked_fill on the input only (variance.py:38-39); pads of hs are live data
    EV_TRY(launch_mask_rows(b.hs, lens, b.pm, B, T, H, st));
    pin = b.pm;
  }
  EV_TRY(run_predictor(ctx, ctx->pitch, pin, b.p1[0], b.p2[0], B, T, lens, conv_lens, 0, pitch_out, nullptr, prefix_mode, st));
  EV_TRY(run_predictor(ctx, ctx->energy, pin, b.p1[1], b.p2[1], B, T, lens, conv_lens, 0, energy_out, nullptr, prefix_mode, st));
  EV_TRY(run_predictor(ctx, ctx->dur, pin, b.p1[2], b.p2[2], B, T, lens, conv_lens, 1, nullptr, dur_out, prefix_mode, st));
  // x = x + pitch_embed + energy_embed (model_open_source.py:131-134), the tracks shifted / scaled per item when prosody is given
  EV_TRY(launch_var_embed_add(b.hs, pitch_out, energy_out, ctx->pemb_w, ctx->pemb_b, ctx->eemb_w, ctx->eemb_b, prosody, conv_lens,
                              B, T, H, g.embed_kernel, st));
  // duration bookkeeping for the length regulator (alignment.py:183-199), durations scaled by alpha = prosody[b*5]
  EV_TRY(launch_duration_scan(dur_out, lens, prosody, 5, invariant, B, T, b.centers, b.ds_f, mel_lens_out, mel_lens_out + B + 1, st));
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
  EV_TRY(set_split_ws(b.part, b.part_cap, 2));
  Range r_phase("ev:am_phase2");
  // length regulator + the decoder's positional encoding (alignment.py:198-211, encoder.py:257-261)
  EV_TRY(launch_gauss_upsample(b1.hs, b1.centers, lens, mel_lens, B, T, H, F, invariant, ctx->pe, ctx->dec.alpha, b.x, st));
  // decoder (model_open_source.py:146: mask None in the reference; per-item lengths under the invariant contract)
  const int mode = body_mode(ctx);
  EV_TRY(run_stack(ctx, ctx->dec, b.x, b.y, b.qkv, b.ctx, b.h, B, F, flens, flens, false, mode, kDecSplits, st));
  g_split_ws.ksplit = 2;
  // to_mel (model_open_source.py:147)
  EV_TRY(conv_x(mode, ctx->mel_w_tc, ctx->mel_w_h, b.y, ctx->mel_w, ctx->mel_b, 0, nullptr, mel_out, B, F, H, g.n_mels, 1, 1, flens, 1,
                EV_ACT_NONE, 0.f, EV_ACT_NONE, EV_ACC_STORE, 1.f, st, ctx->mel_w_x2));
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
  const int mode = body_mode(ctx);
  if (mode != 0 && voc_gp_enabled()) {
    // ---- granule-planar path: [b][C/cpg][l][cpg] activations, bulk-copied A operands, direct coalesced epilogues ----
    Range r_phase("ev:vocoder");
    const int bf = (mode == 2) ? 1 : 0;
    // mel (B,F,n_mels) time-major or (B,n_mels,F) channels-first -> GP
    EV_TRY(launch_to_gp(mel, (long long)F * g.n_mels, mel_time_major ? g.n_mels : 1, mel_time_major ? 1 : F, v.Tm, B, F, g.n_mels, bf, st));
    // conv_pre (hifigan/models.py:116)
    EV_TRY(conv_gp(mode, ctx->pre.w_tc, ctx->pre.w_h, ctx->pre.w_x2, v.Tm, ctx->pre.b, nullptr, v.ACC, B, F, g.n_mels, g.voc_c0, ctx->pre.K, 1, 1, mel_lens, 1,
                   EV_ACT_NONE, 0.f, EV_ACC_STORE, 1.f, st));
    int L = F, mul = 1;
    size_t rb = 0;
    static const char* const kNames[8] = {"voc:stage1", "voc:stage2", "voc:stage3", "voc:stage4", "voc:stage5", "voc:stage6", "voc:stage7", "voc:stage8"};
    for (int s = 0; s < g.n_ups; ++s) {
      Range r_stage(kNames[s & 7]);
      const UpW& u = ctx->ups[s];
      // x = ups[i](leaky_relu(x, 0.1)) (:118-119): polyphase transposed conv, the `rate` output phases are GEMM column groups
      EV_TRY(conv_gp(mode, u.w_tc, u.w_h, u.w_x2, v.ACC, u.b, nullptr, v.X, B, L, u.cin, u.cout_packed, u.K, 1, u.rate, mel_lens, mul, EV_ACT_LRELU, 0.1f,
                     EV_ACC_STORE, 1.f, st));
      L *= u.rate; mul *= u.rate;
      const int C = u.cout;
      int grc = EV_OK;
      if (try_grouped_stage(ctx, v, mode, rb, B, L, C, mel_lens, mul, st, &grc)) {
        EV_TRY(grc);
        rb += (size_t)g.n_resk * g.n_dil;
        continue;
      }
      for (int j = 0; j < g.n_resk; ++j) {
        const float* src = v.X;
        for (int l = 0; l < g.n_dil; ++l, ++rb) {
          const ConvW& c1 = ctx->rb_c1[rb];
          const ConvW& c2 = ctx->rb_c2[rb];
          const bool last = (l == g.n_dil - 1);
          float* dst = last ? v.ACC : ((l & 1) ? v.R2 : v.R1);
          int acc = EV_ACC_STORE;
          if (last && j > 0) acc = (j == g.n_resk - 1) ? EV_ACC_ADD_DIV : EV_ACC_ADD;   // xs += ...; x = xs / n (:120-126)
          if (last && g.n_resk == 1) acc = EV_ACC_STORE;
          // xt = c1(lrelu(x)) ; x = c2(lrelu(xt)) + x   (:50-57): one fused kernel where the shape fits, else two launches
          int frc = EV_OK;
          if (try_gp_pair(mode, c1, c2, src, dst, B, L, C, mel_lens, mul, acc, (float)g.n_resk, st, &frc)) {
            EV_TRY(frc);
            src = dst;
            continue;
          }
          EV_TRY(conv_gp(mode, c1.w_tc, c1.w_h, c1.w_x2, src, c1.b, nullptr, v.Tm, B, L, C, C, c1.K, c1.dil, 1, mel_lens, mul, EV_ACT_LRELU, 0.1f,
                         EV_ACC_STORE, 1.f, st));
          EV_TRY(conv_gp(mode, c2.w_tc, c2.w_h, c2.w_x2, v.Tm, c2.b, src, dst, B, L, C, C, c2.K, 1, 1, mel_lens, mul, EV_ACT_LRELU, 0.1f, acc,
                         (float)g.n_resk, st));
          src = dst;
        }
      }
    }
    EV_CHECK_ARG(mul == ctx->total_up, "ev_vocoder: internal rate mismatch");
    // x = leaky_relu(x) [slope 0.01]; conv_post; tanh (:127-129)
    return launch_conv_post_gp(v.ACC, bf, ctx->post_w, ctx->post_b, mel_lens, mul, B, L, ctx->ups.back().cout, ctx->post_k, 0.01f, wav_out, st);
  }
  EV_TRY(set_split_ws(v.part, v.part_cap, 0));
  const float* m = mel;
  if (!mel_time_major) {
    EV_TRY(launch_transpose_cf_to_tm(mel, v.Tm, B, g.n_mels, F, st));
    m = v.Tm;
  }
  Range r_phase("ev:vocoder");
  // conv_pre (hifigan/models.py:116)
  EV_TRY(conv_x(mode, ctx->pre.w_tc, ctx->pre.w_h, m, ctx->pre.w, ctx->pre.b, 0, nullptr, v.ACC, B, F, g.n_mels, g.voc_c0, ctx->pre.K, 1,
                mel_lens, 1, EV_ACT_NONE, 0.f, EV_ACT_NONE, EV_ACC_STORE, 1.f, st));
  int L = F, mul = 1;
  size_t rb = 0;
  static const char* const kStageNames[8] = {"voc:stage1", "voc:stage2", "voc:stage3", "voc:stage4", "voc:stage5", "voc:stage6",
                                             "voc:stage7", "voc:stage8"};
  for (int s = 0; s < g.n_ups; ++s) {
    Range r_stage(kStageNames[s & 7]);
    const UpW& u = ctx->ups[s];
    // no K-split in the vocoder: outputs are large, the partial-sum traffic costs more than the shorter reduction gains
    // (measured: 2-slice K-split of stage 1 gains 4.6 % at batch 1 and costs 6 % at batch 32)
    g_split_ws.ksplit = 0;
    // x = ups[i](leaky_relu(x, 0.1)) (:118-119): polyphase-packed transposed conv, output viewed (L, rate*Cout)
    EV_TRY(conv_x(mode, u.w_tc, u.w_h, v.ACC, u.w, u.b, 0, nullptr, v.X, B, L, u.cin, u.cout_packed, u.K, 1, mel_lens, mul,
                  EV_ACT_LRELU, 0.1f, EV_ACT_NONE, EV_ACC_STORE, 1.f, st));
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
        const float div = (float)g.n_resk;
        if (last && g.n_resk == 1) acc = EV_ACC_STORE;
        // xt = c1(lrelu(x)) ; x = c2(lrelu(xt)) + x   (:50-57)
        EV_TRY(conv_x(mode, c1.w_tc, c1.w_h, src, c1.w, c1.b, 0, nullptr, v.Tm, B, L, C, C, c1.K, c1.dil, mel_lens, mul,
                      EV_ACT_LRELU, 0.1f, EV_ACT_NONE, EV_ACC_STORE, 1.f, st));
        EV_TRY(conv_x(mode, c2.w_tc, c2.w_h, v.Tm, c2.w, c2.b, 0, src, dst, B, L, C, C, c2.K, 1, mel_lens, mul, EV_ACT_LRELU, 0.1f,
                      EV_ACT_NONE, acc, div, st));
        src = dst;
      }
    }
  }
  // x = leaky_relu(x) [slope 0.01]; conv_post; tanh (:127-129)
  EV_CHECK_ARG(mul == ctx->total_up, "ev_vocoder: internal rate mismatch");
  const int Cl = ctx->ups.back().cout;
  EV_TRY(launch_conv_post(v.ACC, ctx->post_w, ctx->post_b, mel_lens, mul, B, L, Cl, ctx->post_k, 0.01f, wav_out, st));
  return EV_OK;
}

int ev_wav_to_pcm16(const float* wav, int16_t* pcm, size_t n, void* stream) {
  EV_CHECK_ARG(wav && pcm, "ev_wav_to_pcm16: null argument");
  EV_TRY(use_device_of(wav));
  return launch_pcm16(wav, pcm, n, reinterpret_cast<cudaStream_t>(stream));
}

int ev_op_conv1d(const float* x, const float* w, const float* bias, size_t bias_bstride, const float* res, float* out,
                 int B, int L, int Cin, int Cout, int K, int dil, const int32_t* lens, int lens_mul, int in_act,
                 float in_slope, int out_act, int acc, float div, void* stream) {
  EV_CHECK_ARG(x && w && out, "ev_op_conv1d: null argument");
  EV_TRY(use_device_of(x));
  return conv(x, w, bias, (long long)bias_bstride, res, out, B, L, Cin, Cout, K, dil, lens, lens_mul, in_act, in_slope,
              out_act, acc, div, reinterpret_cast<cudaStream_t>(stream));
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
  EV_TRY(use_device_of(x));
  EV_TRY(set_split_ws(splitk_ws, splitk_floats, splitk_ws ? ksplit : 0));
  EV_CHECK_ARG(Cin % 8 == 0 && Cout % 16 == 0 && (Cout <= 128 || Cout % 128 == 0),
               "ev_op_conv1d_tc: needs Cin %% 8 == 0, Cout %% 16 == 0 and Cout <= 128 or a multiple of 128 (Cin=%d Cout=%d)", Cin, Cout);
  EV_CHECK_ARG(split3 < 2 || Cin % 16 == 0, "ev_op_conv1d_tc: the bf16 / bf16x3 modes need Cin %% 16 == 0 (Cin=%d)", Cin);
  if (split3 == 3) {      // bf16x3: w_tc holds the two bf16 planes
    ConvParams p;
    p.x = x; p.w = w_tc; p.bias = bias; p.res = res; p.out = out; p.bias_bs = (long long)bias_bstride;
    p.B = B; p.L = L; p.Cin = Cin; p.Cout = Cout; p.K = K; p.dil = dil; p.lens = lens; p.lens_mul = lens_mul; p.in_act = in_act; p.in_slope = in_slope;
    p.out_act = out_act; p.acc = acc; p.div = div;
    p.splitk_ws = g_split_ws.p; p.splitk_cap = g_split_ws.cap; p.ksplit = g_split_ws.ksplit;
      return launch_conv1d_tc(p, 3, reinterpret_cast<cudaStream_t>(stream));
  }
  return conv_x(split3 == 2 ? 2 : (split3 ? 3 : 1), w_tc, w_tc, x, nullptr, bias, (long long)bias_bstride, res, out, B, L, Cin, Cout, K, dil, lens, lens_mul,
                in_act, in_slope, out_act, acc, div, reinterpret_cast<cudaStream_t>(stream));
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
  GpConvParams p;
  p.x = x; p.w = w; p.bias = bias; p.res = res; p.out = out; p.B = B; p.L = L; p.Cin = Cin; p.Cout = Cout; p.K = K; p.dil = dil; p.rate = rate;
  p.lens = lens; p.lens_mul = lens_mul; p.in_act = in_act; p.in_slope = in_slope; p.acc = acc; p.div = div;
  return launch_conv1d_gp(p, mode, reinterpret_cast<cudaStream_t>(stream));
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
  if (precision != EV_PREC_FP32_FFMA && ctx->bound) {
    bool ok = true;
    if (ctx->has_am) {
      ok = ok && ctx->mel_w_tc && ctx->cond_wx_tc;
      for (const auto* st : {&ctx->enc, &ctx->dec})
        for (const auto& l : st->layers) ok = ok && l.wqkv_tc && l.wo_tc && l.w1_tc && l.w2_tc;
      for (const auto* pr : {&ctx->dur, &ctx->pitch, &ctx->energy})
        for (const float* w : pr->w_tc) ok = ok && w;
    }
    if (ctx->has_voc) {
      ok = ok && ctx->pre.w_tc;
      for (const auto& u : ctx->ups) ok = ok && u.w_tc;
      for (const auto& c1 : ctx->rb_c1) ok = ok && c1.w_tc;
      for (const auto& c2 : ctx->rb_c2) ok = ok && c2.w_tc;
    }
    if (precision == EV_PREC_BF16) {
      if (ctx->has_am) {
        ok = ok && ctx->mel_w_h;
        for (const auto& l : ctx->dec.layers) ok = ok && l.wqkv_h && l.wo_h && l.w1_h && l.w2_h;
      }
      if (ctx->has_voc) {
        ok = ok && ctx->pre.w_h;
        for (const auto& u : ctx->ups) ok = ok && u.w_h;
        for (const auto& c1 : ctx->rb_c1) ok = ok && c1.w_h;
        for (const auto& c2 : ctx->rb_c2) ok = ok && c2.w_h;
      }
    }
    if (!ok) { set_error("ev_set_precision: the bound blob lacks the '.tc' / '.tc16' (tensor-core layout) weights"); return EV_ENOWEIGHT; }
  }
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
  EV_TRY(launch_duration_scan(dur, lens, nullptr, 0, invariant, B, T, centers_tmp, centers_tmp + (size_t)B * T, mel_lens_tmp, nullptr,
                              st));
  return launch_gauss_upsample(hs, centers_tmp, lens, mel_lens_tmp, B, T, H, F, invariant, pe, alpha, out, st);
}

int ev_op_duration_scan(const int64_t* dur, const int32_t* lens, const float* alpha, int invariant, int B, int T, float* centers,
                        float* ds, int32_t* mel_lens, void* stream) {
  EV_CHECK_ARG(dur && centers && ds && mel_lens, "ev_op_duration_scan: null argument");
  EV_CHECK_ARG(B > 0 && T > 0, "ev_op_duration_scan: B=%d T=%d", B, T);
  EV_TRY(use_device_of(dur));
  return launch_duration_scan(dur, lens, alpha, 1, invariant, B, T, centers, ds, mel_lens, nullptr,
                              reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
