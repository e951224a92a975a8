// FLAC (RFC 9639) file images of int16 items (ev_flac_encode): mono, 16 bits, fixed 4096-sample blocks, byte for byte the
// stream oracle/flac_oracle.py defines (its docstring states every rule; this file follows it).
//
// Four launches.
// flac_analyze_kernel: one CTA per (item, block).  It stages the block as int32 in shared memory and scores every candidate
//   subframe by its exact bit count: CONSTANT (the block is constant), FIXED 0-4, LPC 1-12, VERBATIM, in that order, keeping
//   the first of equal costs.  LPC: integer Welch window and autocorrelation (int64, exact), Levinson-Durbin on one thread in
//   fp64 with every operation rounded on its own (__dmul_rn / __dadd_rn / __dsub_rn / IEEE division), then quantisation.  The
//   Rice cost of a residual: each thread folds <= 16 consecutive residuals into sum(u >> k) for k = 0..14 at the finest allowed
//   partition order, the partials are summed per partition, and each coarser order is the pairwise sum of the finer one.
//   All sums are integers, so the decision is independent of the summation order.  Writes a FlacRec (kind, order, LPC
//   coefficients, partition order and Rice parameters) and the frame's byte count.
// flac_stream_kernel: one CTA per item: exclusive scan of its frames' byte counts (the offset of each frame in the image),
//   the image size and the smallest and largest frame.
// flac_offsets_kernel: one CTA: exclusive scan of the image sizes -> out_off (n_items + 1).
// flac_write_kernel: one CTA per (item, block).  It recomputes the chosen residuals, scans the code lengths for bit
//   offsets and builds the frame in a zeroed shared bit buffer, ORing in only the one bits of each code (a Rice code's
//   unary zeros cost nothing).  CRC-16: per-thread chunk CRCs, each moved to its place by multiplying with x^(8 * bytes after
//   it) mod P, XOR-combined (the CRC is linear).  The CTA of block 0 also writes fLaC and STREAMINFO.
// Samples outside [pcm_off[k], pcm_off[k + 1]) are never read, and each image depends only on its own item.
#include <math.h>

#include "ev_common.cuh"

namespace ev {

constexpr int FL_BLOCK = 4096;
constexpr int FL_THREADS = 256;
constexpr int FL_PER_THREAD = FL_BLOCK / FL_THREADS;     // 16 samples per thread
constexpr int FL_MAX_LPC = 12, FL_MAX_FIXED = 4, FL_MAX_PORDER = 8, FL_MAX_RICE = 14, FL_NK = FL_MAX_RICE + 1;
constexpr int FL_HEADER = 42;                            // fLaC + metadata block header + STREAMINFO
constexpr int FL_FRAME_OVERHEAD = 20;                    // >= frame header (<= 16) + subframe header (1) + CRC-16 (2)
constexpr int FL_MIN_RATE = 4000, FL_MAX_RATE = 192000;
constexpr int FL_BUF_WORDS = (FL_BLOCK * 2 + FL_FRAME_OVERHEAD + 3) / 4 + 1;
enum { FL_CONSTANT = 0, FL_VERBATIM = 1, FL_FIXED = 2, FL_LPC = 3 };

struct FlacRec {
  int kind, order, porder, shift, prec, bytes;
  long long sub_bits;
  short q[FL_MAX_LPC];
  unsigned char kp[1 << FL_MAX_PORDER];
};

struct FlacRate {   // frame-header sample rate field: code, and the trailing field's value and bits (0, 8 or 16)
  int code, value, bits;
};

__host__ __device__ inline int utf8_bytes(long long v) {
  if (v < 0x80) return 1;
  int nb = 2;
  while (nb < 7 && v >= (1ll << (5 * nb + 1))) ++nb;
  return nb;
}

__device__ __forceinline__ int frame_header_bytes(long long index, int n, const FlacRate& r) {
  return 4 + utf8_bytes(index) + (n == FL_BLOCK ? 0 : n <= 256 ? 1 : 2) + r.bits / 8 + 1;
}

__device__ __forceinline__ void item_span(const int64_t* pcm_off, int k, long long max_n, long long& start, int& nf, long long& n) {
  start = pcm_off[k];
  n = min(max((long long)pcm_off[k + 1] - start, 0ll), max_n);
  nf = (int)((n + FL_BLOCK - 1) / FL_BLOCK);
}

// exact residual of a FIXED (order <= 4) or LPC predictor at sample i >= order; false if it leaves int32
__device__ __forceinline__ long long predict_residual(const int* x, int i, int kind, int order, const int* q, int shift) {
  long long s = 0;
  if (kind == FL_FIXED) {
    switch (order) {
      case 1: s = x[i - 1]; break;
      case 2: s = 2ll * x[i - 1] - x[i - 2]; break;
      case 3: s = 3ll * x[i - 1] - 3ll * x[i - 2] + x[i - 3]; break;
      case 4: s = 4ll * x[i - 1] - 6ll * x[i - 2] + 4ll * x[i - 3] - x[i - 4]; break;
      default: break;
    }
  } else {
    for (int j = 0; j < order; ++j) s += (long long)q[j] * x[i - 1 - j];
    s >>= shift;
  }
  return (long long)x[i] - s;
}

__device__ __forceinline__ unsigned long long zigzag(long long r) { return r >= 0 ? (unsigned long long)(2 * r) : (unsigned long long)(-2 * r - 1); }

__device__ __forceinline__ int finest_porder(int n, int order) {
  int o = 0;
  while (o < FL_MAX_PORDER && n % (2 << o) == 0 && (n >> (o + 1)) > order) ++o;
  return o;
}

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

struct AnalyzeSmem {
  int x[FL_BLOCK];
  union {
    int y[FL_BLOCK];                                   // windowed samples (autocorrelation only)
    unsigned long long S[FL_THREADS][FL_NK];            // sum(u >> k): per-thread partials, then per partition
  } u;
  long long r[FL_MAX_LPC + 1];
  unsigned long long level_bits[FL_MAX_PORDER + 1];
  int lq[FL_MAX_LPC][FL_MAX_LPC];
  int lshift[FL_MAX_LPC], lprec[FL_MAX_LPC];
  int n_lpc;
  unsigned char kcur[(2 << FL_MAX_PORDER) - 1];         // level o's parameters at [2^o - 1, 2^(o+1) - 1)
  unsigned char kbest[1 << FL_MAX_PORDER];
  long long best_bits;
  int best_kind, best_order, best_porder, best_lpc, cand_porder;
  long long cand_bits;
};

// Rice cost of one predictor (all threads): returns true and sets s.cand_bits / cand_porder / kcur when the residual fits int32.
__device__ bool rice_cost(AnalyzeSmem& s, int n, int kind, int order, const int* q, int shift) {
  const int t = threadIdx.x;
  const int of = finest_porder(n, order);
  const int parts = 1 << of, psize = n >> of, tpp = FL_THREADS / parts;
  const int chunk = (psize + tpp - 1) / tpp;
  const int part = t / tpp, sub = t % tpp;
  const int i0 = part * psize + sub * chunk, i1 = min(i0 + chunk, (part + 1) * psize);
  unsigned long long acc[FL_NK];
#pragma unroll
  for (int k = 0; k < FL_NK; ++k) acc[k] = 0;
  bool bad = false;
  for (int i = max(i0, order); i < i1; ++i) {
    const long long r = predict_residual(s.x, i, kind, order, q, shift);
    bad |= r < -2147483648ll || r > 2147483647ll;
    const unsigned long long u = zigzag(r);
#pragma unroll
    for (int k = 0; k < FL_NK; ++k) acc[k] += u >> k;
  }
  if (t <= FL_MAX_PORDER) s.level_bits[t] = 0;
  __syncthreads();                                      // the previous candidate's readers of S are done
#pragma unroll
  for (int k = 0; k < FL_NK; ++k) s.u.S[t][k] = acc[k];
  if (__syncthreads_or(bad)) return false;
  for (int st = 1; st < tpp; st <<= 1) {                // per-partition sums at the finest order, into S[part * tpp]
    for (int e = t; e < FL_THREADS * FL_NK; e += FL_THREADS) {
      const int row = e / FL_NK, k = e % FL_NK;
      if (row % (2 * st) == 0) s.u.S[row][k] += s.u.S[row + st][k];
    }
    __syncthreads();
  }
  for (int o = of; o >= 0; --o) {
    const int np = 1 << o, stride = tpp << (of - o);
    unsigned long long c = 0;
    if (t < np) {
      const long long m = (n >> o) - (t == 0 ? order : 0);
      unsigned long long best = ~0ull;
      int kb = 0;
      for (int k = 0; k < FL_NK; ++k) {
        const unsigned long long v = (unsigned long long)m * (k + 1) + s.u.S[t * stride][k];
        if (v < best) { best = v; kb = k; }
      }
      s.kcur[np - 1 + t] = (unsigned char)kb;
      c = best + 4;
    }
    c = warp_sum(c);
    if ((t & 31) == 0 && c) atomicAdd(&s.level_bits[o], c);
    __syncthreads();
    if (o > 0) {                                        // level o - 1: pairwise sums
      for (int e = t; e < (np / 2) * FL_NK; e += FL_THREADS) {
        const int j = e / FL_NK, k = e % FL_NK;
        s.u.S[2 * j * stride][k] += s.u.S[(2 * j + 1) * stride][k];
      }
      __syncthreads();
    }
  }
  if (t == 0) {
    int bo = 0;
    for (int o = 1; o <= of; ++o)
      if (s.level_bits[o] < s.level_bits[bo]) bo = o;
    s.cand_porder = bo;
    s.cand_bits = 6 + (long long)s.level_bits[bo];
  }
  __syncthreads();
  return true;
}

__device__ void consider(AnalyzeSmem& s, long long bits, int kind, int order, int lpc, bool with_params) {
  // thread 0 decides, every thread copies the parameters of a new best
  __shared__ int take;
  if (threadIdx.x == 0) {
    take = bits < s.best_bits;
    if (take) {
      s.best_bits = bits; s.best_kind = kind; s.best_order = order; s.best_lpc = lpc;
      s.best_porder = with_params ? s.cand_porder : 0;
    }
  }
  __syncthreads();
  if (take && with_params) {
    const int np = 1 << s.cand_porder;
    for (int j = threadIdx.x; j < np; j += FL_THREADS) s.kbest[j] = s.kcur[np - 1 + j];
  }
  __syncthreads();
}

// order-i coefficients a[1..i] -> quantised q, shift and precision (thread 0)
__device__ void quantise(const double* a, int p, int* q, int& shift, int& prec) {
  prec = min(15, 16 - (32 - __clz(p - 1)));
  double cmax = 0.0;
  for (int j = 1; j <= p; ++j) cmax = fmax(cmax, fabs(a[j]));
  int e;
  frexp(cmax, &e);
  shift = min(max(prec - 1 - e, 0), 15);
  const double lim_hi = (double)((1 << (prec - 1)) - 1), lim_lo = -(double)(1 << (prec - 1));
  for (int j = 1; j <= p; ++j) q[j - 1] = (int)fmin(fmax(rint(ldexp(a[j], shift)), lim_lo), lim_hi);
}

__global__ void __launch_bounds__(FL_THREADS) flac_analyze_kernel(const int16_t* __restrict__ pcm, const int64_t* __restrict__ pcm_off,
                                                                  long long max_n, int max_blocks, FlacRate rate,
                                                                  FlacRec* __restrict__ rec) {
  pdl_entry();
  __shared__ AnalyzeSmem s;
  const int k = blockIdx.y, blk = blockIdx.x, t = threadIdx.x;
  long long start, n_item;
  int nf;
  item_span(pcm_off, k, max_n, start, nf, n_item);
  if (blk >= nf) return;
  const int n = (int)min((long long)FL_BLOCK, n_item - (long long)blk * FL_BLOCK);
  const int16_t* src = pcm + start + (long long)blk * FL_BLOCK;
  for (int i = t; i < n; i += FL_THREADS) s.x[i] = src[i];
  if (t <= FL_MAX_LPC) s.r[t] = 0;
  if (t == 0) s.best_bits = 8 + 16ll * n + 1;          // above VERBATIM: the first candidate always replaces it
  __syncthreads();
  // window and autocorrelation
  const long long d = (long long)(n + 1) * (n + 1);
  for (int i = t; i < n; i += FL_THREADS) {
    const long long w = 2ll * i - n + 1;
    s.u.y[i] = (int)((long long)s.x[i] * (d - w * w) / d);
  }
  const int P = min(FL_MAX_LPC, n - 1);
  bool same = true;
  for (int i = t; i < n; i += FL_THREADS) same &= s.x[i] == s.x[0];
  __syncthreads();
  long long racc[FL_MAX_LPC + 1];
#pragma unroll
  for (int l = 0; l <= FL_MAX_LPC; ++l) racc[l] = 0;
  for (int i = t; i < n; i += FL_THREADS) {
    const long long yi = s.u.y[i];
#pragma unroll
    for (int l = 0; l <= FL_MAX_LPC; ++l)
      if (l <= P && i >= l) racc[l] += yi * s.u.y[i - l];
  }
#pragma unroll
  for (int l = 0; l <= FL_MAX_LPC; ++l) {
    const long long v = warp_sum(racc[l]);
    if ((t & 31) == 0 && v) atomicAdd((unsigned long long*)&s.r[l], (unsigned long long)v);
  }
  const bool constant = __syncthreads_and(same);
  if (t == 0) {                                         // Levinson-Durbin, fp64, no contraction
    int nl = 0;
    if (P >= 1 && s.r[0] != 0) {
      double a[FL_MAX_LPC + 1], na[FL_MAX_LPC + 1];
      for (int j = 0; j <= FL_MAX_LPC; ++j) a[j] = 0.0;
      double err = (double)s.r[0];
      for (int i = 1; i <= P; ++i) {
        double acc = (double)s.r[i];
        for (int j = 1; j < i; ++j) acc = __dsub_rn(acc, __dmul_rn(a[j], (double)s.r[i - j]));
        const double kk = __ddiv_rn(acc, err);
        for (int j = 1; j < i; ++j) na[j] = __dsub_rn(a[j], __dmul_rn(kk, a[i - j]));
        na[i] = kk;
        for (int j = 1; j <= i; ++j) a[j] = na[j];
        err = __dmul_rn(err, __dsub_rn(1.0, __dmul_rn(kk, kk)));
        if (!(err > 0.0)) break;
        quantise(a, i, s.lq[nl], s.lshift[nl], s.lprec[nl]);
        ++nl;
      }
    }
    s.n_lpc = nl;
  }
  __syncthreads();
  if (constant) consider(s, 24, FL_CONSTANT, 0, 0, false);
  for (int p = 0; p <= min(FL_MAX_FIXED, n - 1); ++p)
    if (rice_cost(s, n, FL_FIXED, p, nullptr, 0)) consider(s, 8 + 16ll * p + s.cand_bits, FL_FIXED, p, 0, true);
  for (int l = 0; l < s.n_lpc; ++l) {
    const int p = l + 1;
    if (rice_cost(s, n, FL_LPC, p, s.lq[l], s.lshift[l]))
      consider(s, 8 + 16ll * p + 9 + (long long)p * s.lprec[l] + s.cand_bits, FL_LPC, p, l, true);
  }
  consider(s, 8 + 16ll * n, FL_VERBATIM, 0, 0, false);
  FlacRec* R = rec + (size_t)k * max_blocks + blk;
  const int np = 1 << s.best_porder;
  for (int j = t; j < np; j += FL_THREADS) R->kp[j] = s.kbest[j];
  if (t == 0) {
    R->kind = s.best_kind;
    R->order = s.best_order;
    R->porder = s.best_porder;
    const int l = s.best_lpc;
    R->shift = s.best_kind == FL_LPC ? s.lshift[l] : 0;
    R->prec = s.best_kind == FL_LPC ? s.lprec[l] : 0;
    for (int j = 0; j < FL_MAX_LPC; ++j) R->q[j] = (short)(s.best_kind == FL_LPC && j < s.best_order ? s.lq[l][j] : 0);
    R->sub_bits = s.best_bits;
    R->bytes = frame_header_bytes(blk, n, rate) + (int)((s.best_bits + 7) / 8) + 2;
  }
}

// block-wide exclusive scan of one value per thread (FL_THREADS threads); returns the exclusive prefix, *total the sum
template <typename T>
__device__ T block_exclusive_scan(T v, T* total, T* warp_buf) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  T incl = v;
  for (int o = 1; o < 32; o <<= 1) {
    const T u = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += u;
  }
  if (lane == 31) warp_buf[w] = incl;
  __syncthreads();
  if (w == 0) {
    T x = lane < nw ? warp_buf[lane] : T(0);
    for (int o = 1; o < 32; o <<= 1) {
      const T u = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += u;
    }
    if (lane < nw) warp_buf[lane] = x;
  }
  __syncthreads();
  const T base = w ? warp_buf[w - 1] : T(0);
  *total = warp_buf[nw - 1];
  __syncthreads();
  return base + incl - v;
}

__global__ void __launch_bounds__(FL_THREADS) flac_stream_kernel(const int64_t* __restrict__ pcm_off, long long max_n, int max_blocks,
                                                                 const FlacRec* __restrict__ rec, long long* __restrict__ frame_off,
                                                                 long long* __restrict__ stream_bytes, int* __restrict__ fmin,
                                                                 int* __restrict__ fmax) {
  pdl_entry();
  __shared__ long long wb[FL_THREADS / 32];
  __shared__ int red[2][FL_THREADS / 32];
  const int k = blockIdx.x, t = threadIdx.x;
  long long start, n;
  int nf;
  item_span(pcm_off, k, max_n, start, nf, n);
  long long carry = FL_HEADER;
  int lo = 0x7fffffff, hi = 0;
  for (int j0 = 0; j0 < nf; j0 += FL_THREADS) {
    const int j = j0 + t;
    const int b = j < nf ? rec[(size_t)k * max_blocks + j].bytes : 0;
    if (j < nf) { lo = min(lo, b); hi = max(hi, b); }
    long long tot;
    const long long ex = block_exclusive_scan<long long>(b, &tot, wb);
    if (j < nf) frame_off[(size_t)k * max_blocks + j] = carry + ex;
    carry += tot;
  }
  for (int o = 16; o > 0; o >>= 1) {
    lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  if ((t & 31) == 0) { red[0][t >> 5] = lo; red[1][t >> 5] = hi; }
  __syncthreads();
  if (t == 0) {
    for (int w = 1; w < FL_THREADS / 32; ++w) { lo = min(lo, red[0][w]); hi = max(hi, red[1][w]); }
    stream_bytes[k] = carry;
    fmin[k] = nf ? lo : 0;
    fmax[k] = hi;
  }
}

constexpr int FO_THREADS = 1024;

__global__ void __launch_bounds__(FO_THREADS) flac_offsets_kernel(const long long* __restrict__ stream_bytes, int n_items,
                                                                  int64_t* __restrict__ out_off) {
  pdl_entry();
  __shared__ long long wb[FO_THREADS / 32];
  long long carry = 0;
  for (int k0 = 0; k0 < n_items; k0 += FO_THREADS) {
    const int k = k0 + threadIdx.x;
    long long tot;
    const long long ex = block_exclusive_scan<long long>(k < n_items ? stream_bytes[k] : 0, &tot, wb);
    if (k < n_items) out_off[k] = carry + ex;
    carry += tot;
  }
  if (threadIdx.x == 0) out_off[n_items] = carry;
}

// nb <= 32 bits of v, most significant first, at bit pos of a big-endian bit buffer of 32-bit words (zeroed; ORed in)
__device__ __forceinline__ void put_bits(unsigned* buf, long long pos, unsigned long long v, int nb) {
  if (nb == 0) return;
  v &= (nb == 64 ? ~0ull : ((1ull << nb) - 1));
  if (!v) return;
  const int off = (int)(pos & 31);
  const unsigned long long w = v << (64 - nb - off);
  const unsigned hi = (unsigned)(w >> 32), lo = (unsigned)w;
  if (hi) atomicOr(&buf[pos >> 5], hi);
  if (lo) atomicOr(&buf[(pos >> 5) + 1], lo);
}

__device__ __forceinline__ unsigned get_byte(const unsigned* buf, int i) { return (buf[i >> 2] >> (24 - 8 * (i & 3))) & 0xFFu; }

// a * b mod P(x) = x^16 + x^15 + x^2 + 1 over GF(2)
__device__ __forceinline__ unsigned crc16_mulmod(unsigned a, unsigned b) {
  unsigned r = 0;
  for (int i = 15; i >= 0; --i) {
    r <<= 1;
    if (r & 0x10000u) r ^= 0x18005u;
    if ((b >> i) & 1u) r ^= a;
  }
  return r & 0xFFFFu;
}

// x^(8 L) mod P
__device__ __forceinline__ unsigned crc16_shift(int L) {
  unsigned r = 1, b = 0x100;
  while (L) {
    if (L & 1) r = crc16_mulmod(r, b);
    b = crc16_mulmod(b, b);
    L >>= 1;
  }
  return r;
}

struct WriteSmem {
  int x[FL_BLOCK];
  unsigned buf[FL_BUF_WORDS];
  unsigned short crc_tab[256];
  int wb[FL_THREADS / 32];
  unsigned cx[FL_THREADS / 32];
};

__global__ void __launch_bounds__(FL_THREADS) flac_write_kernel(const int16_t* __restrict__ pcm, const int64_t* __restrict__ pcm_off,
                                                                long long max_n, int max_blocks, FlacRate rate, int sample_rate,
                                                                const FlacRec* __restrict__ rec, const long long* __restrict__ frame_off,
                                                                const long long* __restrict__ stream_bytes, const int* __restrict__ fmin,
                                                                const int* __restrict__ fmax, const int64_t* __restrict__ out_off,
                                                                uint8_t* __restrict__ out, long long out_bytes) {
  pdl_entry();
  __shared__ WriteSmem s;
  const int k = blockIdx.y, blk = blockIdx.x, t = threadIdx.x;
  long long start, n_item;
  int nf;
  item_span(pcm_off, k, max_n, start, nf, n_item);
  if (blk >= nf) return;
  const long long base = out_off[k];
  if (base + stream_bytes[k] > out_bytes) return;       // only when pcm_off disagrees with the sizes the buffer was checked for
  const int n = (int)min((long long)FL_BLOCK, n_item - (long long)blk * FL_BLOCK);
  const FlacRec* R = rec + (size_t)k * max_blocks + blk;
  const int kind = R->kind, order = R->order, porder = R->porder, shift = R->shift, prec = R->prec, nbytes = R->bytes;
  const int16_t* src = pcm + start + (long long)blk * FL_BLOCK;
  for (int i = t; i < n; i += FL_THREADS) s.x[i] = src[i];
  for (int i = t; i < FL_BUF_WORDS; i += FL_THREADS) s.buf[i] = 0;
  {
    unsigned c = (unsigned)t << 8;
    for (int j = 0; j < 8; ++j) c = (c & 0x8000u) ? ((c << 1) ^ 0x8005u) : (c << 1);
    s.crc_tab[t] = (unsigned short)c;
  }
  if (blk == 0 && t == 0) {                             // fLaC, metadata block header, STREAMINFO (RFC 9639 sections 8.1, 8.2)
    unsigned char h[FL_HEADER] = {'f', 'L', 'a', 'C', 0x80, 0, 0, 34};
    const long long total = n_item;
    const unsigned fl = (unsigned)fmin[k], fh = (unsigned)fmax[k];
    h[8] = 0x10; h[9] = 0x00; h[10] = 0x10; h[11] = 0x00;                     // block sizes 4096, 4096
    h[12] = fl >> 16; h[13] = fl >> 8; h[14] = fl;
    h[15] = fh >> 16; h[16] = fh >> 8; h[17] = fh;
    // 20-bit rate, 3-bit channels - 1 (0), 5-bit bits per sample - 1 (15), 36-bit total samples
    h[18] = (unsigned)sample_rate >> 12;
    h[19] = (unsigned)sample_rate >> 4;
    h[20] = (((unsigned)sample_rate & 0xF) << 4) | (0 << 1) | (15 >> 4);
    h[21] = ((15 & 0xF) << 4) | (unsigned)((total >> 32) & 0xF);
    h[22] = (unsigned)(total >> 24); h[23] = (unsigned)(total >> 16); h[24] = (unsigned)(total >> 8); h[25] = (unsigned)total;
    for (int i = 26; i < FL_HEADER; ++i) h[i] = 0;                              // MD5 unknown
    for (int i = 0; i < FL_HEADER; ++i) out[base + i] = h[i];
  }
  __syncthreads();
  // frame header (RFC 9639 section 9.1) and subframe header, warm-up samples, LPC fields, residual header: thread 0
  const int hb = frame_header_bytes(blk, n, rate);
  long long pos = 0;
  if (t == 0) {
    const int bcode = n == FL_BLOCK ? 12 : n <= 256 ? 6 : 7;
    put_bits(s.buf, 0, 0xFFF8, 16);
    put_bits(s.buf, 16, (bcode << 4) | rate.code, 8);
    put_bits(s.buf, 24, 0x08, 8);
    pos = 32;
    const long long v = blk;
    const int ub = utf8_bytes(v);
    if (ub == 1) {
      put_bits(s.buf, pos, (unsigned)v, 8);
    } else {
      const unsigned lead = (0xFF00u >> ub) & 0xFFu;
      put_bits(s.buf, pos, lead | (unsigned)(v >> (6 * (ub - 1))), 8);
      for (int i = ub - 2; i >= 0; --i) put_bits(s.buf, pos + 8 * (ub - 1 - i), 0x80u | (unsigned)((v >> (6 * i)) & 0x3F), 8);
    }
    pos += 8 * ub;
    if (bcode != 12) {
      const int eb = bcode == 6 ? 8 : 16;
      put_bits(s.buf, pos, (unsigned)(n - 1), eb);
      pos += eb;
    }
    if (rate.bits) {
      put_bits(s.buf, pos, (unsigned)rate.value, rate.bits);
      pos += rate.bits;
    }
    unsigned c8 = 0;
    for (int i = 0; i < hb - 1; ++i) {
      c8 ^= get_byte(s.buf, i);
      for (int j = 0; j < 8; ++j) c8 = (c8 & 0x80u) ? ((c8 << 1) ^ 0x07u) & 0xFFu : (c8 << 1) & 0xFFu;
    }
    put_bits(s.buf, pos, c8, 8);
    pos += 8;
    // subframe (section 9.2): zero bit, 6-bit type, wasted-bits flag 0
    const int type = kind == FL_CONSTANT ? 0 : kind == FL_VERBATIM ? 1 : kind == FL_FIXED ? 8 | order : 32 | (order - 1);
    put_bits(s.buf, pos, (unsigned)type << 1, 8);
    pos += 8;
    if (kind == FL_CONSTANT) put_bits(s.buf, pos, (unsigned)s.x[0] & 0xFFFFu, 16);
    if (kind == FL_FIXED || kind == FL_LPC) {
      for (int i = 0; i < order; ++i) put_bits(s.buf, pos + 16 * i, (unsigned)s.x[i] & 0xFFFFu, 16);
      pos += 16 * order;
      if (kind == FL_LPC) {
        put_bits(s.buf, pos, (unsigned)(prec - 1), 4);
        put_bits(s.buf, pos + 4, (unsigned)shift, 5);
        pos += 9;
        for (int j = 0; j < order; ++j) put_bits(s.buf, pos + (long long)prec * j, (unsigned)R->q[j], prec);
        pos += (long long)prec * order;
      }
      put_bits(s.buf, pos, (unsigned)porder, 6);         // coding method 00, 4-bit partition order
      pos += 6;
    }
  }
  if (kind == FL_VERBATIM) {
    const long long b0 = 8ll * hb + 8;
    for (int i = t; i < n; i += FL_THREADS) put_bits(s.buf, b0 + 16ll * i, (unsigned)s.x[i] & 0xFFFFu, 16);
  } else if (kind != FL_CONSTANT) {
    const long long b0 = 8ll * hb + 8 + 16 * order + (kind == FL_LPC ? 9 + (long long)prec * order : 0) + 6;
    int q[FL_MAX_LPC];
    for (int j = 0; j < FL_MAX_LPC; ++j) q[j] = R->q[j];
    const int psize = n >> porder;
    unsigned u[FL_PER_THREAD];
    int len = 0;
    const int i0 = t * FL_PER_THREAD;
#pragma unroll
    for (int e = 0; e < FL_PER_THREAD; ++e) {
      const int i = i0 + e;
      u[e] = 0;
      if (i >= order && i < n) {
        u[e] = (unsigned)zigzag(predict_residual(s.x, i, kind, order, q, shift));
        const int kp = R->kp[i / psize];
        len += (int)(u[e] >> kp) + 1 + kp + ((i == order || (i % psize == 0 && i > order)) ? 4 : 0);
      }
    }
    int tot;
    long long p = b0 + block_exclusive_scan<int>(len, &tot, s.wb);
#pragma unroll
    for (int e = 0; e < FL_PER_THREAD; ++e) {
      const int i = i0 + e;
      if (i >= order && i < n) {
        const int part = i / psize, kp = R->kp[part];
        if (i == order || (i % psize == 0 && i > order)) {
          put_bits(s.buf, p, (unsigned)kp, 4);
          p += 4;
        }
        const long long qv = u[e] >> kp;
        put_bits(s.buf, p + qv, 1, 1);
        put_bits(s.buf, p + qv + 1, u[e], kp);
        p += qv + 1 + kp;
      }
    }
  }
  __syncthreads();
  // CRC-16 of bytes [0, nbytes - 2)
  const int L = nbytes - 2;
  const int chunk = (L + FL_THREADS - 1) / FL_THREADS;
  const int c0 = min(t * chunk, L), c1 = min(c0 + chunk, L);
  unsigned c = 0;
  for (int i = c0; i < c1; ++i) c = ((c << 8) & 0xFFFFu) ^ s.crc_tab[((c >> 8) ^ get_byte(s.buf, i)) & 0xFFu];
  if (c) c = crc16_mulmod(c, crc16_shift(L - c1));
  for (int o = 16; o > 0; o >>= 1) c ^= __shfl_xor_sync(0xffffffffu, c, o);
  if ((t & 31) == 0) s.cx[t >> 5] = c;
  __syncthreads();
  if (t == 0) {
    unsigned crc = 0;
    for (int w = 0; w < FL_THREADS / 32; ++w) crc ^= s.cx[w];
    put_bits(s.buf, 8ll * L, crc, 16);
  }
  __syncthreads();
  uint8_t* dst = out + base + frame_off[(size_t)k * max_blocks + blk];
  for (int i = t; i < nbytes; i += FL_THREADS) dst[i] = (uint8_t)get_byte(s.buf, i);
}

static FlacRate flac_rate(int r) {
  switch (r) {
    case 88200: return {1, 0, 0};
    case 176400: return {2, 0, 0};
    case 192000: return {3, 0, 0};
    case 8000: return {4, 0, 0};
    case 16000: return {5, 0, 0};
    case 22050: return {6, 0, 0};
    case 24000: return {7, 0, 0};
    case 32000: return {8, 0, 0};
    case 44100: return {9, 0, 0};
    case 48000: return {10, 0, 0};
    case 96000: return {11, 0, 0};
    default: break;
  }
  if (r % 1000 == 0 && r / 1000 <= 255) return {12, r / 1000, 8};
  if (r <= 65535) return {13, r, 16};
  if (r % 10 == 0) return {14, r / 10, 16};
  return {0, 0, 0};
}

static long long flac_blocks(long long n) { return (n + FL_BLOCK - 1) / FL_BLOCK; }

static size_t flac_bound(long long n) { return n < 1 ? 0 : (size_t)FL_HEADER + (size_t)flac_blocks(n) * FL_FRAME_OVERHEAD + 2 * (size_t)n; }

static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// records | frame offsets (i64) | image sizes (i64) | min, max frame size (i32)
static size_t flac_ws_bytes(int n_items, long long max_n) {
  const size_t slots = (size_t)n_items * (size_t)flac_blocks(max_n);
  return align256(slots * sizeof(FlacRec)) + align256(slots * sizeof(long long)) + align256((size_t)n_items * sizeof(long long)) +
         align256(2 * (size_t)n_items * sizeof(int));
}

constexpr long long FL_MAX_SAMPLES = (long long)FL_BLOCK << 24;   // 2^36: STREAMINFO's sample count, and frame numbers stay small

}  // namespace ev

using namespace ev;

extern "C" {

size_t ev_flac_bound_bytes(long long n_samples) { return n_samples >= 1 && n_samples <= FL_MAX_SAMPLES ? flac_bound(n_samples) : 0; }

size_t ev_flac_workspace_bytes(int n_items, long long max_n) {
  return n_items >= 1 && n_items <= 65535 && max_n >= 1 && max_n <= FL_MAX_SAMPLES ? flac_ws_bytes(n_items, max_n) : 0;
}

int ev_flac_encode(const int16_t* pcm, const int64_t* pcm_off, int n_items, const int64_t* n_samples, int sample_rate, uint8_t* out,
                   size_t out_bytes, int64_t* out_off, void* ws, size_t ws_bytes, void* stream) {
  EV_CHECK_ARG(pcm && pcm_off && n_samples && out && out_off && ws, "ev_flac_encode: null argument");
  EV_CHECK_ARG(n_items >= 1 && n_items <= 65535, "ev_flac_encode: n_items=%d must lie in [1, 65535]", n_items);
  EV_CHECK_ARG(sample_rate >= FL_MIN_RATE && sample_rate <= FL_MAX_RATE, "ev_flac_encode: sample_rate=%d must lie in [%d, %d]",
               sample_rate, FL_MIN_RATE, FL_MAX_RATE);
  long long max_n = 0;
  size_t need_out = 0;
  for (int k = 0; k < n_items; ++k) {
    EV_CHECK_ARG(n_samples[k] >= 1 && n_samples[k] <= FL_MAX_SAMPLES, "ev_flac_encode: item %d has %lld samples, must be in [1, 2^36]",
                 k, (long long)n_samples[k]);
    max_n = n_samples[k] > max_n ? n_samples[k] : max_n;
    need_out += flac_bound(n_samples[k]);
  }
  EV_CHECK_ARG(out_bytes >= need_out, "ev_flac_encode: output buffer of %zu bytes, %zu needed", out_bytes, need_out);
  const size_t need_ws = flac_ws_bytes(n_items, max_n);
  EV_CHECK_ARG(ws_bytes >= need_ws, "ev_flac_encode: workspace of %zu bytes, %zu needed", ws_bytes, need_ws);
  EV_TRY(use_device_of(pcm));
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long long mb = flac_blocks(max_n);
  EV_CHECK_ARG(mb <= 0x7fffffffll, "ev_flac_encode: item of %lld samples is too long", max_n);
  const size_t slots = (size_t)n_items * (size_t)mb;
  char* w = static_cast<char*>(ws);
  FlacRec* rec = reinterpret_cast<FlacRec*>(w);
  w += align256(slots * sizeof(FlacRec));
  long long* frame_off = reinterpret_cast<long long*>(w);
  w += align256(slots * sizeof(long long));
  long long* sbytes = reinterpret_cast<long long*>(w);
  w += align256((size_t)n_items * sizeof(long long));
  int* fmn = reinterpret_cast<int*>(w);
  int* fmx = fmn + n_items;
  const FlacRate rate = flac_rate(sample_rate);
  const dim3 grid((unsigned)mb, (unsigned)n_items);
  EV_TRY(launch("flac_analyze_kernel", flac_analyze_kernel, grid, FL_THREADS, 0, st, pcm, pcm_off, max_n, (int)mb, rate, rec));
  EV_TRY(launch("flac_stream_kernel", flac_stream_kernel, dim3(n_items), FL_THREADS, 0, st, pcm_off, max_n, (int)mb,
                (const FlacRec*)rec, frame_off, sbytes, fmn, fmx));
  EV_TRY(launch("flac_offsets_kernel", flac_offsets_kernel, dim3(1), FO_THREADS, 0, st, (const long long*)sbytes, n_items, out_off));
  return launch("flac_write_kernel", flac_write_kernel, grid, FL_THREADS, 0, st, pcm, pcm_off, max_n, (int)mb, rate, sample_rate,
                (const FlacRec*)rec, (const long long*)frame_off, (const long long*)sbytes, (const int*)fmn, (const int*)fmx,
                (const int64_t*)out_off, out, (long long)out_bytes);
}

}  // extern "C"
