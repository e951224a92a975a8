// Objective comparison of a synthesis with a recording (ev_eval_compare): cepstral distance after dynamic time warping,
// F0 error and voicing error along the warping path.  Per pair of N syn frames and M ref frames (1 <= N, M <= 4096):
//   cepstra   c_k[f] = (sum_{m=0..79} fp64(L[m, f]) * T[k, m], ascending m, each product and sum rounded) / 80, k = 1..24,
//             T the caller's fp64 table cos(pi k (m + 1/2) / 80).
//   distance  d(i, j) = sqrt(sum_{k=1..24} (c_k[i] - c'_k[j])^2), ascending k, every operation rounded on its own
//             (__dsub_rn / __dmul_rn / __dadd_rn / __dsqrt_rn: no FMA contraction), so the bits are the fp64 oracle's.
//   DTW       D(0,0) = d(0,0); D(i,j) = d(i,j) + min(D(i-1,j-1), D(i-1,j), D(i,j-1)) over the predecessors that exist, ties
//             to the first in that order; the path is the backtrack from (N-1, M-1) to (0,0).
//   stats     mcd = K (D(N-1, M-1) / P), K = 10 sqrt(2) / ln 10, P the path length; D(N-1, M-1) is the sum of d along the
//             path in path order from (0,0) (each D adds one d to its predecessor's D).  vuv_error = (pairs whose voicing
//             differs) / P; voiced_pairs = pairs with both F0 > 0; f0_rmse = sqrt(E / voiced_pairs), E the sum of
//             (1200 log2(f_syn / f_ref))^2 over those pairs in path order (NaN without voiced pairs).
//
// Three launches.  eval_cep_kernel: one CTA per (32 frames, item, side) stages the frames' log-mels and the table.
// eval_cost_kernel: one CTA per (32 x 32 cells, item) stages both sides' cepstra and writes d in anti-diagonal-major order
// (diagonal t = i + j, cells by ascending i), warp w taking the tile's local anti-diagonals w, w + 8, ... so its stores are
// contiguous.  eval_dtw_kernel: one CTA per pair runs the N + M - 1 anti-diagonals with three rolling diagonals of D in shared
// memory (indexed by i) and the next diagonal's distances prefetched into registers, writes a predecessor code per cell, then
// thread 0 backtracks and the CTA forms the statistics.  No kernel reads a frame or cell past its pair's N and M, and every
// pair's arithmetic is the same in any batch or order.
#include <math.h>

#include "ev_common.cuh"

namespace ev {

constexpr int EV_MELS = 80, EV_CEPS = 24, EV_MAX_FRAMES = 4096;
constexpr int EC_FRAMES = 32, EC_THREADS = 256;
constexpr int ET_TILE = 32, ET_THREADS = 256, ET_PAD = EV_CEPS + 1;   // odd row pitch: conflict-free fp64 reads across lanes
constexpr int ED_THREADS = 512, ED_CELLS = EV_MAX_FRAMES / ED_THREADS; // cells of one diagonal per thread
constexpr int ED_MAX_PATH = 2 * EV_MAX_FRAMES;
constexpr double MCD_K = 6.141851463713754;                            // 10 sqrt(2) / ln 10, rounded to fp64
constexpr unsigned char CODE_DIAG = 0, CODE_UP = 1, CODE_LEFT = 2, CODE_START = 3;

// cells of the anti-diagonals before diagonal t of an N x M grid, and the first row i on diagonal t
__host__ __device__ __forceinline__ long long diag_offset(long long t, long long N, long long M) {
  const long long a = N < M ? N : M, b = N < M ? M : N;
  if (t <= a) return t * (t + 1) / 2;
  if (t <= b) return a * (a + 1) / 2 + (t - a) * a;
  const long long u = N + M - 1 - t;                          // diagonals left, of u, u - 1, ..., 1 cells
  return N * M - u * (u + 1) / 2;
}
__host__ __device__ __forceinline__ int diag_lo(int t, int M) { return t - (M - 1) > 0 ? t - (M - 1) : 0; }
__device__ __forceinline__ long long cell_index(int i, int j, int N, int M) {
  return diag_offset(i + j, N, M) + (i - diag_lo(i + j, M));
}
__device__ __forceinline__ int item_frames(const int32_t* n, int b, int max_n) { return min(max(n[b], 1), max_n); }

// cep[side][(b * max_f + f) * 24 + k - 1] = c_k[f] of item b
__global__ void __launch_bounds__(EC_THREADS) eval_cep_kernel(const float* __restrict__ mel_syn, long long syn_frames,
                                                              const int32_t* __restrict__ n_syn, int max_n,
                                                              const float* __restrict__ mel_ref, long long ref_frames,
                                                              const int32_t* __restrict__ n_ref, int max_m,
                                                              const double* __restrict__ table, double* __restrict__ cep_syn,
                                                              double* __restrict__ cep_ref) {
  pdl_entry();
  __shared__ double ts[EV_CEPS * EV_MELS];
  __shared__ float ls[EV_MELS][EC_FRAMES];
  const int b = blockIdx.y, ref = blockIdx.z;
  const int max_f = ref ? max_m : max_n;
  const int n = item_frames(ref ? n_ref : n_syn, b, max_f);
  const int f0 = blockIdx.x * EC_FRAMES;
  if (f0 >= n) return;
  const long long frames = ref ? ref_frames : syn_frames;
  const float* mel = (ref ? mel_ref : mel_syn) + (size_t)b * EV_MELS * frames;
  for (int i = threadIdx.x; i < EV_CEPS * EV_MELS; i += EC_THREADS) ts[i] = table[i];
  for (int i = threadIdx.x; i < EV_MELS * EC_FRAMES; i += EC_THREADS) {
    const int m = i / EC_FRAMES, fl = i % EC_FRAMES;
    ls[m][fl] = f0 + fl < n ? mel[(size_t)m * frames + f0 + fl] : 0.f;
  }
  __syncthreads();
  const int fl = threadIdx.x % EC_FRAMES, f = f0 + fl;
  if (f >= n) return;
  double* out = (ref ? cep_ref : cep_syn) + ((size_t)b * max_f + f) * EV_CEPS;
  for (int k = threadIdx.x / EC_FRAMES; k < EV_CEPS; k += EC_THREADS / EC_FRAMES) {
    const double* t = ts + k * EV_MELS;
    double acc = 0.0;
    for (int m = 0; m < EV_MELS; ++m) acc = __dadd_rn(acc, __dmul_rn((double)ls[m][fl], t[m]));
    out[k] = __ddiv_rn(acc, (double)EV_MELS);
  }
}

// cost[b * max_n * max_m + cell_index(i, j)] = d(i, j); item b's cepstra start syn_rows / ref_rows frames apart
__global__ void __launch_bounds__(ET_THREADS) eval_cost_kernel(const double* __restrict__ cep_syn, long long syn_rows,
                                                               const int32_t* __restrict__ n_syn, int max_n,
                                                               const double* __restrict__ cep_ref, long long ref_rows,
                                                               const int32_t* __restrict__ n_ref, int max_m,
                                                               double* __restrict__ cost) {
  pdl_entry();
  __shared__ double cs[ET_TILE * ET_PAD], cr[ET_TILE * ET_PAD];
  const int b = blockIdx.z;
  const int N = item_frames(n_syn, b, max_n), M = item_frames(n_ref, b, max_m);
  const int i0 = blockIdx.y * ET_TILE, j0 = blockIdx.x * ET_TILE;
  if (i0 >= N || j0 >= M) return;
  const double* a = cep_syn + ((size_t)b * syn_rows + i0) * EV_CEPS;
  const double* r = cep_ref + ((size_t)b * ref_rows + j0) * EV_CEPS;
  const int ni = min(ET_TILE, N - i0), nj = min(ET_TILE, M - j0);
  for (int e = threadIdx.x; e < ET_TILE * EV_CEPS; e += ET_THREADS) {
    const int row = e / EV_CEPS, k = e % EV_CEPS;
    cs[row * ET_PAD + k] = row < ni ? a[e] : 0.0;
    cr[row * ET_PAD + k] = row < nj ? r[e] : 0.0;
  }
  __syncthreads();
  double* out = cost + (size_t)b * max_n * max_m;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int s = w; s < 2 * ET_TILE - 1; s += ET_THREADS / 32) {
    const int il = lane, jl = s - lane;
    if (jl < 0 || jl >= nj || il >= ni) continue;
    const double* x = cs + il * ET_PAD;
    const double* y = cr + jl * ET_PAD;
    double acc = 0.0;
#pragma unroll
    for (int k = 0; k < EV_CEPS; ++k) {
      const double df = __dsub_rn(x[k], y[k]);
      acc = __dadd_rn(acc, __dmul_rn(df, df));
    }
    out[cell_index(i0 + il, j0 + jl, N, M)] = __dsqrt_rn(acc);
  }
}

__device__ __forceinline__ void eval_prefetch(double (&d)[ED_CELLS], const double* cost, int t, int N, int M) {
  const int lo = diag_lo(t, M), hi = min(t, N - 1);
  const double* c = cost + diag_offset(t, N, M) - lo;
#pragma unroll
  for (int q = 0; q < ED_CELLS; ++q) {
    const int i = lo + (int)threadIdx.x + q * ED_THREADS;
    d[q] = i <= hi ? c[i] : 0.0;
  }
}

// stats (3, n_items): mcd, f0_rmse, vuv_error; counts (2, n_items): voiced_pairs, path length
__global__ void __launch_bounds__(ED_THREADS, 2) eval_dtw_kernel(const double* __restrict__ cost, unsigned char* __restrict__ codes,
                                                                 const int32_t* __restrict__ n_syn, int max_n,
                                                                 const int32_t* __restrict__ n_ref, int max_m,
                                                                 const double* __restrict__ f0_syn, long long syn_frames,
                                                                 const double* __restrict__ f0_ref, long long ref_frames,
                                                                 int n_items, double* __restrict__ stats, int32_t* __restrict__ counts,
                                                                 int32_t* __restrict__ path, long long path_stride) {
  pdl_entry();
  extern __shared__ __align__(16) double ed_smem[];          // 3 rolling diagonals of D; then the path and its terms
  __shared__ double total;
  __shared__ int s_len, s_mismatch, s_voiced;
  const int b = blockIdx.x;
  const int N = item_frames(n_syn, b, max_n), M = item_frames(n_ref, b, max_m);
  const size_t base = (size_t)b * max_n * max_m;
  const double* c = cost + base;
  unsigned char* code = codes + base;
  const int T = N + M - 1;
  double dn[ED_CELLS];
  eval_prefetch(dn, c, 0, N, M);
  for (int t = 0; t < T; ++t) {
    double dc[ED_CELLS];
#pragma unroll
    for (int q = 0; q < ED_CELLS; ++q) dc[q] = dn[q];
    if (t + 1 < T) eval_prefetch(dn, c, t + 1, N, M);
    const int lo = diag_lo(t, M), hi = min(t, N - 1);
    const long long off = diag_offset(t, N, M) - lo;
    double* cur = ed_smem + (t % 3) * EV_MAX_FRAMES;
    const double* p1 = ed_smem + ((t + 2) % 3) * EV_MAX_FRAMES;   // diagonal t - 1
    const double* p2 = ed_smem + ((t + 1) % 3) * EV_MAX_FRAMES;   // diagonal t - 2
#pragma unroll
    for (int q = 0; q < ED_CELLS; ++q) {
      const int i = lo + (int)threadIdx.x + q * ED_THREADS;
      if (i > hi) break;
      const int j = t - i;
      double best;
      unsigned char cd;
      if (i > 0 && j > 0) {
        best = p2[i - 1];
        cd = CODE_DIAG;
        if (p1[i - 1] < best) { best = p1[i - 1]; cd = CODE_UP; }
        if (p1[i] < best) { best = p1[i]; cd = CODE_LEFT; }
      } else if (i > 0) {
        best = p1[i - 1];
        cd = CODE_UP;
      } else if (j > 0) {
        best = p1[i];
        cd = CODE_LEFT;
      } else {
        best = 0.0;
        cd = CODE_START;
      }
      const double D = cd == CODE_START ? dc[q] : __dadd_rn(dc[q], best);
      cur[i] = D;
      code[off + i] = cd;
      if (t == T - 1) total = D;
    }
    __syncthreads();
  }
  // backtrack: pk[0 .. P) holds the path from (N-1, M-1) back to (0,0), (i << 16) | j
  int* pk = reinterpret_cast<int*>(ed_smem);
  double* term = ed_smem + ED_MAX_PATH / 2;                   // after pk's 8192 ints
  if (threadIdx.x == 0) {
    int i = N - 1, j = M - 1, p = 0;
    for (;;) {
      pk[p++] = (i << 16) | j;
      const unsigned char cd = code[cell_index(i, j, N, M)];
      if (cd == CODE_START) break;
      if (cd == CODE_DIAG) { --i; --j; }
      else if (cd == CODE_UP) --i;
      else --j;
    }
    s_len = p;
    s_mismatch = 0;
    s_voiced = 0;
  }
  __syncthreads();
  const int P = s_len;
  const double* fs = f0_syn + (size_t)b * syn_frames;
  const double* fr = f0_ref + (size_t)b * ref_frames;
  int mism = 0, voiced = 0;
  for (int p = threadIdx.x; p < P; p += ED_THREADS) {        // term[p]: pair p in path order from (0,0)
    const int v = pk[P - 1 - p], i = v >> 16, j = v & 0xffff;
    const double a = fs[i], r = fr[j];
    const bool va = a > 0.0, vr = r > 0.0;
    mism += va != vr;
    voiced += va && vr;
    double e = 0.0;
    if (va && vr) {
      const double cents = 1200.0 * log2(a / r);
      e = __dmul_rn(cents, cents);
    }
    term[p] = e;
    if (path) {
      path[((size_t)b * path_stride + p) * 2] = i;
      path[((size_t)b * path_stride + p) * 2 + 1] = j;
    }
  }
  if (path)
    for (long long p = P + threadIdx.x; p < path_stride; p += ED_THREADS) {
      path[((size_t)b * path_stride + p) * 2] = -1;
      path[((size_t)b * path_stride + p) * 2 + 1] = -1;
    }
  for (int o = 16; o > 0; o >>= 1) {
    mism += __shfl_xor_sync(0xffffffffu, mism, o);
    voiced += __shfl_xor_sync(0xffffffffu, voiced, o);
  }
  if ((threadIdx.x & 31) == 0) {                              // integer counts: exact in any order
    atomicAdd(&s_mismatch, mism);
    atomicAdd(&s_voiced, voiced);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double e = 0.0;
    for (int p = 0; p < P; ++p) e = __dadd_rn(e, term[p]);   // unvoiced pairs add +0, which leaves the sum's bits alone
    const int nv = s_voiced;
    stats[b] = MCD_K * (total / (double)P);
    stats[n_items + b] = nv > 0 ? sqrt(e / (double)nv) : NAN;
    stats[2 * n_items + b] = (double)s_mismatch / (double)P;
    counts[b] = nv;
    counts[n_items + b] = P;
  }
}

static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// cepstra of both sides (f64) | d of every cell (f64) | predecessor codes (u8)
static size_t eval_ws_bytes(int n_items, int max_n, int max_m) {
  const size_t cells = (size_t)n_items * (size_t)max_n * (size_t)max_m;
  return align256((size_t)n_items * max_n * EV_CEPS * sizeof(double)) + align256((size_t)n_items * max_m * EV_CEPS * sizeof(double)) +
         align256(cells * sizeof(double)) + align256(cells);
}

static bool eval_args_ok(int n_items, int max_n, int max_m) {
  return n_items >= 1 && n_items <= 65535 && max_n >= 1 && max_n <= EV_MAX_FRAMES && max_m >= 1 && max_m <= EV_MAX_FRAMES;
}

// the cost and DTW launches of ev_eval_compare and ev_eval_align, from cepstra (n_items, *_rows, 24) f64
static int eval_align_tail(const double* cep_syn, long long syn_rows, const double* f0_syn, long long syn_frames, const int32_t* n_syn,
                           int max_n, const double* cep_ref, long long ref_rows, const double* f0_ref, long long ref_frames,
                           const int32_t* n_ref, int max_m, int n_items, double* stats, int32_t* counts, int32_t* path,
                           long long path_stride, char* w, cudaStream_t st) {
  w += align256((size_t)n_items * max_n * EV_CEPS * sizeof(double));
  w += align256((size_t)n_items * max_m * EV_CEPS * sizeof(double));
  double* cost = reinterpret_cast<double*>(w);
  w += align256((size_t)n_items * max_n * max_m * sizeof(double));
  unsigned char* codes = reinterpret_cast<unsigned char*>(w);
  const size_t smem = 3 * EV_MAX_FRAMES * sizeof(double);
  static std::atomic<uint64_t> attr_devs{0};
  if (first_use_on_device(attr_devs))
    cudaFuncSetAttribute(eval_dtw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  EV_TRY(launch("eval_cost_kernel", eval_cost_kernel, dim3((max_m + ET_TILE - 1) / ET_TILE, (max_n + ET_TILE - 1) / ET_TILE, n_items),
                ET_THREADS, 0, st, cep_syn, syn_rows, n_syn, max_n, cep_ref, ref_rows, n_ref, max_m, cost));
  return launch("eval_dtw_kernel", eval_dtw_kernel, dim3(n_items), ED_THREADS, smem, st, (const double*)cost, codes, n_syn, max_n, n_ref,
                max_m, f0_syn, syn_frames, f0_ref, ref_frames, n_items, stats, counts, path, path_stride);
}

// the argument checks ev_eval_compare and ev_eval_align share
static int eval_args_check(const char* what, int n_items, int max_n, int max_m, long long syn_frames, long long ref_frames,
                           const int32_t* path, long long path_stride, size_t ws_bytes) {
  EV_CHECK_ARG(n_items >= 1 && n_items <= 65535, "%s: n_items=%d must lie in [1, 65535]", what, n_items);
  EV_CHECK_ARG(max_n >= 1 && max_n <= EV_MAX_FRAMES && max_m >= 1 && max_m <= EV_MAX_FRAMES,
               "%s: max_n=%d, max_m=%d must lie in [1, %d]", what, max_n, max_m, EV_MAX_FRAMES);
  EV_CHECK_ARG(syn_frames >= max_n && ref_frames >= max_m, "%s: %lld / %lld frames per row hold fewer than %d / %d", what,
               syn_frames, ref_frames, max_n, max_m);
  EV_CHECK_ARG(!path || path_stride >= (long long)max_n + max_m - 1, "%s: path_stride=%lld must be at least %d", what,
               path_stride, max_n + max_m - 1);
  const size_t need = eval_ws_bytes(n_items, max_n, max_m);
  EV_CHECK_ARG(ws_bytes >= need, "%s: workspace of %zu bytes, %zu needed", what, ws_bytes, need);
  return EV_OK;
}

}  // namespace ev

using namespace ev;

extern "C" {

size_t ev_eval_workspace_bytes(int n_items, int max_n, int max_m) {
  return eval_args_ok(n_items, max_n, max_m) ? eval_ws_bytes(n_items, max_n, max_m) : 0;
}

int ev_eval_compare(const float* mel_syn, const double* f0_syn, long long syn_frames, const int32_t* n_syn, int max_n,
                    const float* mel_ref, const double* f0_ref, long long ref_frames, const int32_t* n_ref, int max_m, int n_items,
                    const double* table, double* stats, int32_t* counts, int32_t* path, long long path_stride, void* ws,
                    size_t ws_bytes, void* stream) {
  EV_CHECK_ARG(mel_syn && f0_syn && n_syn && mel_ref && f0_ref && n_ref && table && stats && counts && ws,
               "ev_eval_compare: null argument");
  EV_TRY(eval_args_check("ev_eval_compare", n_items, max_n, max_m, syn_frames, ref_frames, path, path_stride, ws_bytes));
  EV_TRY(use_device_of(mel_syn));
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  char* w = static_cast<char*>(ws);
  double* cep_syn = reinterpret_cast<double*>(w);
  double* cep_ref = reinterpret_cast<double*>(w + align256((size_t)n_items * max_n * EV_CEPS * sizeof(double)));
  const int max_f = max_n > max_m ? max_n : max_m;
  EV_TRY(launch("eval_cep_kernel", eval_cep_kernel, dim3((max_f + EC_FRAMES - 1) / EC_FRAMES, n_items, 2), EC_THREADS, 0, st, mel_syn,
                syn_frames, n_syn, max_n, mel_ref, ref_frames, n_ref, max_m, table, cep_syn, cep_ref));
  return eval_align_tail(cep_syn, max_n, f0_syn, syn_frames, n_syn, max_n, cep_ref, max_m, f0_ref, ref_frames, n_ref, max_m, n_items,
                         stats, counts, path, path_stride, w, st);
}

int ev_eval_align(const double* cep_syn, const double* f0_syn, long long syn_frames, const int32_t* n_syn, int max_n,
                  const double* cep_ref, const double* f0_ref, long long ref_frames, const int32_t* n_ref, int max_m, int n_items,
                  double* stats, int32_t* counts, int32_t* path, long long path_stride, void* ws, size_t ws_bytes, void* stream) {
  EV_CHECK_ARG(cep_syn && f0_syn && n_syn && cep_ref && f0_ref && n_ref && stats && counts && ws, "ev_eval_align: null argument");
  EV_TRY(eval_args_check("ev_eval_align", n_items, max_n, max_m, syn_frames, ref_frames, path, path_stride, ws_bytes));
  EV_TRY(use_device_of(cep_syn));
  return eval_align_tail(cep_syn, syn_frames, f0_syn, syn_frames, n_syn, max_n, cep_ref, ref_frames, f0_ref, ref_frames, n_ref, max_m,
                         n_items, stats, counts, path, path_stride, static_cast<char*>(ws), reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
