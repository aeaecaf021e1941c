// ctc_lexicon.cu -- lexicon-constrained CTC decoding: every entry of a caller's word list is scored by its exact CTC
// forward log-probability over the 48 kept steps, and the P best entries of each crop are returned.
//   q[t,c] = softmax(l_t)_c + 1e-7 (= exp(lp[t,c]) of the beam decoder), blank = K-1.  An entry l_1..l_L has the states
//   ext = (blank, l_1, blank, ..., l_L, blank), S = 2L+1; alpha_0 = (q[0,blank], q[0,l_1], 0, ...), and
//   alpha_t[s] = (alpha_{t-1}[s] + alpha_{t-1}[s-1] + [skip_s] alpha_{t-1}[s-2]) q[t, ext_s], where skip_s holds for a
//   label that differs from the label before it.  score = log(alpha_47[S-2] + alpha_47[S-1]).  An entry that is empty,
//   longer than 48, has a label outside [0, K-2] or needs more than 48 steps (L + adjacent repeats > 48) scores -inf.
//
// lex_forward_kernel<NL>: grid (crops, chunks of kChunk entries), one thread per entry.  The CTA computes its crop's q
//   into shared memory (48 rows of K+1 floats; column K is 0).  A thread keeps alpha in registers in the linear domain:
//   three additions and a multiplication per state and step, no exp / log.  Whenever its largest state leaves
//   [2^32, 2^100) the thread multiplies every state by an exact power of two and keeps the exponent E apart, so a score
//   of e^-774 or below stays representable and the scaling adds no rounding.  States that can no longer reach the end
//   in the steps left are zeroed first (exact: they never flow into one that can), so the largest state is one that
//   counts; its mass passes to a successor that still counts, multiplied by at least 1e-7, and no state grows by more
//   than 3 (1 + 1e-7) per step, so the largest never leaves the normal range between two checks and every alignable
//   entry's score is finite.  (A state more than 2^134 below the largest would lose bits as a subnormal; no test input
//   comes near that.)  States past the entry's end read the zero column and stay 0, so the register array can be longer
//   than the entry: the result does not depend on NL.  Each of the three launches (NL = 8, 16, 48 labels) takes the warps whose longest entry falls in its
//   range, so a warp costs what its own entries need.  The fp32 sum alpha is turned into log(sum) - E ln 2 in fp64 and
//   rounded once; the result is stored as the order-preserving key okey(score), 0 for -inf.
// lex_select_kernel: one CTA per crop.  The P best keys by an exact radix select; keys equal to the P-th take the
//   smallest entry indices (a second radix select, on the complemented index); the selected entries are ranked by
//   (key descending, index ascending) and their labels copied from the lexicon.
// A score is a function of the crop's logits and the entry alone (fixed reduction orders, no atomics on values) and the
// selection works on exact keys, so a crop's result is bit-identical in any batch, on every run, and whatever else the
// lexicon holds or in which order.
#include <math.h>

#include "common.cuh"
#include "ctc_q.cuh"

namespace {

using ctcq::kT;
constexpr int kThreads = 128, kChunk = 1024, kSelThreads = 256;
constexpr int kMaxLabelEnd = 1 << 24;            // entries whose labels end beyond 2^24 score -inf (B2O_MAX_LEXICON_LABELS)

__device__ __forceinline__ unsigned okey(float f) {           // order-preserving uint32 of a float
  const unsigned b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float unokey(unsigned k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// Entry i's length, 0 when its offsets do not describe 1..48 labels inside [0, 2^24).
__device__ __forceinline__ int entry_len(const int* __restrict__ offsets, int i, int* off) {
  const int o0 = offsets[i], o1 = offsets[i + 1];
  *off = o0;
  return (o0 >= 0 && o1 <= kMaxLabelEnd && o1 - o0 >= 1 && o1 - o0 <= kT) ? o1 - o0 : 0;
}

// q of one crop's 48 steps into s (row stride K+1, column K = 0): one warp per step, fixed-order reductions
// (ctc_q.cuh, shared with the training loss).
__device__ void stage_probs(const float* __restrict__ logits, int K, float* s) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int t = warp; t < kT; t += kThreads / 32) {
    const float* row = logits + t * K;
    float* out = s + t * (K + 1);
    float m, se;
    ctcq::ctc_step_norm(row, K, lane, &m, &se);
    for (int c = lane; c < K; c += 32) out[c] = ctcq::ctc_q(row[c], m, se);
    if (lane == 0) out[K] = 0.f;
  }
}

using ctcq::ctc_prune;
using ctcq::ctc_rescale;

// okey of the entry's CTC forward log-probability over q (row stride K+1), 0 for -inf.
template <int NL>
__device__ unsigned entry_key(const float* q, int K, const short* __restrict__ labels, int off, int L) {
  constexpr int NS = 2 * NL + 1;
  if (L <= 0) return 0u;
  int col[NL];
  bool bad = false;
#pragma unroll
  for (int i = 0; i < NL; ++i) {
    int c = K;                                                   // past the end: the zero column
    if (i < L) {
      c = labels[off + i];
      if (c < 0 || c > K - 2) { bad = true; c = K; }
    }
    col[i] = c;
  }
  if (bad) return 0u;
  unsigned long long rep = 0;                                    // bit i (0 < i < L): label i repeats label i-1
#pragma unroll
  for (int i = 1; i < NL; ++i)
    if (i < L && col[i] == col[i - 1]) rep |= 1ull << i;
  if (L + __popcll(rep) > kT) return 0u;                         // cannot be aligned in 48 steps
  float a[NS];
#pragma unroll
  for (int s = 0; s < NS; ++s) a[s] = 0.f;
  a[0] = q[K - 1];
  a[1] = q[col[0]];
  int e_sum = 0, live = 0;
  ctc_prune(a, live, kT - 1, L, rep);
  ctc_rescale(a, e_sum);
  for (int t = 1; t < kT; ++t) {
    const float* r = q + t * (K + 1);
    const float qb = r[K - 1];
#pragma unroll
    for (int s = NS - 1; s >= 1; --s) {                          // descending: a[s-1], a[s-2] are still step t-1's
      float v = __fadd_rn(a[s], a[s - 1]);
      if (s & 1) {
        const int i = s >> 1;
        if (i > 0 && !((rep >> i) & 1ull)) v = __fadd_rn(v, a[s - 2]);
        v = __fmul_rn(v, r[col[i]]);
      } else {
        v = __fmul_rn(v, qb);
      }
      a[s] = v;
    }
    a[0] = __fmul_rn(a[0], qb);
    ctc_prune(a, live, kT - 1 - t, L, rep);
    ctc_rescale(a, e_sum);
  }
  const int S = 2 * L + 1;
  float x2 = 0.f, x1 = 0.f;
#pragma unroll
  for (int s = 0; s < NS; ++s) {
    if (s == S - 2) x2 = a[s];
    if (s == S - 1) x1 = a[s];
  }
  const float x = __fadd_rn(x2, x1);
  if (!(x > 0.f)) return 0u;
  const double v = log(static_cast<double>(x)) - static_cast<double>(e_sum) * 0.69314718055994530942;
  return okey(__double2float_rn(v));
}

template <int NL>
__global__ void __launch_bounds__(kThreads)
lex_forward_kernel(const float* __restrict__ logits /*[B][48][K]*/, int K, const int* __restrict__ offsets,
                   const short* __restrict__ labels, int n_words, int lo, unsigned* __restrict__ keys /*[B][n_words]*/) {
  extern __shared__ float q[];                                   // [48][K+1]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, b = blockIdx.x;
  const int base = blockIdx.y * kChunk, end = min(n_words, base + kChunk);
  // a warp group of 32 entries is this launch's when its longest entry has lo < L <= NL (invalid entries count as 1)
  bool any = false;
  for (int g = base + warp * 32; g < end; g += kThreads) {
    int off, len = 1;
    if (g + lane < end) len = max(1, entry_len(offsets, g + lane, &off));
    const int mx = __reduce_max_sync(0xffffffffu, len);
    any |= mx > lo && mx <= NL;
  }
  if (!__syncthreads_or(any)) return;
  stage_probs(logits + static_cast<size_t>(b) * kT * K, K, q);
  __syncthreads();
  for (int g = base + warp * 32; g < end; g += kThreads) {
    const int i = g + lane;
    int off = 0, len = 0;
    if (i < end) len = entry_len(offsets, i, &off);
    const int mx = __reduce_max_sync(0xffffffffu, max(1, i < end ? len : 1));
    if (mx <= lo || mx > NL) continue;
    const unsigned k = entry_key<NL>(q, K, labels, off, len);
    if (i < end) keys[static_cast<size_t>(b) * n_words + i] = k;
  }
}

// The k-th largest nonzero key(i), i < n (1 <= k <= number of nonzero keys), by an MSB-first radix select: returns it;
// *take = how many keys equal to it belong to the k largest, *equal = how many keys equal it.
template <class F>
__device__ unsigned radix_select(int n, int k, F key, unsigned* hist, int* misc, int* take, int* equal) {
  const int lane = threadIdx.x & 31;
  unsigned prefix = 0, mask = 0;
  int kk = k, eq = 0;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += kSelThreads) hist[i] = 0;
    __syncthreads();
    for (int i0 = 0; i0 < n; i0 += kSelThreads) {
      const int i = i0 + threadIdx.x;
      const unsigned v = i < n ? key(i) : 0u;
      const bool ok = v != 0u && (v & mask) == prefix;
      const unsigned d = (v >> shift) & 255u;
      const unsigned peers = __match_any_sync(0xffffffffu, ok ? d : 0x100u);
      if (ok && lane == __ffs(peers) - 1) atomicAdd(&hist[d], static_cast<unsigned>(__popc(peers)));
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned c = 0;
      for (int d = 255; d >= 0; --d) {
        if (c + hist[d] >= static_cast<unsigned>(kk)) {
          misc[0] = d;
          misc[1] = kk - static_cast<int>(c);
          misc[2] = static_cast<int>(hist[d]);
          break;
        }
        c += hist[d];
      }
    }
    __syncthreads();
    prefix |= static_cast<unsigned>(misc[0]) << shift;
    mask |= 255u << shift;
    kk = misc[1];
    eq = misc[2];
    __syncthreads();
  }
  *take = kk;
  *equal = eq;
  return prefix;
}

__global__ void __launch_bounds__(kSelThreads)
lex_select_kernel(const unsigned* __restrict__ keys /*[B][n]*/, int n, const int* __restrict__ offsets,
                  const short* __restrict__ labels, int P, int* __restrict__ out /*[B][P][48]*/,
                  float* __restrict__ logp /*[B][P] or null*/) {
  __shared__ unsigned hist[256], sel_key[B2O_MAX_LEXICON_TOP_PATHS];
  __shared__ int sel_idx[B2O_MAX_LEXICON_TOP_PATHS], misc[4], count[2];
  const int b = blockIdx.x;
  const unsigned* key = keys + static_cast<size_t>(b) * n;
  if (threadIdx.x == 0) count[0] = count[1] = 0;
  __syncthreads();
  int valid = 0;
  for (int i = threadIdx.x; i < n; i += kSelThreads) valid += key[i] != 0u;
  atomicAdd(&count[0], valid);
  __syncthreads();
  const int nvalid = count[0];
  unsigned theta = 1u, tie = 0u;                                 // all nonzero keys when there are at most P of them
  if (nvalid > P) {
    int take, equal;
    theta = radix_select(n, P, [&](int i) { return key[i]; }, hist, misc, &take, &equal);
    if (take < equal) {                                          // ties with the P-th: the smallest indices
      int t2, e2;
      const unsigned th = theta;
      tie = radix_select(n, take, [&](int i) { return key[i] == th ? ~static_cast<unsigned>(i) : 0u; }, hist, misc,
                         &t2, &e2);
    }
  }
  for (int i = threadIdx.x; i < n; i += kSelThreads) {
    const unsigned k = key[i];
    if (k != 0u && (k > theta || (k == theta && ~static_cast<unsigned>(i) >= tie))) {
      const int slot = atomicAdd(&count[1], 1);
      sel_key[slot] = k;
      sel_idx[slot] = i;
    }
  }
  __syncthreads();
  const int nsel = count[1];
  for (int j = threadIdx.x; j < nsel; j += kSelThreads) {      // rank: key descending, index ascending
    const unsigned k = sel_key[j];
    const int idx = sel_idx[j];
    int rank = 0;
    for (int m = 0; m < nsel; ++m) rank += sel_key[m] > k || (sel_key[m] == k && sel_idx[m] < idx);
    int* o = out + (static_cast<size_t>(b) * P + rank) * kT;
    const int o0 = offsets[idx], len = offsets[idx + 1] - o0;
    for (int u = 0; u < kT; ++u) o[u] = u < len ? labels[o0 + u] : -1;
    if (logp) logp[static_cast<size_t>(b) * P + rank] = unokey(k);
  }
  for (int r = nsel + threadIdx.x; r < P; r += kSelThreads) {   // fewer finite-score entries than paths asked for
    int* o = out + (static_cast<size_t>(b) * P + r) * kT;
    for (int u = 0; u < kT; ++u) o[u] = -1;
    if (logp) logp[static_cast<size_t>(b) * P + r] = -INFINITY;
  }
}

template <int NL>
int forward_launch(b2o_ctx* ctx, const float* logits, int B, int K, const int* offsets, const short* labels, int n_words,
                   int lo, unsigned* keys, cudaStream_t st) {
  const size_t bytes = static_cast<size_t>(kT) * (K + 1) * sizeof(float);
  B2O_CUDA_CHECK(ctx, cudaFuncSetAttribute(lex_forward_kernel<NL>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           static_cast<int>(bytes)));
  const dim3 grid(B, (n_words + kChunk - 1) / kChunk);
  lex_forward_kernel<NL><<<grid, kThreads, bytes, st>>>(logits, K, offsets, labels, n_words, lo, keys);
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}

}  // namespace

size_t ctc_lexicon_workspace_bytes(int B, int n_words) {
  return (static_cast<size_t>(B) * n_words * sizeof(unsigned) + 255) / 256 * 256;
}

int ctc_lexicon_run(b2o_ctx* ctx, const float* logits, int B, int K, const int* offsets, const short* labels,
                    int n_words, int top_paths, int* labels_out, float* logp, void* ws, cudaStream_t st) {
  if (B <= 0) return B2O_OK;
  unsigned* keys = reinterpret_cast<unsigned*>(ws);
  B2O_RETURN_IF(forward_launch<8>(ctx, logits, B, K, offsets, labels, n_words, 0, keys, st));
  B2O_RETURN_IF(forward_launch<16>(ctx, logits, B, K, offsets, labels, n_words, 8, keys, st));
  B2O_RETURN_IF(forward_launch<48>(ctx, logits, B, K, offsets, labels, n_words, 16, keys, st));
  lex_select_kernel<<<B, kSelThreads, 0, st>>>(keys, n_words, offsets, labels, top_paths, labels_out, logp);
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}
