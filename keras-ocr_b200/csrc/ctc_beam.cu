// ctc_beam.cu -- CTC prefix beam search over the fc_12 logits (the greedy=False form of keras.backend.ctc_decode that
// the reference's CTCDecoder does not use, recognition.py:169-184).  Graves 2012 / Hannun et al. 2014:
//   lp[t,c] = log(softmax(l_t)_c + 1e-7), blank = K-1.  A beam is a label prefix with log-probabilities p_b (ending in
//   blank) and p_nb (ending in a label); score = logaddexp(p_b, p_nb).  Start: the empty prefix, p_b = 0, p_nb = -inf.
//   Per step every beam b yields: b via blank (p_b' = score + lp[blank]), b via its last label (p_nb' = p_nb + lp[last]),
//   and b+c for every label c (p_nb' = (c == last ? p_b : score) + lp[c]); equal prefixes merge with logaddexp and the
//   W best survive.  Order: score descending, equal scores by label sequence ascending, a prefix before its extensions.
//   Repeated letters stay as the prefix search yields them (no merge_repeated post-pass).
//
// ctc_beam_kernel: one CTA per crop, everything in shared memory.  Per step:
//   1. lp of the step in fp32 (block max, fixed-order sum-exp);
//   2. the shortlist: the S = min(W+1, K-1) labels with the largest lp (ties: smaller label first);
//   3. parent links: beam b = a + last(b) with a a beam (64-bit prefix hashes, confirmed by comparing the prefixes);
//   4. candidate i = a * (S+1) + x: x = 0 is beam a itself -- via blank, via its last label, and via the extension of its
//      parent, whatever the label -- and x > 0 the extension of a by shortlist label x-1, unless that is already a beam;
//   5. the W best by an exact radix select on the order-preserving key of the fp32 score; candidates that tie with the
//      W-th take the remaining places in label-sequence order; the survivors are compacted in candidate order.
// Why the shortlist loses nothing: let c be outside it and a+c not a beam.  The only candidate that yields a+c is a's
// extension by c, of score (c == last(a) ? p_b(a) : score(a)) + lp[c].  S = W+1 labels c' rank above c (lp[c'] > lp[c],
// or equal with c' < c); at most one of them is last(a), so at least W of them give a+c' a contribution score(a) + lp[c']
// >= the score of a+c (p_b <= score), and merging only adds to it.  Each of those W prefixes beats a+c -- strictly, or
// tied and ranked first because a+c' < a+c -- so a+c is not among the W best.  In fp32 the inequalities hold too (the
// additions round monotonically and logaddexp(x, y) >= max(x, y)); only two candidates whose fp32 scores round to the
// same value can be ordered differently from exact arithmetic, which is a near-tie the tests bound (tests/test_gpu_beam.py).
// Everything is a function of the crop's logits alone (fixed reduction orders, exact keys, ordered compaction): a crop
// decodes bit-identically in any batch and on every run.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kT = 48, kThreads = 256, kWarps = kThreads / 32;
constexpr unsigned long long kHashMul = 0x100000001B3ull, kHashRoot = 0xcbf29ce484222325ull;

__device__ __forceinline__ unsigned okey(float f) {           // order-preserving uint32 of a float
  const unsigned b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float unokey(unsigned k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

__device__ __forceinline__ float lae(float a, float b) {     // log(exp(a) + exp(b))
  if (a == -INFINITY) return b;
  if (b == -INFINITY) return a;
  return __fadd_rn(fmaxf(a, b), log1pf(expf(-fabsf(__fsub_rn(a, b)))));
}

// Shared-memory plan, the same on the host (sizes) and the device (pointers).
struct Smem {
  float* lp;                       // [K]
  short* pos;                      // [K] shortlist position of a label, -1 when not in it
  int* shortl;                     // [S]
  short* pre[2];                   // [W][48] prefixes, double-buffered
  int* len[2];
  float *pb[2], *pnb[2], *sc[2];   // [W]
  unsigned long long *h[2], *ph[2];  // [W] hash of the prefix and of the prefix without its last label
  int* parent;                     // [W]
  unsigned char* excl;             // [W][S] extension a+shortl[x] is already a beam
  unsigned* key;                   // [W][S+1] candidate keys (0: no candidate)
  unsigned char* sel;              // [W][S+1]
  unsigned* hist;                  // [256]
  int* red;                        // [kWarps + 8] scratch of the block reductions
};

__host__ __device__ inline int shortlist_size(int W, int K) { return W + 1 < K - 1 ? W + 1 : K - 1; }

__host__ __device__ inline size_t smem_plan(int W, int K, unsigned char* base, Smem* s) {
  const int S = shortlist_size(W, K), S1 = S + 1;
  size_t off = 0;
#define B2O_TAKE(ptr, type, count)                                                    \
  do {                                                                                \
    if (base) (ptr) = reinterpret_cast<type*>(base + off);                            \
    off += (static_cast<size_t>(count) * sizeof(type) + 15) / 16 * 16;                \
  } while (0)
  Smem d;
  Smem* p = s ? s : &d;
  B2O_TAKE(p->lp, float, K);
  B2O_TAKE(p->pos, short, K);
  B2O_TAKE(p->shortl, int, S);
  for (int i = 0; i < 2; ++i) {
    B2O_TAKE(p->pre[i], short, W * kT);
    B2O_TAKE(p->len[i], int, W);
    B2O_TAKE(p->pb[i], float, W);
    B2O_TAKE(p->pnb[i], float, W);
    B2O_TAKE(p->sc[i], float, W);
    B2O_TAKE(p->h[i], unsigned long long, W);
    B2O_TAKE(p->ph[i], unsigned long long, W);
  }
  B2O_TAKE(p->parent, int, W);
  B2O_TAKE(p->excl, unsigned char, W * S);
  B2O_TAKE(p->key, unsigned, W * S1);
  B2O_TAKE(p->sel, unsigned char, W * S1);
  B2O_TAKE(p->hist, unsigned, 256);
  B2O_TAKE(p->red, int, kWarps + 8);
#undef B2O_TAKE
  return off;
}

// Exclusive prefix sum of v over the block in thread order; *total = the sum.
__device__ int block_scan(int v, int* red, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) red[warp] = x;
  __syncthreads();
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int w = 0; w < kWarps; ++w) { const int t = red[w]; red[w] = acc; acc += t; }
    red[kWarps] = acc;
  }
  __syncthreads();
  const int r = red[warp] + x - v;
  *total = red[kWarps];
  __syncthreads();
  return r;
}

// The k-th largest (1 <= k <= number of nonzero keys) of key(i), i < n, by an MSB-first radix select: returns it as
// theta; *take = how many keys equal to theta belong to the k largest, *equal = how many keys equal theta.
template <class F>
__device__ unsigned radix_select(int n, int k, F key, unsigned* hist, int* red, int* take, int* equal) {
  unsigned prefix = 0, mask = 0;
  int kk = k;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += kThreads) hist[i] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += kThreads) {
      const unsigned v = key(i);
      if ((v & mask) == prefix) atomicAdd(&hist[(v >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (threadIdx.x < 32) {                         // lane l scans digits 255-8l .. 248-8l, from the top
      const int lane = threadIdx.x;
      unsigned s = 0;
      for (int j = 0; j < 8; ++j) s += hist[255 - 8 * lane - j];
      unsigned inc = s;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned y = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += y;
      }
      unsigned c = inc - s;
      if (c < static_cast<unsigned>(kk) && inc >= static_cast<unsigned>(kk)) {
        for (int j = 0; j < 8; ++j) {
          const int d = 255 - 8 * lane - j;
          if (c + hist[d] >= static_cast<unsigned>(kk)) {
            red[kWarps + 1] = d;
            red[kWarps + 2] = kk - static_cast<int>(c);
            red[kWarps + 3] = static_cast<int>(hist[d]);
            break;
          }
          c += hist[d];
        }
      }
    }
    __syncthreads();
    prefix |= static_cast<unsigned>(red[kWarps + 1]) << shift;
    mask |= 255u << shift;
    kk = red[kWarps + 2];
    __syncthreads();
  }
  *take = kk;
  *equal = red[kWarps + 3];
  return prefix;
}

struct Beams {
  const Smem& s;
  int cur, S1;
  __device__ int len(int a) const { return s.len[cur][a]; }
  __device__ int last(int a) const { const int l = s.len[cur][a]; return l ? s.pre[cur][a * kT + l - 1] : -1; }
  // label sequence of candidate i at position t (t < its length)
  __device__ int at(int i, int t) const {
    const int a = i / S1, x = i - a * S1;
    return t < s.len[cur][a] ? s.pre[cur][a * kT + t] : s.shortl[x - 1];
  }
  __device__ int clen(int i) const { const int a = i / S1; return s.len[cur][a] + (i - a * S1 > 0); }
  // candidate i's label sequence before candidate j's (a prefix before its extensions)
  __device__ bool lex_less(int i, int j) const {
    const int li = clen(i), lj = clen(j), n = li < lj ? li : lj;
    for (int t = 0; t < n; ++t) {
      const int u = at(i, t), v = at(j, t);
      if (u != v) return u < v;
    }
    return li < lj;
  }
  // contribution of beam a's extension by label c
  __device__ float ext(int a, int c) const {
    return __fadd_rn(c == last(a) ? s.pb[cur][a] : s.sc[cur][a], s.lp[c]);
  }
  __device__ void eval(int i, int blank, float* pb, float* pnb) const {
    const int a = i / S1, x = i - a * S1;
    if (x == 0) {
      const int l = last(a);
      *pb = __fadd_rn(s.sc[cur][a], s.lp[blank]);
      float nb = l >= 0 ? __fadd_rn(s.pnb[cur][a], s.lp[l]) : -INFINITY;
      if (s.parent[a] >= 0) nb = lae(nb, ext(s.parent[a], l));
      *pnb = nb;
    } else {
      *pb = -INFINITY;
      *pnb = ext(a, s.shortl[x - 1]);
    }
  }
};

__global__ void __launch_bounds__(kThreads)
ctc_beam_kernel(const float* __restrict__ logits /*[B][48][K]*/, int K, int W, int P, int* __restrict__ labels /*[B][P][48]*/,
                float* __restrict__ logp /*[B][P] or null*/) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Smem s;
  smem_plan(W, K, smem_raw, &s);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int blank = K - 1, S = shortlist_size(W, K), S1 = S + 1;
  int cur = 0, nb = 1;
  if (tid == 0) {
    s.len[0][0] = 0; s.pb[0][0] = 0.f; s.pnb[0][0] = -INFINITY; s.sc[0][0] = 0.f;
    s.h[0][0] = kHashRoot; s.ph[0][0] = 0;
  }
  for (int t = 0; t < kT; ++t) {
    // ---- 1. lp of step t
    const float* row = logits + (static_cast<size_t>(blockIdx.x) * kT + t) * K;
    float m = -INFINITY;
    for (int c = tid; c < K; c += kThreads) { const float v = row[c]; s.lp[c] = v; m = fmaxf(m, v); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float* redf = reinterpret_cast<float*>(s.red);
    if (lane == 0) redf[warp] = m;
    __syncthreads();
    m = redf[0];
    for (int w = 1; w < kWarps; ++w) m = fmaxf(m, redf[w]);
    float se = 0.f;
    for (int c = tid; c < K; c += kThreads) se = __fadd_rn(se, expf(__fsub_rn(s.lp[c], m)));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) se = __fadd_rn(se, __shfl_xor_sync(0xffffffffu, se, o));
    __syncthreads();
    if (lane == 0) redf[warp] = se;
    __syncthreads();
    se = redf[0];
    for (int w = 1; w < kWarps; ++w) se = __fadd_rn(se, redf[w]);
    for (int c = tid; c < K; c += kThreads)
      s.lp[c] = logf(__fadd_rn(__fdiv_rn(expf(__fsub_rn(s.lp[c], m)), se), 1e-7f));
    __syncthreads();

    // ---- 2. shortlist: labels in ascending order, a thread owns a contiguous range
    {
      const int n = K - 1, chunk = (n + kThreads - 1) / kThreads, c0 = min(n, tid * chunk), c1 = min(n, c0 + chunk);
      unsigned theta = 0;
      int take = n, equal = 0;
      if (S < n) theta = radix_select(n, S, [&](int c) { return okey(s.lp[c]); }, s.hist, s.red, &take, &equal);
      int eq = 0;
      for (int c = c0; c < c1; ++c) eq += okey(s.lp[c]) == theta;
      int total;
      const int eq0 = block_scan(eq, s.red, &total);   // labels tied with theta before this thread's range
      int eq_before = eq0, cnt = 0;
      for (int c = c0; c < c1; ++c) {
        const unsigned k = okey(s.lp[c]);
        cnt += S == n || k > theta || (k == theta && eq_before++ < take);
      }
      eq_before = eq0;
      int at = block_scan(cnt, s.red, &total);
      for (int c = c0; c < c1; ++c) {
        const unsigned k = okey(s.lp[c]);
        const bool in = S == n || k > theta || (k == theta && eq_before++ < take);
        s.pos[c] = in ? static_cast<short>(at) : static_cast<short>(-1);
        if (in) s.shortl[at++] = c;
      }
      if (tid == 0) s.pos[blank] = -1;
    }

    // ---- 3. parent links and the extensions that are already beams
    const Beams bm{s, cur, S1};
    for (int i = tid; i < nb * S; i += kThreads) s.excl[i] = 0;
    if (tid < nb) {
      int par = -1;
      const int l = s.len[cur][tid];
      if (l > 0)
        for (int a = 0; a < nb && par < 0; ++a) {
          if (s.len[cur][a] != l - 1 || s.h[cur][a] != s.ph[cur][tid]) continue;
          bool same = true;
          for (int u = 0; u < l - 1 && same; ++u) same = s.pre[cur][a * kT + u] == s.pre[cur][tid * kT + u];
          if (same) par = a;
        }
      s.parent[tid] = par;
    }
    __syncthreads();
    if (tid < nb && s.parent[tid] >= 0) {
      const int q = s.pos[bm.last(tid)];
      if (q >= 0) s.excl[s.parent[tid] * S + q] = 1;
    }
    __syncthreads();

    // ---- 4. candidate keys
    const int n = nb * S1;
    int valid = 0;
    for (int i = tid; i < n; i += kThreads) {
      const int a = i / S1, x = i - a * S1;
      unsigned k = 0;
      if (x == 0 || !s.excl[a * S + x - 1]) {
        float pb, pnb;
        bm.eval(i, blank, &pb, &pnb);
        k = okey(lae(pb, pnb));
        ++valid;
      }
      s.key[i] = k;
      s.sel[i] = 0;
    }
    int nvalid;
    block_scan(valid, s.red, &nvalid);

    // ---- 5. the W best
    if (nvalid <= W) {
      for (int i = tid; i < n; i += kThreads) s.sel[i] = s.key[i] != 0;
    } else {
      int take, equal;
      const unsigned theta = radix_select(n, W, [&](int i) { return s.key[i]; }, s.hist, s.red, &take, &equal);
      for (int i = tid; i < n; i += kThreads) s.sel[i] = s.key[i] > theta || (take == equal && s.key[i] == theta);
      __syncthreads();
      // ties with the W-th score: the label-sequence order picks `take` of them, one block-wide minimum at a time
      for (int r = 0; r < take && take < equal; ++r) {
        int best = -1;
        for (int i = tid; i < n; i += kThreads)
          if (s.key[i] == theta && !s.sel[i] && (best < 0 || bm.lex_less(i, best))) best = i;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const int other = __shfl_xor_sync(0xffffffffu, best, o);
          if (other >= 0 && (best < 0 || bm.lex_less(other, best))) best = other;
        }
        if (lane == 0) s.red[warp] = best;
        __syncthreads();
        if (tid == 0) {
          int b = -1;
          for (int w = 0; w < kWarps; ++w) {
            const int o = s.red[w];
            if (o >= 0 && (b < 0 || bm.lex_less(o, b))) b = o;
          }
          s.sel[b] = 1;
        }
        __syncthreads();
      }
    }
    __syncthreads();

    // ---- 6. compaction in candidate order into the other buffer
    {
      const int chunk = (n + kThreads - 1) / kThreads, i0 = min(n, tid * chunk), i1 = min(n, i0 + chunk);
      int cnt = 0;
      for (int i = i0; i < i1; ++i) cnt += s.sel[i];
      int total;
      int slot = block_scan(cnt, s.red, &total);
      const int nx = cur ^ 1;
      for (int i = i0; i < i1; ++i) {
        if (!s.sel[i]) continue;
        const int a = i / S1, x = i - a * S1, l = s.len[cur][a];
        float pb, pnb;
        bm.eval(i, blank, &pb, &pnb);
        for (int u = 0; u < l; ++u) s.pre[nx][slot * kT + u] = s.pre[cur][a * kT + u];
        if (x > 0) {
          const int c = s.shortl[x - 1];
          s.pre[nx][slot * kT + l] = static_cast<short>(c);
          s.h[nx][slot] = s.h[cur][a] * kHashMul + static_cast<unsigned long long>(c + 1);
          s.ph[nx][slot] = s.h[cur][a];
        } else {
          s.h[nx][slot] = s.h[cur][a];
          s.ph[nx][slot] = s.ph[cur][a];
        }
        s.len[nx][slot] = l + (x > 0);
        s.pb[nx][slot] = pb;
        s.pnb[nx][slot] = pnb;
        s.sc[nx][slot] = unokey(s.key[i]);        // the selection key's score, bit for bit
        ++slot;
      }
      nb = total;
      cur = nx;
      __syncthreads();
    }
  }

  // ---- the P best of the final beams, best first
  const Beams fin{s, cur, 1};                      // S1 = 1: candidate i is beam i itself
  const int b = blockIdx.x;
  if (tid < nb) {
    const unsigned k = okey(s.sc[cur][tid]);
    int rank = 0;
    for (int a = 0; a < nb; ++a) {
      const unsigned ka = okey(s.sc[cur][a]);
      rank += ka > k || (ka == k && a != tid && fin.lex_less(a, tid));
    }
    if (rank < P) {
      int* o = labels + (static_cast<size_t>(b) * P + rank) * kT;
      const int l = s.len[cur][tid];
      for (int u = 0; u < kT; ++u) o[u] = u < l ? s.pre[cur][tid * kT + u] : -1;
      if (logp) logp[static_cast<size_t>(b) * P + rank] = s.sc[cur][tid];
    }
  }
  for (int r = nb + tid; r < P; r += kThreads) {   // fewer distinct prefixes than paths asked for (tiny K)
    int* o = labels + (static_cast<size_t>(b) * P + r) * kT;
    for (int u = 0; u < kT; ++u) o[u] = -1;
    if (logp) logp[static_cast<size_t>(b) * P + r] = -INFINITY;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// ctc_beam_lm_kernel: the same search ranked by a character language model (DESIGN.md section 1, "Language model").
//   A beam also carries G(a) in fp32: G(empty) = 0, G(a + c) = G(a) + (alpha * l(c | hist(a)) + beta), hist(a) the last
//   order-1 symbols of "<s> a" and l the fp32 row value of its longest listed suffix.  Candidates are ranked by
//   F = A + G (rounded once), A = logaddexp(p_b, p_nb) the acoustic score; G is a function of the prefix, so merging
//   equal prefixes is unchanged.  After the last step F_end = F + alpha * l(</s> | hist) ranks the returned paths.
// Per step, besides steps 1-6 above:
//   2'. the shortlist is per beam: the S = min(W+1, K-1) labels with the largest lp[c] + alpha * l(c | hist(a)) (ties:
//       smaller label first), one warp per beam (a 32-round bitwise radix select over the order-preserving keys);
//   6'. a beam whose history changed (an extension) looks up its row once: the longest listed suffix of its history by
//       binary search over the sorted keys (at most order-1 searches), then reads K floats of that row per use from
//       global memory (L2-resident).  A beam kept via blank or its last label keeps its parent's row.
// Why the per-beam shortlist loses nothing: let c be outside a's shortlist and a+c not a beam.  The only candidate that
// yields a+c is a's extension by c: F(a+c) = (c == last(a) ? p_b(a) : A(a)) + lp[c] + G(a) + alpha l(c | hist(a)) + beta.
// S = W+1 labels c' rank above c in lp[c'] + alpha l(c' | hist(a)); at most one of them is last(a), so at least W of
// them give a+c' an F >= A(a) + lp[c'] + G(a) + alpha l(c' | hist(a)) + beta >= F(a+c) (p_b <= A, merging only adds,
// and F is monotone in A), and each of those W prefixes beats a+c or ties and precedes it.  In fp32 the three sums are
// split differently from the shortlist key, so two candidates within a few ulps of F can be ordered differently from
// exact arithmetic: a near-tie, which tests/test_gpu_lm.py counts and bounds.
// With alpha = beta = 0 every alpha * l is +-0, so the shortlist key is lp, G = +0, F = A and F_end = A bit for bit: the
// per-beam shortlists equal the global one and the search returns ctc_beam_kernel's labels and scores exactly.
//
// Hotwords (kHot, DESIGN.md section 1, "Hotwords"): the same kernel also ranks by a bonus for a caller's word list.
//   A prefix is live when it is a prefix of a listed word (the empty prefix is); H(a) = gamma |a| when a is live, else 0,
//   and H_end(a) = gamma |a| when a is a listed word, else 0.  Candidates rank by F = (A + G) + H and the returned paths
//   by F_end = ((A + G) + alpha l(</s> | hist)) + H_end, each addition of H or H_end skipped when it is 0 (so gamma = 0,
//   or an empty list, gives the kernel without kHot bit for bit).  H is a function of the prefix: merging is unchanged.
//   A beam also carries its trie node (-1 once it is not live): a beam kept via blank or its last label keeps its
//   parent's node, an extension a+c looks up the child of a's node by c once, by binary search over the sorted edge
//   keys (parent << 8) | label, whose children of one node are contiguous.
//   2''. the shortlist key of c is lp[c] + alpha l(c | hist(a)) + H(a+c) (the addition skipped when H(a+c) = 0): F(a+c)
//       less the per-beam terms A(a) or p_b(a), G(a) and beta.  A live a finds its children's range once, and each lane
//       its labels in that range; the shortlist records which of its labels keep a+c live.
// Why the per-beam shortlist still loses nothing: F(a+c) = (c == last(a) ? p_b(a) : A(a)) + G(a) + beta + key(c) in
// exact arithmetic.  S = W+1 labels c' rank above c by key; at most one of them is last(a), so at least W of them give
// a+c' an F >= A(a) + G(a) + beta + key(c') >= F(a+c) (H(a+c') enters F(a+c') exactly as it enters key(c'), merging
// only adds to A, and F is monotone in A), and each of those W prefixes beats a+c or ties and precedes it.  In fp32
// the key and F group the sums differently, so candidates within a few ulps of F can be ordered differently from exact
// arithmetic: a near-tie, which tests/test_gpu_hotwords.py counts and bounds.
constexpr unsigned kLmBos = 127u;                 // the code of <s> in a packed history (labels are < 126)

struct Trie {                                     // b2o_hotwords on the device (kHot only)
  const unsigned long long* keys;                 // [n_edges] (parent << 8) | label, ascending
  const int* child;                               // [n_edges] the child node of each edge
  const unsigned char* fin;                       // [n_nodes] 1: the node's prefix is a listed word
  int n_edges;
  float gamma;
};

// The first index in [lo, hi) whose key is >= k.
__device__ __forceinline__ int lower_key(const unsigned long long* __restrict__ keys, int lo, int hi,
                                         unsigned long long k) {
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(keys + mid) < k) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// The child of live node u by label c, or -1.
__device__ int trie_child(const Trie& tr, int u, int c) {
  const unsigned long long k = (static_cast<unsigned long long>(u) << 8) | static_cast<unsigned>(c);
  const int j = lower_key(tr.keys, 0, tr.n_edges, k);
  return j < tr.n_edges && __ldg(tr.keys + j) == k ? __ldg(tr.child + j) : -1;
}

struct SmemLm {
  short* shl;                      // [W][S] per-beam shortlist, ascending labels
  float *g[2], *f[2];              // [W] G and F of each beam
  int* row[2];                     // [W] the beam's LM row
  unsigned char* chg;              // [W] the beam's history changed this step
};

__host__ __device__ inline size_t smem_plan_lm(int W, int K, unsigned char* base, Smem* s, SmemLm* l) {
  size_t off = smem_plan(W, K, base, s);
  const int S = shortlist_size(W, K);
  SmemLm d;
  SmemLm* p = l ? l : &d;
#define B2O_TAKE(ptr, type, count)                                                    \
  do {                                                                                \
    if (base) (ptr) = reinterpret_cast<type*>(base + off);                            \
    off += (static_cast<size_t>(count) * sizeof(type) + 15) / 16 * 16;                \
  } while (0)
  B2O_TAKE(p->shl, short, W * S);
  for (int i = 0; i < 2; ++i) {
    B2O_TAKE(p->g[i], float, W);
    B2O_TAKE(p->f[i], float, W);
    B2O_TAKE(p->row[i], int, W);
  }
  B2O_TAKE(p->chg, unsigned char, W);
#undef B2O_TAKE
  return off;
}

struct SmemHot {
  int* node[2];                    // [W] the beam's trie node, -1 once its prefix is not live
  unsigned char* kid;              // [W][S] shl[x] keeps the beam's prefix live
};

__host__ __device__ inline size_t smem_plan_hot(int W, int K, unsigned char* base, Smem* s, SmemLm* l, SmemHot* h) {
  size_t off = smem_plan_lm(W, K, base, s, l);
  const int S = shortlist_size(W, K);
  SmemHot d;
  SmemHot* p = h ? h : &d;
#define B2O_TAKE(ptr, type, count)                                                    \
  do {                                                                                \
    if (base) (ptr) = reinterpret_cast<type*>(base + off);                            \
    off += (static_cast<size_t>(count) * sizeof(type) + 15) / 16 * 16;                \
  } while (0)
  for (int i = 0; i < 2; ++i) B2O_TAKE(p->node[i], int, W);
  B2O_TAKE(p->kid, unsigned char, W * S);
#undef B2O_TAKE
  return off;
}

// The row of the longest listed suffix of the history of "<s> pre[0..L)": keys sorted ascending, (n << 56) | the n
// symbols packed 8 bits each, oldest highest; keys[0] = 0 is the empty history.
__device__ int lm_row(const unsigned long long* __restrict__ keys, int H, int order, const short* pre, int L) {
  const int top = min(order - 1, L + 1);
  for (int n = top; n >= 1; --n) {
    unsigned long long k = static_cast<unsigned long long>(n) << 56;
    for (int i = 0; i < n; ++i) {
      const int p = L + 1 - n + i;                // position in "<s> a"
      const unsigned sym = p == 0 ? kLmBos : static_cast<unsigned>(pre[p - 1]);
      k |= static_cast<unsigned long long>(sym) << (8 * (n - 1 - i));
    }
    int lo = 0, hi = H;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (__ldg(keys + mid) < k) lo = mid + 1; else hi = mid;
    }
    if (lo < H && __ldg(keys + lo) == k) return lo;
  }
  return 0;
}

// One warp: the S labels c < n with the largest lp[c] + alpha * lrow[c] (ties: smaller label), ascending, into out[S].
// kHot: plus hb = H(a+c) for the labels that keep the beam's prefix live (node >= 0: its trie node); kid[S] then flags
// those labels of out.
template <bool kHot>
__device__ void lm_shortlist(const float* lp, const float* __restrict__ lrow, float alpha, int n, int S, short* out,
                             const Trie& tr, int node, float hb, unsigned char* kid) {
  const int lane = threadIdx.x & 31;
  const unsigned lt = (1u << lane) - 1u;
  unsigned kv[4];
  unsigned live = 0;                              // kHot: bit i set when lane + 32 i keeps the prefix live
  if constexpr (kHot) {
    int lo = 0, hi = 0;
    const unsigned long long base = static_cast<unsigned long long>(node) << 8;
    if (node >= 0) {                              // the node's children: one contiguous key range
      lo = lower_key(tr.keys, 0, tr.n_edges, base);
      hi = lower_key(tr.keys, lo, tr.n_edges, base + 256);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = lane + 32 * i;
      float v = 0.f;
      if (c < n) {
        v = __fadd_rn(lp[c], __fmul_rn(alpha, __ldg(lrow + c)));
        if (lo < hi) {
          const int j = lower_key(tr.keys, lo, hi, base | static_cast<unsigned>(c));
          if (j < hi && __ldg(tr.keys + j) == (base | static_cast<unsigned>(c))) {
            live |= 1u << i;
            if (hb != 0.f) v = __fadd_rn(v, hb);
          }
        }
      }
      kv[i] = c < n ? okey(v) : 0u;
    }
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = lane + 32 * i;
      kv[i] = c < n ? okey(__fadd_rn(lp[c], __fmul_rn(alpha, __ldg(lrow + c)))) : 0u;
    }
  }
  unsigned theta = 0;
  int take = 0;
  if (S < n) {
    for (int bit = 31; bit >= 0; --bit) {         // the largest theta with at least S keys >= theta: the S-th key
      const unsigned t = theta | (1u << bit);
      int cnt = 0;
#pragma unroll
      for (int i = 0; i < 4; ++i) cnt += kv[i] >= t;
      if (__reduce_add_sync(0xffffffffu, cnt) >= S) theta = t;
    }
    int gt = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) gt += kv[i] > theta;
    take = S - __reduce_add_sync(0xffffffffu, gt);
  }
  int at = 0, eq_before = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = lane + 32 * i;
    const bool eq = S < n && kv[i] == theta && c < n;
    const unsigned eqm = __ballot_sync(0xffffffffu, eq);
    const bool in = c < n && (S == n || kv[i] > theta || (eq && eq_before + __popc(eqm & lt) < take));
    const unsigned m = __ballot_sync(0xffffffffu, in);
    if (in) out[at + __popc(m & lt)] = static_cast<short>(c);
    if constexpr (kHot) {
      if (in) kid[at + __popc(m & lt)] = static_cast<unsigned char>((live >> i) & 1u);
    }
    at += __popc(m);
    eq_before += __popc(eqm);
  }
}

struct LmOrder {                                  // candidate label sequences with per-beam shortlists
  const Smem& s;
  const short* shl;
  int cur, S, S1;
  __device__ int at(int i, int t) const {
    const int a = i / S1, x = i - a * S1;
    return t < s.len[cur][a] ? s.pre[cur][a * kT + t] : shl[a * S + x - 1];
  }
  __device__ int clen(int i) const { const int a = i / S1; return s.len[cur][a] + (i - a * S1 > 0); }
  __device__ bool lex_less(int i, int j) const {
    const int li = clen(i), lj = clen(j), n = li < lj ? li : lj;
    for (int t = 0; t < n; ++t) {
      const int u = at(i, t), v = at(j, t);
      if (u != v) return u < v;
    }
    return li < lj;
  }
};

template <bool kHot>
__global__ void __launch_bounds__(kThreads)
ctc_beam_lm_kernel(const float* __restrict__ logits /*[B][48][K]*/, int K, int W, int P,
                   const unsigned long long* __restrict__ lm_keys /*[H]*/, const float* __restrict__ lm_rows /*[H][K]*/,
                   int H, int order, float alpha, float beta, int* __restrict__ labels /*[B][P][48]*/,
                   float* __restrict__ logp /*[B][P] or null*/, float* __restrict__ fused /*[B][P] or null*/,
                   Trie tr /*kHot only*/) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Smem s;
  SmemLm l;
  SmemHot hw;
  if constexpr (kHot) smem_plan_hot(W, K, smem_raw, &s, &l, &hw);
  else smem_plan_lm(W, K, smem_raw, &s, &l);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int blank = K - 1, S = shortlist_size(W, K), S1 = S + 1;
  int cur = 0, nb = 1;
  if (tid == 0) {
    s.len[0][0] = 0; s.pb[0][0] = 0.f; s.pnb[0][0] = -INFINITY; s.sc[0][0] = 0.f;
    s.h[0][0] = kHashRoot; s.ph[0][0] = 0;
    l.g[0][0] = 0.f; l.f[0][0] = 0.f;
    l.row[0][0] = lm_row(lm_keys, H, order, s.pre[0], 0);
    if constexpr (kHot) hw.node[0][0] = 0;         // the trie's root: the empty prefix is live
  }
  for (int t = 0; t < kT; ++t) {
    // ---- 1. lp of step t (as ctc_beam_kernel)
    const float* row = logits + (static_cast<size_t>(blockIdx.x) * kT + t) * K;
    float m = -INFINITY;
    for (int c = tid; c < K; c += kThreads) { const float v = row[c]; s.lp[c] = v; m = fmaxf(m, v); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float* redf = reinterpret_cast<float*>(s.red);
    if (lane == 0) redf[warp] = m;
    __syncthreads();
    m = redf[0];
    for (int w = 1; w < kWarps; ++w) m = fmaxf(m, redf[w]);
    float se = 0.f;
    for (int c = tid; c < K; c += kThreads) se = __fadd_rn(se, expf(__fsub_rn(s.lp[c], m)));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) se = __fadd_rn(se, __shfl_xor_sync(0xffffffffu, se, o));
    __syncthreads();
    if (lane == 0) redf[warp] = se;
    __syncthreads();
    se = redf[0];
    for (int w = 1; w < kWarps; ++w) se = __fadd_rn(se, redf[w]);
    for (int c = tid; c < K; c += kThreads)
      s.lp[c] = logf(__fadd_rn(__fdiv_rn(expf(__fsub_rn(s.lp[c], m)), se), 1e-7f));
    __syncthreads();

    // ---- 2'. per-beam shortlists, one warp per beam
    for (int a = warp; a < nb; a += kWarps) {
      if constexpr (kHot)
        lm_shortlist<true>(s.lp, lm_rows + static_cast<size_t>(l.row[cur][a]) * K, alpha, K - 1, S, l.shl + a * S, tr,
                           hw.node[cur][a], __fmul_rn(tr.gamma, static_cast<float>(s.len[cur][a] + 1)), hw.kid + a * S);
      else
        lm_shortlist<false>(s.lp, lm_rows + static_cast<size_t>(l.row[cur][a]) * K, alpha, K - 1, S, l.shl + a * S,
                            tr, -1, 0.f, nullptr);
    }

    // ---- 3. parent links and the extensions that are already beams
    const Beams bm{s, cur, S1};
    const LmOrder ord{s, l.shl, cur, S, S1};
    for (int i = tid; i < nb * S; i += kThreads) s.excl[i] = 0;
    if (tid < nb) {
      int par = -1;
      const int len = s.len[cur][tid];
      if (len > 0)
        for (int a = 0; a < nb && par < 0; ++a) {
          if (s.len[cur][a] != len - 1 || s.h[cur][a] != s.ph[cur][tid]) continue;
          bool same = true;
          for (int u = 0; u < len - 1 && same; ++u) same = s.pre[cur][a * kT + u] == s.pre[cur][tid * kT + u];
          if (same) par = a;
        }
      s.parent[tid] = par;
    }
    __syncthreads();
    if (tid < nb && s.parent[tid] >= 0) {          // last(tid) in its parent's shortlist (ascending): binary search
      const short* sl = l.shl + s.parent[tid] * S;
      const int c = bm.last(tid);
      int lo = 0, hi = S;
      while (lo < hi) { const int mid = (lo + hi) >> 1; if (sl[mid] < c) lo = mid + 1; else hi = mid; }
      if (lo < S && sl[lo] == c) s.excl[s.parent[tid] * S + lo] = 1;
    }
    __syncthreads();

    // ---- 4. candidate keys: F = A + G (kHot: F = (A + G) + H)
    auto candidate = [&](int i, float* pb, float* pnb, float* g) {
      const int a = i / S1, x = i - a * S1;
      if (x == 0) {
        bm.eval(i, blank, pb, pnb);
        *g = l.g[cur][a];
      } else {
        const int c = l.shl[a * S + x - 1];
        *pb = -INFINITY;
        *pnb = bm.ext(a, c);
        const float lv = __ldg(lm_rows + static_cast<size_t>(l.row[cur][a]) * K + c);
        *g = __fadd_rn(l.g[cur][a], __fadd_rn(__fmul_rn(alpha, lv), beta));
      }
    };
    const int n = nb * S1;
    int valid = 0;
    for (int i = tid; i < n; i += kThreads) {
      const int a = i / S1, x = i - a * S1;
      unsigned k = 0;
      if (x == 0 || !s.excl[a * S + x - 1]) {
        float pb, pnb, g;
        candidate(i, &pb, &pnb, &g);
        if constexpr (kHot) {
          float f = __fadd_rn(lae(pb, pnb), g);
          const int len = s.len[cur][a];
          const bool live = x == 0 ? hw.node[cur][a] >= 0 : hw.kid[a * S + x - 1] != 0;
          const float h = live ? __fmul_rn(tr.gamma, static_cast<float>(len + (x > 0))) : 0.f;
          if (h != 0.f) f = __fadd_rn(f, h);
          k = okey(f);
        } else {
          k = okey(__fadd_rn(lae(pb, pnb), g));
        }
        ++valid;
      }
      s.key[i] = k;
      s.sel[i] = 0;
    }
    int nvalid;
    block_scan(valid, s.red, &nvalid);

    // ---- 5. the W best (as ctc_beam_kernel, the tie order over per-beam shortlists)
    if (nvalid <= W) {
      for (int i = tid; i < n; i += kThreads) s.sel[i] = s.key[i] != 0;
    } else {
      int take, equal;
      const unsigned theta = radix_select(n, W, [&](int i) { return s.key[i]; }, s.hist, s.red, &take, &equal);
      for (int i = tid; i < n; i += kThreads) s.sel[i] = s.key[i] > theta || (take == equal && s.key[i] == theta);
      __syncthreads();
      for (int r = 0; r < take && take < equal; ++r) {
        int best = -1;
        for (int i = tid; i < n; i += kThreads)
          if (s.key[i] == theta && !s.sel[i] && (best < 0 || ord.lex_less(i, best))) best = i;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const int other = __shfl_xor_sync(0xffffffffu, best, o);
          if (other >= 0 && (best < 0 || ord.lex_less(other, best))) best = other;
        }
        if (lane == 0) s.red[warp] = best;
        __syncthreads();
        if (tid == 0) {
          int b = -1;
          for (int w = 0; w < kWarps; ++w) {
            const int o = s.red[w];
            if (o >= 0 && (b < 0 || ord.lex_less(o, b))) b = o;
          }
          s.sel[b] = 1;
        }
        __syncthreads();
      }
    }
    __syncthreads();

    // ---- 6. compaction in candidate order into the other buffer; 6'. new histories look up their row
    {
      const int chunk = (n + kThreads - 1) / kThreads, i0 = min(n, tid * chunk), i1 = min(n, i0 + chunk);
      int cnt = 0;
      for (int i = i0; i < i1; ++i) cnt += s.sel[i];
      int total;
      int slot = block_scan(cnt, s.red, &total);
      const int nx = cur ^ 1;
      for (int i = i0; i < i1; ++i) {
        if (!s.sel[i]) continue;
        const int a = i / S1, x = i - a * S1, len = s.len[cur][a];
        float pb, pnb, g;
        candidate(i, &pb, &pnb, &g);
        for (int u = 0; u < len; ++u) s.pre[nx][slot * kT + u] = s.pre[cur][a * kT + u];
        if (x > 0) {
          const int c = l.shl[a * S + x - 1];
          s.pre[nx][slot * kT + len] = static_cast<short>(c);
          s.h[nx][slot] = s.h[cur][a] * kHashMul + static_cast<unsigned long long>(c + 1);
          s.ph[nx][slot] = s.h[cur][a];
        } else {
          s.h[nx][slot] = s.h[cur][a];
          s.ph[nx][slot] = s.ph[cur][a];
          l.row[nx][slot] = l.row[cur][a];
        }
        l.chg[slot] = x > 0;
        s.len[nx][slot] = len + (x > 0);
        s.pb[nx][slot] = pb;
        s.pnb[nx][slot] = pnb;
        s.sc[nx][slot] = lae(pb, pnb);
        l.g[nx][slot] = g;
        if constexpr (kHot) {
          l.f[nx][slot] = __fadd_rn(lae(pb, pnb), g);   // A + G: F_end adds H_end, not H
          // the parent's node for now; an extension that stays live steps to its child in 6'
          hw.node[nx][slot] = x == 0 || hw.kid[a * S + x - 1] ? hw.node[cur][a] : -1;
        } else {
          l.f[nx][slot] = unokey(s.key[i]);         // the selection key's F, bit for bit
        }
        ++slot;
      }
      nb = total;
      cur = nx;
      __syncthreads();
      if (tid < nb && l.chg[tid]) {
        l.row[cur][tid] = lm_row(lm_keys, H, order, s.pre[cur] + tid * kT, s.len[cur][tid]);
        if constexpr (kHot) {
          const int u = hw.node[cur][tid];
          if (u >= 0) hw.node[cur][tid] = trie_child(tr, u, s.pre[cur][tid * kT + s.len[cur][tid] - 1]);
        }
      }
      __syncthreads();
    }
  }

  // ---- the P best of the final beams by F_end, best first
  const Beams fin{s, cur, 1};
  const int b = blockIdx.x;
  float* fend = l.g[cur ^ 1];                      // free: the other buffer's G
  if (tid < nb) {
    float fe = __fadd_rn(l.f[cur][tid],
                         __fmul_rn(alpha, __ldg(lm_rows + static_cast<size_t>(l.row[cur][tid]) * K + blank)));
    if constexpr (kHot) {                          // + H_end: the bonus stays only on a listed word
      const int u = hw.node[cur][tid];
      const float he = u >= 0 && __ldg(tr.fin + u) ? __fmul_rn(tr.gamma, static_cast<float>(s.len[cur][tid])) : 0.f;
      if (he != 0.f) fe = __fadd_rn(fe, he);
    }
    fend[tid] = fe;
  }
  __syncthreads();
  if (tid < nb) {
    const unsigned k = okey(fend[tid]);
    int rank = 0;
    for (int a = 0; a < nb; ++a) {
      const unsigned ka = okey(fend[a]);
      rank += ka > k || (ka == k && a != tid && fin.lex_less(a, tid));
    }
    if (rank < P) {
      int* o = labels + (static_cast<size_t>(b) * P + rank) * kT;
      const int len = s.len[cur][tid];
      for (int u = 0; u < kT; ++u) o[u] = u < len ? s.pre[cur][tid * kT + u] : -1;
      if (logp) logp[static_cast<size_t>(b) * P + rank] = s.sc[cur][tid];
      if (fused) fused[static_cast<size_t>(b) * P + rank] = fend[tid];
    }
  }
  for (int r = nb + tid; r < P; r += kThreads) {
    int* o = labels + (static_cast<size_t>(b) * P + r) * kT;
    for (int u = 0; u < kT; ++u) o[u] = -1;
    if (logp) logp[static_cast<size_t>(b) * P + r] = -INFINITY;
    if (fused) fused[static_cast<size_t>(b) * P + r] = -INFINITY;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// ctc_beam_pattern_kernel: the same search constrained to the readings a DFA accepts (DESIGN.md section 1, "Patterns").
//   The DFA: states 0 .. n-1, trans[q][c] the successor of q by label c (-1: none), dist[q] the fewest labels from q to
//   an accepting state (0: q accepts).  A beam also carries its state q(a) = delta*(start, a); the empty beam starts in
//   start.  Equal prefixes have equal states, so merging is unchanged.  After step t a candidate in state q is kept only
//   if dist[q] <= 47 - t -- a beam kept via blank or its last label and an extension alike -- so after the last step
//   every survivor accepts.  Ranking, merging, the tie order and the returned scores are those of ctc_beam_kernel.
// Per step, besides steps 1-6 above:
//   2'. the shortlist is per beam: of the labels c with delta(q(a), c) defined and dist[delta(q(a), c)] <= 47 - t (the
//       beam's allowed labels), the min(S, their count) with the largest lp[c] (ties: smaller label), ascending, one
//       warp per beam; slots past the count are not candidates;
//   6'. an extension's state is read from trans; trans and dist are read from global memory (L2-resident).
// Why the per-beam shortlist loses nothing: a label outside the allowed set yields a prefix that either the DFA rejects
// or that cannot reach acceptance in the steps left, so it is never a candidate.  Let c be allowed, outside a's
// shortlist and a+c not a beam.  The shortlist then holds S = W+1 allowed labels c' ranked above c (lp[c'] > lp[c], or
// equal with c' < c); at most one of them is last(a), so at least W of them give a+c' a contribution score(a) + lp[c']
// >= the score of a+c.  Each a+c' is a candidate in the same step: as a's extension, or, if a+c' is already a beam, as
// that beam kept -- whose state is delta(q(a), c') too, so it is feasible, and whose score includes the extension's
// contribution.  So W candidates beat a+c or tie and precede it, and a+c is not among the W best.  The fp32 argument of
// ctc_beam_kernel carries over unchanged.
// A candidate of score -inf (an extension by the last label of a beam whose p_b is -inf) is no candidate here: its
// prefix has probability 0, and left in, it would walk the DFA without the blanks a repeated label needs (a{30} would
// "survive" in 30 steps).  ctc_beam_kernel keeps such candidates while there is room, which only ever fills places no
// finite candidate wants; a -inf beam later becomes finite only through its parent's extension, whose contribution
// lae(-inf, x) = x is bit for bit the score that extension gets here as a new beam.  So with a one-state DFA that
// accepts everything (".*") every label is allowed at every step, the per-beam shortlists equal the global one, and
// the search returns ctc_beam_kernel's readings and scores bit for bit; only slots that ctc_beam_kernel fills with
// -inf readings (fewer finite ones than paths asked for, at tiny K) are -1 with -inf here.
struct SmemPat {
  short* shl;                      // [W][S] per-beam shortlist, ascending labels
  int* cnt;                        // [W] its length
  int* q[2];                       // [W] the beam's DFA state
};

__host__ __device__ inline size_t smem_plan_pattern(int W, int K, unsigned char* base, Smem* s, SmemPat* l) {
  size_t off = smem_plan(W, K, base, s);
  const int S = shortlist_size(W, K);
  SmemPat d;
  SmemPat* p = l ? l : &d;
#define B2O_TAKE(ptr, type, count)                                                    \
  do {                                                                                \
    if (base) (ptr) = reinterpret_cast<type*>(base + off);                            \
    off += (static_cast<size_t>(count) * sizeof(type) + 15) / 16 * 16;                \
  } while (0)
  B2O_TAKE(p->shl, short, W * S);
  B2O_TAKE(p->cnt, int, W);
  for (int i = 0; i < 2; ++i) B2O_TAKE(p->q[i], int, W);
#undef B2O_TAKE
  return off;
}

// One warp: of the labels c < n with trow[c] >= 0 and dist[trow[c]] <= limit, the min(S, their count) with the largest
// lp[c] (ties: smaller label), ascending, into out; returns how many.  Not inlined: inlined, the kernel spills.
__device__ __noinline__ int pattern_shortlist(const float* lp, const short* __restrict__ trow, const unsigned char* __restrict__ dist,
                                 int limit, int n, int S, short* out) {
  const int lane = threadIdx.x & 31;
  const unsigned lt = (1u << lane) - 1u;
  unsigned kv[4];
  int allowed = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = lane + 32 * i;
    bool ok = false;
    if (c < n) {
      const int q = __ldg(trow + c);
      ok = q >= 0 && static_cast<int>(__ldg(dist + q)) <= limit;
    }
    kv[i] = ok ? okey(lp[c]) : 0u;                 // okey of a finite lp is never 0
    allowed += ok;
  }
  const int m = __reduce_add_sync(0xffffffffu, allowed), Sa = S < m ? S : m;
  unsigned theta = 0;
  int take = 0;
  if (Sa < m) {
    for (int bit = 31; bit >= 0; --bit) {         // the largest theta with at least Sa keys >= theta: the Sa-th key
      const unsigned t = theta | (1u << bit);
      int cnt = 0;
#pragma unroll
      for (int i = 0; i < 4; ++i) cnt += kv[i] >= t;
      if (__reduce_add_sync(0xffffffffu, cnt) >= Sa) theta = t;
    }
    int gt = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) gt += kv[i] > theta;
    take = Sa - __reduce_add_sync(0xffffffffu, gt);
  }
  int at = 0, eq_before = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const bool eq = Sa < m && kv[i] == theta;
    const unsigned eqm = __ballot_sync(0xffffffffu, eq);
    const bool in = kv[i] != 0u && (Sa == m || kv[i] > theta || (eq && eq_before + __popc(eqm & lt) < take));
    const unsigned msk = __ballot_sync(0xffffffffu, in);
    if (in) out[at + __popc(msk & lt)] = static_cast<short>(lane + 32 * i);
    at += __popc(msk);
    eq_before += __popc(eqm);
  }
  return Sa;
}

__global__ void __launch_bounds__(kThreads)
ctc_beam_pattern_kernel(const float* __restrict__ logits /*[B][48][K]*/, int K, int W, int P,
                        const short* __restrict__ trans /*[n][K-1]*/, const unsigned char* __restrict__ dist /*[n]*/,
                        int start, int* __restrict__ labels /*[B][P][48]*/, float* __restrict__ logp /*[B][P] or null*/) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Smem s;
  SmemPat l;
  smem_plan_pattern(W, K, smem_raw, &s, &l);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int blank = K - 1, S = shortlist_size(W, K), S1 = S + 1;
  int cur = 0, nb = 1;
  if (tid == 0) {
    s.len[0][0] = 0; s.pb[0][0] = 0.f; s.pnb[0][0] = -INFINITY; s.sc[0][0] = 0.f;
    s.h[0][0] = kHashRoot; s.ph[0][0] = 0;
    l.q[0][0] = start;
  }
  for (int t = 0; t < kT; ++t) {
    const int limit = kT - 1 - t;                  // labels that can still follow after this step
    // ---- 1. lp of step t (as ctc_beam_kernel)
    const float* row = logits + (static_cast<size_t>(blockIdx.x) * kT + t) * K;
    float m = -INFINITY;
    for (int c = tid; c < K; c += kThreads) { const float v = row[c]; s.lp[c] = v; m = fmaxf(m, v); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float* redf = reinterpret_cast<float*>(s.red);
    if (lane == 0) redf[warp] = m;
    __syncthreads();
    m = redf[0];
    for (int w = 1; w < kWarps; ++w) m = fmaxf(m, redf[w]);
    float se = 0.f;
    for (int c = tid; c < K; c += kThreads) se = __fadd_rn(se, expf(__fsub_rn(s.lp[c], m)));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) se = __fadd_rn(se, __shfl_xor_sync(0xffffffffu, se, o));
    __syncthreads();
    if (lane == 0) redf[warp] = se;
    __syncthreads();
    se = redf[0];
    for (int w = 1; w < kWarps; ++w) se = __fadd_rn(se, redf[w]);
    for (int c = tid; c < K; c += kThreads)
      s.lp[c] = logf(__fadd_rn(__fdiv_rn(expf(__fsub_rn(s.lp[c], m)), se), 1e-7f));
    __syncthreads();

    // ---- 2'. per-beam shortlists over the allowed labels, one warp per beam
    for (int a = warp; a < nb; a += kWarps) {
      const int c = pattern_shortlist(s.lp, trans + static_cast<size_t>(l.q[cur][a]) * (K - 1), dist, limit, K - 1, S,
                                      l.shl + a * S);
      if (lane == 0) l.cnt[a] = c;
    }

    // ---- 3. parent links and the extensions that are already beams
    const Beams bm{s, cur, S1};
    const LmOrder ord{s, l.shl, cur, S, S1};
    for (int i = tid; i < nb * S; i += kThreads) s.excl[i] = 0;
    if (tid < nb) {
      int par = -1;
      const int len = s.len[cur][tid];
      if (len > 0)
        for (int a = 0; a < nb && par < 0; ++a) {
          if (s.len[cur][a] != len - 1 || s.h[cur][a] != s.ph[cur][tid]) continue;
          bool same = true;
          for (int u = 0; u < len - 1 && same; ++u) same = s.pre[cur][a * kT + u] == s.pre[cur][tid * kT + u];
          if (same) par = a;
        }
      s.parent[tid] = par;
    }
    __syncthreads();
    if (tid < nb && s.parent[tid] >= 0) {          // last(tid) in its parent's shortlist (ascending): binary search
      const int pa = s.parent[tid], n_sl = l.cnt[pa];
      const short* sl = l.shl + pa * S;
      const int c = bm.last(tid);
      int lo = 0, hi = n_sl;
      while (lo < hi) { const int mid = (lo + hi) >> 1; if (sl[mid] < c) lo = mid + 1; else hi = mid; }
      if (lo < n_sl && sl[lo] == c) s.excl[pa * S + lo] = 1;
    }
    __syncthreads();

    // ---- 4. candidate keys: a beam kept only while it can still reach acceptance, extensions by its shortlist
    const int n = nb * S1;
    int valid = 0;
    for (int i = tid; i < n; i += kThreads) {
      const int a = i / S1, x = i - a * S1;
      const bool cand = x == 0 ? static_cast<int>(__ldg(dist + l.q[cur][a])) <= limit
                               : x - 1 < l.cnt[a] && !s.excl[a * S + x - 1];
      unsigned k = 0;
      if (cand) {
        float pb, pnb;
        if (x == 0) {
          bm.eval(i, blank, &pb, &pnb);
        } else {
          pb = -INFINITY;
          pnb = bm.ext(a, l.shl[a * S + x - 1]);
        }
        const float a_i = lae(pb, pnb);
        if (a_i > -INFINITY) {                     // a zero-probability prefix (a repeat without a blank) is none
          k = okey(a_i);
          ++valid;
        }
      }
      s.key[i] = k;
      s.sel[i] = 0;
    }
    int nvalid;
    block_scan(valid, s.red, &nvalid);

    // ---- 5. the W best (as ctc_beam_kernel, the tie order over per-beam shortlists)
    if (nvalid <= W) {
      for (int i = tid; i < n; i += kThreads) s.sel[i] = s.key[i] != 0;
    } else {
      int take, equal;
      const unsigned theta = radix_select(n, W, [&](int i) { return s.key[i]; }, s.hist, s.red, &take, &equal);
      for (int i = tid; i < n; i += kThreads) s.sel[i] = s.key[i] > theta || (take == equal && s.key[i] == theta);
      __syncthreads();
      for (int r = 0; r < take && take < equal; ++r) {
        int best = -1;
        for (int i = tid; i < n; i += kThreads)
          if (s.key[i] == theta && !s.sel[i] && (best < 0 || ord.lex_less(i, best))) best = i;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const int other = __shfl_xor_sync(0xffffffffu, best, o);
          if (other >= 0 && (best < 0 || ord.lex_less(other, best))) best = other;
        }
        if (lane == 0) s.red[warp] = best;
        __syncthreads();
        if (tid == 0) {
          int b = -1;
          for (int w = 0; w < kWarps; ++w) {
            const int o = s.red[w];
            if (o >= 0 && (b < 0 || ord.lex_less(o, b))) b = o;
          }
          s.sel[b] = 1;
        }
        __syncthreads();
      }
    }
    __syncthreads();

    // ---- 6. compaction in candidate order into the other buffer; 6'. an extension steps its DFA state
    {
      const int chunk = (n + kThreads - 1) / kThreads, i0 = min(n, tid * chunk), i1 = min(n, i0 + chunk);
      int cnt = 0;
      for (int i = i0; i < i1; ++i) cnt += s.sel[i];
      int total;
      int slot = block_scan(cnt, s.red, &total);
      const int nx = cur ^ 1;
      for (int i = i0; i < i1; ++i) {
        if (!s.sel[i]) continue;
        const int a = i / S1, x = i - a * S1, len = s.len[cur][a];
        float pb, pnb;
        if (x == 0) {
          bm.eval(i, blank, &pb, &pnb);
        } else {
          pb = -INFINITY;
          pnb = bm.ext(a, l.shl[a * S + x - 1]);
        }
        for (int u = 0; u < len; ++u) s.pre[nx][slot * kT + u] = s.pre[cur][a * kT + u];
        if (x > 0) {
          const int c = l.shl[a * S + x - 1];
          s.pre[nx][slot * kT + len] = static_cast<short>(c);
          s.h[nx][slot] = s.h[cur][a] * kHashMul + static_cast<unsigned long long>(c + 1);
          s.ph[nx][slot] = s.h[cur][a];
          l.q[nx][slot] = __ldg(trans + static_cast<size_t>(l.q[cur][a]) * (K - 1) + c);
        } else {
          s.h[nx][slot] = s.h[cur][a];
          s.ph[nx][slot] = s.ph[cur][a];
          l.q[nx][slot] = l.q[cur][a];
        }
        s.len[nx][slot] = len + (x > 0);
        s.pb[nx][slot] = pb;
        s.pnb[nx][slot] = pnb;
        s.sc[nx][slot] = unokey(s.key[i]);        // the selection key's score, bit for bit
        ++slot;
      }
      nb = total;
      cur = nx;
      __syncthreads();
    }
  }

  // ---- the P best of the final beams (every one accepts), best first; -1 labels and -inf past the survivors
  const Beams fin{s, cur, 1};
  const int b = blockIdx.x;
  if (tid < nb) {
    const unsigned k = okey(s.sc[cur][tid]);
    int rank = 0;
    for (int a = 0; a < nb; ++a) {
      const unsigned ka = okey(s.sc[cur][a]);
      rank += ka > k || (ka == k && a != tid && fin.lex_less(a, tid));
    }
    if (rank < P) {
      int* o = labels + (static_cast<size_t>(b) * P + rank) * kT;
      const int len = s.len[cur][tid];
      for (int u = 0; u < kT; ++u) o[u] = u < len ? s.pre[cur][tid * kT + u] : -1;
      if (logp) logp[static_cast<size_t>(b) * P + rank] = s.sc[cur][tid];
    }
  }
  for (int r = nb + tid; r < P; r += kThreads) {
    int* o = labels + (static_cast<size_t>(b) * P + r) * kT;
    for (int u = 0; u < kT; ++u) o[u] = -1;
    if (logp) logp[static_cast<size_t>(b) * P + r] = -INFINITY;
  }
}

}  // namespace

int ctc_beam_pattern_run(b2o_ctx* ctx, const float* logits, int B, int K, int beam_width, int top_paths,
                         const b2o_pattern* pat, int* labels, float* logp, cudaStream_t st) {
  if (B <= 0) return B2O_OK;
  const size_t bytes = smem_plan_pattern(beam_width, K, nullptr, nullptr, nullptr);
  B2O_CUDA_CHECK(ctx, cudaFuncSetAttribute(ctc_beam_pattern_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           static_cast<int>(bytes)));
  ctc_beam_pattern_kernel<<<B, kThreads, bytes, st>>>(logits, K, beam_width, top_paths,
                                                      reinterpret_cast<const short*>(pat->trans_dev), pat->dist_dev,
                                                      pat->start, labels, logp);
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}

int ctc_beam_lm_run(b2o_ctx* ctx, const float* logits, int B, int K, int beam_width, int top_paths,
                    const b2o_char_lm* lm, int* labels, float* logp, float* fused, cudaStream_t st) {
  if (B <= 0) return B2O_OK;
  const size_t bytes = smem_plan_lm(beam_width, K, nullptr, nullptr, nullptr);
  B2O_CUDA_CHECK(ctx, cudaFuncSetAttribute(ctc_beam_lm_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           static_cast<int>(bytes)));
  ctc_beam_lm_kernel<false><<<B, kThreads, bytes, st>>>(logits, K, beam_width, top_paths,
                                                        reinterpret_cast<const unsigned long long*>(lm->keys_dev),
                                                        lm->rows_dev, lm->n_histories, lm->order, lm->alpha, lm->beta,
                                                        labels, logp, fused, Trie{});
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}

int ctc_beam_hotword_run(b2o_ctx* ctx, const float* logits, int B, int K, int beam_width, int top_paths,
                         const b2o_char_lm* lm, const b2o_hotwords* hw, int* labels, float* logp, float* fused,
                         cudaStream_t st) {
  if (B <= 0) return B2O_OK;
  const size_t bytes = smem_plan_hot(beam_width, K, nullptr, nullptr, nullptr, nullptr);
  B2O_CUDA_CHECK(ctx, cudaFuncSetAttribute(ctc_beam_lm_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           static_cast<int>(bytes)));
  const Trie tr{reinterpret_cast<const unsigned long long*>(hw->keys_dev), hw->child_dev, hw->final_dev, hw->n_edges,
                hw->weight};
  ctc_beam_lm_kernel<true><<<B, kThreads, bytes, st>>>(logits, K, beam_width, top_paths,
                                                       reinterpret_cast<const unsigned long long*>(lm->keys_dev),
                                                       lm->rows_dev, lm->n_histories, lm->order, lm->alpha, lm->beta,
                                                       labels, logp, fused, tr);
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}

int ctc_beam_run(b2o_ctx* ctx, const float* logits, int B, int K, int beam_width, int top_paths, int* labels, float* logp,
                 cudaStream_t st) {
  if (B <= 0) return B2O_OK;
  const size_t bytes = smem_plan(beam_width, K, nullptr, nullptr);
  B2O_CUDA_CHECK(ctx, cudaFuncSetAttribute(ctc_beam_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           static_cast<int>(bytes)));
  ctc_beam_kernel<<<B, kThreads, bytes, st>>>(logits, K, beam_width, top_paths, labels, logp);
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}
