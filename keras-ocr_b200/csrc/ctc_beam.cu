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

}  // namespace

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
