// ctc_train.cu -- training the recognizer's output layer (fc_12: Dense 256 -> K plus bias) on frozen CRNN features with
// the loss the reference trains with, Keras ctc_batch_cost on the softmax output (recognition.py:334-349):
//   x_{b,t} = the 256 BiLSTM features of kept step t of crop b, after Dropout(rate) (recognition.py:321);
//   l_{b,t} = x_{b,t} W + bias;  q[t,c] = softmax(l_t)_c + 1e-7;  blank = K-1;
//   L_b = -log sum over the alignments of the crop's text of prod_t q[t, path_t]  (48 steps);
//   grad_W = (1/B) sum_{b,t} x_{b,t}^T g_{b,t},  grad_bias = (1/B) sum_{b,t} g_{b,t},  g = dL_b/dl.
//
// Dropout.  Feature c of step t of cached row r is kept iff  mix64(key0 ^ (r * 12288 + t * 256 + c)) >> 40  (24 bits) is
//   >= thr = floor(rate * 2^24), with key0 = mix64(mix64(seed) ^ step) and mix64 the splitmix64 finaliser (z += golden
//   gamma, two xor-shift-multiplies, a final xor-shift).  A kept feature is multiplied by scale = 1 / (1 - rate) (both fp32
//   operations), a dropped one is 0.  rate = 0 takes the no-dropout code: the features as they are.
//
// ctc_loss_kernel: one CTA (8 warps) per crop.
//   Logits: exactly fc_ctc_kernel's arithmetic -- warp w owns steps 6w..6w+5, lane l the classes l, l+32, ...; each logit
//   is the serial fmaf chain from the bias over the 256 features in ascending order -- so with rate 0 they are bit for bit
//   the logits inference decodes.  They stay in shared memory (48 rows of K floats) and, for tests, may be copied out.
//   q: ctc_step_norm + ctc_q of ctc_q.cuh, the same numbers the lexicon and beam decoders use.
//   alpha (forward, including q_t) runs in the linear domain as the lexicon kernel's does: the same updates
//   (a[s] + a[s-1]) [+ a[s-2]], times q, in the same order, states that cannot reach the end zeroed, exact power-of-two
//   rescaling when the largest state leaves [2^32, 2^100).  One warp runs it, lane l owning states l, l+32, l+64, l+96,
//   so L_b is computed on the same fp32 values as the lexicon score of the text, and L_b = log(alpha_47[S-2] +
//   alpha_47[S-1]) - E ln 2, negated and rounded to fp32 once.  Error (the lexicon kernel's argument): every state is
//   within sum_t (3u + delta_t) relative of exact, delta_t the error of q, u = 2^-24; L_b within 1.01 (sum_t (3u +
//   delta_t) + u) + u |L_b| absolute.
//   beta (steps t+1..47, not including q_t) runs backwards first on the same warp: (b[s] q[s] + b[s+1] q[s+1]) [+ b[s+2]
//   q[s+2]], states that the start cannot reach by step t zeroed (exact: they never flow into one that can), the same
//   rescaling (its exponent is not needed); it has the same relative error bound.  Its rows stay in shared memory.
//   Posterior: per step, gamma_t[c] = sum over s with ext_s = c of alpha_t[s] beta_t[s] / Z_t, Z_t = sum_s alpha_t[s]
//   beta_t[s] (= P = exp(-L_b) up to the scale factors, which cancel).  The products and sums are formed in fp64 in
//   ascending s, so gamma carries the alpha and beta errors (2 sum_t (3u + delta_t)) and one rounding.
//   Gradient through softmax + 1e-7: d_c = dL/dq[t,c] = -gamma_t[c] / q[t,c], so
//     g[t,k] = p_k (d_k - sum_c p_c d_c) = p_k (D_t - r_t[k]),  r_t[k] = gamma_t[k] / q[t,k],  D_t = sum_c gamma_t[c] p_c / q[t,c]
//   (r and D in fp64 over the text's distinct classes and blank, rounded to fp32; p = softmax as in ctc_q.cuh).
//   A crop whose text is empty, longer than 48, has a label outside [0, K-2], cannot be aligned in 48 steps (L + adjacent
//   repeats > 48) or has labels beyond index 2^24 gets L_b = +inf; one whose row index is outside [0, n_rows) gets NaN;
//   their g rows are 0 and they add nothing to the gradient.
// grad_partial_kernel: grad_W by split-K -- the B*48 rows in fixed chunks of kChunkRows, each 64 x 64 tile of a chunk a
//   serial fmaf chain over its rows in ascending order; bias_partial_kernel the same for grad_bias; grad_final_kernel
//   adds the chunks in ascending order and divides by B.  No atomics: a step is bit-identical run to run.
// Workspace (ctc_train_workspace_bytes): g (B, 48, K) float32 first, then the grad_W chunk partials (chunks, 256, K) and
//   the grad_bias ones (chunks, K), each 256-byte aligned.
// rmsprop_kernel: Keras RMSprop with momentum 0 (optimizer_v2/rmsprop.py): acc = rho acc + (1 - rho) g^2,
//   param -= lr g / (sqrt(acc) + eps), every operation rounded in fp32 in that order.
#include <math.h>

#include "common.cuh"
#include "ctc_dropout.cuh"
#include "ctc_q.cuh"

using ctcq::kT;
using ctcdrop::Dropout;
using ctcdrop::kept;

namespace {

constexpr int kFeat = 256, kWarps = 8, kThreads = 32 * kWarps, kStepsPerWarp = kT / kWarps;
constexpr int kMaxS = 2 * kT + 1;                  // 97 states
constexpr int kMaxLabelEnd = 1 << 24;
constexpr int kChunkRows = 16 * kT;                // split-K chunk: 16 crops
constexpr int kTile = 64, kSub = 32;               // grad_partial_kernel: 64 x 64 outputs, 32 rows per stage

// Where crop b's 48 x 256 features start: at row index[b] of an (n_rows, 48, 256) cache (fit_top), or, by_batch, at
// entry b of the batch's own rows `stride` halves apart (the recurrent training's l2, whose 48 kept steps lie inside a
// 50-step row).  Either way the dropout mask stays keyed on the dataset row index[b].
struct FeatRows {
  long long stride;
  bool by_batch;
  __device__ __forceinline__ size_t of(int b, int row) const {
    return static_cast<size_t>(by_batch ? b : row) * static_cast<size_t>(stride);
  }
};

// The feature value x' the logits and grad_W use.
__device__ __forceinline__ float feat_value(const __half h, bool keep, const Dropout& d) {
  const float x = __half2float(h);
  if (!d.on) return x;
  return keep ? __fmul_rn(x, d.scale) : 0.f;
}

// Shared memory of ctc_loss_kernel: the logits (48 x K floats), then a region that first holds the features and the
// dropout mask and then the alpha / beta rows, then small per-step arrays.
struct LossSmem {
  static constexpr size_t kFeatBytes = kT * kFeat * 2 + kT * kFeat / 8;                       // 26112
  static constexpr size_t kBeta = 0, kAlpha = kBeta + 18624, kProd = kAlpha + 784, kG = kProd + 784,
                          kTerm = kG + 400, kRecBytes = kTerm + 400;                           // 20992
  static constexpr size_t kUnion = kFeatBytes > kRecBytes ? kFeatBytes : kRecBytes;
  static size_t bytes(int K) { return static_cast<size_t>(kT) * K * 4 + kUnion + 3 * kT * 4 + 1024 + 2 * kT * 4 + 16; }
};

template <bool DROP>
__global__ void __launch_bounds__(kThreads)
ctc_loss_kernel(const __half* __restrict__ features, FeatRows fr, int n_rows, const int* __restrict__ index,
                int K, const float* __restrict__ w /*[256][K]*/, const float* __restrict__ bias,
                const int* __restrict__ offsets, const short* __restrict__ labels, Dropout drop,
                float* __restrict__ loss, float* __restrict__ g /*[B][48][K] or null*/,
                float* __restrict__ logits_out /*[B][48][K] or null*/) {
  extern __shared__ __align__(16) unsigned char smem[];
  float* lg = reinterpret_cast<float*>(smem);                                          // [48][K]
  unsigned char* un = smem + static_cast<size_t>(kT) * K * 4;
  __half* xs = reinterpret_cast<__half*>(un);                                          // [48][256]
  unsigned* mask = reinterpret_cast<unsigned*>(un + kT * kFeat * 2);                   // [48][8]
  float* beta = reinterpret_cast<float*>(un + LossSmem::kBeta);                        // [48][97], later r rows
  float* alpha = reinterpret_cast<float*>(un + LossSmem::kAlpha);                      // [2][97]
  double* prod = reinterpret_cast<double*>(un + LossSmem::kProd);                      // [97]
  double* gsum = reinterpret_cast<double*>(un + LossSmem::kG);                         // [49]
  double* term = reinterpret_cast<double*>(un + LossSmem::kTerm);                      // [49]
  float* mt = reinterpret_cast<float*>(un + LossSmem::kUnion);                         // [48]
  float* set = mt + kT;                                                                // [48]
  float* dt = set + kT;                                                                // [48]
  signed char* slot_of = reinterpret_cast<signed char*>(dt + kT);                      // [1024]
  int* lab = reinterpret_cast<int*>(slot_of + 1024);                                   // [48]
  int* first = lab + kT;                                                               // [48]
  __shared__ int s_len, s_row, s_bad;
  __shared__ unsigned long long s_rep;

  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) {
    const int row = index ? index[b] : b;
    const int o0 = offsets[b], o1 = offsets[b + 1];
    int L = (o0 >= 0 && o1 <= kMaxLabelEnd && o1 - o0 >= 1 && o1 - o0 <= kT) ? o1 - o0 : 0;
    unsigned long long rep = 0;
    for (int i = 0; i < L; ++i) {
      const int c = labels[o0 + i];
      if (c < 0 || c > K - 2) { L = 0; break; }
      lab[i] = c;
      if (i > 0 && c == lab[i - 1]) rep |= 1ull << i;
    }
    if (L > 0 && L + __popcll(rep) > kT) L = 0;
    s_len = L;
    s_rep = rep;
    s_row = row;
    s_bad = (row < 0 || row >= n_rows) ? 2 : (L == 0 ? 1 : 0);
  }
  __syncthreads();
  const int L = s_len, row = s_row, bad = s_bad;
  const unsigned long long rep = s_rep;
  if (bad) {
    if (tid == 0) loss[b] = bad == 2 ? __int_as_float(0x7fc00000) : INFINITY;
    for (int i = tid; i < kT * K; i += kThreads) {
      if (g) g[static_cast<size_t>(b) * kT * K + i] = 0.f;
      if (logits_out) logits_out[static_cast<size_t>(b) * kT * K + i] = __int_as_float(0x7fc00000);   // no logits: NaN
    }
    return;
  }
  // ---- features (and the dropout mask) into shared memory
  {
    const uint4* src = reinterpret_cast<const uint4*>(features + fr.of(b, row));
    uint4* dst = reinterpret_cast<uint4*>(xs);
    for (int i = tid; i < kT * kFeat / 8; i += kThreads) dst[i] = src[i];
    if (DROP) {
      for (int i = tid; i < kT * kFeat; i += kThreads) {           // a warp covers 32 consecutive features of one step
        const unsigned bits = __ballot_sync(0xffffffffu, kept(drop, row, i / kFeat, i % kFeat));
        if (lane == 0) mask[i / 32] = bits;
      }
    }
  }
  __syncthreads();
  // ---- logits: fc_ctc_kernel's chains
  {
    const int t0 = warp * kStepsPerWarp;
    for (int k = lane; k < K; k += 32) {
      float acc[kStepsPerWarp];
      const float bk = bias[k];
#pragma unroll
      for (int j = 0; j < kStepsPerWarp; ++j) acc[j] = bk;
#pragma unroll 4
      for (int c = 0; c < kFeat; ++c) {
        const float wv = __ldg(w + static_cast<size_t>(c) * K + k);
#pragma unroll
        for (int j = 0; j < kStepsPerWarp; ++j) {
          const int t = t0 + j;
          const bool keep = DROP ? ((mask[t * 8 + (c >> 5)] >> (c & 31)) & 1u) != 0 : true;
          acc[j] = fmaf(feat_value(xs[t * kFeat + c], keep, drop), wv, acc[j]);
        }
      }
#pragma unroll
      for (int j = 0; j < kStepsPerWarp; ++j) {
        lg[(t0 + j) * K + k] = acc[j];
        if (logits_out) logits_out[(static_cast<size_t>(b) * kT + t0 + j) * K + k] = acc[j];
      }
    }
  }
  __syncthreads();
  // ---- per-step normalisers; the class -> slot map (the first position of a label in the text, L for blank)
  for (int t = warp; t < kT; t += kWarps) {
    float m, se;
    ctcq::ctc_step_norm(lg + t * K, K, lane, &m, &se);
    if (lane == 0) { mt[t] = m; set[t] = se; }
  }
  for (int c = tid; c < K; c += kThreads) slot_of[c] = c == K - 1 ? static_cast<signed char>(L) : -1;
  if (tid < L) {
    int f = 0;                                                     // the smallest j with lab[j] == lab[tid]
    while (lab[f] != lab[tid]) ++f;
    first[tid] = f;
  }
  __syncthreads();
  if (tid < L && first[tid] == tid) slot_of[lab[tid]] = static_cast<signed char>(tid);
  __syncthreads();
  if (warp != 0) {
    if (!g) return;
  } else {
    const int S = 2 * L + 1, blank = K - 1;
    auto qv = [&](int t, int s) {                                  // q[t, ext_s]
      const int c = (s & 1) ? lab[s >> 1] : blank;
      return ctcq::ctc_q(lg[t * K + c], mt[t], set[t]);
    };
    auto slot = [&](int s) { return (s & 1) ? first[s >> 1] : L; };
    if (g) {
      // beta, backwards; minsteps(s) = the first step at which the start reaches s
      auto minsteps = [&](int s) {
        if (s == 0) return 0;
        const int j = (s - 1) >> 1;                                 // label j of state 2j+1, or the one before blank 2j+2
        return j + __popcll(rep & ((2ull << j) - 1)) + ((s & 1) ? 0 : 1);
      };
      for (int t = kT - 1; t >= 0; --t) {
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int s = lane + 32 * j;
          float x = 0.f;
          if (s < S && minsteps(s) <= t) {
            if (t == kT - 1) {
              x = (s >= S - 2) ? 1.f : 0.f;
            } else {
              const float* nb = beta + (t + 1) * kMaxS;
              x = __fmul_rn(nb[s], qv(t + 1, s));
              if (s + 1 < S) x = __fadd_rn(x, __fmul_rn(nb[s + 1], qv(t + 1, s + 1)));
              if (s + 2 < S && (s & 1) && !((rep >> ((s + 2) >> 1)) & 1ull))
                x = __fadd_rn(x, __fmul_rn(nb[s + 2], qv(t + 1, s + 2)));
            }
          }
          v[j] = x;
        }
        float m = fmaxf(fmaxf(v[0], v[1]), fmaxf(v[2], v[3]));
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        const int sh = ctcq::ctc_rescale_shift(m);
        const float f = __int_as_float((127 + sh) << 23);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int s = lane + 32 * j;
          if (s < kMaxS) beta[t * kMaxS + s] = sh ? __fmul_rn(v[j], f) : v[j];
        }
        __syncwarp();
      }
    }
    // alpha, forwards (the lexicon kernel's entry_key, one state per lane and slot)
    int e_sum = 0, live = 0;
    float a[4];
    for (int t = 0; t < kT; ++t) {
      const float* pa = alpha + ((t + 1) & 1) * kMaxS;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int s = lane + 32 * j;
        float v = 0.f;
        if (s < S) {
          if (t == 0) {
            v = s == 0 ? qv(0, 0) : (s == 1 ? qv(0, 1) : 0.f);
          } else if (s == 0) {
            v = __fmul_rn(pa[0], qv(t, 0));
          } else {
            v = __fadd_rn(pa[s], pa[s - 1]);
            if ((s & 1) && (s >> 1) > 0 && !((rep >> (s >> 1)) & 1ull)) v = __fadd_rn(v, pa[s - 2]);
            v = __fmul_rn(v, qv(t, s));
          }
        }
        a[j] = v;
      }
      while (live < 2 * L - 1 && ctcq::ctc_need_steps(live, L, rep) > kT - 1 - t) ++live;
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (lane + 32 * j < live) a[j] = 0.f;
      float m = fmaxf(fmaxf(a[0], a[1]), fmaxf(a[2], a[3]));
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
      const int sh = ctcq::ctc_rescale_shift(m);
      if (sh) {
        const float f = __int_as_float((127 + sh) << 23);
#pragma unroll
        for (int j = 0; j < 4; ++j) a[j] = __fmul_rn(a[j], f);
        e_sum += sh;
      }
      float* na = alpha + (t & 1) * kMaxS;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int s = lane + 32 * j;
        if (s < kMaxS) na[s] = a[j];
      }
      __syncwarp();
      if (g) {
        // posterior of step t over the text's distinct classes and blank
        const float* bt = beta + t * kMaxS;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int s = lane + 32 * j;
          if (s < S) prod[s] = static_cast<double>(na[s]) * static_cast<double>(bt[s]);
        }
        __syncwarp();
        for (int u = lane; u <= L; u += 32) {
          double acc = 0.0;
          for (int s = 0; s < S; ++s)
            if (slot(s) == u) acc += prod[s];
          gsum[u] = acc;
        }
        __syncwarp();
        double z = 0.0;
        for (int u = 0; u <= L; ++u) z += gsum[u];
        float* rt = beta + t * kMaxS;                               // beta_t is used up: r_t takes its row
        for (int u = lane; u <= L; u += 32) {
          double tm = 0.0;
          float r = 0.f;
          if (u == L || first[u] == u) {
            const int c = u == L ? blank : lab[u];
            const float p = ctcq::ctc_p(lg[t * K + c], mt[t], set[t]);
            const float q = __fadd_rn(p, 1e-7f);
            const double gam = gsum[u] / z;
            tm = gam * (static_cast<double>(p) / static_cast<double>(q));
            r = static_cast<float>(gam / static_cast<double>(q));
          }
          term[u] = tm;
          rt[u] = r;
        }
        __syncwarp();
        if (lane == 0) {
          double d = 0.0;
          for (int u = 0; u <= L; ++u) d += term[u];
          dt[t] = static_cast<float>(d);
        }
        __syncwarp();
      }
    }
    if (lane == 0) {
      const float* fa = alpha + ((kT - 1) & 1) * kMaxS;
      const float x = __fadd_rn(fa[S - 2], fa[S - 1]);
      float v = INFINITY;
      if (x > 0.f) v = __double2float_rn(-(log(static_cast<double>(x)) - static_cast<double>(e_sum) * 0.69314718055994530942));
      loss[b] = v;
    }
    if (!g) return;
  }
  __syncthreads();
  // ---- g[t,k] = p_k (D_t - r_t[k])
  float* gb = g + static_cast<size_t>(b) * kT * K;
  for (int i = tid; i < kT * K; i += kThreads) {
    const int t = i / K, k = i - t * K;
    const float p = ctcq::ctc_p(lg[i], mt[t], set[t]);
    const int sl = slot_of[k];
    const float r = sl >= 0 ? beta[t * kMaxS + sl] : 0.f;
    gb[i] = __fmul_rn(p, __fsub_rn(dt[t], r));
  }
}

// partial[chunk][c][k] = sum over the chunk's rows r (ascending) of x'[r][c] g[r][k], one 64 x 64 tile per CTA.
template <bool DROP>
__global__ void __launch_bounds__(256)
grad_partial_kernel(const __half* __restrict__ features, FeatRows fr, int n_rows, const int* __restrict__ index, int B, int K,
                    const float* __restrict__ g, Dropout drop, float* __restrict__ partial) {
  __shared__ float xs[kSub][kTile], gs[kSub][kTile];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int k0 = blockIdx.x * kTile, c0 = blockIdx.y * kTile, chunk = blockIdx.z;
  const int r_begin = chunk * kChunkRows, r_end = min(B * kT, r_begin + kChunkRows);
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int r0 = r_begin; r0 < r_end; r0 += kSub) {
    for (int e = threadIdx.x; e < kSub * kTile; e += 256) {
      const int rr = e / kTile, cc = e % kTile, r = r0 + rr;
      float xv = 0.f, gv = 0.f;
      if (r < r_end) {
        const int bi = r / kT, t = r - bi * kT;
        const int row = index ? index[bi] : bi;
        if (row >= 0 && row < n_rows) {
          const int c = c0 + cc;
          const bool keep = DROP ? kept(drop, row, t, c) : true;
          xv = feat_value(features[fr.of(bi, row) + static_cast<size_t>(t) * kFeat + c], keep, drop);
        }
        const int k = k0 + cc;
        if (k < K) gv = g[static_cast<size_t>(r) * K + k];
      }
      xs[rr][cc] = xv;
      gs[rr][cc] = gv;
    }
    __syncthreads();
    const int n = min(kSub, r_end - r0);
    for (int rr = 0; rr < n; ++rr) {
      float xv[4], gv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { xv[i] = xs[rr][ty * 4 + i]; gv[i] = gs[rr][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(xv[i], gv[j], acc[i][j]);
    }
    __syncthreads();
  }
  float* out = partial + static_cast<size_t>(chunk) * kFeat * K;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = k0 + tx * 4 + j;
      if (k < K) out[static_cast<size_t>(c0 + ty * 4 + i) * K + k] = acc[i][j];
    }
}

// partial_b[chunk][k] = sum over the chunk's rows (ascending) of g[r][k].
__global__ void bias_partial_kernel(const float* __restrict__ g, int B, int K, float* __restrict__ partial_b) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x, chunk = blockIdx.y;
  if (k >= K) return;
  const int r_begin = chunk * kChunkRows, r_end = min(B * kT, r_begin + kChunkRows);
  float s = 0.f;
  for (int r = r_begin; r < r_end; ++r) s = __fadd_rn(s, g[static_cast<size_t>(r) * K + k]);
  partial_b[static_cast<size_t>(chunk) * K + k] = s;
}

// out[e] = (sum over chunks, ascending, of partial[chunk][e]) / B.
__global__ void grad_final_kernel(const float* __restrict__ partial, int n, int chunks, int B, float* __restrict__ out) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  float s = 0.f;
  for (int ch = 0; ch < chunks; ++ch) s = __fadd_rn(s, partial[static_cast<size_t>(ch) * n + e]);
  out[e] = __fdiv_rn(s, static_cast<float>(B));
}

__global__ void rmsprop_kernel(float* __restrict__ param, const float* __restrict__ grad, float* __restrict__ acc,
                               long long n, float lr, float rho, float eps) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float gv = grad[i];
  const float a = __fadd_rn(__fmul_rn(rho, acc[i]), __fmul_rn(__fsub_rn(1.f, rho), __fmul_rn(gv, gv)));
  acc[i] = a;
  param[i] = __fsub_rn(param[i], __fdiv_rn(__fmul_rn(lr, gv), __fadd_rn(__fsqrt_rn(a), eps)));
}

size_t align256(size_t x) { return (x + 255) / 256 * 256; }
int chunks_of(int B) { return (B * kT + kChunkRows - 1) / kChunkRows; }

}  // namespace

size_t ctc_train_workspace_bytes(int B, int K) {
  const size_t nch = static_cast<size_t>(chunks_of(B));
  return align256(static_cast<size_t>(B) * kT * K * 4) + align256(nch * kFeat * K * 4) + align256(nch * K * 4);
}

size_t ctc_train_smem_bytes(int K) { return LossSmem::bytes(K); }

int ctc_loss_grad_run(b2o_ctx* ctx, const __half* features, long long feat_stride, bool feat_by_batch, int n_rows,
                      const int* index, int B, int K, const float* w, const float* bias, const int* offsets,
                      const short* labels, float rate, uint64_t seed, uint64_t step, float* loss, float* grad_w,
                      float* grad_b, float* logits, void* ws, cudaStream_t st) {
  const Dropout d = ctcdrop::make_dropout(rate, seed, step);
  const FeatRows fr = {feat_stride, feat_by_batch};
  const bool grads = grad_w != nullptr;
  uint8_t* base = reinterpret_cast<uint8_t*>(ws);
  float* g = grads ? reinterpret_cast<float*>(base) : nullptr;
  const size_t smem = LossSmem::bytes(K);
  auto kern = d.on ? ctc_loss_kernel<true> : ctc_loss_kernel<false>;
  B2O_CUDA_CHECK(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  kern<<<B, kThreads, smem, st>>>(features, fr, n_rows, index, K, w, bias, offsets, labels, d, loss, g, logits);
  B2O_LAUNCH_CHECK(ctx);
  if (!grads) return B2O_OK;
  const int nch = chunks_of(B);
  float* partial = reinterpret_cast<float*>(base + align256(static_cast<size_t>(B) * kT * K * 4));
  float* partial_b = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(partial) +
                                              align256(static_cast<size_t>(nch) * kFeat * K * 4));
  const dim3 grid((K + kTile - 1) / kTile, kFeat / kTile, nch);
  if (d.on) grad_partial_kernel<true><<<grid, 256, 0, st>>>(features, fr, n_rows, index, B, K, g, d, partial);
  else grad_partial_kernel<false><<<grid, 256, 0, st>>>(features, fr, n_rows, index, B, K, g, d, partial);
  B2O_LAUNCH_CHECK(ctx);
  bias_partial_kernel<<<dim3((K + 127) / 128, nch), 128, 0, st>>>(g, B, K, partial_b);
  B2O_LAUNCH_CHECK(ctx);
  grad_final_kernel<<<(kFeat * K + 255) / 256, 256, 0, st>>>(partial, kFeat * K, nch, B, grad_w);
  B2O_LAUNCH_CHECK(ctx);
  grad_final_kernel<<<(K + 255) / 256, 256, 0, st>>>(partial_b, K, nch, B, grad_b);
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}

int rmsprop_run(b2o_ctx* ctx, float* param, const float* grad, float* acc, long long n, float lr, float rho, float eps,
                cudaStream_t st) {
  if (n <= 0) return B2O_OK;
  rmsprop_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, st>>>(param, grad, acc, n, lr, rho, eps);
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}
