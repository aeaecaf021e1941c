// ctc_char_scores.cu -- how sure the model is of each character of a reading, and what it would read there instead:
// the posterior of every one-character edit at each position, from CTC forward-backward over the 48 kept steps
// (include/b2ocr.h, DESIGN.md section 1, "Character scores").
//
// ctc_char_scores_kernel: one CTA per crop, one warp per reading (min(P, 4) warps).
//   1. The 48 per-step normalisers (max m_t and sum-exp s_t of the logits), one warp per step in a fixed order, exactly
//      as ctc_align.cu forms them; lp[t,c] = logf(expf(l - m_t) / s_t + 1e-7) is then formed where it is needed.
//   2. The reading y_0..y_{n-1} has the states ext = (blank, y_0, blank, ..., y_{n-1}, blank), S = 2n + 1 <= 97; lane L
//      holds states 4L .. 4L+3.  The forward alpha_t(s) and the backward beta_t(s) (both including lp at t) go to the
//      warp's shared tables, log domain, one fp32 logsumexp per transition.
//   3. F(y[k->e]) for every position k and edit e, one lane per (k, e), lanes strided over the positions of a chunk of
//      at most kFCap / K positions:
//        substitution by c:  A(t) = alpha_t(2k) (+) [c != y_{k-1}] alpha_t(2k-1),  B(t) = beta_t(2k+2) (+) [c != y_{k+1}]
//          beta_t(2k+3), with A(-1) = 0 for an empty prefix and B(48) = 0 for an empty suffix (else -inf);
//          g_t = lp[t,c] + (g_{t-1} (+) A(t-1)),  F = (+)_t g_t + B(t+1);
//        deletion: tau the step at which y_{k+1} starts, F = (+)_tau A'(tau-1) + beta_tau(2k+3) with A' as A for
//          c = y_{k+1}; without a suffix F = A'(47), the prefix's end.
//      The F of a chunk go to shared memory; per position the warp forms m = max_e F, s = sum_e exp(F - m) (lane-strided
//      in label order, then a butterfly), the confidence exp(F(y) - m) / s, and the top A edits by A warp arg-max rounds
//      (larger F first, equal F by smaller label).
//   No atomics and fixed reduction orders: a crop's result is a function of its logits and labels alone, whichever warp
//   of whichever launch shape handles it.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kT = 48, kMaxWarps = 4, kPerLane = 4;
constexpr int kStride = 100;                 // states per table row: S <= 97, float4 rows
constexpr int kFCap = 2048;                  // F values per warp: every position for K <= 42, at least two for K <= 1024
constexpr int kWarpFloats = 2 * kT * kStride + kFCap;

__device__ __forceinline__ float step_lp(const float* row, int c, float m, float s) {
  return logf(__fadd_rn(__fdiv_rn(expf(__fsub_rn(row[c], m)), s), 1e-7f));
}

__device__ __forceinline__ float lse2(float a, float b) {
  const float m = fmaxf(a, b);
  if (!(m > -INFINITY)) return -INFINITY;
  return __fadd_rn(m, log1pf(expf(__fsub_rn(fminf(a, b), m))));
}

__device__ __forceinline__ float lse3(float a, float b, float c) {
  const float m = fmaxf(a, fmaxf(b, c));
  if (!(m > -INFINITY)) return -INFINITY;
  return __fadd_rn(m, logf(__fadd_rn(__fadd_rn(expf(__fsub_rn(a, m)), expf(__fsub_rn(b, m))), expf(__fsub_rn(c, m)))));
}

// (value, label) arg-max: larger value, equal values by smaller label; label < 0 is "none yet".
__device__ __forceinline__ bool better(float v, int e, float bv, int be) {
  return be < 0 || (e >= 0 && (v > bv || (v == bv && e < be)));
}

__global__ void __launch_bounds__(32 * kMaxWarps)
ctc_char_scores_kernel(const float* __restrict__ logits /*[B][48][K]*/, int K, const int32_t* __restrict__ labels
                       /*[B][P][48]*/, int P, int A, float* __restrict__ conf /*[B][P][48]*/,
                       int32_t* __restrict__ alt_labels /*[B][P][48][A]*/, float* __restrict__ alt_post /*[B][P][48][A]*/,
                       float* __restrict__ logp /*[B][P] or null*/) {
  extern __shared__ __align__(16) float smem[];
  __shared__ float mx[kT], se[kT];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5, b = blockIdx.x;
  const float* lg = logits + static_cast<size_t>(b) * kT * K;
  for (int t = warp; t < kT; t += nw) {
    const float* row = lg + static_cast<size_t>(t) * K;
    float m = -INFINITY;
    for (int c = lane; c < K; c += 32) m = fmaxf(m, row[c]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float s = 0.f;
    for (int c = lane; c < K; c += 32) s = __fadd_rn(s, expf(__fsub_rn(row[c], m)));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
    if (lane == 0) { mx[t] = m; se[t] = s; }
  }
  __syncthreads();
  float* alpha = smem + static_cast<size_t>(warp) * kWarpFloats;     // [48][kStride]
  float* beta = alpha + kT * kStride;                                // [48][kStride]
  float* fbuf = beta + kT * kStride;                                 // [kFCap]
  const int blank = K - 1;
  const float nan = __int_as_float(0x7fc00000);
  for (int p = warp; p < P; p += nw) {
    const size_t row_id = static_cast<size_t>(b) * P + p;
    const int32_t* lab = labels + row_id * kT;
    float* cf = conf + row_id * kT;
    int32_t* al = alt_labels ? alt_labels + row_id * kT * A : nullptr;
    float* ap = alt_post ? alt_post + row_id * kT * A : nullptr;
    // n = labels before the first negative one; a label outside [0, K-2] makes the reading's outputs the L = -inf ones
    const int v0 = lab[lane], v1 = lane < kT - 32 ? lab[32 + lane] : -1;
    const unsigned neg0 = __ballot_sync(0xffffffffu, v0 < 0), neg1 = __ballot_sync(0xffffffffu, lane < kT - 32 && v1 < 0);
    const int n = neg0 ? __ffs(neg0) - 1 : (neg1 ? 32 + __ffs(neg1) - 1 : kT);
    const bool bad = __any_sync(0xffffffffu, (lane < n && v0 > K - 2) || (32 + lane < n && v1 > K - 2));
    // padding past the reading, and a bad reading's positions
    for (int i = lane; i < kT; i += 32) cf[i] = i < n ? 0.f : nan;
    for (int i = lane; i < kT * A; i += 32) {
      if (al) al[i] = -1;
      if (ap) ap[i] = i / A < n ? 0.f : nan;
    }
    if (bad) {
      if (logp && lane == 0) logp[row_id] = -INFINITY;
      __syncwarp();
      continue;
    }
    const int S = 2 * n + 1;
    const int i0 = 2 * lane;
    const int cm = (i0 >= 1 && i0 - 1 < n) ? lab[i0 - 1] : -1;
    const int ca = i0 < n ? lab[i0] : blank, cb = i0 + 1 < n ? lab[i0 + 1] : blank;
    const bool skip1 = i0 >= 1 && i0 < n && ca != cm;               // state 4L+1 may come from 4L-1
    const bool skip3 = i0 + 1 < n && cb != ca;                      // state 4L+3 may come from 4L+1
    // forward
    float d[kPerLane];
    {
      d[0] = lane == 0 ? step_lp(lg, blank, mx[0], se[0]) : -INFINITY;
      d[1] = (lane == 0 && n >= 1) ? step_lp(lg, ca, mx[0], se[0]) : -INFINITY;
      d[2] = d[3] = -INFINITY;
    }
    if (lane < kStride / 4) *reinterpret_cast<float4*>(alpha + 4 * lane) = make_float4(d[0], d[1], d[2], d[3]);
    for (int t = 1; t < kT; ++t) {
      const float* row = lg + static_cast<size_t>(t) * K;
      const float m = mx[t], s = se[t];
      const float lpb = step_lp(row, blank, m, s), lpa = step_lp(row, ca, m, s), lpc = step_lp(row, cb, m, s);
      float up3 = __shfl_up_sync(0xffffffffu, d[3], 1), up2 = __shfl_up_sync(0xffffffffu, d[2], 1);
      if (lane == 0) up3 = up2 = -INFINITY;
      const float p1[kPerLane] = {up3, d[0], d[1], d[2]};
      const float p2[kPerLane] = {up2, up3, d[0], d[1]};
      const bool sk[kPerLane] = {false, skip1, false, skip3};
      const float e[kPerLane] = {lpb, lpa, lpb, lpc};
      float nd[kPerLane];
#pragma unroll
      for (int j = 0; j < kPerLane; ++j) {
        const float prev = lse3(d[j], p1[j], sk[j] ? p2[j] : -INFINITY);
        nd[j] = 4 * lane + j < S && prev > -INFINITY ? __fadd_rn(prev, e[j]) : -INFINITY;
      }
#pragma unroll
      for (int j = 0; j < kPerLane; ++j) d[j] = nd[j];
      if (lane < kStride / 4)
        *reinterpret_cast<float4*>(alpha + t * kStride + 4 * lane) = make_float4(d[0], d[1], d[2], d[3]);
    }
    // backward: beta_t(s) = lp[t, ext_s] + (beta_{t+1}(s) (+) beta_{t+1}(s+1) (+) [skip] beta_{t+1}(s+2)); the skip
    // into state s+2 is the one the forward allows into it
    const bool skip5 = __shfl_down_sync(0xffffffffu, skip1, 1) && lane < 31;    // state 4L+5 may come from 4L+3
    {
      const float* row = lg + static_cast<size_t>(kT - 1) * K;
      const float m = mx[kT - 1], s = se[kT - 1];
      const float e[kPerLane] = {step_lp(row, blank, m, s), step_lp(row, ca, m, s), step_lp(row, blank, m, s),
                                 step_lp(row, cb, m, s)};
#pragma unroll
      for (int j = 0; j < kPerLane; ++j) d[j] = (4 * lane + j == S - 1 || 4 * lane + j == S - 2) ? e[j] : -INFINITY;
    }
    if (lane < kStride / 4)
      *reinterpret_cast<float4*>(beta + (kT - 1) * kStride + 4 * lane) = make_float4(d[0], d[1], d[2], d[3]);
    for (int t = kT - 2; t >= 0; --t) {
      const float* row = lg + static_cast<size_t>(t) * K;
      const float m = mx[t], s = se[t];
      const float lpb = step_lp(row, blank, m, s), lpa = step_lp(row, ca, m, s), lpc = step_lp(row, cb, m, s);
      float dn0 = __shfl_down_sync(0xffffffffu, d[0], 1), dn1 = __shfl_down_sync(0xffffffffu, d[1], 1);
      if (lane == 31) dn0 = dn1 = -INFINITY;
      const float n1[kPerLane] = {d[1], d[2], d[3], dn0};          // beta_{t+1}(s+1)
      const float n2[kPerLane] = {d[2], d[3], dn0, dn1};           // beta_{t+1}(s+2)
      const bool sk[kPerLane] = {false, skip3, false, skip5};
      const float e[kPerLane] = {lpb, lpa, lpb, lpc};
      float nd[kPerLane];
#pragma unroll
      for (int j = 0; j < kPerLane; ++j) {
        const float next = lse3(d[j], n1[j], sk[j] ? n2[j] : -INFINITY);
        nd[j] = 4 * lane + j < S && next > -INFINITY ? __fadd_rn(next, e[j]) : -INFINITY;
      }
#pragma unroll
      for (int j = 0; j < kPerLane; ++j) d[j] = nd[j];
      if (lane < kStride / 4)
        *reinterpret_cast<float4*>(beta + t * kStride + 4 * lane) = make_float4(d[0], d[1], d[2], d[3]);
    }
    __syncwarp();
    if (logp && lane == 0) {
      const float* last = alpha + (kT - 1) * kStride;
      logp[row_id] = n >= 1 ? lse2(last[S - 1], last[S - 2]) : last[0];
    }
    // the edits, a chunk of positions at a time
    const int chunk = kFCap / K;
    for (int k0 = 0; k0 < n; k0 += chunk) {
      const int k1 = min(n, k0 + chunk), items = (k1 - k0) * K;
      for (int i = lane; i < items; i += 32) {
        const int k = k0 + i / K, e = i - (i / K) * K;
        const int prevc = k >= 1 ? lab[k - 1] : -1, nextc = k + 1 < n ? lab[k + 1] : -1;
        const float* a0 = alpha + 2 * k;                   // alpha_t(2k) at a0[t * kStride]
        float f = -INFINITY;
        if (e < blank) {
          const bool use_am = k >= 1 && e != prevc, use_bp = k + 1 < n && e != nextc;
          float g = -INFINITY;
          for (int t = 0; t < kT; ++t) {
            const float ain = t == 0 ? (k == 0 ? 0.f : -INFINITY)
                                     : (use_am ? lse2(a0[(t - 1) * kStride], a0[(t - 1) * kStride - 1])
                                               : a0[(t - 1) * kStride]);
            const float* row = lg + static_cast<size_t>(t) * K;
            const float prev = lse2(g, ain);
            g = prev > -INFINITY ? __fadd_rn(step_lp(row, e, mx[t], se[t]), prev) : -INFINITY;
            float bout;
            if (t + 1 == kT) {
              bout = k + 1 == n ? 0.f : -INFINITY;
            } else {
              const float* b2 = beta + (t + 1) * kStride + 2 * k + 2;
              bout = use_bp ? lse2(b2[0], b2[1]) : b2[0];
            }
            f = lse2(f, __fadd_rn(g, bout));
          }
        } else if (k + 1 == n) {                           // deletion of the last character: the prefix's end
          const float* a = a0 + (kT - 1) * kStride;
          f = k >= 1 ? lse2(a[0], a[-1]) : a[0];
        } else {                                           // deletion: the suffix's first label starts at step tau
          const bool use_am = k >= 1 && prevc != nextc;
          for (int tau = 0; tau < kT; ++tau) {
            const float ain = tau == 0 ? (k == 0 ? 0.f : -INFINITY)
                                       : (use_am ? lse2(a0[(tau - 1) * kStride], a0[(tau - 1) * kStride - 1])
                                                 : a0[(tau - 1) * kStride]);
            f = lse2(f, __fadd_rn(ain, beta[tau * kStride + 2 * k + 3]));
          }
        }
        fbuf[i] = f;
      }
      __syncwarp();
      for (int k = k0; k < k1; ++k) {
        float* fk = fbuf + (k - k0) * K;
        float m = -INFINITY;
        for (int e = lane; e < K; e += 32) m = fmaxf(m, fk[e]);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        if (!(m > -INFINITY)) continue;                    // L = -inf: confidence 0, labels -1, posteriors 0
        float s = 0.f;
        for (int e = lane; e < K; e += 32) s = __fadd_rn(s, expf(__fsub_rn(fk[e], m)));
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
        if (lane == 0) cf[k] = __fdiv_rn(expf(__fsub_rn(fk[lab[k]], m)), s);
        for (int a = 0; a < A; ++a) {
          float bv = -INFINITY;
          int be = -1;
          for (int e = lane; e < K; e += 32) {
            const float v = fk[e];
            if (v == v && better(v, e, bv, be)) { bv = v; be = e; }
          }
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const int oe = __shfl_xor_sync(0xffffffffu, be, o);
            if (better(ov, oe, bv, be)) { bv = ov; be = oe; }
          }
          __syncwarp();
          if (be < 0) break;                               // fewer than A edits (K < A): the rest stay -1 / 0
          if (lane == 0) {
            if (al) al[k * A + a] = be;
            if (ap) ap[k * A + a] = __fdiv_rn(expf(__fsub_rn(bv, m)), s);
            fk[be] = nan;                                  // taken
          }
          __syncwarp();
        }
      }
      __syncwarp();
    }
  }
}

}  // namespace

int ctc_char_scores_run(b2o_ctx* ctx, const float* logits, int B, int K, const int32_t* labels, int P, int A, float* conf,
                        int32_t* alt_labels, float* alt_post, float* logp, cudaStream_t st) {
  if (B <= 0) return B2O_OK;
  const int warps = P < kMaxWarps ? P : kMaxWarps;
  const int bytes = warps * kWarpFloats * static_cast<int>(sizeof(float));
  B2O_CUDA_CHECK(ctx, cudaFuncSetAttribute(ctc_char_scores_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  ctc_char_scores_kernel<<<B, 32 * warps, bytes, st>>>(logits, K, labels, P, A, conf, alt_labels, alt_post, logp);
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}

bool ctc_char_scores_args(int k, int top_paths, int alternatives) {
  return k >= 2 && k <= B2O_MAX_CLASSES && top_paths >= 1 && top_paths <= B2O_MAX_ALIGN_PATHS && alternatives >= 0 &&
         alternatives <= B2O_MAX_CHAR_ALTERNATIVES;
}

extern "C" int b2o_ctc_char_scores(b2o_ctx* ctx, const float* logits_dev, int b, int k, const int32_t* labels_dev,
                                   int top_paths, int alternatives, float* conf_dev, int32_t* alt_labels_dev,
                                   float* alt_post_dev, float* logp_dev, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  if (!ctc_char_scores_args(k, top_paths, alternatives) || b < 0 ||
      (b > 0 && (!logits_dev || !labels_dev || !conf_dev ||
                 (alternatives > 0 && (!alt_labels_dev || !alt_post_dev))))) {
    ctx->set_error("b2o_ctc_char_scores: bad argument (2 <= k <= 1024, 1 <= top_paths <= 128, 0 <= alternatives <= 8)");
    return B2O_ERR_ARG;
  }
  DeviceGuard guard(ctx->device);
  return ctc_char_scores_run(ctx, logits_dev, b, k, labels_dev, top_paths, alternatives, conf_dev,
                             alternatives > 0 ? alt_labels_dev : nullptr, alternatives > 0 ? alt_post_dev : nullptr,
                             logp_dev, reinterpret_cast<cudaStream_t>(stream));
}
