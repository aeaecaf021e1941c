// ctc_align.cu -- where each character of a reading lies: CTC Viterbi forced alignment of the reading's labels over the
// 48 kept steps, and the character cells that alignment cuts from the word box, mapped back through the STN and warpBox
// into detector-input pixels (include/b2ocr.h, DESIGN.md section 1).
//
// ctc_align_kernel: one CTA per crop, 4 warps.
//   1. The 48 per-step normalisers (max m_t and sum-exp s_t of the logits), one warp per step in a fixed order, as
//      ctc_lexicon.cu's stage_probs; lp[t,c] = logf(expf(l - m_t) / s_t + 1e-7) is then formed where it is needed.
//   2. One warp per reading.  The reading l_0..l_{n-1} has the states ext = (blank, l_0, blank, ..., l_{n-1}, blank),
//      S = 2n + 1 <= 97; lane L holds states 4L .. 4L+3 in registers.  delta_0 = (lp[0,blank], lp[0,l_0], -inf, ...),
//      delta_t[s] = lp[t, ext_s] + max(delta_{t-1}[s], delta_{t-1}[s-1], [skip_s] delta_{t-1}[s-2]), skip_s for a label
//      that differs from the label before it.  Ties go to the earlier candidate of that list: staying beats advancing
//      by one, which beats skipping a blank.  The choice per (t, s) goes to shared memory (48 x 128 bytes per warp).
//      The alignment ends in the last label's state S-2 or the trailing blank S-1, the blank only when strictly better.
//      Lane 0 walks the backpointers from step 47 to 0 and writes each character's first and last step.
//   No atomics and fixed reduction orders: a crop's result is a function of its logits and labels alone.
// char_cells_kernel: one CTA per crop; thread 0 plans the crop's warp (common.cuh's warp_extent / plan_warp, the turn
//   the crop was read in), then one thread per (reading, character) forms the cuts and maps its cell in fp64.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kT = 48, kDiscard = 2, kWarps = 4, kThreads = 32 * kWarps, kPerLane = 4;
constexpr int kCropW = 200, kCropH = 31, kCellThreads = 128;

__device__ __forceinline__ float step_lp(const float* row, int c, float m, float s) {
  return logf(__fadd_rn(__fdiv_rn(expf(__fsub_rn(row[c], m)), s), 1e-7f));
}

__global__ void __launch_bounds__(kThreads)
ctc_align_kernel(const float* __restrict__ logits /*[B][48][K]*/, int K, const int32_t* __restrict__ labels /*[B][P][48]*/,
                 int P, int32_t* __restrict__ spans /*[B][P][48][2]*/, float* __restrict__ logp /*[B][P] or null*/) {
  __shared__ float mx[kT], se[kT];
  __shared__ __align__(4) unsigned char bp[kWarps][kT][32 * kPerLane];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, b = blockIdx.x;
  const float* lg = logits + static_cast<size_t>(b) * kT * K;
  for (int t = warp; t < kT; t += kWarps) {
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
  const int blank = K - 1;
  for (int p = warp; p < P; p += kWarps) {
    const size_t row_id = static_cast<size_t>(b) * P + p;
    const int32_t* lab = labels + row_id * kT;
    int32_t* sp = spans + row_id * kT * 2;
    // n = labels before the first negative one; a label outside [0, K-2] makes the reading unalignable
    const int v0 = lab[lane], v1 = lane < kT - 32 ? lab[32 + lane] : -1;
    const unsigned neg0 = __ballot_sync(0xffffffffu, v0 < 0), neg1 = __ballot_sync(0xffffffffu, lane < kT - 32 && v1 < 0);
    const int n = neg0 ? __ffs(neg0) - 1 : (neg1 ? 32 + __ffs(neg1) - 1 : kT);
    const bool bad = __any_sync(0xffffffffu, (lane < n && v0 > K - 2) || (32 + lane < n && v1 > K - 2));
    const int S = 2 * n + 1;
    // this lane's labels l_{2L-1}, l_{2L}, l_{2L+1} (states 4L-1 .. 4L+3); past the reading: the blank, never read
    const int i0 = 2 * lane;
    const int cm = (!bad && i0 >= 1 && i0 - 1 < n) ? lab[i0 - 1] : -1;
    const int ca = (!bad && i0 < n) ? lab[i0] : blank, cb = (!bad && i0 + 1 < n) ? lab[i0 + 1] : blank;
    const bool skip1 = i0 >= 1 && i0 < n && ca != cm;               // state 4L+1 may come from 4L-1
    const bool skip3 = i0 + 1 < n && cb != ca;                      // state 4L+3 may come from 4L+1
    for (int i = lane; i < 2 * kT; i += 32) sp[i] = -1;
    float d[kPerLane];
    {
      const float* row = lg;
      d[0] = lane == 0 ? step_lp(row, blank, mx[0], se[0]) : -INFINITY;
      d[1] = (lane == 0 && n >= 1 && !bad) ? step_lp(row, ca, mx[0], se[0]) : -INFINITY;
      d[2] = d[3] = -INFINITY;
    }
    if (bad) d[0] = -INFINITY;
    for (int t = 1; t < kT; ++t) {
      const float* row = lg + static_cast<size_t>(t) * K;
      const float m = mx[t], s = se[t];
      const float lpb = step_lp(row, blank, m, s);
      const float lpa = step_lp(row, ca, m, s), lpc = step_lp(row, cb, m, s);
      float up3 = __shfl_up_sync(0xffffffffu, d[3], 1), up2 = __shfl_up_sync(0xffffffffu, d[2], 1);
      if (lane == 0) up3 = up2 = -INFINITY;
      const float p1[kPerLane] = {up3, d[0], d[1], d[2]};        // delta_{t-1}[s-1]
      const float p2[kPerLane] = {up2, up3, d[0], d[1]};         // delta_{t-1}[s-2]
      const bool sk[kPerLane] = {false, skip1, false, skip3};
      const float e[kPerLane] = {lpb, lpa, lpb, lpc};
      unsigned packed = 0;
      float nd[kPerLane];
#pragma unroll
      for (int j = 0; j < kPerLane; ++j) {
        float best = d[j];
        unsigned ch = 0;
        if (p1[j] > best) { best = p1[j]; ch = 1; }
        if (sk[j] && p2[j] > best) { best = p2[j]; ch = 2; }
        nd[j] = 4 * lane + j < S ? __fadd_rn(best, e[j]) : -INFINITY;
        packed |= ch << (8 * j);
      }
#pragma unroll
      for (int j = 0; j < kPerLane; ++j) d[j] = nd[j];
      *reinterpret_cast<unsigned*>(&bp[warp][t][4 * lane]) = packed;
    }
    // the end: S-2 (the last label) unless the trailing blank S-1 is strictly better; an empty reading ends on blank
    float last = -INFINITY, tail = -INFINITY;
#pragma unroll
    for (int j = 0; j < kPerLane; ++j) {
      if (4 * lane + j == S - 2) last = d[j];
      if (4 * lane + j == S - 1) tail = d[j];
    }
    last = n >= 1 ? __shfl_sync(0xffffffffu, last, (S - 2) >> 2) : -INFINITY;
    tail = __shfl_sync(0xffffffffu, tail, (S - 1) >> 2);
    const int s_end = tail > last ? S - 1 : S - 2;
    const float score = tail > last ? tail : last;
    __syncwarp();
    if (lane == 0) {
      if (logp) logp[row_id] = score > -INFINITY ? score : -INFINITY;   // NaN logits: -inf
      if (score > -INFINITY && n >= 1) {
        int s = s_end, prev = -1;
        for (int t = kT - 1; t >= 0; --t) {
          if (s & 1) {
            const int k = s >> 1;
            if (s != prev) sp[2 * k + 1] = t;
            sp[2 * k] = t;
          }
          prev = s;
          if (t > 0) s -= bp[warp][t][s];
        }
      }
    }
    __syncwarp();
  }
}

// Crop x of the cut before character j (1 <= j < n): grid row r = (l_{j-1} + f_j) / 2 + 2 (common.cuh's stn_crop_x).
__device__ __forceinline__ double cut_x(const int32_t* sp, int j, const float* th) {
  const double r = 0.5 * static_cast<double>(sp[2 * (j - 1) + 1] + sp[2 * j]) + kDiscard;
  return stn_crop_x(r, th);
}

__global__ void __launch_bounds__(kCellThreads)
char_cells_kernel(const int32_t* __restrict__ spans /*[B][P][48][2]*/, int P, const float* __restrict__ theta /*[B][6]*/,
                  const float* __restrict__ boxes /*[B][4][2]*/, const int32_t* __restrict__ turns /*[B]*/,
                  float* __restrict__ cells /*[B][P][48][4][2]*/) {
  __shared__ b2o_warp_plan plan;
  __shared__ float box[8];
  __shared__ double ext[2];
  const int b = blockIdx.x;
  if (threadIdx.x == 0) {
    if (boxes) {
      const int turn = turns ? (turns[b] & 3) : 0;
      double sw = 0.0, sh = 0.0;
      const bool ok = warp_extent(boxes + static_cast<size_t>(b) * 8, turn, kCropW, kCropH, box, &sw, &sh);
      plan_warp(boxes + static_cast<size_t>(b) * 8, turn, kCropW, kCropH, &plan);
      if (!ok) plan.valid = 0;
      ext[0] = static_cast<float>(sw);            // the destination corners the homography maps the box onto
      ext[1] = static_cast<float>(sh);
    } else {                                      // the crop frame itself
      const float frame[8] = {0.f, 0.f, static_cast<float>(kCropW), 0.f, static_cast<float>(kCropW),
                              static_cast<float>(kCropH), 0.f, static_cast<float>(kCropH)};
      for (int i = 0; i < 8; ++i) box[i] = frame[i];
      plan.valid = 1;
      ext[0] = kCropW;
      ext[1] = kCropH;
    }
  }
  __syncthreads();
  const float* th = theta ? theta + static_cast<size_t>(b) * 6 : nullptr;
  const double sw = ext[0], sh = ext[1];
  for (int i = threadIdx.x; i < P * kT; i += kCellThreads) {
    const int p = i / kT, k = i - p * kT;
    const int32_t* sp = spans + (static_cast<size_t>(b) * P + p) * kT * 2;
    float* o = cells + ((static_cast<size_t>(b) * P + p) * kT + k) * 8;
    if (!plan.valid || sp[2 * k] < 0) {
#pragma unroll
      for (int c = 0; c < 8; ++c) o[c] = __int_as_float(0x7fc00000);
      continue;
    }
    const bool last = k == kT - 1 || sp[2 * k + 2] < 0;
    // cuts 1..k+1 clamped to [0, sw] with a running max (non-decreasing even where theta flips time)
    double run = 0.0, a = 0.0, c1 = sw;
    for (int j = 1; j <= k + (last ? 0 : 1); ++j) {
      run = fmax(run, fmin(fmax(cut_x(sp, j, th), 0.0), sw));
      if (j == k) a = run;
      if (j == k + 1) c1 = run;
    }
    const double xs[4] = {a, c1, c1, a}, ys[4] = {0.0, 0.0, sh, sh};
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      if ((k == 0 && (c == 0 || c == 3)) || (last && (c == 1 || c == 2))) {    // outer edges: the box's own corners
        o[2 * c] = box[2 * c];
        o[2 * c + 1] = box[2 * c + 1];
      } else if (!boxes) {
        o[2 * c] = static_cast<float>(xs[c]);
        o[2 * c + 1] = static_cast<float>(ys[c]);
      } else {
        const double* m = plan.m;
        const double X = __dadd_rn(__dadd_rn(__dmul_rn(m[0], xs[c]), __dmul_rn(m[1], ys[c])), m[2]);
        const double Y = __dadd_rn(__dadd_rn(__dmul_rn(m[3], xs[c]), __dmul_rn(m[4], ys[c])), m[5]);
        const double W = __dadd_rn(__dadd_rn(__dmul_rn(m[6], xs[c]), __dmul_rn(m[7], ys[c])), m[8]);
        o[2 * c] = static_cast<float>(__ddiv_rn(X, W));
        o[2 * c + 1] = static_cast<float>(__ddiv_rn(Y, W));
      }
    }
  }
}

}  // namespace

int ctc_align_run(b2o_ctx* ctx, const float* logits, int B, int K, const int32_t* labels, int P, int32_t* spans,
                  float* logp, cudaStream_t st) {
  if (B <= 0) return B2O_OK;
  ctc_align_kernel<<<B, kThreads, 0, st>>>(logits, K, labels, P, spans, logp);
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}

extern "C" int b2o_ctc_align(b2o_ctx* ctx, const float* logits_dev, int b, int k, const int32_t* labels_dev,
                             int top_paths, int32_t* spans_dev, float* logp_dev, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  if (k < 2 || k > B2O_MAX_CLASSES || top_paths < 1 || top_paths > B2O_MAX_ALIGN_PATHS || b < 0 ||
      (b > 0 && (!logits_dev || !labels_dev || !spans_dev))) {
    ctx->set_error("b2o_ctc_align: bad argument (2 <= k <= 1024, 1 <= top_paths <= 128)");
    return B2O_ERR_ARG;
  }
  DeviceGuard guard(ctx->device);
  return ctc_align_run(ctx, logits_dev, b, k, labels_dev, top_paths, spans_dev, logp_dev,
                       reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int b2o_char_cells(b2o_ctx* ctx, const int32_t* spans_dev, int b, int top_paths, const float* theta_dev,
                              const float* boxes_dev, const int32_t* turns_dev, float* cells_dev, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  if (top_paths < 1 || top_paths > B2O_MAX_ALIGN_PATHS || b < 0 || (b > 0 && (!spans_dev || !cells_dev)) ||
      (turns_dev && !boxes_dev)) {
    ctx->set_error("b2o_char_cells: bad argument");
    return B2O_ERR_ARG;
  }
  if (b == 0) return B2O_OK;
  DeviceGuard guard(ctx->device);
  char_cells_kernel<<<b, kCellThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(spans_dev, top_paths, theta_dev,
                                                                                   boxes_dev, turns_dev, cells_dev);
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}
