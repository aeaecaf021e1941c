// windows.cu -- wide words (DESIGN.md section 1, "Wide words"): a box wider than the 200 x 31 crop at full height is
// read as K overlapping 200-column windows at the scale min(T / w, 31 / h), T = 200 + (M - 1) S, and the windows'
// CTC steps are stitched into one reading (include/b2ocr.h).
//   window_counts_kernel : one thread per box: K (1 for a word that fits, as warpBox reads it today).
//   warp_windows_kernel  : one CTA per window: thread 0 finds the window's word in the CSR of window starts and plans
//                          the window's homography; then warp_kernel's sampling (common.cuh's warp_sample).
//   stitch_kernel        : one warp per wide word: per-step argmax, log max-probability and position of every window,
//                          the cuts between windows, and greedy CTC over the kept steps.
// Every value is fp64 with a fixed operation order, or fp32 in a fixed order: a word's result is a function of its box,
// logits and theta alone, whatever the batch.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kCropH = kWarpCropH, kCropW = kWarpCropW, kT = 48, kDiscard = 2;
constexpr int kStride = B2O_WINDOW_STRIDE, kShrink = B2O_WINDOW_SHRINK, kMaxWindows = B2O_MAX_WINDOWS;

// The word frame: warp_extent in turn 0 with the target width T = 200 + (M - 1) S, so wc = scale w and sh = scale h with
// scale = min(T / w, 31 / h) in warp_extent's own fp64 expressions.  K = 1 where the word fits (wc <= 200) or warpBox
// raises (then ok is false); otherwise 1 + ceil((wc - 200) / S), at most M (wc may exceed T by an ulp).
__device__ inline int window_extent(const float* q, int max_windows, float box[8], double* wc, double* sh, bool* ok) {
  *wc = *sh = 0.0;
  *ok = warp_extent(q, 0, kCropW + (max_windows - 1) * kStride, kCropH, box, wc, sh);
  if (!*ok || *wc <= kCropW) return 1;
  const int k = 1 + static_cast<int>(ceil(__ddiv_rn(__dsub_rn(*wc, static_cast<double>(kCropW)), kStride)));
  return k < max_windows ? k : max_windows;
}

// a_k: k S for all but the last window, which ends flush with the word (wc - 200); 0 for a word that fits.
__device__ __forceinline__ double window_start(int k, int K, double wc) {
  if (K == 1) return 0.0;
  return k < K - 1 ? static_cast<double>(k * kStride) : __dsub_rn(wc, static_cast<double>(kCropW));
}

// Window k of the box: the ordered box onto (-a, 0), (wc - a, 0), (wc - a, sh), (-a, sh), each rounded to float32, dsize
// (200, int(sh)).  A word that fits (K = 1) gets plan_warp's plan: a = 0 and dsize (int(wc), int(sh)).
__device__ inline void plan_window(const float* q, int max_windows, int k, b2o_window_plan* p) {
  float box[8];
  double wc, sh;
  bool ok;
  const int K = window_extent(q, max_windows, box, &wc, &sh, &ok);
  for (int i = 0; i < 9; ++i) p->m[i] = 0.0;
  p->wc = wc;
  p->sh = sh;
  p->k = K;
  p->a = 0.0;
  p->dw = p->dh = p->valid = 0;
  if (!ok || k >= K) return;
  const double a = window_start(k, K, wc);
  const float x0 = static_cast<float>(__dsub_rn(0.0, a)), x1 = static_cast<float>(__dsub_rn(wc, a));
  const float y1 = static_cast<float>(sh);
  const float dst[8] = {x0, 0.f, x1, 0.f, x1, y1, x0, y1};
  p->a = a;
  p->dw = K == 1 ? static_cast<int>(wc) : kCropW;
  p->dh = static_cast<int>(sh);
  if (persp_inverse(box, dst, p->m)) p->valid = 1;
}

// K of box j of image i, j < counts[i] (counts null: every slot); slots past the count are not written.
__global__ void window_counts_kernel(const float* __restrict__ boxes, const int32_t* __restrict__ counts, int n,
                                     int max_boxes, int max_windows, int32_t* __restrict__ windows) {
  const long long g = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (g >= static_cast<long long>(n) * max_boxes) return;
  const int i = static_cast<int>(g / max_boxes), j = static_cast<int>(g - static_cast<long long>(i) * max_boxes);
  if (counts && j >= counts[i]) return;
  float box[8];
  double wc, sh;
  bool ok;
  windows[g] = window_extent(boxes + g * 8, max_windows, box, &wc, &sh, &ok);
}

// the word whose windows hold window j: the last i with win_start[i] <= j
__device__ __forceinline__ int word_of(const int32_t* __restrict__ win_start, int n_words, int j) {
  int lo = 0, hi = n_words - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (win_start[mid] <= j) lo = mid; else hi = mid - 1;
  }
  return lo;
}

template <int CH>
__global__ void __launch_bounds__(256)
warp_windows_kernel(const uint8_t* __restrict__ img_all, int n, int H, int W, const float* __restrict__ boxes,
                    const int32_t* __restrict__ image_index, const int32_t* __restrict__ words,
                    const int32_t* __restrict__ win_start, int n_words, int max_windows, int first,
                    uint8_t* __restrict__ crops, __half* __restrict__ crnn_in) {
  __shared__ b2o_window_plan plan;
  __shared__ int word_box;
  __shared__ uint8_t tile[kCropH * kCropW * CH];
  const int slot = blockIdx.x, j = first + slot;
  if (threadIdx.x == 0) {
    const int i = word_of(win_start, n_words, j);
    word_box = words[i];
    plan_window(boxes + static_cast<size_t>(word_box) * 8, max_windows, j - win_start[i], &plan);
  }
  __syncthreads();
  int img = image_index[word_box];
  img = min(max(img, 0), n - 1);
  const uint8_t* g = img_all + static_cast<size_t>(img) * H * W * CH;
  const int dw = plan.valid ? min(plan.dw, kCropW) : 0, dh = plan.valid ? min(plan.dh, kCropH) : 0;
  const int bw0 = warp_block_width(dw, dh);
  warp_crop<CH>(dw, dh, [&](int x, int y, int (&v)[CH]) { warp_sample<CH>(g, H, W, plan.m, x, y, bw0, v); },
                tile, slot, crops, crnn_in);
}

__global__ void __launch_bounds__(32)
stitch_kernel(const float* __restrict__ logits /*[W][48][C]*/, int C, const float* __restrict__ theta /*[W][6]*/,
              const float* __restrict__ boxes, const int32_t* __restrict__ words, const int32_t* __restrict__ win_start,
              int max_windows, int32_t* __restrict__ labels /*[.][48 M]*/, float* __restrict__ logp) {
  __shared__ int best[kMaxWindows][kT];
  __shared__ float term[kMaxWindows][kT];
  __shared__ double pos[kMaxWindows][kT];
  __shared__ double cut[kMaxWindows];
  __shared__ int kept;
  const int lane = threadIdx.x, word = blockIdx.x, blank = C - 1;
  const int w0 = win_start[word], box_id = words[word];
  const int K = min(max(win_start[word + 1] - w0, 1), max_windows);
  double wc = 0.0;
  if (lane == 0) {
    float box[8];
    double sh;
    bool ok;
    window_extent(boxes + static_cast<size_t>(box_id) * 8, max_windows, box, &wc, &sh, &ok);
  }
  wc = __shfl_sync(0xffffffffu, wc, 0);
  // 1. every window's steps: first maximum, log(max p + 1e-7) with max p = 1 / sum_c exp(l_c - l_max) summed in
  //    ascending c, and the position a_k + x in the word, x clamped to [0, 200] and made non-decreasing
  for (int k = 0; k < K; ++k) {
    const float* lg = logits + static_cast<size_t>(w0 + k) * kT * C;
    const float* th = theta ? theta + static_cast<size_t>(w0 + k) * 6 : nullptr;
    for (int t = lane; t < kT; t += 32) {
      const float* row = lg + static_cast<size_t>(t) * C;
      float m = -INFINITY;
      int arg = -1;
      for (int c = 0; c < C; ++c)
        if (row[c] > m) { m = row[c]; arg = c; }
      float s = 0.f;
      for (int c = 0; c < C; ++c) s = __fadd_rn(s, expf(__fsub_rn(row[c], m)));
      best[k][t] = arg < 0 ? 0 : arg;                    // all-NaN row: argmax 0, as fc_ctc_kernel
      term[k][t] = logf(__fadd_rn(__frcp_rn(s), 1e-7f));
      pos[k][t] = fmin(fmax(stn_crop_x(static_cast<double>(t + kDiscard), th), 0.0), static_cast<double>(kCropW));
    }
    __syncwarp();
    if (lane == 0) {
      const double a = window_start(k, K, wc);
      double run = 0.0;
      for (int t = 0; t < kT; ++t) {
        run = fmax(run, pos[k][t]);
        pos[k][t] = __dadd_rn(a, run);
      }
    }
    __syncwarp();
  }
  // 2. the cut between windows k and k + 1: the candidate of window k+1 nearest the overlap's centre (the lower step on
  //    a tie) where both windows emit a blank, else the centre itself; raised to the previous cut where it falls below
  for (int k = 0; k + 1 < K; ++k) {
    const double a0 = window_start(k, K, wc), a1 = window_start(k + 1, K, wc);
    const double end = __dadd_rn(a0, static_cast<double>(kCropW));
    const double mid = __dmul_rn(0.5, __dadd_rn(a1, end));
    const double lo = __dadd_rn(a1, static_cast<double>(kShrink)), hi = __dsub_rn(end, static_cast<double>(kShrink));
    double bd = INFINITY;
    int bt = kT;
    for (int t = lane; t < kT; t += 32) {
      const double p = pos[k + 1][t];
      if (!(p >= lo && p <= hi) || best[k + 1][t] != blank) continue;
      double nd = INFINITY;
      int nt = 0;
      for (int u = 0; u < kT; ++u) {
        const double d = fabs(__dsub_rn(pos[k][u], p));
        if (d < nd) { nd = d; nt = u; }
      }
      if (best[k][nt] != blank) continue;
      const double d = fabs(__dsub_rn(p, mid));
      if (d < bd || (d == bd && t < bt)) { bd = d; bt = t; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double od = __shfl_xor_sync(0xffffffffu, bd, o);
      const int ot = __shfl_xor_sync(0xffffffffu, bt, o);
      if (od < bd || (od == bd && ot < bt)) { bd = od; bt = ot; }
    }
    if (lane == 0) {                                     // never below the previous cut: no range is read twice
      const double c = bt < kT ? pos[k + 1][bt] : mid;
      cut[k] = k ? fmax(c, cut[k - 1]) : c;
    }
    __syncwarp();
  }
  // 3. window k keeps cut_{k-1} <= P < cut_k; greedy CTC over the kept steps in order
  int32_t* out = labels + static_cast<size_t>(box_id) * kT * max_windows;
  if (lane == 0) {
    int n = 0, prev = -1;
    float S = 0.f;
    for (int k = 0; k < K; ++k) {
      const double from = k ? cut[k - 1] : -INFINITY, to = k + 1 < K ? cut[k] : INFINITY;
      for (int t = 0; t < kT; ++t) {
        const double p = pos[k][t];
        if (!(p >= from && p < to)) continue;
        const int c = best[k][t];
        S = __fadd_rn(S, term[k][t]);
        if (c != blank && c != prev) out[n++] = c;
        prev = c;
      }
    }
    if (logp) logp[box_id] = S;
    kept = n;
  }
  __syncwarp();
  for (int i = kept + lane; i < kT * max_windows; i += 32) out[i] = -1;
}

// b2o_window_plan_test: plan_window of every (box, window) slot, one thread each.
__global__ void window_plan_kernel(const float* __restrict__ boxes, int n, int max_windows,
                                   b2o_window_plan* __restrict__ plans) {
  const long long g = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (g >= static_cast<long long>(n) * max_windows) return;
  b2o_window_plan p;
  plan_window(boxes + (g / max_windows) * 8, max_windows, static_cast<int>(g % max_windows), &p);
  plans[g] = p;
}

}  // namespace

static bool windows_ok(int max_windows) { return max_windows >= 1 && max_windows <= B2O_MAX_WINDOWS; }

extern "C" int b2o_window_counts(b2o_ctx* ctx, const float* boxes_dev, const int32_t* counts_dev, int n, int max_boxes,
                                 int max_windows, int32_t* windows_dev, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  if (!windows_ok(max_windows) || n < 0 || max_boxes < 0 || (n > 0 && max_boxes > 0 && (!boxes_dev || !windows_dev))) {
    ctx->set_error("b2o_window_counts: bad argument (1 <= max_windows <= 16)");
    return B2O_ERR_ARG;
  }
  const long long total = static_cast<long long>(n) * max_boxes;
  if (total == 0) return B2O_OK;
  DeviceGuard guard(ctx->device);
  window_counts_kernel<<<static_cast<unsigned>((total + 127) / 128), 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      boxes_dev, counts_dev, n, max_boxes, max_windows, windows_dev);
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}

extern "C" int b2o_warp_windows(b2o_ctx* ctx, const uint8_t* img_dev, int channels, int n, int h, int w,
                                const float* boxes_dev, const int32_t* image_index_dev, const int32_t* words_dev,
                                const int32_t* win_start_dev, int n_words, int max_windows, int first, int count,
                                uint8_t* crops_dev, void* crnn_in_dev, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  if (channels != 1 && channels != 3) { ctx->set_error("b2o_warp_windows: channels must be 1 or 3"); return B2O_ERR_ARG; }
  if (!windows_ok(max_windows) || count < 0 || first < 0 || n_words < 0) {
    ctx->set_error("b2o_warp_windows: bad argument (1 <= max_windows <= 16)");
    return B2O_ERR_ARG;
  }
  if (count == 0) return B2O_OK;
  if (!img_dev || !boxes_dev || !image_index_dev || !words_dev || !win_start_dev || n_words == 0 || n <= 0 || h <= 0 ||
      w <= 0 || (!crops_dev && !crnn_in_dev)) {
    ctx->set_error("b2o_warp_windows: bad argument");
    return B2O_ERR_ARG;
  }
  DeviceGuard guard(ctx->device);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  __half* x = reinterpret_cast<__half*>(crnn_in_dev);
  if (channels == 3)
    warp_windows_kernel<3><<<count, 256, 0, st>>>(img_dev, n, h, w, boxes_dev, image_index_dev, words_dev, win_start_dev,
                                                  n_words, max_windows, first, crops_dev, x);
  else
    warp_windows_kernel<1><<<count, 256, 0, st>>>(img_dev, n, h, w, boxes_dev, image_index_dev, words_dev, win_start_dev,
                                                  n_words, max_windows, first, crops_dev, x);
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}

extern "C" int b2o_stitch_windows(b2o_ctx* ctx, const float* logits_dev, int k, const float* theta_dev,
                                  const float* boxes_dev, const int32_t* words_dev, const int32_t* win_start_dev,
                                  int n_words, int max_windows, int32_t* labels_dev, float* logp_dev, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  if (k < 2 || k > B2O_MAX_CLASSES || !windows_ok(max_windows) || n_words < 0 ||
      (n_words > 0 && (!logits_dev || !boxes_dev || !words_dev || !win_start_dev || !labels_dev))) {
    ctx->set_error("b2o_stitch_windows: bad argument (2 <= k <= 1024, 1 <= max_windows <= 16)");
    return B2O_ERR_ARG;
  }
  if (n_words == 0) return B2O_OK;
  DeviceGuard guard(ctx->device);
  stitch_kernel<<<n_words, 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(logits_dev, k, theta_dev, boxes_dev, words_dev,
                                                                           win_start_dev, max_windows, labels_dev,
                                                                           logp_dev);
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}

extern "C" int b2o_window_plan_test(b2o_ctx* ctx, const float* boxes_dev, int n, int max_windows,
                                    b2o_window_plan* plans_dev, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  if (!windows_ok(max_windows) || n < 0 || (n > 0 && (!boxes_dev || !plans_dev))) {
    ctx->set_error("b2o_window_plan_test: bad argument");
    return B2O_ERR_ARG;
  }
  if (n == 0) return B2O_OK;
  DeviceGuard guard(ctx->device);
  const long long total = static_cast<long long>(n) * max_windows;
  window_plan_kernel<<<static_cast<unsigned>((total + 127) / 128), 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      boxes_dev, n, max_windows, plans_dev);
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}
