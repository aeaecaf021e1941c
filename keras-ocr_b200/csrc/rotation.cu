// rotation.cu -- reading every word in several quarter turns: b2o_select_rotation picks, per word or per image, the turn
// whose best reading is the most probable, gathers that turn's readings and rolls the word's box so that it starts at
// the text's own top-left corner (include/b2ocr.h).  The per-turn readings come from b2o_warp_boxes_turned followed by
// any of the CRNN decoders; this kernel only compares and copies, so a result is exact.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kSteps = 48;
constexpr int kThreads = 256;

struct Turns {
  int t[4];
};

// One CTA per image, so the page sums run in a fixed order whatever else is in the batch; one warp per word after that.
__global__ void __launch_bounds__(kThreads)
select_rotation_kernel(const int32_t* __restrict__ labels, const float* __restrict__ logp,
                       const int32_t* __restrict__ image_index, int b, int P, Turns turns, int R, int vote,
                       int32_t* __restrict__ labels_out, float* __restrict__ logp_out, int32_t* __restrict__ turn_out,
                       float* __restrict__ boxes, float* __restrict__ table, int max_boxes) {
  __shared__ int range[2];
  __shared__ float page[4];
  __shared__ int page_pick;
  const int img = blockIdx.x;
  if (threadIdx.x < 2) {                     // [lo, hi) of this image's words: lower bounds in the sorted image_index
    const int key = img + threadIdx.x;
    int lo = 0, hi = b;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (image_index[mid] < key) lo = mid + 1; else hi = mid;
    }
    range[threadIdx.x] = lo;
  }
  __syncthreads();
  const int w0 = range[0], w1 = range[1];
  if (w0 >= w1) return;
  const size_t plane = static_cast<size_t>(b) * P;                // one turn's (b, P) scores
  if (vote == B2O_ROTATION_VOTE_PAGE) {
    if (threadIdx.x < R) {                   // float32 sum in word order, one thread per turn
      float s = 0.f;
      for (int k = w0; k < w1; ++k) s = __fadd_rn(s, logp[threadIdx.x * plane + static_cast<size_t>(k) * P]);
      page[threadIdx.x] = s;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int best = 0;                          // strict >: ties and an all -inf image keep the turn listed first
      for (int j = 1; j < R; ++j)
        if (page[j] > page[best]) best = j;
      page_pick = best;
    }
    __syncthreads();
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int k = w0 + warp; k < w1; k += kThreads / 32) {
    int pick = 0;
    if (vote == B2O_ROTATION_VOTE_PAGE) {
      pick = page_pick;
    } else {
      float best = logp[static_cast<size_t>(k) * P];
      for (int j = 1; j < R; ++j) {
        const float v = logp[j * plane + static_cast<size_t>(k) * P];
        if (v > best) { best = v; pick = j; }
      }
    }
    const size_t src = pick * plane + static_cast<size_t>(k) * P;
    for (int i = lane; i < P * kSteps; i += 32) labels_out[static_cast<size_t>(k) * P * kSteps + i] = labels[src * kSteps + i];
    for (int i = lane; i < P; i += 32) logp_out[static_cast<size_t>(k) * P + i] = logp[src + i];
    if (lane == 0) {
      const int r = turns.t[pick];
      turn_out[k] = r;
      if (boxes) {                           // the box the crop was cut from: the ordered corners rolled by r
        float q[8], o[8];
        for (int i = 0; i < 8; ++i) q[i] = boxes[static_cast<size_t>(k) * 8 + i];
        int ord[4];
        order_corners(q, ord);
        for (int i = 0; i < 4; ++i) {
          o[2 * i] = q[2 * ord[(i + r) & 3]];
          o[2 * i + 1] = q[2 * ord[(i + r) & 3] + 1];
        }
        for (int i = 0; i < 8; ++i) boxes[static_cast<size_t>(k) * 8 + i] = o[i];
        const int slot = k - w0;
        if (table && slot < max_boxes)
          for (int i = 0; i < 8; ++i) table[(static_cast<size_t>(img) * max_boxes + slot) * 8 + i] = o[i];
      }
    }
  }
}

}  // namespace

extern "C" int b2o_select_rotation(b2o_ctx* ctx, const int32_t* labels_dev, const float* logp_dev,
                                   const int32_t* image_index_dev, int n_images, int b, int top_paths,
                                   const int32_t* turns_host, int n_turns, int vote, int32_t* labels_out_dev,
                                   float* logp_out_dev, int32_t* turn_out_dev, float* boxes_dev, float* table_dev,
                                   int max_boxes, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  DeviceGuard guard(ctx->device);
  if (!turns_host || n_turns < 1 || n_turns > 4 || (vote != B2O_ROTATION_VOTE_WORD && vote != B2O_ROTATION_VOTE_PAGE)) {
    ctx->set_error("b2o_select_rotation: 1 to 4 turns and a vote of B2O_ROTATION_VOTE_WORD or _PAGE are required");
    return B2O_ERR_ARG;
  }
  Turns turns = {{0, 0, 0, 0}};
  for (int j = 0; j < n_turns; ++j) {
    turns.t[j] = turns_host[j];
    bool dup = false;
    for (int i = 0; i < j; ++i) dup = dup || turns.t[i] == turns.t[j];
    if (turns.t[j] < 0 || turns.t[j] > 3 || dup) {
      ctx->set_error("b2o_select_rotation: turns must be distinct values in 0..3");
      return B2O_ERR_ARG;
    }
  }
  if (b == 0) return B2O_OK;
  if (b < 0 || n_images <= 0 || top_paths < 1 || !labels_dev || !logp_dev || !image_index_dev || !labels_out_dev ||
      !logp_out_dev || !turn_out_dev || (table_dev && (!boxes_dev || max_boxes < 1))) {
    ctx->set_error("b2o_select_rotation: bad argument");
    return B2O_ERR_ARG;
  }
  select_rotation_kernel<<<n_images, kThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      labels_dev, logp_dev, image_index_dev, b, top_paths, turns, n_turns, vote, labels_out_dev, logp_out_dev,
      turn_out_dev, boxes_dev, table_dev, max_boxes);
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}
