// image.cu -- the OpenCV image stages of Pipeline.recognize as CUDA kernels, bit-compatible with
// OpenCV 4.x fixed-point arithmetic (models of the arithmetic are pinned against cv2 in
// tests/test_cv_models.py and tests/test_image_refs.py; these kernels against the models, plan included, in
// tests/test_gpu_image_stages.py):
//   resize_pad_kernel : cv2.resize INTER_LINEAR on uint8 (tools.py:394-396) + tools.pad(255) (356-375)
//   gray_kernel       : cv2.cvtColor(RGB2GRAY) (recognition.py:510)
//   warp_kernel       : tools.warpBox (tools.py:61-117): get_rotated_box ordering (533-581, rectangle
//                       branch), get_rotated_width_height (41-57), cv2.getPerspectiveTransform (8x8 LU,
//                       fp64), cv2.warpPerspective INTER_LINEAR (1/32-pixel coordinates, 15-bit weights); in quarter
//                       turn r the ordered box is rolled by r first (warpBox(skip_rotate=True), b2o_warp_boxes_turned)
#include <math.h>

#include "common.cuh"

namespace {

// ------------------------------------------------------------------------------------ resize + pad
// blockIdx.z = image of a batch of equally sized sources (strides 0 for the one-image entry point); `gray`,
// when given, also receives cv2.cvtColor(RGB2GRAY) of the padded result (recognition.py:510), which saves the
// recognizer a second pass over the batch.
__device__ __forceinline__ uint8_t gray_of(int r, int g, int b) {
  return static_cast<uint8_t>((9798 * r + 19235 * g + 3735 * b + 16384) >> 15);
}

// scale_x / scale_y = 1 / (dsize / ssize) in fp64, computed once on the host exactly as OpenCV does: two fp64
// divisions per pixel cost more than everything else in this kernel.
__global__ void resize_pad_kernel(const uint8_t* __restrict__ src, int hs, int ws, int hr, int wr,
                                  uint8_t* __restrict__ dst, int hp, int wp, uint8_t* __restrict__ gray,
                                  double scale_x, double scale_y) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y;
  if (x >= wp) return;
  src += static_cast<size_t>(blockIdx.z) * hs * ws * 3;
  const size_t opix = (static_cast<size_t>(blockIdx.z) * hp + y) * wp + x;
  uint8_t* o = dst + opix * 3;
  if (x >= wr || y >= hr) {
    o[0] = 255; o[1] = 255; o[2] = 255;
    if (gray) gray[opix] = gray_of(255, 255, 255);
    return;
  }
  // OpenCV: scale = 1 / (dsize / ssize), source coordinate at pixel centres, float fractions,
  // 11-bit coefficients (INTER_RESIZE_COEF_BITS), horizontal pass first.  (x + 0.5) * scale - 0.5 rounds the
  // product and the difference separately, as OpenCV does: a contracted DFMA would round once.
  float fx = static_cast<float>(__dadd_rn(__dmul_rn(x + 0.5, scale_x), -0.5));
  int sx = static_cast<int>(floorf(fx));
  fx -= sx;
  if (sx < 0) { fx = 0.f; sx = 0; }
  if (sx >= ws - 1) { fx = 0.f; sx = ws - 1; }
  const int sx1 = min(sx + 1, ws - 1);
  const int a0 = __float2int_rn((1.f - fx) * 2048.f), a1 = __float2int_rn(fx * 2048.f);
  float fy = static_cast<float>(__dadd_rn(__dmul_rn(y + 0.5, scale_y), -0.5));
  const int sy = static_cast<int>(floorf(fy));
  fy -= sy;
  const int b0 = __float2int_rn((1.f - fy) * 2048.f), b1 = __float2int_rn(fy * 2048.f);
  const int y0 = min(max(sy, 0), hs - 1), y1 = min(max(sy + 1, 0), hs - 1);
  const uint8_t* r0 = src + static_cast<size_t>(y0) * ws * 3;
  const uint8_t* r1 = src + static_cast<size_t>(y1) * ws * 3;
  int rgb[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int s0 = r0[sx * 3 + c] * a0 + r0[sx1 * 3 + c] * a1;
    const int s1 = r1[sx * 3 + c] * a0 + r1[sx1 * 3 + c] * a1;
    const int v = (((b0 * (s0 >> 4)) >> 16) + ((b1 * (s1 >> 4)) >> 16) + 2) >> 2;
    rgb[c] = min(max(v, 0), 255);
    o[c] = static_cast<uint8_t>(rgb[c]);
  }
  if (gray) gray[opix] = gray_of(rgb[0], rgb[1], rgb[2]);
}

// ------------------------------------------------------------------------------------ RGB -> gray
__global__ void gray_kernel(const uint8_t* __restrict__ img, long long total, uint8_t* __restrict__ gray) {
  const long long p = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p >= total) return;
  const uint8_t* q = img + p * 3;
  gray[p] = gray_of(q[0], q[1], q[2]);
}

// ------------------------------------------------------------------------------------ warpBox
// plan_warp / warp_extent (common.cuh): the WarpPlan of a box in quarter turn r.
using WarpPlan = b2o_warp_plan;

constexpr int kCropH = 31, kCropW = 200;
constexpr int kMaxPolySegments = B2O_MAX_POLY_SEGMENTS;

// warp_sample, warp_block_width and warp_crop: common.cuh.

// CH = 1: gray image (n,H,W), crops (k,31,200), CRNN input (k,200,31).  CH = 3 (build_model(color=True),
// recognition.py:214, 508-510: no gray conversion): RGB image (n,H,W,3), crops (k,31,200,3), CRNN input (k,200,31,3);
// cv2.warpPerspective samples every channel with the same coordinates and weights.
template <int CH>
__global__ void __launch_bounds__(256)
warp_kernel(const uint8_t* __restrict__ gray, int n, int H, int W, const float* __restrict__ boxes,
            const int* __restrict__ image_index, int turn, uint8_t* __restrict__ crops, __half* __restrict__ crnn_in) {
  __shared__ WarpPlan plan;
  __shared__ uint8_t tile[kCropH * kCropW * CH];
  const int k = blockIdx.x;
  if (threadIdx.x == 0) plan_warp(boxes + static_cast<size_t>(k) * 8, turn, kCropW, kCropH, &plan);
  __syncthreads();
  int img = image_index[k];
  img = min(max(img, 0), n - 1);
  const uint8_t* g = gray + static_cast<size_t>(img) * H * W * CH;
  const int dw = plan.valid ? min(plan.dw, kCropW) : 0, dh = plan.valid ? min(plan.dh, kCropH) : 0;
  const int bw0 = warp_block_width(dw, dh);
  warp_crop<CH>(dw, dh, [&](int x, int y, int (&v)[CH]) { warp_sample<CH>(g, H, W, plan.m, x, y, bw0, v); },
                tile, k, crops, crnn_in);
}

// ------------------------------------------------------------------------------------ piecewise warpBox
// One polygon of s segments (b2o_warp_polys): top edge t_0..t_s = poly[0..s], bottom edge b_i = poly[2s+1-i].
// w = int(sum_i (|t_i t_i+1| + |b_i b_i+1|) / 2), h = int(mean_j |t_j b_j|), scale = min(200 / w, 31 / h), dsize =
// (int(scale w), int(scale h)); segment i maps onto x in [X_i, X_i+1], X_i = float32(scale w * cum_i / cum_s) with cum
// the running edge-mean length, y in [0, float32(scale h)].  A 4-point entry is warpBox itself (plan_warp).
struct PolyPlan {
  double m[kMaxPolySegments][9];
  float X[kMaxPolySegments + 1];
  int seg_ok[kMaxPolySegments];
  int s, dw, dh, valid;
};

__device__ void plan_poly(const float* poly, int points, PolyPlan* p) {
  p->valid = 0;
  p->s = 1;
  if (points == 4) {
    b2o_warp_plan wp;
    wp.dw = wp.dh = 0;
    plan_warp(poly, 0, kCropW, kCropH, &wp);
    if (!wp.valid) return;
    for (int i = 0; i < 9; ++i) p->m[0][i] = wp.m[i];
    p->seg_ok[0] = 1;
    p->dw = wp.dw; p->dh = wp.dh; p->valid = 1;
    return;
  }
  if (points < 6 || points > 2 * (kMaxPolySegments + 1) || (points & 1)) return;
  const int s = points / 2 - 1;
  const float* t = poly;
  double cum[kMaxPolySegments + 1];
  cum[0] = 0.0;
  for (int i = 0; i < s; ++i) {
    const double dt = corner_dist(t + 2 * i, t + 2 * (i + 1));
    const double db = corner_dist(poly + 2 * (points - 1 - i), poly + 2 * (points - 2 - i));
    cum[i + 1] = __dadd_rn(cum[i], __dadd_rn(dt, db) / 2);
  }
  double hs = 0.0;
  for (int j = 0; j <= s; ++j) hs = __dadd_rn(hs, corner_dist(t + 2 * j, poly + 2 * (points - 1 - j)));
  const int w = static_cast<int>(cum[s]);
  const int h = static_cast<int>(hs / (s + 1));
  if (w <= 0 || h <= 0) return;
  const double sa = static_cast<double>(kCropW) / w, sb = static_cast<double>(kCropH) / h;
  const double scale = sa < sb ? sa : sb;
  const double sw = __dmul_rn(scale, w), sh = __dmul_rn(scale, h);
  for (int i = 0; i <= s; ++i) p->X[i] = static_cast<float>(__dmul_rn(sw, cum[i] / cum[s]));
  const float fsh = static_cast<float>(sh);
  for (int i = 0; i < s; ++i) {
    const float* ti = t + 2 * i;
    const float* bi = poly + 2 * (points - 1 - i);
    const float src[8] = {ti[0], ti[1], ti[2], ti[3], bi[-2], bi[-1], bi[0], bi[1]};
    const float dst[8] = {p->X[i], 0.f, p->X[i + 1], 0.f, p->X[i + 1], fsh, p->X[i], fsh};
    p->seg_ok[i] = persp_inverse(src, dst, p->m[i]) ? 1 : 0;
  }
  p->s = s;
  p->dw = static_cast<int>(sw);
  p->dh = static_cast<int>(sh);
  p->valid = 1;
}

template <int CH>
__global__ void __launch_bounds__(256)
warp_polys_kernel(const uint8_t* __restrict__ img_all, int n, int H, int W, const float* __restrict__ polys,
                  const int* __restrict__ points, const int* __restrict__ image_index, uint8_t* __restrict__ crops,
                  __half* __restrict__ crnn_in) {
  __shared__ PolyPlan plan;
  __shared__ uint8_t tile[kCropH * kCropW * CH];
  const int k = blockIdx.x;
  if (threadIdx.x == 0) plan_poly(polys + static_cast<size_t>(k) * 4 * (kMaxPolySegments + 1), points[k], &plan);
  __syncthreads();
  int img = image_index[k];
  img = min(max(img, 0), n - 1);
  const uint8_t* g = img_all + static_cast<size_t>(img) * H * W * CH;
  const int dw = plan.valid ? min(plan.dw, kCropW) : 0, dh = plan.valid ? min(plan.dh, kCropH) : 0;
  const int bw0 = warp_block_width(dw, dh);
  warp_crop<CH>(dw, dh, [&](int x, int y, int (&v)[CH]) {
    int seg = 0;
    const float fx = static_cast<float>(x);
    for (int j = 1; j < plan.s; ++j) if (plan.X[j] <= fx) seg = j;
    if (plan.seg_ok[seg]) warp_sample<CH>(g, H, W, plan.m[seg], x, y, bw0, v);
  }, tile, k, crops, crnn_in);
}

// b2o_warp_plan_test: plan_warp alone, one thread per box.  A degenerate box leaves m, dw and dh zero.
__global__ void warp_plan_kernel(const float* __restrict__ boxes, int n, WarpPlan* __restrict__ plans) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  WarpPlan p = {};
  plan_warp(boxes + static_cast<size_t>(k) * 8, 0, kCropW, kCropH, &p);
  plans[k] = p;
}

// crops (k,31,200[,ch]) u8 -> CRNN input (k,200,31[,ch]) fp16 = crop / 255 after Permute((2,1,3)) and the axis flip
__global__ void crops_to_input_kernel(const uint8_t* __restrict__ crops, long long total, int ch, __half* __restrict__ out) {
  const long long p = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p >= total) return;
  const int per = kCropH * kCropW * ch;
  const long long k = p / per;
  const int i = static_cast<int>(p - k * per);
  const int c = i % ch, q = i / ch;
  const int t = q / kCropH, j = q - t * kCropH;
  out[p] = __float2half_rn(static_cast<float>(crops[k * per + ((kCropH - 1 - j) * kCropW + t) * ch + c]) / 255.0f);
}

}  // namespace

extern "C" int b2o_resize_pad(b2o_ctx* ctx, const uint8_t* src, int hs, int ws, int hr, int wr, uint8_t* dst,
                              int index, int hp, int wp, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  DeviceGuard guard(ctx->device);
  if (!src || !dst || hs <= 0 || ws <= 0 || hr <= 0 || wr <= 0 || hr > hp || wr > wp || index < 0) {
    ctx->set_error("b2o_resize_pad: bad argument (resized image must fit the padded size)");
    return B2O_ERR_ARG;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  resize_pad_kernel<<<dim3((wp + 127) / 128, hp), 128, 0, st>>>(src, hs, ws, hr, wr,
                                                                dst + static_cast<size_t>(index) * hp * wp * 3, hp, wp,
                                                                nullptr, 1.0 / (static_cast<double>(wr) / ws),
                                                                1.0 / (static_cast<double>(hr) / hs));
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}

extern "C" int b2o_resize_pad_batch(b2o_ctx* ctx, const uint8_t* src, int n, int hs, int ws, int hr, int wr,
                                    uint8_t* dst, int hp, int wp, uint8_t* gray, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  DeviceGuard guard(ctx->device);
  if (!src || !dst || n <= 0 || n > 65535 || hs <= 0 || ws <= 0 || hr <= 0 || wr <= 0 || hr > hp || wr > wp || hp > 65535) {
    ctx->set_error("b2o_resize_pad_batch: bad argument (resized image must fit the padded size)");
    return B2O_ERR_ARG;
  }
  resize_pad_kernel<<<dim3((wp + 127) / 128, hp, n), 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      src, hs, ws, hr, wr, dst, hp, wp, gray, 1.0 / (static_cast<double>(wr) / ws), 1.0 / (static_cast<double>(hr) / hs));
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}

extern "C" int b2o_rgb_to_gray(b2o_ctx* ctx, const uint8_t* img, int n, int h, int w, uint8_t* gray, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  DeviceGuard guard(ctx->device);
  if (!img || !gray || n <= 0 || h <= 0 || w <= 0) { ctx->set_error("b2o_rgb_to_gray: bad argument"); return B2O_ERR_ARG; }
  const long long total = static_cast<long long>(n) * h * w;
  gray_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(img, total, gray);
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}

static int warp_boxes_impl(b2o_ctx* ctx, const uint8_t* img, int ch, int n, int h, int w, const float* boxes,
                           const int32_t* image_index, int n_boxes, int turn, uint8_t* crops, void* crnn_in,
                           void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  DeviceGuard guard(ctx->device);
  if (ch != 1 && ch != 3) { ctx->set_error("b2o_warp_boxes: channels must be 1 or 3"); return B2O_ERR_ARG; }
  if (turn < 0 || turn > 3) { ctx->set_error("b2o_warp_boxes_turned: turn must be 0, 1, 2 or 3"); return B2O_ERR_ARG; }
  if (n_boxes == 0) return B2O_OK;
  if (!img || !boxes || !image_index || n <= 0 || h <= 0 || w <= 0 || n_boxes < 0 || (!crops && !crnn_in)) {
    ctx->set_error("b2o_warp_boxes: bad argument");
    return B2O_ERR_ARG;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (ch == 3) warp_kernel<3><<<n_boxes, 256, 0, st>>>(img, n, h, w, boxes, image_index, turn, crops, reinterpret_cast<__half*>(crnn_in));
  else warp_kernel<1><<<n_boxes, 256, 0, st>>>(img, n, h, w, boxes, image_index, turn, crops, reinterpret_cast<__half*>(crnn_in));
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}

extern "C" int b2o_warp_boxes(b2o_ctx* ctx, const uint8_t* gray, int n, int h, int w, const float* boxes,
                              const int32_t* image_index, int n_boxes, uint8_t* crops, void* crnn_in, void* stream) {
  return warp_boxes_impl(ctx, gray, 1, n, h, w, boxes, image_index, n_boxes, 0, crops, crnn_in, stream);
}

extern "C" int b2o_warp_boxes_color(b2o_ctx* ctx, const uint8_t* rgb, int n, int h, int w, const float* boxes,
                                    const int32_t* image_index, int n_boxes, uint8_t* crops, void* crnn_in, void* stream) {
  return warp_boxes_impl(ctx, rgb, 3, n, h, w, boxes, image_index, n_boxes, 0, crops, crnn_in, stream);
}

extern "C" int b2o_warp_boxes_turned(b2o_ctx* ctx, const uint8_t* img, int channels, int n, int h, int w,
                                     const float* boxes, const int32_t* image_index, int n_boxes, int turn,
                                     uint8_t* crops, void* crnn_in, void* stream) {
  return warp_boxes_impl(ctx, img, channels, n, h, w, boxes, image_index, n_boxes, turn, crops, crnn_in, stream);
}

extern "C" int b2o_warp_polys(b2o_ctx* ctx, const uint8_t* img, int channels, int n, int h, int w, const float* polys,
                              const int32_t* points, const int32_t* image_index, int n_polys, uint8_t* crops,
                              void* crnn_in, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  DeviceGuard guard(ctx->device);
  if (channels != 1 && channels != 3) { ctx->set_error("b2o_warp_polys: channels must be 1 or 3"); return B2O_ERR_ARG; }
  if (n_polys == 0) return B2O_OK;
  if (!img || !polys || !points || !image_index || n <= 0 || h <= 0 || w <= 0 || n_polys < 0 || (!crops && !crnn_in)) {
    ctx->set_error("b2o_warp_polys: bad argument");
    return B2O_ERR_ARG;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (channels == 3)
    warp_polys_kernel<3><<<n_polys, 256, 0, st>>>(img, n, h, w, polys, points, image_index, crops,
                                                  reinterpret_cast<__half*>(crnn_in));
  else
    warp_polys_kernel<1><<<n_polys, 256, 0, st>>>(img, n, h, w, polys, points, image_index, crops,
                                                  reinterpret_cast<__half*>(crnn_in));
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}

extern "C" int b2o_warp_plan_test(b2o_ctx* ctx, const float* boxes, int n, b2o_warp_plan* plans, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  DeviceGuard guard(ctx->device);
  if (n == 0) return B2O_OK;
  if (!boxes || !plans || n < 0) { ctx->set_error("b2o_warp_plan_test: bad argument"); return B2O_ERR_ARG; }
  warp_plan_kernel<<<(n + 127) / 128, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(boxes, n, plans);
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}

static int crops_to_input_impl(b2o_ctx* ctx, const uint8_t* crops, int ch, int b, void* crnn_in, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  DeviceGuard guard(ctx->device);
  if (b == 0) return B2O_OK;
  if (!crops || !crnn_in || b < 0) { ctx->set_error("b2o_crops_to_input: bad argument"); return B2O_ERR_ARG; }
  const long long total = static_cast<long long>(b) * kCropH * kCropW * ch;
  crops_to_input_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      crops, total, ch, reinterpret_cast<__half*>(crnn_in));
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}

extern "C" int b2o_crops_to_input(b2o_ctx* ctx, const uint8_t* crops, int b, void* crnn_in, void* stream) {
  return crops_to_input_impl(ctx, crops, 1, b, crnn_in, stream);
}

extern "C" int b2o_crops_to_input_color(b2o_ctx* ctx, const uint8_t* crops, int b, void* crnn_in, void* stream) {
  return crops_to_input_impl(ctx, crops, 3, b, crnn_in, stream);
}
