// conv_simt.cu -- CUDA-core kernels around the tensor-core conv engine:
//   * conv_simt_kernel : generic direct convolution (debug cross-check of conv_tc.cu, and the
//                        production path for the few layers whose channel counts are not multiples
//                        of 64: CRAFT conv_cls.*, STN 5x5 16->32)
//   * stem_rgb_kernel  : compute_input (detection.py:34-42) fused with basenet.slice1.0 + BN + ReLU
//   * stem_crnn_kernel : CRNN conv_1 (1->64, recognition.py:217-219)
//   * maxpool2 / maxpool3s1 / upsample (MaxPooling2D detection.py:100-102,365-367; UpsampleLike 290-309)
//   * head_tail_kernel : conv_cls.6 (1x1 16->16 ReLU) + conv_cls.8 (1x1 16->2) fused, fp32 scores
#include <string.h>

#include "common.cuh"

namespace {

__device__ __forceinline__ float apply_epilogue(float acc, const float* s1, const float* t1, const float* s2,
                                                const float* t2, int relu, int c) {
  float y = fmaf(acc, s1[c], t1[c]);
  if (relu) y = fmaxf(y, 0.0f);
  if (s2 != nullptr) y = fmaf(y, s2[c], t2[c]);
  return y;
}

template <int CO_T>
__global__ void __launch_bounds__(128)
conv_simt_kernel(const __half* __restrict__ in, int in_ld, int N, int H, int W, int cin,
                 const float* __restrict__ wgt, int cout, int ksize, int dil, const float* __restrict__ s1,
                 const float* __restrict__ t1, const float* __restrict__ s2, const float* __restrict__ t2, int relu,
                 void* __restrict__ out, int out_ld, int out_f32) {
  const long long total = static_cast<long long>(N) * H * W;
  const long long pix = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (pix >= total) return;
  const int co0 = blockIdx.y * CO_T;
  const int w = static_cast<int>(pix % W);
  const int h = static_cast<int>((pix / W) % H);
  const int n = static_cast<int>(pix / (static_cast<long long>(W) * H));
  float acc[CO_T];
#pragma unroll
  for (int j = 0; j < CO_T; ++j) acc[j] = 0.0f;
  const int hk = ksize >> 1;
  for (int ky = 0; ky < ksize; ++ky) {
    const int ih = h + (ky - hk) * dil;
    if (ih < 0 || ih >= H) continue;
    for (int kx = 0; kx < ksize; ++kx) {
      const int iw = w + (kx - hk) * dil;
      if (iw < 0 || iw >= W) continue;
      const __half* ip = in + ((static_cast<size_t>(n) * H + ih) * W + iw) * in_ld;
      const float* wp = wgt + static_cast<size_t>(ky * ksize + kx) * cin * cout + co0;
      for (int ci = 0; ci < cin; ci += 8) {
        const uint4 raw = *reinterpret_cast<const uint4*>(ip + ci);
        const __half2* h2 = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 xv = __half22float2(h2[e]);
          const float* w0 = wp + static_cast<size_t>(ci + 2 * e) * cout;
          const float* w1 = w0 + cout;
          if (CO_T % 4 == 0) {
#pragma unroll
            for (int j = 0; j < CO_T; j += 4) {
              const float4 a = __ldg(reinterpret_cast<const float4*>(w0 + j));
              const float4 b = __ldg(reinterpret_cast<const float4*>(w1 + j));
              acc[j + 0] = fmaf(xv.x, a.x, acc[j + 0]); acc[j + 1] = fmaf(xv.x, a.y, acc[j + 1]);
              acc[j + 2] = fmaf(xv.x, a.z, acc[j + 2]); acc[j + 3] = fmaf(xv.x, a.w, acc[j + 3]);
              acc[j + 0] = fmaf(xv.y, b.x, acc[j + 0]); acc[j + 1] = fmaf(xv.y, b.y, acc[j + 1]);
              acc[j + 2] = fmaf(xv.y, b.z, acc[j + 2]); acc[j + 3] = fmaf(xv.y, b.w, acc[j + 3]);
            }
          } else {
#pragma unroll
            for (int j = 0; j < CO_T; ++j) {
              acc[j] = fmaf(xv.x, __ldg(w0 + j), acc[j]);
              acc[j] = fmaf(xv.y, __ldg(w1 + j), acc[j]);
            }
          }
        }
      }
    }
  }
  if (out_f32) {
    float* o = reinterpret_cast<float*>(out) + static_cast<size_t>(pix) * out_ld + co0;
#pragma unroll
    for (int j = 0; j < CO_T; ++j) o[j] = apply_epilogue(acc[j], s1, t1, s2, t2, relu, co0 + j);
  } else {
    __half* o = reinterpret_cast<__half*>(out) + static_cast<size_t>(pix) * out_ld + co0;
#pragma unroll
    for (int j = 0; j < CO_T; j += 2) {
      const float a = apply_epilogue(acc[j], s1, t1, s2, t2, relu, co0 + j);
      const float b = apply_epilogue(acc[j + 1], s1, t1, s2, t2, relu, co0 + j + 1);
      *reinterpret_cast<__half2*>(o + j) = __floats2half2_rn(a, b);
    }
  }
}

// compute_input + 3x3 conv 3->64 + folded BN + ReLU.  One thread per pixel, weights in smem.
__global__ void __launch_bounds__(128)
stem_rgb_kernel(const uint8_t* __restrict__ img, int N, int H, int W, const float* __restrict__ wgt /*[27][64]*/,
                const float* __restrict__ s1, const float* __restrict__ t1, __half* __restrict__ out, int out_ld) {
  __shared__ float sw[27 * 64];
  __shared__ float ss[64], st[64];
  for (int i = threadIdx.x; i < 27 * 64; i += blockDim.x) sw[i] = wgt[i];
  if (threadIdx.x < 64) { ss[threadIdx.x] = s1[threadIdx.x]; st[threadIdx.x] = t1[threadIdx.x]; }
  __syncthreads();
  const long long total = static_cast<long long>(N) * H * W;
  const long long pix = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (pix >= total) return;
  const int w = static_cast<int>(pix % W);
  const int h = static_cast<int>((pix / W) % H);
  const int n = static_cast<int>(pix / (static_cast<long long>(W) * H));
  // numpy semantics of compute_input: float32 array, in-place ops against float64 constants
  const double mean[3] = {0.485 * 255, 0.456 * 255, 0.406 * 255};
  const double stdv[3] = {0.229 * 255, 0.224 * 255, 0.225 * 255};
  float x[27];
#pragma unroll
  for (int ky = 0; ky < 3; ++ky)
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {
      const int ih = h + ky - 1, iw = w + kx - 1;
      const bool ok = ih >= 0 && ih < H && iw >= 0 && iw < W;
      const uint8_t* ip = img + ((static_cast<size_t>(n) * H + (ok ? ih : 0)) * W + (ok ? iw : 0)) * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        float v = static_cast<float>(static_cast<double>(ip[c]) - mean[c]);
        v = static_cast<float>(static_cast<double>(v) / stdv[c]);
        x[(ky * 3 + kx) * 3 + c] = ok ? v : 0.0f;
      }
    }
  __half* o = out + static_cast<size_t>(pix) * out_ld;
#pragma unroll 1
  for (int cb = 0; cb < 64; cb += 8) {
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.0f;
#pragma unroll
    for (int k = 0; k < 27; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&sw[k * 64 + cb]);
      const float4 b = *reinterpret_cast<const float4*>(&sw[k * 64 + cb + 4]);
      acc[0] = fmaf(x[k], a.x, acc[0]); acc[1] = fmaf(x[k], a.y, acc[1]);
      acc[2] = fmaf(x[k], a.z, acc[2]); acc[3] = fmaf(x[k], a.w, acc[3]);
      acc[4] = fmaf(x[k], b.x, acc[4]); acc[5] = fmaf(x[k], b.y, acc[5]);
      acc[6] = fmaf(x[k], b.z, acc[6]); acc[7] = fmaf(x[k], b.w, acc[7]);
    }
    uint4 pk;
    __half2 h;
    h = __floats2half2_rn(fmaxf(fmaf(acc[0], ss[cb + 0], st[cb + 0]), 0.f), fmaxf(fmaf(acc[1], ss[cb + 1], st[cb + 1]), 0.f));
    pk.x = *reinterpret_cast<uint32_t*>(&h);
    h = __floats2half2_rn(fmaxf(fmaf(acc[2], ss[cb + 2], st[cb + 2]), 0.f), fmaxf(fmaf(acc[3], ss[cb + 3], st[cb + 3]), 0.f));
    pk.y = *reinterpret_cast<uint32_t*>(&h);
    h = __floats2half2_rn(fmaxf(fmaf(acc[4], ss[cb + 4], st[cb + 4]), 0.f), fmaxf(fmaf(acc[5], ss[cb + 5], st[cb + 5]), 0.f));
    pk.z = *reinterpret_cast<uint32_t*>(&h);
    h = __floats2half2_rn(fmaxf(fmaf(acc[6], ss[cb + 6], st[cb + 6]), 0.f), fmaxf(fmaf(acc[7], ss[cb + 7], st[cb + 7]), 0.f));
    pk.w = *reinterpret_cast<uint32_t*>(&h);
    *reinterpret_cast<uint4*>(o + cb) = pk;
  }
}

// compute_input (detection.py:34-42) into a 16-channel fp16 image (r, g, b, 0 x 13): the A operand of
// the tensor-core stem convolution (3x3, 16 -> 64 with the 13 padding channels weighted 0).
__global__ void normalize16_kernel(const uint8_t* __restrict__ img, long long total, __half* __restrict__ out) {
  const long long p = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p >= total) return;
  const double mean[3] = {0.485 * 255, 0.456 * 255, 0.406 * 255};
  const double stdv[3] = {0.229 * 255, 0.224 * 255, 0.225 * 255};
  const uint8_t* ip = img + p * 3;
  float v[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float t = static_cast<float>(static_cast<double>(ip[c]) - mean[c]);
    v[c] = static_cast<float>(static_cast<double>(t) / stdv[c]);
  }
  const __half2 rg = __floats2half2_rn(v[0], v[1]), b0 = __floats2half2_rn(v[2], 0.0f);
  uint4 lo, hi = make_uint4(0u, 0u, 0u, 0u);
  lo.x = *reinterpret_cast<const uint32_t*>(&rg);
  lo.y = *reinterpret_cast<const uint32_t*>(&b0);
  lo.z = 0u; lo.w = 0u;
  uint4* o = reinterpret_cast<uint4*>(out + p * 16);
  o[0] = lo;
  o[1] = hi;
}

// CRNN conv_1: x (B,200,31[,CIN]) fp16 -> (B,200,31,64) fp16, 3x3 same, bias + ReLU.  CIN = 1 (gray, the default) or 3
// (build_model(color=True), recognition.py:214).  Weights [tap][cin][64].
// (The 576 filter taps stay in shared memory: read as a kernel parameter through the constant cache they would be 576
// scalar constant loads per thread; the constant bank only pays for a few dozen reads.)
// Each thread computes PIX consecutive pixels, so one shared-memory read of a filter tap feeds PIX FMAs (with one pixel
// per thread the kernel is bound by shared-memory reads).
template <int CIN, int PIX>
__global__ void __launch_bounds__(128)
stem_crnn_kernel(const __half* __restrict__ x, int B, int H, int W, const float* __restrict__ wgt /*[9*CIN][64]*/,
                 const float* __restrict__ t1, __half* __restrict__ out, int out_ld) {
  constexpr int K = 9 * CIN;
  __shared__ float sw[K * 64];
  __shared__ float sb[64];
  for (int i = threadIdx.x; i < K * 64; i += blockDim.x) sw[i] = wgt[i];
  if (threadIdx.x < 64) sb[threadIdx.x] = t1[threadIdx.x];
  __syncthreads();
  const long long total = static_cast<long long>(B) * H * W;
  const long long pix0 = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * PIX;
  if (pix0 >= total) return;
  float v[PIX][K];
#pragma unroll
  for (int q = 0; q < PIX; ++q) {
    const long long pix = pix0 + q < total ? pix0 + q : total - 1;      // a tail thread recomputes the last pixel (not stored)
    const int w = static_cast<int>(pix % W);
    const int h = static_cast<int>((pix / W) % H);
    const int n = static_cast<int>(pix / (static_cast<long long>(W) * H));
#pragma unroll
    for (int ky = 0; ky < 3; ++ky)
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int ih = h + ky - 1, iw = w + kx - 1;
        const bool ok = ih >= 0 && ih < H && iw >= 0 && iw < W;
#pragma unroll
        for (int c = 0; c < CIN; ++c)
          v[q][(ky * 3 + kx) * CIN + c] = ok ? __half2float(x[((static_cast<size_t>(n) * H + ih) * W + iw) * CIN + c]) : 0.0f;
      }
  }
#pragma unroll 1
  for (int cb = 0; cb < 64; cb += 16) {                    // 16 channels = one 32-byte sector per 256-bit store
    float acc[PIX][16];
#pragma unroll
    for (int q = 0; q < PIX; ++q)
#pragma unroll
      for (int j = 0; j < 16; ++j) acc[q][j] = sb[cb + j];
#pragma unroll
    for (int k = 0; k < K; ++k)
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float wv = sw[k * 64 + cb + j];
#pragma unroll
        for (int q = 0; q < PIX; ++q) acc[q][j] = fmaf(v[q][k], wv, acc[q][j]);
      }
#pragma unroll
    for (int q = 0; q < PIX; ++q) {
      if (pix0 + q >= total) break;
      uint32_t pk[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const __half2 h = __floats2half2_rn(fmaxf(acc[q][2 * j], 0.f), fmaxf(acc[q][2 * j + 1], 0.f));
        pk[j] = *reinterpret_cast<const uint32_t*>(&h);
      }
      uint4* o = reinterpret_cast<uint4*>(out + static_cast<size_t>(pix0 + q) * out_ld + cb);
      o[0] = make_uint4(pk[0], pk[1], pk[2], pk[3]);
      o[1] = make_uint4(pk[4], pk[5], pk[6], pk[7]);
    }
  }
}

__device__ __forceinline__ uint4 hmax8(uint4 a, uint4 b) {
  uint4 r;
  __half2* ra = reinterpret_cast<__half2*>(&a);
  __half2* rb = reinterpret_cast<__half2*>(&b);
  __half2* rr = reinterpret_cast<__half2*>(&r);
#pragma unroll
  for (int i = 0; i < 4; ++i) rr[i] = __hmax2(ra[i], rb[i]);
  return r;
}

// 2x2 / stride 2 "valid" max pool, 8 channels per thread.
__global__ void maxpool2_kernel(const __half* __restrict__ in, int in_ld, int N, int H, int W, int C,
                                __half* __restrict__ out, int out_ld) {
  const int OH = H / 2, OW = W / 2, CV = C / 8;
  const long long total = static_cast<long long>(N) * OH * OW * CV;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cv = static_cast<int>(idx % CV);
  const long long op = idx / CV;
  const int ow = static_cast<int>(op % OW);
  const int oh = static_cast<int>((op / OW) % OH);
  const int n = static_cast<int>(op / (static_cast<long long>(OW) * OH));
  const __half* p = in + ((static_cast<size_t>(n) * H + 2 * oh) * W + 2 * ow) * in_ld + cv * 8;
  const uint4 a = *reinterpret_cast<const uint4*>(p);
  const uint4 b = *reinterpret_cast<const uint4*>(p + in_ld);
  const uint4 c = *reinterpret_cast<const uint4*>(p + static_cast<size_t>(W) * in_ld);
  const uint4 d = *reinterpret_cast<const uint4*>(p + static_cast<size_t>(W) * in_ld + in_ld);
  *reinterpret_cast<uint4*>(out + static_cast<size_t>(op) * out_ld + cv * 8) = hmax8(hmax8(a, b), hmax8(c, d));
}

// 3x3 / stride 1 "same" max pool (padding never wins the max).  blockIdx.y walks the images so that the index
// inside one image fits 32 bits (64-bit div/mod was most of this kernel's instructions).
__global__ void __launch_bounds__(256, 4)
maxpool3s1_kernel(const __half* __restrict__ in, int in_ld, int N, int H, int W, int C, __half* __restrict__ out,
                  int out_ld) {
  const unsigned CV = C / 8;
  const unsigned per_image = static_cast<unsigned>(H) * W * CV;
  const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= per_image) return;
  const unsigned cv = idx % CV, op = idx / CV;
  const int w = static_cast<int>(op % W), h = static_cast<int>(op / W);
  for (int n = blockIdx.y; n < N; n += gridDim.y) {
    const __half* src = in + static_cast<size_t>(n) * H * W * in_ld + cv * 8;
    uint4 m = *reinterpret_cast<const uint4*>(src + (static_cast<size_t>(h) * W + w) * in_ld);
    for (int dy = -1; dy <= 1; ++dy)
      for (int dx = -1; dx <= 1; ++dx) {
        const int ih = h + dy, iw = w + dx;
        if (ih < 0 || ih >= H || iw < 0 || iw >= W) continue;
        m = hmax8(m, *reinterpret_cast<const uint4*>(src + (static_cast<size_t>(ih) * W + iw) * in_ld));
      }
    *reinterpret_cast<uint4*>(out + (static_cast<size_t>(n) * H * W + op) * out_ld + cv * 8) = m;
  }
}

// Bilinear resize with half-pixel centres (tf resize_bilinear(half_pixel_centers=True) ==
// torch interpolate(align_corners=False)), written into a channel slice of the concat buffer.
__global__ void upsample_kernel(const __half* __restrict__ in, int in_ld, int N, int IH, int IW, int C,
                                __half* __restrict__ out, int out_ld, int OH, int OW) {
  const int CV = C / 8;
  const long long total = static_cast<long long>(N) * OH * OW * CV;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cv = static_cast<int>(idx % CV);
  const long long op = idx / CV;
  const int ow = static_cast<int>(op % OW);
  const int oh = static_cast<int>((op / OW) % OH);
  const int n = static_cast<int>(op / (static_cast<long long>(OW) * OH));
  const float sh = static_cast<float>(IH) / static_cast<float>(OH);
  const float sw = static_cast<float>(IW) / static_cast<float>(OW);
  float fy = fmaxf((oh + 0.5f) * sh - 0.5f, 0.0f);
  float fx = fmaxf((ow + 0.5f) * sw - 0.5f, 0.0f);
  const int y0 = static_cast<int>(fy), x0 = static_cast<int>(fx);
  const int y1 = min(y0 + 1, IH - 1), x1 = min(x0 + 1, IW - 1);
  const float ly = fy - y0, lx = fx - x0;
  const float hy = 1.0f - ly, hx = 1.0f - lx;
  const __half* base = in + static_cast<size_t>(n) * IH * IW * in_ld + cv * 8;
  const uint4 a = *reinterpret_cast<const uint4*>(base + (static_cast<size_t>(y0) * IW + x0) * in_ld);
  const uint4 b = *reinterpret_cast<const uint4*>(base + (static_cast<size_t>(y0) * IW + x1) * in_ld);
  const uint4 c = *reinterpret_cast<const uint4*>(base + (static_cast<size_t>(y1) * IW + x0) * in_ld);
  const uint4 d = *reinterpret_cast<const uint4*>(base + (static_cast<size_t>(y1) * IW + x1) * in_ld);
  const __half2* pa = reinterpret_cast<const __half2*>(&a);
  const __half2* pb = reinterpret_cast<const __half2*>(&b);
  const __half2* pc = reinterpret_cast<const __half2*>(&c);
  const __half2* pd = reinterpret_cast<const __half2*>(&d);
  uint4 r;
  __half2* pr = reinterpret_cast<__half2*>(&r);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 fa = __half22float2(pa[i]), fb = __half22float2(pb[i]);
    const float2 fc = __half22float2(pc[i]), fd = __half22float2(pd[i]);
    const float vx = hy * (hx * fa.x + lx * fb.x) + ly * (hx * fc.x + lx * fd.x);
    const float vy = hy * (hx * fa.y + lx * fb.y) + ly * (hx * fc.y + lx * fd.y);
    pr[i] = __floats2half2_rn(vx, vy);
  }
  *reinterpret_cast<uint4*>(out + static_cast<size_t>(op) * out_ld + cv * 8) = r;
}

// Exact 2x case (OH == 2*IH, OW == 2*IW; every CRAFT decoder level when the input is a multiple of 32):
// one thread per (quad, 8-channel vector).  Quad (qy, qx) in [0, IH] x [0, IW] sits between input rows
// qy-1 / qy and columns qx-1 / qx (clamped) and produces output rows 2qy-1, 2qy and columns 2qx-1, 2qx
// from ONE set of four loads.  Weights are those of upsample_kernel (0.25 / 0.75, and 0 on the first
// row/column where the source coordinate clamps to 0), and the expression has the same form, so both
// kernels give identical bits.
__global__ void upsample2x_v1_kernel(const __half* __restrict__ in, int in_ld, int N, int IH, int IW, int C,
                                  __half* __restrict__ out, int out_ld) {
  const int CV = C / 8;
  const int QW = IW + 1, QH = IH + 1;
  const long long total = static_cast<long long>(N) * QH * QW * CV;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cv = static_cast<int>(idx % CV);
  const long long q = idx / CV;
  const int qx = static_cast<int>(q % QW);
  const int qy = static_cast<int>((q / QW) % QH);
  const int n = static_cast<int>(q / (static_cast<long long>(QW) * QH));
  const int ya = max(qy - 1, 0), yb = min(qy, IH - 1);
  const int xa = max(qx - 1, 0), xb = min(qx, IW - 1);
  const __half* base = in + static_cast<size_t>(n) * IH * IW * in_ld + cv * 8;
  const uint4 a = *reinterpret_cast<const uint4*>(base + (static_cast<size_t>(ya) * IW + xa) * in_ld);
  const uint4 b = *reinterpret_cast<const uint4*>(base + (static_cast<size_t>(ya) * IW + xb) * in_ld);
  const uint4 c = *reinterpret_cast<const uint4*>(base + (static_cast<size_t>(yb) * IW + xa) * in_ld);
  const uint4 d = *reinterpret_cast<const uint4*>(base + (static_cast<size_t>(yb) * IW + xb) * in_ld);
  const __half2* pa = reinterpret_cast<const __half2*>(&a);
  const __half2* pb = reinterpret_cast<const __half2*>(&b);
  const __half2* pc = reinterpret_cast<const __half2*>(&c);
  const __half2* pd = reinterpret_cast<const __half2*>(&d);
  const int OH = 2 * IH, OW = 2 * IW;
#pragma unroll
  for (int ry = 0; ry < 2; ++ry) {
    const int oh = 2 * qy - 1 + ry;
    if (oh < 0 || oh >= OH) continue;
    const float ly = ry == 0 ? 0.25f : (qy == 0 ? 0.0f : 0.75f), hy = 1.0f - ly;
#pragma unroll
    for (int rx = 0; rx < 2; ++rx) {
      const int ow = 2 * qx - 1 + rx;
      if (ow < 0 || ow >= OW) continue;
      const float lx = rx == 0 ? 0.25f : (qx == 0 ? 0.0f : 0.75f), hx = 1.0f - lx;
      uint4 r;
      __half2* pr = reinterpret_cast<__half2*>(&r);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 fa = __half22float2(pa[i]), fb = __half22float2(pb[i]);
        const float2 fc = __half22float2(pc[i]), fd = __half22float2(pd[i]);
        const float vx = hy * (hx * fa.x + lx * fb.x) + ly * (hx * fc.x + lx * fd.x);
        const float vy = hy * (hx * fa.y + lx * fb.y) + ly * (hx * fc.y + lx * fd.y);
        pr[i] = __floats2half2_rn(vx, vy);
      }
      *reinterpret_cast<uint4*>(out + ((static_cast<size_t>(n) * OH + oh) * OW + ow) * out_ld + cv * 8) = r;
    }
  }
}

// The same quads with a third of the instructions (the v1 kernel is bound by instruction issue, not by memory):
// blockIdx.y walks the images so the decomposition of the index is 32-bit, and the two
// horizontal blends of a quad column (rows ya and yb) are formed once and shared by its two output rows.  Every
// product and sum is the one v1 forms (same operands, same association), so the bits are v1's (B2O_GLUE=v1 A/B test).
__global__ void __launch_bounds__(256, 4)
upsample2x_kernel(const __half* __restrict__ in, int in_ld, int N, int IH, int IW, int C, __half* __restrict__ out,
                  int out_ld) {
  const unsigned CV = C / 8;
  const unsigned QW = IW + 1, QH = IH + 1;
  const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= QH * QW * CV) return;
  const unsigned cv = idx % CV, q = idx / CV;
  const int qx = static_cast<int>(q % QW), qy = static_cast<int>(q / QW);
  const int ya = max(qy - 1, 0), yb = min(qy, IH - 1);
  const int xa = max(qx - 1, 0), xb = min(qx, IW - 1);
  const int OH = 2 * IH, OW = 2 * IW;
  const int oh0 = 2 * qy - 1, ow0 = 2 * qx - 1;
  for (int n = blockIdx.y; n < N; n += gridDim.y) {
    const __half* base = in + static_cast<size_t>(n) * IH * IW * in_ld + cv * 8;
    const uint4 a = *reinterpret_cast<const uint4*>(base + (static_cast<size_t>(ya) * IW + xa) * in_ld);
    const uint4 b = *reinterpret_cast<const uint4*>(base + (static_cast<size_t>(ya) * IW + xb) * in_ld);
    const uint4 c = *reinterpret_cast<const uint4*>(base + (static_cast<size_t>(yb) * IW + xa) * in_ld);
    const uint4 d = *reinterpret_cast<const uint4*>(base + (static_cast<size_t>(yb) * IW + xb) * in_ld);
    float fa[8], fb[8], fc[8], fd[8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 va = __half22float2(reinterpret_cast<const __half2*>(&a)[i]);
      const float2 vb = __half22float2(reinterpret_cast<const __half2*>(&b)[i]);
      const float2 vc = __half22float2(reinterpret_cast<const __half2*>(&c)[i]);
      const float2 vd = __half22float2(reinterpret_cast<const __half2*>(&d)[i]);
      fa[2 * i] = va.x; fa[2 * i + 1] = va.y; fb[2 * i] = vb.x; fb[2 * i + 1] = vb.y;
      fc[2 * i] = vc.x; fc[2 * i + 1] = vc.y; fd[2 * i] = vd.x; fd[2 * i + 1] = vd.y;
    }
    __half* obase = out + static_cast<size_t>(n) * OH * OW * out_ld + cv * 8;
#pragma unroll
    for (int rx = 0; rx < 2; ++rx) {
      const int ow = ow0 + rx;
      if (ow < 0 || ow >= OW) continue;
      const float lx = rx == 0 ? 0.25f : (qx == 0 ? 0.0f : 0.75f), hx = 1.0f - lx;
      float top[8], bot[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        top[i] = hx * fa[i] + lx * fb[i];
        bot[i] = hx * fc[i] + lx * fd[i];
      }
#pragma unroll
      for (int ry = 0; ry < 2; ++ry) {
        const int oh = oh0 + ry;
        if (oh < 0 || oh >= OH) continue;
        const float ly = ry == 0 ? 0.25f : (qy == 0 ? 0.0f : 0.75f), hy = 1.0f - ly;
        uint4 r;
        __half2* pr = reinterpret_cast<__half2*>(&r);
#pragma unroll
        for (int i = 0; i < 4; ++i)
          pr[i] = __floats2half2_rn(hy * top[2 * i] + ly * bot[2 * i], hy * top[2 * i + 1] + ly * bot[2 * i + 1]);
        *reinterpret_cast<uint4*>(obase + (static_cast<size_t>(oh) * OW + ow) * out_ld) = r;
      }
    }
  }
}

// conv_cls.6 (16->16, ReLU) + conv_cls.8 (16->2, linear): fp32 scores (n,h,w,2).
__global__ void __launch_bounds__(256)
head_tail_kernel(const __half* __restrict__ in, int in_ld, long long total, const float* __restrict__ w6 /*[16][16]*/,
                 const float* __restrict__ b6, const float* __restrict__ w8 /*[16][2]*/, const float* __restrict__ b8,
                 float* __restrict__ scores) {
  __shared__ float s6[256], sb6[16], s8[32], sb8[2];
  if (threadIdx.x < 256) s6[threadIdx.x] = w6[threadIdx.x];
  if (threadIdx.x < 16) sb6[threadIdx.x] = b6[threadIdx.x];
  if (threadIdx.x < 32) s8[threadIdx.x] = w8[threadIdx.x];
  if (threadIdx.x < 2) sb8[threadIdx.x] = b8[threadIdx.x];
  __syncthreads();
  const long long pix = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (pix >= total) return;
  const __half* ip = in + static_cast<size_t>(pix) * in_ld;
  float x[16];
  const uint4 r0 = *reinterpret_cast<const uint4*>(ip);
  const uint4 r1 = *reinterpret_cast<const uint4*>(ip + 8);
  const __half2* h0 = reinterpret_cast<const __half2*>(&r0);
  const __half2* h1 = reinterpret_cast<const __half2*>(&r1);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 a = __half22float2(h0[i]), b = __half22float2(h1[i]);
    x[2 * i] = a.x; x[2 * i + 1] = a.y; x[8 + 2 * i] = b.x; x[8 + 2 * i + 1] = b.y;
  }
  float o0 = sb8[0], o1 = sb8[1];
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    float a = sb6[j];
#pragma unroll
    for (int c = 0; c < 16; ++c) a = fmaf(x[c], s6[c * 16 + j], a);
    a = fmaxf(a, 0.0f);                         // kept in fp32 between the two fused layers
    o0 = fmaf(a, s8[j * 2 + 0], o0);
    o1 = fmaf(a, s8[j * 2 + 1], o1);
  }
  reinterpret_cast<float2*>(scores)[pix] = make_float2(o0, o1);
}

inline unsigned blocks_for(long long total, int threads) { return static_cast<unsigned>((total + threads - 1) / threads); }

}  // namespace

int conv_simt_run(b2o_ctx* ctx, const ConvLayer& L, const TensorView& in, const TensorView& out, int out_f32,
                  cudaStream_t st) {
  if (in.c != L.cin || out.c != L.cout || L.cin % 8 != 0 || L.w_simt == nullptr) {
    ctx->set_error("conv_simt_run: unsupported layer " + L.name);
    return B2O_ERR_ARG;
  }
  const long long total = static_cast<long long>(in.n) * in.h * in.w;
  dim3 block(128);
#define B2O_SIMT_LAUNCH(CO)                                                                                   \
  conv_simt_kernel<CO><<<dim3(blocks_for(total, 128), L.cout / CO), block, 0, st>>>(                          \
      in.ptr, in.ld, in.n, in.h, in.w, L.cin, L.w_simt, L.cout, L.ksize, L.dil, L.s1, L.t1, L.s2, L.t2, L.relu, \
      out.ptr, out.ld, out_f32)
  if (L.cout % 16 == 0) B2O_SIMT_LAUNCH(16);
  else if (L.cout % 8 == 0) B2O_SIMT_LAUNCH(8);
  else if (L.cout % 2 == 0) B2O_SIMT_LAUNCH(2);
  else { ctx->set_error("conv_simt_run: odd cout"); return B2O_ERR_ARG; }
#undef B2O_SIMT_LAUNCH
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}

bool conv_pool_fused(const b2o_ctx* ctx, const ConvLayer& L) {
  return ctx->conv_engine == B2O_CONV_AUTO && L.block_n != 0;      // generic tiles and SIMT pool in a kernel of its own
}

int conv_run(b2o_ctx* ctx, const ConvLayer& L, const TensorView& in, const TensorView& out, int out_f32,
             cudaStream_t st, const TensorView* pool_out, int write_full) {
  if (ctx->conv_engine != B2O_CONV_SIMT && L.block_n != 0) {
    if (pool_out != nullptr && !conv_pool_fused(ctx, L)) {      // generic tiles: unfused pool
      B2O_RETURN_IF(conv_tc_run(ctx, L, in, out, out_f32, st));
      return maxpool2_run(ctx, out, *pool_out, st);
    }
    return conv_tc_run(ctx, L, in, out, out_f32, st, pool_out, write_full);
  }
  B2O_RETURN_IF(conv_simt_run(ctx, L, in, out, out_f32, st));
  if (pool_out != nullptr) return maxpool2_run(ctx, out, *pool_out, st);
  return B2O_OK;
}

int stem_rgb_run(b2o_ctx* ctx, const ConvLayer& L, const uint8_t* img, int n, int h, int w, const TensorView& out,
                 cudaStream_t st) {
  const long long total = static_cast<long long>(n) * h * w;
  stem_rgb_kernel<<<blocks_for(total, 128), 128, 0, st>>>(img, n, h, w, L.w_f32, L.s1, L.t1, out.ptr, out.ld);
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}

int normalize16_run(b2o_ctx* ctx, const uint8_t* img, int n, int h, int w, __half* out, cudaStream_t st) {
  const long long total = static_cast<long long>(n) * h * w;
  normalize16_kernel<<<blocks_for(total, 256), 256, 0, st>>>(img, total, out);
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}

int stem_crnn_run(b2o_ctx* ctx, const ConvLayer& L, const __half* x, int b, const TensorView& out, cudaStream_t st) {
  const long long total = static_cast<long long>(b) * out.h * out.w;
  if (L.cin == 3) stem_crnn_kernel<3, 2><<<blocks_for((total + 1) / 2, 128), 128, 0, st>>>(x, b, out.h, out.w, L.w_f32, L.t1, out.ptr, out.ld);
  else stem_crnn_kernel<1, 4><<<blocks_for((total + 3) / 4, 128), 128, 0, st>>>(x, b, out.h, out.w, L.w_f32, L.t1, out.ptr, out.ld);
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}

int maxpool2_run(b2o_ctx* ctx, const TensorView& in, const TensorView& out, cudaStream_t st) {
  const long long total = static_cast<long long>(in.n) * (in.h / 2) * (in.w / 2) * (in.c / 8);
  if (total == 0) return B2O_OK;
  maxpool2_kernel<<<blocks_for(total, 256), 256, 0, st>>>(in.ptr, in.ld, in.n, in.h, in.w, in.c, out.ptr, out.ld);
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}

int maxpool3s1_run(b2o_ctx* ctx, const TensorView& in, const TensorView& out, cudaStream_t st) {
  const long long per_image = static_cast<long long>(in.h) * in.w * (in.c / 8);
  if (per_image == 0 || in.n == 0) return B2O_OK;
  maxpool3s1_kernel<<<dim3(blocks_for(per_image, 256), std::min(in.n, 65535)), 256, 0, st>>>(
      in.ptr, in.ld, in.n, in.h, in.w, in.c, out.ptr, out.ld);
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}

int upsample_run(b2o_ctx* ctx, const TensorView& in, const TensorView& out, cudaStream_t st) {
  if (in.n == 0 || out.h == 0 || out.w == 0) return B2O_OK;
  if (out.h == 2 * in.h && out.w == 2 * in.w) {
    const long long per_image = static_cast<long long>(in.h + 1) * (in.w + 1) * (in.c / 8);
    if (ctx->glue_v1)
      upsample2x_v1_kernel<<<blocks_for(per_image * in.n, 256), 256, 0, st>>>(in.ptr, in.ld, in.n, in.h, in.w, in.c,
                                                                            out.ptr, out.ld);
    else
      upsample2x_kernel<<<dim3(blocks_for(per_image, 256), std::min(in.n, 65535)), 256, 0, st>>>(
          in.ptr, in.ld, in.n, in.h, in.w, in.c, out.ptr, out.ld);
    B2O_LAUNCH_CHECK(ctx);
    return B2O_OK;
  }
  const long long total = static_cast<long long>(out.n) * out.h * out.w * (in.c / 8);
  upsample_kernel<<<blocks_for(total, 256), 256, 0, st>>>(in.ptr, in.ld, in.n, in.h, in.w, in.c, out.ptr, out.ld,
                                                          out.h, out.w);
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}

int head_tail_run(b2o_ctx* ctx, const ConvLayer& L6, const ConvLayer& L8, const TensorView& in, float* scores,
                  cudaStream_t st) {
  const long long total = static_cast<long long>(in.n) * in.h * in.w;
  head_tail_kernel<<<blocks_for(total, 256), 256, 0, st>>>(in.ptr, in.ld, total, L6.w_simt, L6.t1, L8.w_simt, L8.t1,
                                                           scores);
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}
