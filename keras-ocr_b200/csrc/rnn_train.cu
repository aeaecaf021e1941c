// rnn_train.cu -- training the recognizer's BiLSTM (lstm_10, lstm_10_back, lstm_11, lstm_11_back) and fc_12 on frozen
// fc_9 features with Keras ctc_batch_cost (recognition.py:292-349): the forward of the inference network, then
// backpropagation through time in all four directions.
//
// Parameters: one flat fp32 vector, per direction d = 0..3 (lstm_10, lstm_10_back, lstm_11, lstm_11_back) the kernel W
//   (128, 512), the recurrent kernel U (128, 512) and the bias (512) at d * kDirFloats, then fc_12.kernel (256, K) and
//   fc_12.bias (K) at kLstmFloats.  The gradient has the same layout.
//
// Forward, the inference arithmetic (api.cu's crnn_forward after fc_9):
//   pack_kernel       W and U rounded to fp16 from the masters, as b2o_load_crnn packs them.
//   proj_kernel       xw = x W + b per direction: mma.sync m16n8k16 (exact fp16 products, fp32 accumulation; the
//                     reduction order is the MMA's, the same on every call), plus the bias in one fp32 addition.
//   lstm_save_kernel  lstm_kernel's recurrence and gate arithmetic, that also stores per processing step the gate
//                     activations i, f, g = tanh(z_c), o and the cell c in fp32.  h is rounded to fp16 between steps.
//   l1 = fp16(hf + hb) (add_run), both in processing order (the reference's go_backwards quirk, recognition.py:298-319);
//   l2 = [h11f, h11b], again in processing order; fc_12 + CTC on l2's steps 2..49 by ctc_train.cu's kernels, with the
//   dropout mask keyed on the dataset row.
// Backward (rounding to fp16 treated as the identity):
//   l2_grad_kernel    dL/dl2[s] = mask * scale * (g_{s-2} w_fc12^T), 0 for the two discarded steps; g = dL/dlogits.
//   bptt_kernel       one CTA = 8 crops of one direction, 512 threads, s = 49 .. 0:
//                       dh = dh_out[s] + U dz[s+1]  (the recurrent product in fp32 FMAs, U's fp16 values exact in fp32)
//                       dc = dc' + dh o (1 - tanh(c)^2);  dz_o = dh tanh(c) o (1 - o);  dz_i = dc g i (1 - i);
//                       dz_f = dc c_prev f (1 - f);  dz_g = dc i (1 - g^2);  dc' = dc f.
//                     Thread (k, q) keeps U[k][4j + q] (j = 0..127) in registers and sums its quarter of the gates in
//                     ascending j for all 8 crops; the quarters are added by two xor shuffles, a fixed order.
//   dl1_kernel        dL/dl1[t] = dz_11f[t] W_11f^T + dz_11b[49 - t] W_11b^T (lstm_11_back reads l1 reversed), one
//                     serial fp32 FMA chain per element, forward direction first.  Both directions of layer 1 then get
//                     dL/dl1[s] at their processing step s (the quirk: l1[s] = hf[s] + hb[s]).
//   wgrad_partial_kernel / bias_partial_kernel / wgrad_final_kernel: dW = x^T dz, dU = h_prev^T dz, db = sum dz over the
//                     batch's rows in fixed chunks of kChunkCrops crops, each chunk a serial FMA chain in ascending row,
//                     the chunks added in ascending order and divided by B.  No atomics: bit-identical run to run.
#include <math.h>

#include "common.cuh"
#include "ctc_dropout.cuh"
#include "ctc_q.cuh"

using ctcdrop::Dropout;

size_t ctc_train_workspace_bytes(int B, int K);
int ctc_loss_grad_run(b2o_ctx* ctx, const __half* features, long long feat_stride, bool feat_by_batch, int n_rows,
                      const int* index, int B, int K, const float* w, const float* bias, const int* offsets,
                      const short* labels, float rate, uint64_t seed, uint64_t step, float* loss, float* grad_w,
                      float* grad_b, float* logits, void* ws, cudaStream_t st);
int add_run(b2o_ctx* ctx, const __half* a, const __half* b, __half* o, long long n, cudaStream_t st);

namespace {

constexpr int kUnits = 128, kGates = 512, kSteps = 50, kDiscard = 2, kKeep = 48, kL2 = 256;
constexpr int kCropsPerCta = 8;
constexpr int kHPitch = kUnits + 8;
constexpr int kActs = 5;                                          // i, f, g, o, c
constexpr long long kDirFloats = 2LL * kUnits * kGates + kGates;  // 131584
constexpr long long kLstmFloats = 4 * kDirFloats;                 // 526336
constexpr int kChunkCrops = 16;

__device__ __forceinline__ float sigmoidf_acc(float x) { return 1.0f / (1.0f + expf(-x)); }

__device__ __forceinline__ void mma_m16n8k16(float* d, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// w16t[d][n][k] = fp16(W_d[k][n]) (transposed for the MMA's B fragments), u16[d][k][g] = fp16(U_d[k][g]).
__global__ void pack_kernel(const float* __restrict__ params, __half* __restrict__ w16t, __half* __restrict__ u16) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 4 * kUnits * kGates) return;
  const int d = i / (kUnits * kGates), e = i % (kUnits * kGates), k = e / kGates, n = e % kGates;
  const float* p = params + d * kDirFloats;
  w16t[static_cast<size_t>(d) * kUnits * kGates + n * kUnits + k] = __float2half_rn(p[e]);
  u16[i] = __float2half_rn(p[kUnits * kGates + e]);
}

// Where a layer's input rows come from: layer 1 reads row index[b] of the caller's (n_rows, 50, 128) fc_9 cache (a row
// outside [0, n_rows) reads as zeros; the CTC kernel gives that crop NaN), layer 2 the batch's own l1.
struct XRows {
  const __half* x;
  const int* index;     // null: row b
  int n_rows;
  __device__ __forceinline__ const __half* row(int b) const {
    const int r = index ? index[b] : b;
    return (r >= 0 && r < n_rows) ? x + static_cast<size_t>(r) * kSteps * kUnits : nullptr;
  }
};

// xw[d][b*50 + t][n] = sum_k x[b][t][k] W16[k][n] + bias[n] for the two directions d0, d0 + 1 (blockIdx.z).  A CTA of 4
// warps owns 64 rows x 64 columns, a warp 16 rows x 64 columns (8 MMA tiles), k in 8 steps of 16.
__global__ void __launch_bounds__(128) proj_kernel(XRows xr, int B, int d0, const __half* __restrict__ w16t,
                                                   const float* __restrict__ params, float* __restrict__ xw) {
  const int d = d0 + blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, tq = lane & 3;
  const int rows = B * kSteps;
  const int r0 = blockIdx.x * 64 + warp * 16, n0 = blockIdx.y * 64;
  const __half* wt = w16t + static_cast<size_t>(d) * kUnits * kGates;
  auto xrow = [&](int r) -> const __half* {
    if (r >= rows) return nullptr;
    const __half* p = xr.row(r / kSteps);
    return p ? p + (r % kSteps) * kUnits : nullptr;
  };
  const __half* xa = xrow(r0 + g);
  const __half* xb = xrow(r0 + g + 8);
  auto ld2 = [](const __half* p, int k) -> uint32_t { return p ? *reinterpret_cast<const uint32_t*>(p + k) : 0u; };
  float acc[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[j][e] = 0.f;
#pragma unroll
  for (int kt = 0; kt < kUnits / 16; ++kt) {
    const int k0 = kt * 16 + 2 * tq;
    const uint32_t a[4] = {ld2(xa, k0), ld2(xb, k0), ld2(xa, k0 + 8), ld2(xb, k0 + 8)};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const __half* wr = wt + static_cast<size_t>(n0 + j * 8 + g) * kUnits;
      mma_m16n8k16(acc[j], a, *reinterpret_cast<const uint32_t*>(wr + k0), *reinterpret_cast<const uint32_t*>(wr + k0 + 8));
    }
  }
  const float* bias = params + d * kDirFloats + 2 * kUnits * kGates;
  float* out = xw + static_cast<size_t>(d) * rows * kGates;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int n = n0 + j * 8 + 2 * tq;
    const float b0 = bias[n], b1 = bias[n + 1];
    if (r0 + g < rows) {
      out[static_cast<size_t>(r0 + g) * kGates + n] = __fadd_rn(acc[j][0], b0);
      out[static_cast<size_t>(r0 + g) * kGates + n + 1] = __fadd_rn(acc[j][1], b1);
    }
    if (r0 + g + 8 < rows) {
      out[static_cast<size_t>(r0 + g + 8) * kGates + n] = __fadd_rn(acc[j][2], b0);
      out[static_cast<size_t>(r0 + g + 8) * kGates + n + 1] = __fadd_rn(acc[j][3], b1);
    }
  }
}

// Per direction: where its h goes (processing order) and where its gradient dL/dh comes from.
struct DirIO {
  __half* out[2];        // (B, 50, out_ld) fp16 at channel out_off[j]
  int out_ld, out_off[2];
  const float* dh[2];    // (B, 50, dh_ld) fp32 at channel dh_off[j]
  int dh_ld, dh_off[2];
};

// lstm_kernel's recurrence (crnn_tail.cu: the same fragments, MMAs, gate arithmetic and fp16 h) for directions d0, d0 + 1
// (blockIdx.y; odd directions go backwards), that also stores acts[d][b][s][{i, f, g, o, c}][unit] in fp32.  The U^T
// fragments live in shared memory (afs[tile * 8 + kt][thread], 128 kB) rather than in registers: lstm_kernel already
// uses all 128 registers a 512-thread CTA allows, and the stores of the activations need some.
__global__ void __launch_bounds__(kGates, 1)
lstm_save_kernel(const float* __restrict__ xw_all, const __half* __restrict__ u16, int B, int d0, DirIO io,
                 float* __restrict__ acts_all) {
  __shared__ __align__(16) __half h_s[2][kCropsPerCta][kHPitch];
  extern __shared__ __align__(16) uint4 afs[];                       // [16][512]
  const int j = blockIdx.y, d = d0 + j, backwards = d & 1;
  const float* xw = xw_all + static_cast<size_t>(d) * B * kSteps * kGates;
  const __half* u = u16 + static_cast<size_t>(d) * kUnits * kGates;
  float* acts = acts_all + static_cast<size_t>(d) * B * kSteps * kActs * kUnits;
  __half* out = j ? io.out[1] : io.out[0];
  const int out_ld = io.out_ld, out_off = j ? io.out_off[1] : io.out_off[0];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = lane >> 2, q = lane & 3;
  const int unit = warp * 8 + r;
  const int cA = q * 2;
  const int b0 = blockIdx.x * kCropsPerCta;
  const int nb = min(kCropsPerCta, B - b0);

#pragma unroll 1
  for (int tile = 0; tile < 2; ++tile)
#pragma unroll 1
    for (int kt = 0; kt < kUnits / 16; ++kt) {
      const int col_lo = (2 * tile) * kUnits + unit, col_hi = (2 * tile + 1) * kUnits + unit;
      const int k0 = kt * 16 + q * 2;
      auto pack = [&](int k, int col) {
        const __half2 v = __halves2half2(u[k * kGates + col], u[(k + 1) * kGates + col]);
        return *reinterpret_cast<const uint32_t*>(&v);
      };
      afs[(tile * 8 + kt) * kGates + threadIdx.x] = make_uint4(pack(k0, col_lo), pack(k0, col_hi), pack(k0 + 8, col_lo),
                                                               pack(k0 + 8, col_hi));
    }
  for (int i = threadIdx.x; i < 2 * kCropsPerCta * kHPitch; i += blockDim.x) (&h_s[0][0][0])[i] = __float2half_rn(0.0f);

  const bool okA = cA < nb, okB = cA + 1 < nb;
  auto load_x = [&](int t, float* z) {
    const float* pa = xw + (static_cast<size_t>(b0 + cA) * kSteps + t) * kGates + unit;
    const float* pb = pa + static_cast<size_t>(kSteps) * kGates;
#pragma unroll
    for (int gidx = 0; gidx < 4; ++gidx) {
      z[2 * gidx] = okA ? pa[gidx * kUnits] : 0.0f;
      z[2 * gidx + 1] = okB ? pb[gidx * kUnits] : 0.0f;
    }
  };
  float xnext[8];
  load_x(backwards ? kSteps - 1 : 0, xnext);
  float c_state[2] = {0.0f, 0.0f};
  __syncthreads();
  for (int step = 0; step < kSteps; ++step) {
    float d0f[4] = {xnext[0], xnext[1], xnext[2], xnext[3]};
    float d1f[4] = {xnext[4], xnext[5], xnext[6], xnext[7]};
    if (step + 1 < kSteps) load_x(backwards ? (kSteps - 2 - step) : (step + 1), xnext);
    const __half* hrow = &h_s[step & 1][r][q * 2];
#pragma unroll
    for (int kt = 0; kt < kUnits / 16; ++kt) {
      const uint32_t b0r = *reinterpret_cast<const uint32_t*>(hrow + kt * 16);
      const uint32_t b1r = *reinterpret_cast<const uint32_t*>(hrow + kt * 16 + 8);
      const uint4 f0 = afs[kt * kGates + threadIdx.x], f1 = afs[(8 + kt) * kGates + threadIdx.x];
      const uint32_t a0[4] = {f0.x, f0.y, f0.z, f0.w}, a1[4] = {f1.x, f1.y, f1.z, f1.w};
      mma_m16n8k16(d0f, a0, b0r, b1r);
      mma_m16n8k16(d1f, a1, b0r, b1r);
    }
#pragma unroll
    for (int e = 0; e < 2; ++e) {                         // e = 0: crop cA, e = 1: crop cA + 1
      const float zi = d0f[e], zf = d0f[2 + e], zc = d1f[e], zo = d1f[2 + e];
      const float ig = sigmoidf_acc(zi), fg = sigmoidf_acc(zf), gg = tanhf(zc), og = sigmoidf_acc(zo);
      const float c = fg * c_state[e] + ig * gg;
      const __half h = __float2half_rn(og * tanhf(c));
      c_state[e] = c;
      h_s[(step + 1) & 1][cA + e][unit] = h;
      if (cA + e < nb) {
        const size_t row = static_cast<size_t>(b0 + cA + e) * kSteps + step;
        out[row * out_ld + out_off + unit] = h;
        float* a = acts + row * kActs * kUnits + unit;
        a[0] = ig; a[kUnits] = fg; a[2 * kUnits] = gg; a[3 * kUnits] = og; a[4 * kUnits] = c;
      }
    }
    __syncthreads();
  }
}

// dl2[b][s][c] = 0 for s < 2, else mask * scale * sum_k g[b][s-2][k] w[c][k] (serial fmaf chain, ascending k).  One CTA
// per crop, thread c keeps the 48 steps' sums; w and g are staged through shared memory 32 classes at a time.
template <bool DROP>
__global__ void __launch_bounds__(kL2) l2_grad_kernel(const float* __restrict__ g, const float* __restrict__ w, int K,
                                                      const int* __restrict__ index, Dropout drop,
                                                      float* __restrict__ dl2) {
  constexpr int kTk = 32;
  __shared__ float ws_[kL2][kTk + 1];
  __shared__ float gs[kKeep][kTk];
  const int b = blockIdx.x, c = threadIdx.x;
  float acc[kKeep];
#pragma unroll
  for (int t = 0; t < kKeep; ++t) acc[t] = 0.f;
  const float* gb = g + static_cast<size_t>(b) * kKeep * K;
  for (int k0 = 0; k0 < K; k0 += kTk) {
    const int nk = min(kTk, K - k0);
    for (int i = threadIdx.x; i < kL2 * kTk; i += blockDim.x) {
      const int cc = i / kTk, kk = i % kTk;
      ws_[cc][kk] = kk < nk ? w[static_cast<size_t>(cc) * K + k0 + kk] : 0.f;
    }
    for (int i = threadIdx.x; i < kKeep * kTk; i += blockDim.x) {
      const int t = i / kTk, kk = i % kTk;
      gs[t][kk] = kk < nk ? gb[static_cast<size_t>(t) * K + k0 + kk] : 0.f;
    }
    __syncthreads();
    for (int kk = 0; kk < nk; ++kk) {
      const float wv = ws_[c][kk];
#pragma unroll
      for (int t = 0; t < kKeep; ++t) acc[t] = fmaf(gs[t][kk], wv, acc[t]);
    }
    __syncthreads();
  }
  float* o = dl2 + static_cast<size_t>(b) * kSteps * kL2;
  o[c] = 0.f;
  o[kL2 + c] = 0.f;
  const int row = index ? index[b] : b;
#pragma unroll
  for (int t = 0; t < kKeep; ++t) {
    float v = acc[t];
    if (DROP) v = ctcdrop::kept(drop, row, t, c) ? __fmul_rn(v, drop.scale) : 0.f;
    o[(kDiscard + t) * kL2 + c] = v;
  }
}

// Backpropagation through time for directions d0, d0 + 1 (blockIdx.y), 8 crops per CTA.  dz[d][b][s][gate*128 + k]
// (processing step s) is written over the direction's xw, which the backward no longer needs.
__global__ void __launch_bounds__(kGates, 1)
bptt_kernel(const float* __restrict__ acts_all, const __half* __restrict__ u16, int B, int d0, DirIO io,
            float* __restrict__ dz_all) {
  __shared__ __align__(16) float dz_s[2][kGates][kCropsPerCta];    // [buffer][gate][crop]
  extern __shared__ __align__(16) __half2 us[];                     // [64][512]: thread t's U pairs at us[jj * 512 + t]
  const int j = blockIdx.y, d = d0 + j;
  const float* acts = acts_all + static_cast<size_t>(d) * B * kSteps * kActs * kUnits;
  const __half* u = u16 + static_cast<size_t>(d) * kUnits * kGates;
  float* dz = dz_all + static_cast<size_t>(d) * B * kSteps * kGates;
  const float* dh_out = j ? io.dh[1] : io.dh[0];
  const int dh_ld = io.dh_ld, dh_off = j ? io.dh_off[1] : io.dh_off[0];
  const int k = threadIdx.x >> 2, q = threadIdx.x & 3;
  const int b0 = blockIdx.x * kCropsPerCta;
  const int nb = min(kCropsPerCta, B - b0);
  // U[k][4j + q], j = 0..127, as 64 half2 (j even, j odd) in this thread's column of `us`
#pragma unroll 1
  for (int jj = 0; jj < 64; ++jj)
    us[jj * kGates + threadIdx.x] = __halves2half2(u[k * kGates + 4 * (2 * jj) + q], u[k * kGates + 4 * (2 * jj + 1) + q]);
  for (int i = threadIdx.x; i < kGates * kCropsPerCta; i += blockDim.x) (&dz_s[1][0][0])[i] = 0.f;
  const int e0 = 2 * q;                                           // this thread's crops e0, e0 + 1 (unit k)
  float dc_next[2] = {0.f, 0.f};
  __syncthreads();
  for (int s = kSteps - 1; s >= 0; --s) {
    const int cur = s & 1, nxt = cur ^ 1;                         // dz of step s + 1 is in dz_s[nxt]
    float rec[kCropsPerCta];
#pragma unroll
    for (int e = 0; e < kCropsPerCta; ++e) rec[e] = 0.f;
    if (s < kSteps - 1) {
#pragma unroll 4
      for (int jj = 0; jj < 64; ++jj) {
        const float2 uf = __half22float2(us[jj * kGates + threadIdx.x]);
        const float4* p0 = reinterpret_cast<const float4*>(&dz_s[nxt][4 * (2 * jj) + q][0]);
        const float4* p1 = reinterpret_cast<const float4*>(&dz_s[nxt][4 * (2 * jj + 1) + q][0]);
        const float4 a0 = p0[0], a1 = p0[1], c0 = p1[0], c1 = p1[1];
        rec[0] = fmaf(uf.x, a0.x, rec[0]); rec[1] = fmaf(uf.x, a0.y, rec[1]);
        rec[2] = fmaf(uf.x, a0.z, rec[2]); rec[3] = fmaf(uf.x, a0.w, rec[3]);
        rec[4] = fmaf(uf.x, a1.x, rec[4]); rec[5] = fmaf(uf.x, a1.y, rec[5]);
        rec[6] = fmaf(uf.x, a1.z, rec[6]); rec[7] = fmaf(uf.x, a1.w, rec[7]);
        rec[0] = fmaf(uf.y, c0.x, rec[0]); rec[1] = fmaf(uf.y, c0.y, rec[1]);
        rec[2] = fmaf(uf.y, c0.z, rec[2]); rec[3] = fmaf(uf.y, c0.w, rec[3]);
        rec[4] = fmaf(uf.y, c1.x, rec[4]); rec[5] = fmaf(uf.y, c1.y, rec[5]);
        rec[6] = fmaf(uf.y, c1.z, rec[6]); rec[7] = fmaf(uf.y, c1.w, rec[7]);
      }
#pragma unroll
      for (int e = 0; e < kCropsPerCta; ++e) {                   // (p0 + p1) + (p2 + p3) in every lane of the quad
        rec[e] = __fadd_rn(rec[e], __shfl_xor_sync(0xffffffffu, rec[e], 1));
        rec[e] = __fadd_rn(rec[e], __shfl_xor_sync(0xffffffffu, rec[e], 2));
      }
    }
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int cr = e0 + e;
      float zi = 0.f, zf = 0.f, zg = 0.f, zo = 0.f;
      if (cr < nb) {
        const size_t row = static_cast<size_t>(b0 + cr) * kSteps + s;
        const float* a = acts + row * kActs * kUnits + k;
        const float ig = a[0], fg = a[kUnits], gg = a[2 * kUnits], og = a[3 * kUnits], c = a[4 * kUnits];
        const float cp = s > 0 ? a[4 * kUnits - kActs * kUnits] : 0.f;
        const float rv = cr == 0 ? rec[0] : cr == 1 ? rec[1] : cr == 2 ? rec[2] : cr == 3 ? rec[3]
                       : cr == 4 ? rec[4] : cr == 5 ? rec[5] : cr == 6 ? rec[6] : rec[7];
        const float dh = __fadd_rn(dh_out[row * dh_ld + dh_off + k], rv);
        const float tc = tanhf(c);
        const float dc = fmaf(__fmul_rn(dh, og), fmaf(-tc, tc, 1.f), dc_next[e]);
        zo = __fmul_rn(__fmul_rn(dh, tc), __fmul_rn(og, __fsub_rn(1.f, og)));
        zi = __fmul_rn(__fmul_rn(dc, gg), __fmul_rn(ig, __fsub_rn(1.f, ig)));
        zf = __fmul_rn(__fmul_rn(dc, cp), __fmul_rn(fg, __fsub_rn(1.f, fg)));
        zg = __fmul_rn(__fmul_rn(dc, ig), fmaf(-gg, gg, 1.f));
        dc_next[e] = __fmul_rn(dc, fg);
        float* o = dz + row * kGates + k;
        o[0] = zi; o[kUnits] = zf; o[2 * kUnits] = zg; o[3 * kUnits] = zo;
      }
      dz_s[cur][k][cr] = zi;
      dz_s[cur][kUnits + k][cr] = zf;
      dz_s[cur][2 * kUnits + k][cr] = zg;
      dz_s[cur][3 * kUnits + k][cr] = zo;
    }
    __syncthreads();
  }
}

// dl1[b][t][m] = sum_n dz_2[b][t][n] W16_2[m][n], then + sum_n dz_3[b][49-t][n] W16_3[m][n]: one serial fmaf chain per
// element.  A CTA owns 32 rows x 128 outputs, a thread 4 rows x 4 outputs; 64 gates staged per round.
__global__ void __launch_bounds__(256) dl1_kernel(const float* __restrict__ dz_all, const __half* __restrict__ w16t,
                                                  int B, float* __restrict__ dl1) {
  constexpr int kR = 32, kN = 64;
  __shared__ float zs[kR][kN + 1];
  __shared__ float wsh[kN][kUnits + 4];
  const int rows = B * kSteps, r0 = blockIdx.x * kR;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;         // outputs m = tx + 32 i, rows ty + 8 j
  float acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[a][c] = 0.f;
  for (int dd = 2; dd < 4; ++dd) {
    const float* dz = dz_all + static_cast<size_t>(dd) * rows * kGates;
    const __half* wt = w16t + static_cast<size_t>(dd) * kUnits * kGates;   // [n][m]
    for (int n0 = 0; n0 < kGates; n0 += kN) {
      for (int i = threadIdx.x; i < kR * kN; i += blockDim.x) {
        const int rr = i / kN, nn = i % kN, r = r0 + rr;
        float v = 0.f;
        if (r < rows) {
          const int b = r / kSteps, t = r % kSteps, s = dd == 2 ? t : kSteps - 1 - t;
          v = dz[(static_cast<size_t>(b) * kSteps + s) * kGates + n0 + nn];
        }
        zs[rr][nn] = v;
      }
      for (int i = threadIdx.x; i < kN * kUnits; i += blockDim.x) {
        const int nn = i / kUnits, m = i % kUnits;
        wsh[nn][m] = __half2float(wt[static_cast<size_t>(n0 + nn) * kUnits + m]);
      }
      __syncthreads();
      for (int nn = 0; nn < kN; ++nn) {
        float wv[4], zv[4];
#pragma unroll
        for (int a = 0; a < 4; ++a) { wv[a] = wsh[nn][tx + 32 * a]; zv[a] = zs[ty + 8 * a][nn]; }
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
          for (int c = 0; c < 4; ++c) acc[a][c] = fmaf(zv[a], wv[c], acc[a][c]);
      }
      __syncthreads();
    }
  }
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const int r = r0 + ty + 8 * a;
    if (r < rows)
#pragma unroll
      for (int c = 0; c < 4; ++c) dl1[static_cast<size_t>(r) * kUnits + tx + 32 * c] = acc[a][c];
  }
}

// The inputs of direction d's weight gradients at processing step s of crop b: x (the layer input the step read) and
// h_prev (the direction's output one step earlier, 0 at s = 0), both fp16 rows of 128.
struct GradIn {
  XRows x;               // layer 1: the fc_9 cache; layer 2: l1 (index null)
  const __half* h[2];    // (B, 50, h_ld) at channel h_off[j]
  int h_ld, h_off[2];
};

// partial[chunk][d * kDirFloats + which * 65536 + m * 512 + n] = sum over the chunk's rows r = (b, s), ascending, of
// A_which(r)[m] dz[r][n] with A_0 = x at input time (s, or 49 - s going backwards), A_1 = h_prev.  blockIdx.y =
// (j * 2 + which) * 2 + m-tile, blockIdx.x = n-tile, blockIdx.z = chunk.
__global__ void __launch_bounds__(256) wgrad_partial_kernel(GradIn gi, const float* __restrict__ dz_all, int B, int d0,
                                                            float* __restrict__ partial) {
  constexpr int kTile = 64, kSub = 32;
  __shared__ float as[kSub][kTile], zs[kSub][kTile];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int mt = blockIdx.y & 1, which = (blockIdx.y >> 1) & 1, j = blockIdx.y >> 2, d = d0 + j;
  const int n0 = blockIdx.x * kTile, m0 = mt * kTile, chunk = blockIdx.z;
  const int rows = B * kSteps;
  const int r_begin = chunk * kChunkCrops * kSteps, r_end = min(rows, r_begin + kChunkCrops * kSteps);
  const float* dz = dz_all + static_cast<size_t>(d) * rows * kGates;
  float acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[a][c] = 0.f;
  for (int r0 = r_begin; r0 < r_end; r0 += kSub) {
    for (int e = threadIdx.x; e < kSub * kTile; e += 256) {
      const int rr = e / kTile, cc = e % kTile, r = r0 + rr;
      float av = 0.f, zv = 0.f;
      if (r < r_end) {
        const int b = r / kSteps, s = r % kSteps;
        if (which == 0) {
          const __half* xr = gi.x.row(b);
          const int t = (d & 1) ? kSteps - 1 - s : s;
          if (xr) av = __half2float(xr[t * kUnits + m0 + cc]);
        } else if (s > 0) {
          const __half* h = j ? gi.h[1] : gi.h[0];
          av = __half2float(h[(static_cast<size_t>(b) * kSteps + s - 1) * gi.h_ld + (j ? gi.h_off[1] : gi.h_off[0]) + m0 + cc]);
        }
        zv = dz[static_cast<size_t>(r) * kGates + n0 + cc];
      }
      as[rr][cc] = av;
      zs[rr][cc] = zv;
    }
    __syncthreads();
    const int n = min(kSub, r_end - r0);
    for (int rr = 0; rr < n; ++rr) {
      float av[4], zv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { av[i] = as[rr][ty * 4 + i]; zv[i] = zs[rr][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[i][c] = fmaf(av[i], zv[c], acc[i][c]);
    }
    __syncthreads();
  }
  float* out = partial + static_cast<size_t>(chunk) * kLstmFloats + d * kDirFloats + which * kUnits * kGates;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int c = 0; c < 4; ++c) out[static_cast<size_t>(m0 + ty * 4 + i) * kGates + n0 + tx * 4 + c] = acc[i][c];
}

// partial[chunk][d * kDirFloats + 2 * 65536 + n] = sum over the chunk's rows (ascending) of dz[r][n].
__global__ void bias_partial_kernel(const float* __restrict__ dz_all, int B, int d0, float* __restrict__ partial) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x, d = d0 + blockIdx.y, chunk = blockIdx.z;
  const int rows = B * kSteps;
  const int r_begin = chunk * kChunkCrops * kSteps, r_end = min(rows, r_begin + kChunkCrops * kSteps);
  const float* dz = dz_all + static_cast<size_t>(d) * rows * kGates;
  float s = 0.f;
  for (int r = r_begin; r < r_end; ++r) s = __fadd_rn(s, dz[static_cast<size_t>(r) * kGates + n]);
  partial[static_cast<size_t>(chunk) * kLstmFloats + d * kDirFloats + 2 * kUnits * kGates + n] = s;
}

// grad[e] = (sum over chunks, ascending, of partial[chunk][e]) / B for the 526,336 LSTM entries.
__global__ void wgrad_final_kernel(const float* __restrict__ partial, int chunks, int B, float* __restrict__ grad) {
  const long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (e >= kLstmFloats) return;
  float s = 0.f;
  for (int ch = 0; ch < chunks; ++ch) s = __fadd_rn(s, partial[static_cast<size_t>(ch) * kLstmFloats + e]);
  grad[e] = __fdiv_rn(s, static_cast<float>(B));
}

size_t align256(size_t x) { return (x + 255) / 256 * 256; }
int chunks_of(int B) { return (B + kChunkCrops - 1) / kChunkCrops; }

// The workspace, slot after slot, each 256-byte aligned (the sizes are per batch of B crops):
enum Slot { kW16, kU16, kXz, kActsSlot, kH1, kL1, kL2Slot, kDl2, kDl1, kPartial, kCtc, kSlots };
struct RnnPlan {
  size_t off[kSlots + 1];
};
RnnPlan plan_rnn(int B, int K) {
  const size_t rows = static_cast<size_t>(B) * kSteps;
  const size_t bytes[kSlots] = {
      4ull * kUnits * kGates * 2,              // w16t  [4][512][128] fp16
      4ull * kUnits * kGates * 2,              // u16   [4][128][512] fp16
      4ull * rows * kGates * 4,                // xw, then dz: [4][B][50][512] fp32
      4ull * rows * kActs * kUnits * 4,        // acts  [4][B][50][5][128] fp32 (i, f, g, o, c)
      2ull * rows * kUnits * 2,                // hf, hb [2][B][50][128] fp16
      rows * kUnits * 2,                       // l1    [B][50][128] fp16
      rows * kL2 * 2,                          // l2    [B][50][256] fp16
      rows * kL2 * 4,                          // dl2   [B][50][256] fp32
      rows * kUnits * 4,                       // dl1   [B][50][128] fp32
      static_cast<size_t>(chunks_of(B)) * kLstmFloats * 4,
      ctc_train_workspace_bytes(B, K)};
  RnnPlan p;
  size_t off = 0;
  for (int i = 0; i < kSlots; ++i) { p.off[i] = off; off += align256(bytes[i]); }
  p.off[kSlots] = off;
  return p;
}

}  // namespace

size_t rnn_train_workspace_bytes(int B, int K) { return plan_rnn(B, K).off[kSlots]; }
size_t rnn_train_acts_offset(int B, int K) { return plan_rnn(B, K).off[kActsSlot]; }

int rnn_loss_grad_run(b2o_ctx* ctx, const __half* x, int n_rows, const int* index, int B, int K, const float* params,
                      const int* offsets, const short* labels, float rate, uint64_t seed, uint64_t step, float* loss,
                      float* grad, void* ws, cudaStream_t st) {
  const RnnPlan p = plan_rnn(B, K);
  uint8_t* base = reinterpret_cast<uint8_t*>(ws);
  __half* w16t = reinterpret_cast<__half*>(base + p.off[kW16]);
  __half* u16 = reinterpret_cast<__half*>(base + p.off[kU16]);
  float* xz = reinterpret_cast<float*>(base + p.off[kXz]);
  float* acts = reinterpret_cast<float*>(base + p.off[kActsSlot]);
  __half* h1 = reinterpret_cast<__half*>(base + p.off[kH1]);
  __half* l1 = reinterpret_cast<__half*>(base + p.off[kL1]);
  __half* l2 = reinterpret_cast<__half*>(base + p.off[kL2Slot]);
  float* dl2 = reinterpret_cast<float*>(base + p.off[kDl2]);
  float* dl1 = reinterpret_cast<float*>(base + p.off[kDl1]);
  float* partial = reinterpret_cast<float*>(base + p.off[kPartial]);
  void* ctc_ws = base + p.off[kCtc];
  const size_t rows = static_cast<size_t>(B) * kSteps;
  const float* fc_w = params + kLstmFloats;
  const float* fc_b = fc_w + static_cast<size_t>(kL2) * K;
  const XRows x1 = {x, index, n_rows}, x2 = {l1, nullptr, B};
  DirIO io1 = {{h1, h1 + rows * kUnits}, kUnits, {0, 0}, {dl1, dl1}, kUnits, {0, 0}};
  DirIO io2 = {{l2, l2}, kL2, {0, kUnits}, {dl2, dl2}, kL2, {0, kUnits}};
  const dim3 proj_grid((static_cast<unsigned>(rows) + 63) / 64, kGates / 64, 2);
  const dim3 rec_grid((B + kCropsPerCta - 1) / kCropsPerCta, 2);
  // ---- forward
  pack_kernel<<<4 * kUnits * kGates / 256, 256, 0, st>>>(params, w16t, u16);
  B2O_LAUNCH_CHECK(ctx);
  proj_kernel<<<proj_grid, 128, 0, st>>>(x1, B, 0, w16t, params, xz);
  B2O_LAUNCH_CHECK(ctx);
  constexpr int kFragSmem = 16 * kGates * 16;
  B2O_CUDA_CHECK(ctx, cudaFuncSetAttribute(lstm_save_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kFragSmem));
  lstm_save_kernel<<<rec_grid, kGates, kFragSmem, st>>>(xz, u16, B, 0, io1, acts);
  B2O_LAUNCH_CHECK(ctx);
  B2O_RETURN_IF(add_run(ctx, h1, h1 + rows * kUnits, l1, static_cast<long long>(rows) * kUnits, st));
  proj_kernel<<<proj_grid, 128, 0, st>>>(x2, B, 2, w16t, params, xz);
  B2O_LAUNCH_CHECK(ctx);
  lstm_save_kernel<<<rec_grid, kGates, kFragSmem, st>>>(xz, u16, B, 2, io2, acts);
  B2O_LAUNCH_CHECK(ctx);
  // ---- fc_12 + CTC on l2's kept steps (and, with grad, fc_12's gradients and g = dL/dlogits in the CTC workspace)
  float* grad_w = grad ? grad + kLstmFloats : nullptr;
  float* grad_b = grad ? grad_w + static_cast<size_t>(kL2) * K : nullptr;
  B2O_RETURN_IF(ctc_loss_grad_run(ctx, l2 + kDiscard * kL2, static_cast<long long>(kSteps) * kL2, true, n_rows, index, B,
                                  K, fc_w, fc_b, offsets, labels, rate, seed, step, loss, grad_w, grad_b, nullptr,
                                  ctc_ws, st));
  if (!grad) return B2O_OK;
  // ---- backward
  const Dropout d = ctcdrop::make_dropout(rate, seed, step);
  const float* g = reinterpret_cast<const float*>(ctc_ws);      // ctc_train.cu's workspace starts with g (B, 48, K)
  if (d.on) l2_grad_kernel<true><<<B, kL2, 0, st>>>(g, fc_w, K, index, d, dl2);
  else l2_grad_kernel<false><<<B, kL2, 0, st>>>(g, fc_w, K, index, d, dl2);
  B2O_LAUNCH_CHECK(ctx);
  constexpr int kBpttSmem = 64 * kGates * 4;
  B2O_CUDA_CHECK(ctx, cudaFuncSetAttribute(bptt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kBpttSmem));
  bptt_kernel<<<rec_grid, kGates, kBpttSmem, st>>>(acts, u16, B, 2, io2, xz);
  B2O_LAUNCH_CHECK(ctx);
  dl1_kernel<<<(static_cast<unsigned>(rows) + 31) / 32, 256, 0, st>>>(xz, w16t, B, dl1);
  B2O_LAUNCH_CHECK(ctx);
  bptt_kernel<<<rec_grid, kGates, kBpttSmem, st>>>(acts, u16, B, 0, io1, xz);
  B2O_LAUNCH_CHECK(ctx);
  const int nch = chunks_of(B);
  const GradIn g1 = {x1, {h1, h1 + rows * kUnits}, kUnits, {0, 0}};
  const GradIn g2 = {x2, {l2, l2}, kL2, {0, kUnits}};
  for (int layer = 0; layer < 2; ++layer) {
    const int d0 = 2 * layer;
    wgrad_partial_kernel<<<dim3(kGates / 64, 8, nch), 256, 0, st>>>(layer ? g2 : g1, xz, B, d0, partial);
    B2O_LAUNCH_CHECK(ctx);
    bias_partial_kernel<<<dim3(kGates / 128, 2, nch), 128, 0, st>>>(xz, B, d0, partial);
    B2O_LAUNCH_CHECK(ctx);
  }
  wgrad_final_kernel<<<static_cast<unsigned>((kLstmFloats + 255) / 256), 256, 0, st>>>(partial, nch, B, grad);
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}
