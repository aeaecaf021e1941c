// Shared declarations for the b2ocr CUDA library (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <map>
#include <set>
#include <string>
#include <vector>

#include "../../include/b2ocr.h"

#define B2O_CUDA_CHECK(ctx, expr)                                                              \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess) {                                                                   \
      (ctx)->set_error(std::string(#expr) + ": " + cudaGetErrorString(_e));                    \
      return B2O_ERR_CUDA;                                                                     \
    }                                                                                          \
  } while (0)

#define B2O_LAUNCH_CHECK(ctx)                                                                  \
  do {                                                                                         \
    (ctx)->launches++;                                                                         \
    cudaError_t _e = cudaGetLastError();                                                       \
    if (_e != cudaSuccess) {                                                                   \
      (ctx)->set_error(std::string(__FILE__) + ":" + std::to_string(__LINE__) + " launch: " +  \
                       cudaGetErrorString(_e));                                                \
      return B2O_ERR_CUDA;                                                                     \
    }                                                                                          \
  } while (0)

// Every entry point that touches the device runs with the context's device current and puts the caller's device
// back on return (the caller -- torch -- may be driving another GPU of the box in the same process).
struct DeviceGuard {
  int prev = -1;
  bool changed = false;
  explicit DeviceGuard(int device) {
    if (cudaGetDevice(&prev) == cudaSuccess && prev != device) changed = cudaSetDevice(device) == cudaSuccess;
  }
  ~DeviceGuard() {
    if (changed) cudaSetDevice(prev);
  }
  DeviceGuard(const DeviceGuard&) = delete;
  DeviceGuard& operator=(const DeviceGuard&) = delete;
};

#define B2O_RETURN_IF(expr)                                                                    \
  do {                                                                                         \
    int _s = (expr);                                                                           \
    if (_s != B2O_OK) return _s;                                                               \
  } while (0)

// Epilogue applied by every convolution / dense kernel, per output channel n:
//   y = acc * s1[n] + t1[n];  if (relu) y = max(y, 0);  if (s2) y = y * s2[n] + t2[n]
// CRAFT conv+BN(+ReLU): s1 = gamma/sqrt(var+eps), t1 = (bias-mean)*s1+beta   (detection.py:87-103)
// CRNN  conv+ReLU+BN  : s1 = 1, t1 = bias, relu, s2 = gamma/sqrt(var+eps), t2 = beta-mean*s2
//                       (recognition.py:223-242 -- BN comes AFTER the ReLU there)
struct ConvLayer {
  std::string name;
  int cin = 0, cout = 0, ksize = 1, dil = 1, relu = 0;
  __half* w_kmajor = nullptr;  // [cout][taps*cin] fp16, K index = tap*cin + c   (wgmma B operand)
  float* w_simt = nullptr;     // [taps][cin][cout] fp32 holding the fp16-rounded values (SIMT engine)
  float* w_f32 = nullptr;      // [taps][cin][cout] fp32 (only for the 3-channel / 1-channel stems)
  float *s1 = nullptr, *t1 = nullptr, *s2 = nullptr, *t2 = nullptr;
  std::vector<float> h_w_f32;                  // host copy of w_f32 (the 1- / 3-channel CRNN stem: kernel-parameter filter bank)
  std::vector<float> h_w_simt;                 // host copy of w_simt for layers of <= 1024 weights (fused into other kernels' parameters)
  std::vector<float> h_s1, h_t1, h_s2, h_t2;   // host copies: passed to the tensor-core kernel as a kernel parameter (constant bank)
  CUtensorMap wmap;            // TMA map over w_kmajor (box kch x block_n)
  CUtensorMap wmap_pair;       // the same with box kch x block_n/2: the half of a B tile one CTA of a pair fetches
  bool pair_ok = false;        // wmap_pair is valid (64-channel chunks, block_n >= 64)
  int block_n = 0;             // tensor-core N tile; 0 = layer not eligible for the tensor-core engine
  int kch = 0;                 // tensor-core K chunk (channels per stage): 64 / 32 / 16
  // channels of the layer the reference defines, where the tensor-core form pads them (3 -> 16 input channels of the
  // CRAFT stem, 400 -> 512 columns of the STN GEMM): what the roofline's algorithmic FLOP count uses.  0 = cin / cout.
  int alg_cin = 0, alg_cout = 0;
};

struct TensorView {            // NHWC fp16 activation living inside a (possibly wider) buffer
  __half* ptr = nullptr;       // address of channel 0 of the slice
  int n = 0, h = 0, w = 0, c = 0;
  int ld = 0;                  // channel stride of the underlying buffer (elements)
};

struct b2o_ctx {
  int device = 0;
  int sm_count = 132;
  int conv_engine = B2O_CONV_AUTO;
  // CTA pairs (2-CTA clusters sharing B tiles by TMA multicast), opt-in with B2O_TC_PAIR=1 (halo-tile layers) or 2 (all
  // eligible layers): bit-identical, but measured slower on H100 (bench: 141 against 202 img/s, 700 W H100 80GB HBM3)
  bool tc_pair = false;
  bool tc_pair_generic = false;   // B2O_TC_PAIR=2: also pair the generic tiles (1x1 / dilated layers)
  // Decoder glue: B2O_UPCONV_COMMUTE=1 commutes the 2x upsampling behind the decoder half of upconvN.conv.0 (low-res GEMM +
  // upsample-add in the full-resolution layer's epilogue).  Numerically validated; opt-in.  Default: explicit UpsampleLike
  // kernels, as the reference graph has them.
  bool tc_aff_const = true;    // epilogue constants as a kernel parameter (constant cache); B2O_TC_AFF=smem: staging in shared memory / global loads
  bool no_commute = true;
  bool glue_v1 = false;        // B2O_GLUE=v1: the round-1 upsample2x kernel (64-bit index chain, unshared blends) for A/B runs and the bit-identity test
  bool no_fused_tail = false;  // B2O_FUSED_TAIL=0: conv_cls.6/.8 as the separate head_tail_kernel instead of conv_cls.4's epilogue
  bool tc_swap = true;         // 64-channel fp16 layers, and the streamed 128-channel halo layers on 16 x 16 tiles, as channels x
                               // pixels GEMMs (bit-identical); B2O_TC_SWAP=0: pixels x channels
  int64_t tc_tile256_launches = 0;   // conv launches that took the 16 x 16-tile channels-by-pixels body (b2o_tc_tile256_launches)
  int64_t tc_coop_n_launches = 0;    // conv launches that ran paired n-tiles (b2o_tc_coop_n_launches)
  std::set<const void*> configured;   // kernels whose per-device launch attributes are set on this device
  int64_t launches = 0;
  std::string error;
  std::map<std::string, ConvLayer> craft, crnn;
  bool craft_loaded = false, crnn_loaded = false;
  int crnn_in_ch = 1;              // 1 = gray crops (default), 3 = RGB crops (build_model(color=True))
  bool crnn_stn = true;            // the loaded CRNN has a spatial transformer (build_model(stn=True), the default)
  bool quads_configured = false;   // quads_kernel's dynamic shared-memory opt-in done on this device
  // CRNN tail parameters (device)
  float *stn_d2_w = nullptr, *stn_d2_b = nullptr;              // dense 64 -> 6, fp32
  __half* lstm_u[4] = {nullptr, nullptr, nullptr, nullptr};    // recurrent kernels [128][512] fp16
  float *fc12_w = nullptr, *fc12_b = nullptr;                  // [256][K], [K] fp32, K = len(alphabet) + 1
  int n_classes = 37;                                          // K (last index = CTC blank), <= B2O_MAX_CLASSES
  std::vector<void*> owned;    // device allocations freed in b2o_destroy
  b2o_char_lm zero_lm{};       // hotwords without a model: order 2, one empty-history row of zeros (uploaded on first use)
  // optional per-launch timing of the tensor-core conv kernel (bench.py's roofline leg)
  bool debug_taps = false;     // b2o_set_debug_taps: the CRNN forward also writes its fp32 logits (tests only)
  int craft_step = -1;         // last step of the most recent successful CRAFT forward (b2o_craft_tap), -1: none
  const void* craft_ws = nullptr;   // ... and its workspace and input shape, which b2o_craft_tap must be given again
  int craft_n = 0, craft_h = 0, craft_w = 0;
  // the most recent successful CRNN forward (b2o_crnn_tap, b2o_crnn_align): its workspace and batch, and bit i set for
  // every workspace slot rb::i (api.cu) it wrote; 0: none since creation, or the last forward failed after it started
  const void* crnn_ws = nullptr;
  int crnn_b = 0;
  uint32_t crnn_written = 0;
  bool profile = false;
  std::vector<cudaEvent_t> prof_events;   // (start, stop) pairs
  double prof_flop = 0.0;
  void* jpeg = nullptr;        // nvJPEG handle + state, created on first use (jpeg.cu)
  bool jpeg_failed = false;    // nvJPEG could not be opened on this box: do not try again
  void set_error(const std::string& e) { error = e; }
};
void jpeg_release(b2o_ctx* ctx);

// CRAFT tail fused into the epilogue of a 16-channel tensor-core layer: conv_cls.6 (1x1 16->16, ReLU) and conv_cls.8
// (1x1 16->2) on the 16 channels a thread already holds; fp32 (text, link) scores out (detection.py:404-410).
struct ConvTail {
  const float *w6, *b6, *w8, *b8;   // [cin 16][cout 16] fp32 (fp16-rounded values), [16], [16][2], [2] -- device
  float* scores;                    // (n,h,w,2)
  const float *h_w6 = nullptr, *h_b6 = nullptr, *h_w8 = nullptr, *h_b8 = nullptr;   // the same on the host (kernel-parameter path)
};

// ---- engines (conv_tc.cu, conv_simt.cu) -------------------------------------------------------
int conv_tc_prepare(b2o_ctx* ctx, ConvLayer& L);   // builds wmap / picks block_n (0 if ineligible)
// pool_out != null: also write the 2x2/2 max-pooled output (fused epilogue); write_full = 0 skips `out`
int conv_tc_run(b2o_ctx* ctx, const ConvLayer& L, const TensorView& in, const TensorView& out,
                int out_f32, cudaStream_t st, const TensorView* pool_out = nullptr, int write_full = 1,
                const ConvTail* tail = nullptr, const TensorView* up_add = nullptr);
// up_add (1x1 layers, 64-channel chunks): a (n, h/2, w/2, cout) fp16 tensor whose exact-2x bilinear upsampling is added to
// the accumulator before the affine/ReLU -- the decoder's UpsampleLike + Concatenate + 1x1 conv with the upsampling
// commuted behind the (linear) convolution of the low-resolution half (detection.py:290-309, 380-390)
int conv_simt_run(b2o_ctx* ctx, const ConvLayer& L, const TensorView& in, const TensorView& out,
                  int out_f32, cudaStream_t st);
int conv_run(b2o_ctx* ctx, const ConvLayer& L, const TensorView& in, const TensorView& out,
             int out_f32, cudaStream_t st, const TensorView* pool_out = nullptr, int write_full = 1);
// conv_run of L with a pool_out fuses the pool into the convolution (then write_full = 0 leaves `out` unwritten)
bool conv_pool_fused(const b2o_ctx* ctx, const ConvLayer& L);
int stem_rgb_run(b2o_ctx* ctx, const ConvLayer& L, const uint8_t* img, int n, int h, int w,
                 const TensorView& out, cudaStream_t st);
int normalize16_run(b2o_ctx* ctx, const uint8_t* img, int n, int h, int w, __half* out, cudaStream_t st);
int stem_crnn_run(b2o_ctx* ctx, const ConvLayer& L, const __half* x, int b, const TensorView& out,
                  cudaStream_t st);
int maxpool2_run(b2o_ctx* ctx, const TensorView& in, const TensorView& out, cudaStream_t st);
int maxpool3s1_run(b2o_ctx* ctx, const TensorView& in, const TensorView& out, cudaStream_t st);
int upsample_run(b2o_ctx* ctx, const TensorView& in, const TensorView& out, cudaStream_t st);
int head_tail_run(b2o_ctx* ctx, const ConvLayer& L6, const ConvLayer& L8, const TensorView& in,
                  float* scores, cudaStream_t st);

// ---- atomic union-find (boxes.cu's connected components, lines.cu's text lines) ----------------------------
// L[a] is a's parent; a root is its own parent.  uf_unite hangs the larger root under the smaller one, so every root is
// the smallest index of its set, whatever order the unions run in.
static __device__ __forceinline__ int uf_find(const int* L, int a) {
  while (true) {
    const int p = *reinterpret_cast<const volatile int*>(L + a);
    if (p == a) return a;
    a = p;
  }
}
static __device__ __forceinline__ void uf_unite(int* L, int a, int b) {
  while (true) {
    a = uf_find(L, a);
    b = uf_find(L, b);
    if (a == b) return;
    if (a < b) { const int t = a; a = b; b = t; }
    const int old = atomicMin(L + a, b);     // hang the larger root under the smaller one
    if (old == a) return;
    a = old;
  }
}

// ---- one-CTA sorts and scans on total-order keys (lines.cu's text lines, blocks.cu's text blocks) ----------------
struct SortKey {                     // lexicographic (a, b, c); p travels with the key
  unsigned long long a, b;
  unsigned c, p;
};

static __device__ __forceinline__ bool key_less(const SortKey& x, const SortKey& y) {
  if (x.a != y.a) return x.a < y.a;
  if (x.b != y.b) return x.b < y.b;
  return x.c < y.c;
}

// order-preserving map of a double onto uint64; -0.0 and +0.0 map to the same key (an exact tie)
static __device__ __forceinline__ unsigned long long dkey(double x) {
  if (x == 0.0) x = 0.0;
  const unsigned long long b = static_cast<unsigned long long>(__double_as_longlong(x));
  return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}

// a . b = a.x b.x + a.y b.y in fp64, in that order, without contraction
static __device__ __forceinline__ double dot2(double ax, double ay, double bx, double by) {
  return __dadd_rn(__dmul_rn(ax, bx), __dmul_rn(ay, by));
}

// exclusive block-wide scan of v; returns the prefix and leaves the block total in *total (smem scratch: 32 ints + 1)
static __device__ int block_exclusive_scan(int v, int* scratch, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  int x = v;
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) scratch[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int s = lane < nw ? scratch[lane] : 0;
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    if (lane < nw) scratch[lane] = s;
    if (lane == nw - 1) scratch[32] = s;
  }
  __syncthreads();
  const int r = x - v + (warp ? scratch[warp - 1] : 0);
  *total = scratch[32];
  __syncthreads();
  return r;
}

// ascending bitonic sort of keys[0, p) (p a power of two) by the whole CTA, in global memory
static __device__ void block_sort(SortKey* keys, int p) {
  for (int k = 2; k <= p; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = threadIdx.x; t < (p >> 1); t += blockDim.x) {
        const int lo = 2 * t - (t & (j - 1));          // index whose bit j is clear
        const int hi = lo + j;
        const bool up = (lo & k) == 0;
        const SortKey x = keys[lo], y = keys[hi];
        if (key_less(y, x) == up) { keys[lo] = y; keys[hi] = x; }
      }
      __syncthreads();
    }
  }
}

// keys[from, p) = the largest key, so that padding sorts last
static __device__ __forceinline__ void pad_keys(SortKey* keys, int from, int p) {
  for (int t = from + threadIdx.x; t < p; t += blockDim.x) {
    SortKey s;
    s.a = s.b = ~0ull;
    s.c = s.p = ~0u;
    keys[t] = s;
  }
}

// ---- box corner order (image.cu's warp, rotation.cu's box roll, ctc_align.cu's cells) ------------
// fp64 Euclidean distance of two float32 points, as scipy's cdist computes it (tools.py:41-57)
static __device__ inline double corner_dist(const float* a, const float* b) {
  const double dx = static_cast<double>(a[0]) - static_cast<double>(b[0]);
  const double dy = static_cast<double>(a[1]) - static_cast<double>(b[1]);
  return sqrt(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));
}

// get_rotated_box on a rectangle (tools.py:533-581): ord = the indices of q (4x2) in the order tl, tr, br, bl -- stable
// sort by x, the two left corners split by y, the right ones by distance from tl.
static __device__ inline void order_corners(const float* q, int ord[4]) {
  int idx[4] = {0, 1, 2, 3};
  for (int i = 1; i < 4; ++i) {              // insertion sort == numpy's argsort(kind="stable")
    const int v = idx[i];
    int j = i - 1;
    while (j >= 0 && q[2 * idx[j]] > q[2 * v]) { idx[j + 1] = idx[j]; --j; }
    idx[j + 1] = v;
  }
  int l0 = idx[0], l1 = idx[1];
  if (q[2 * l0 + 1] > q[2 * l1 + 1]) { const int t = l0; l0 = l1; l1 = t; }
  const int r0 = idx[2], r1 = idx[3];
  const double d0 = corner_dist(q + 2 * l0, q + 2 * r0), d1 = corner_dist(q + 2 * l0, q + 2 * r1);
  ord[0] = l0;                               // tl
  ord[3] = l1;                               // bl
  // (br, tr) = rightMost[argsort(D)[::-1]]
  if (d0 <= d1) { ord[2] = r1; ord[1] = r0; } else { ord[2] = r0; ord[1] = r1; }
}

// ---- warpBox geometry (image.cu's warp, ctc_align.cu's character cells) ------------------------------
// turn r (0..3): warpBox(skip_rotate=True) of the ordered box rolled by r, np.roll(c, -r, axis=0) -- the crop starts at
// corner c[r] and odd turns swap width and height.  Turn 0 is tools.warpBox itself.
// warp_extent: the rolled box (get_rotated_box on a rectangle, then the roll), get_rotated_width_height and the scaled
// content size sw x sh of the crop in fp64; the homography maps the box onto (0,0), (sw,0), (sw,sh), (0,sh) rounded to
// float32.  False where the reference raises ZeroDivisionError (w or h is 0).
static __device__ inline bool warp_extent(const float* q /*4x2*/, int turn, int target_w, int target_h, float box[8],
                                          double* sw, double* sh) {
  // --- get_rotated_box on a rectangle, then the roll -----------------------------------------------
  int ord[4];
  order_corners(q, ord);
  for (int i = 0; i < 4; ++i) {
    box[2 * i] = q[2 * ord[(i + turn) & 3]];
    box[2 * i + 1] = q[2 * ord[(i + turn) & 3] + 1];
  }
  // --- get_rotated_width_height --------------------------------------------------------------------
  const int w = static_cast<int>((corner_dist(box + 0, box + 2) + corner_dist(box + 4, box + 6)) / 2);
  const int h = static_cast<int>((corner_dist(box + 0, box + 6) + corner_dist(box + 2, box + 4)) / 2);
  if (w <= 0 || h <= 0) return false;        // the reference raises ZeroDivisionError here
  const double sa = static_cast<double>(target_w) / w, sb = static_cast<double>(target_h) / h;
  const double scale = sa < sb ? sa : sb;
  *sw = scale * w;
  *sh = scale * h;
  return true;
}

// cv2.getPerspectiveTransform(src, dst) (8x8 system, LU with partial pivoting, fp64) followed by cv::invert of the
// 3x3 (closed form): m[9] = the inverse homography, destination -> source.  False where the system is singular.
static __device__ inline bool persp_inverse(const float* src /*4x2*/, const float* dst /*4x2*/, double m[9]) {
  double A[8][8], b[8];
  for (int i = 0; i < 4; ++i) {
    const double sxx = src[2 * i], syy = src[2 * i + 1], dx = dst[2 * i], dy = dst[2 * i + 1];
    for (int k = 0; k < 8; ++k) { A[i][k] = 0.0; A[i + 4][k] = 0.0; }
    A[i][0] = A[i + 4][3] = sxx;
    A[i][1] = A[i + 4][4] = syy;
    A[i][2] = A[i + 4][5] = 1.0;
    A[i][6] = __dmul_rn(-sxx, dx);
    A[i][7] = __dmul_rn(-syy, dx);
    A[i + 4][6] = __dmul_rn(-sxx, dy);
    A[i + 4][7] = __dmul_rn(-syy, dy);
    b[i] = dx;
    b[i + 4] = dy;
  }
  for (int i = 0; i < 8; ++i) {
    int k = i;
    for (int j = i + 1; j < 8; ++j)
      if (fabs(A[j][i]) > fabs(A[k][i])) k = j;
    if (fabs(A[k][i]) < 2.220446049250313e-14) return false;     // DBL_EPSILON*100: singular
    if (k != i) {
      for (int j = i; j < 8; ++j) { const double t = A[i][j]; A[i][j] = A[k][j]; A[k][j] = t; }
      const double t = b[i]; b[i] = b[k]; b[k] = t;
    }
    const double d = -1.0 / A[i][i];
    for (int j = i + 1; j < 8; ++j) {
      const double alpha = __dmul_rn(A[j][i], d);
      for (int kk = i + 1; kk < 8; ++kk) A[j][kk] = __dadd_rn(A[j][kk], __dmul_rn(alpha, A[i][kk]));
      b[j] = __dadd_rn(b[j], __dmul_rn(alpha, b[i]));
    }
  }
  for (int i = 7; i >= 0; --i) {
    double s = b[i];
    for (int kk = i + 1; kk < 8; ++kk) s = __dsub_rn(s, __dmul_rn(A[i][kk], b[kk]));
    b[i] = s / A[i][i];
  }
  const double M[9] = {b[0], b[1], b[2], b[3], b[4], b[5], b[6], b[7], 1.0};
#define MM(r, c) M[(r) * 3 + (c)]
#define DET2(a, b, c, d) __dsub_rn(__dmul_rn(a, b), __dmul_rn(c, d))
  const double det = __dadd_rn(
      __dsub_rn(__dmul_rn(MM(0, 0), DET2(MM(1, 1), MM(2, 2), MM(1, 2), MM(2, 1))),
                __dmul_rn(MM(0, 1), DET2(MM(1, 0), MM(2, 2), MM(1, 2), MM(2, 0)))),
      __dmul_rn(MM(0, 2), DET2(MM(1, 0), MM(2, 1), MM(1, 1), MM(2, 0))));
  if (det == 0.0) return false;
  const double id = 1.0 / det;
  m[0] = __dmul_rn(DET2(MM(1, 1), MM(2, 2), MM(1, 2), MM(2, 1)), id);
  m[1] = __dmul_rn(DET2(MM(0, 2), MM(2, 1), MM(0, 1), MM(2, 2)), id);
  m[2] = __dmul_rn(DET2(MM(0, 1), MM(1, 2), MM(0, 2), MM(1, 1)), id);
  m[3] = __dmul_rn(DET2(MM(1, 2), MM(2, 0), MM(1, 0), MM(2, 2)), id);
  m[4] = __dmul_rn(DET2(MM(0, 0), MM(2, 2), MM(0, 2), MM(2, 0)), id);
  m[5] = __dmul_rn(DET2(MM(0, 2), MM(1, 0), MM(0, 0), MM(1, 2)), id);
  m[6] = __dmul_rn(DET2(MM(1, 0), MM(2, 1), MM(1, 1), MM(2, 0)), id);
  m[7] = __dmul_rn(DET2(MM(0, 1), MM(2, 0), MM(0, 0), MM(2, 1)), id);
  m[8] = __dmul_rn(DET2(MM(0, 0), MM(1, 1), MM(0, 1), MM(1, 0)), id);
#undef MM
#undef DET2
  return true;
}

// b2o_warp_plan (include/b2ocr.h): m[9] = inverse homography (destination -> source), fp64 like cv2; dw, dh = dsize
// of warpPerspective; valid = 0 where warpBox raises ZeroDivisionError (or the system is singular).
static __device__ inline void plan_warp(const float* q /*4x2*/, int turn, int target_w, int target_h, b2o_warp_plan* plan) {
  plan->valid = 0;
  float box[8];
  double sw, sh;
  if (!warp_extent(q, turn, target_w, target_h, box, &sw, &sh)) return;
  const float dst[8] = {0.f, 0.f, static_cast<float>(sw), 0.f, static_cast<float>(sw), static_cast<float>(sh),
                        0.f, static_cast<float>(sh)};
  plan->dw = static_cast<int>(sw);
  plan->dh = static_cast<int>(sh);
  if (persp_inverse(box, dst, plan->m)) plan->valid = 1;
}

// ---- warpBox sampling (image.cu's box and polygon warps, windows.cu's wide-word windows) ----------------------
constexpr int kWarpCropH = 31, kWarpCropW = 200;

// cv2.warpPerspective INTER_LINEAR (BORDER_CONSTANT 0) of one crop pixel (x, y) through the inverse map m, with
// cv::WarpPerspectiveInvoker's block width bw0 (x is re-based at multiples of it): 1/32-pixel coordinates, 15-bit
// weights.
template <int CH>
static __device__ __forceinline__ void warp_sample(const uint8_t* __restrict__ g, int H, int W, const double* m, int x,
                                                   int y, int bw0, int v[CH]) {
  const int bx = (x / bw0) * bw0, x1 = x - bx;
  const double X0 = __dadd_rn(__dadd_rn(__dmul_rn(m[0], bx), __dmul_rn(m[1], y)), m[2]);
  const double Y0 = __dadd_rn(__dadd_rn(__dmul_rn(m[3], bx), __dmul_rn(m[4], y)), m[5]);
  const double W0 = __dadd_rn(__dadd_rn(__dmul_rn(m[6], bx), __dmul_rn(m[7], y)), m[8]);
  double Wv = __dadd_rn(W0, __dmul_rn(m[6], x1));
  Wv = Wv != 0.0 ? 32.0 / Wv : 0.0;
  const double fX = fmax(-2147483648.0, fmin(2147483647.0, __dmul_rn(__dadd_rn(X0, __dmul_rn(m[0], x1)), Wv)));
  const double fY = fmax(-2147483648.0, fmin(2147483647.0, __dmul_rn(__dadd_rn(Y0, __dmul_rn(m[3], x1)), Wv)));
  const int X = __double2int_rn(fX), Y = __double2int_rn(fY);
  const int sx = min(max(X >> 5, -32768), 32767), sy = min(max(Y >> 5, -32768), 32767);
  const int ax = X & 31, ay = Y & 31;
  const bool x0ok = sx >= 0 && sx < W, x1ok = sx + 1 >= 0 && sx + 1 < W;
  const bool y0ok = sy >= 0 && sy < H, y1ok = sy + 1 >= 0 && sy + 1 < H;
  // BilinearTab_i: (1-fx)(1-fy) ... scaled to 2^15; exact for 1/32 steps
  const int w00 = (32 - ax) * (32 - ay) * 32, w01 = ax * (32 - ay) * 32;
  const int w10 = (32 - ax) * ay * 32, w11 = ax * ay * 32;
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    const int p00 = (x0ok && y0ok) ? g[(static_cast<size_t>(sy) * W + sx) * CH + c] : 0;
    const int p01 = (x1ok && y0ok) ? g[(static_cast<size_t>(sy) * W + sx + 1) * CH + c] : 0;
    const int p10 = (x0ok && y1ok) ? g[(static_cast<size_t>(sy + 1) * W + sx) * CH + c] : 0;
    const int p11 = (x1ok && y1ok) ? g[(static_cast<size_t>(sy + 1) * W + sx + 1) * CH + c] : 0;
    v[c] = (p00 * w00 + p01 * w01 + p10 * w10 + p11 * w11 + 16384) >> 15;
  }
}

// The crop tile of one word -> the CRNN input slot k.  Layout (recognition.py:215-216): x[t][j] = crop[30-j][t] / 255.
// Called by all threads after the tile is written.
template <int CH>
static __device__ __forceinline__ void store_crnn_in(const uint8_t* tile, int k, __half* __restrict__ crnn_in) {
  __half* o = crnn_in + static_cast<size_t>(k) * kWarpCropH * kWarpCropW * CH;
  for (int i = threadIdx.x; i < kWarpCropH * kWarpCropW * CH; i += blockDim.x) {
    const int c = i % CH, q = i / CH;
    const int t = q / kWarpCropH, j = q - t * kWarpCropH;
    o[i] = __float2half_rn(static_cast<float>(tile[((kWarpCropH - 1 - j) * kWarpCropW + t) * CH + c]) / 255.0f);
  }
}

// cv::WarpPerspectiveInvoker's block width for a dsize dw x dh (clamped to the crop): x is re-based at its multiples
static __device__ __forceinline__ int warp_block_width(int dw, int dh) {
  const int bh0 = min(16, max(dh, 1));
  return min(1024 / bh0, max(dw, 1));
}

// The crop of one word, shared by the box, polygon and window warps: sample(x, y, v) for x < dw, y < dh (the dsize
// clamped to the crop, 0 where the plan is invalid) and 0 elsewhere, into tile (31 x 200 x CH, shared memory) and crop
// slot k of crops (optional); then the CRNN input slot k (optional).
template <int CH, typename Sample>
static __device__ __forceinline__ void warp_crop(int dw, int dh, Sample sample, uint8_t* tile, int k,
                                                 uint8_t* __restrict__ crops, __half* __restrict__ crnn_in) {
  for (int i = threadIdx.x; i < kWarpCropH * kWarpCropW; i += blockDim.x) {
    const int y = i / kWarpCropW, x = i - y * kWarpCropW;
    int v[CH];
#pragma unroll
    for (int c = 0; c < CH; ++c) v[c] = 0;
    if (x < dw && y < dh) sample(x, y, v);
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      tile[i * CH + c] = static_cast<uint8_t>(v[c]);
      if (crops) crops[(static_cast<size_t>(k) * kWarpCropH * kWarpCropW + i) * CH + c] = static_cast<uint8_t>(v[c]);
    }
  }
  if (crnn_in == nullptr) return;
  __syncthreads();
  store_crnn_in<CH>(tile, k, crnn_in);
}

// ---- the STN's time axis (ctc_align.cu's character cuts, windows.cu's stitch) -----------------------------------
// Crop column of grid row r (r = kept step + 2 discarded steps): through the STN's time coordinate on the grid's centre
// column, u = 0.5 (theta[4] gy + theta[5] + 1) 50 with gy = -1 + 2r/49, or u = r without an STN (th null); 4 crop
// columns per pooled step, pixel centres at integers: x = 4u + 1.5.  fp64 without contraction.
static __device__ __forceinline__ double stn_crop_x(double r, const float* th) {
  double u = r;
  if (th) {
    const double gy = __dadd_rn(-1.0, __ddiv_rn(__dmul_rn(2.0, r), 49.0));
    u = __dmul_rn(__dmul_rn(0.5, __dadd_rn(__dadd_rn(__dmul_rn(static_cast<double>(th[4]), gy),
                                                     static_cast<double>(th[5])), 1.0)), 50.0);
  }
  return __dadd_rn(__dmul_rn(4.0, u), 1.5);
}

static inline TensorView make_view(void* base, int n, int h, int w, int c, int ld = 0, int coff = 0) {
  TensorView v;
  v.ptr = reinterpret_cast<__half*>(base) + coff;
  v.n = n; v.h = h; v.w = w; v.c = c; v.ld = ld ? ld : c;
  return v;
}
