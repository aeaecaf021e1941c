// api.cu -- C-ABI entry points (include/b2ocr.h): context, weight packing, network orchestration.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <functional>

#include "common.cuh"

int stn_theta_run(b2o_ctx* ctx, const __half* d1, int B, float* theta, cudaStream_t st);
int stn_col2im_run(b2o_ctx* ctx, const __half* y, const float* bias, int B, __half* out, cudaStream_t st);
int stn_sample_run(b2o_ctx* ctx, const __half* feat, const float* theta, int B, __half* out, cudaStream_t st);
int lstm_run(b2o_ctx* ctx, const float* xw, int xw_ld, int xw_off, const __half* u, int B, int backwards, __half* out,
             int out_ld, int out_off, cudaStream_t st);
int add_run(b2o_ctx* ctx, const __half* a, const __half* b, __half* o, long long n, cudaStream_t st);
int fc_ctc_run(b2o_ctx* ctx, const __half* l2, int B, float* logits, int* labels, float* logp, cudaStream_t st);
int ctc_beam_run(b2o_ctx* ctx, const float* logits, int B, int K, int beam_width, int top_paths, int* labels, float* logp,
                 cudaStream_t st);
int ctc_beam_lm_run(b2o_ctx* ctx, const float* logits, int B, int K, int beam_width, int top_paths,
                    const b2o_char_lm* lm, int* labels, float* logp, float* fused, cudaStream_t st);
int ctc_beam_hotword_run(b2o_ctx* ctx, const float* logits, int B, int K, int beam_width, int top_paths,
                         const b2o_char_lm* lm, const b2o_hotwords* hw, int* labels, float* logp, float* fused,
                         cudaStream_t st);
int ctc_beam_pattern_run(b2o_ctx* ctx, const float* logits, int B, int K, int beam_width, int top_paths,
                         const b2o_pattern* pat, int* labels, float* logp, cudaStream_t st);
size_t ctc_lexicon_workspace_bytes(int B, int n_words);
int ctc_lexicon_run(b2o_ctx* ctx, const float* logits, int B, int K, const int* offsets, const short* labels,
                    int n_words, int top_paths, int* labels_out, float* logp, void* ws, cudaStream_t st);
int ctc_align_run(b2o_ctx* ctx, const float* logits, int B, int K, const int32_t* labels, int P, int32_t* spans,
                  float* logp, cudaStream_t st);
int ctc_char_scores_run(b2o_ctx* ctx, const float* logits, int B, int K, const int32_t* labels, int P, int A, float* conf,
                        int32_t* alt_labels, float* alt_post, float* logp, cudaStream_t st);
bool ctc_char_scores_args(int k, int top_paths, int alternatives);
size_t ctc_train_workspace_bytes(int B, int K);
int ctc_loss_grad_run(b2o_ctx* ctx, const __half* features, long long feat_stride, bool feat_by_batch, int n_rows,
                      const int* index, int B, int K, const float* w, const float* bias, const int* offsets,
                      const short* labels, float rate, uint64_t seed, uint64_t step, float* loss, float* grad_w,
                      float* grad_b, float* logits, void* ws, cudaStream_t st);
size_t rnn_train_workspace_bytes(int B, int K);
int rnn_loss_grad_run(b2o_ctx* ctx, const __half* x, int n_rows, const int* index, int B, int K, const float* params,
                      const int* offsets, const short* labels, float rate, uint64_t seed, uint64_t step, float* loss,
                      float* grad, void* ws, cudaStream_t st);
int rmsprop_run(b2o_ctx* ctx, float* param, const float* grad, float* acc, long long n, float lr, float rho, float eps,
                cudaStream_t st);

namespace {

typedef std::map<std::string, const b2o_tensor*> TensorMap;

const b2o_tensor* need(b2o_ctx* ctx, const TensorMap& m, const std::string& name, int ndim, const int64_t* shape) {
  auto it = m.find(name);
  if (it == m.end()) { ctx->set_error("missing weight tensor: " + name); return nullptr; }
  const b2o_tensor* t = it->second;
  if (t->ndim != ndim) { ctx->set_error("bad rank for " + name); return nullptr; }
  for (int i = 0; i < ndim; ++i)
    if (t->shape[i] != shape[i]) { ctx->set_error("bad shape for " + name); return nullptr; }
  return t;
}

template <typename T>
T* dev_alloc(b2o_ctx* ctx, size_t count) {
  void* p = nullptr;
  if (cudaMalloc(&p, count * sizeof(T)) != cudaSuccess) { ctx->set_error("cudaMalloc failed"); return nullptr; }
  ctx->owned.push_back(p);
  return reinterpret_cast<T*>(p);
}

template <typename T>
T* dev_upload(b2o_ctx* ctx, const std::vector<T>& host) {
  T* p = dev_alloc<T>(ctx, host.size());
  if (!p) return nullptr;
  if (cudaMemcpy(p, host.data(), host.size() * sizeof(T), cudaMemcpyHostToDevice) != cudaSuccess) {
    ctx->set_error("cudaMemcpy (weights) failed");
    return nullptr;
  }
  return p;
}

// Build one layer.  wget(o, c, ky, kx) returns the fp32 weight.
int build_layer(b2o_ctx* ctx, ConvLayer& L, const std::string& name, int cin, int cout, int ksize, int dil, int relu,
                const std::function<float(int, int, int, int)>& wget, const std::vector<float>& s1,
                const std::vector<float>& t1, const std::vector<float>* s2, const std::vector<float>* t2,
                bool keep_f32_stem) {
  L = ConvLayer();
  L.name = name; L.cin = cin; L.cout = cout; L.ksize = ksize; L.dil = dil; L.relu = relu;
  const int taps = ksize * ksize;
  if (keep_f32_stem) {
    std::vector<float> wf(static_cast<size_t>(taps) * cin * cout);
    for (int ky = 0; ky < ksize; ++ky)
      for (int kx = 0; kx < ksize; ++kx)
        for (int c = 0; c < cin; ++c)
          for (int o = 0; o < cout; ++o)
            wf[(static_cast<size_t>(ky * ksize + kx) * cin + c) * cout + o] = wget(o, c, ky, kx);
    if (!(L.w_f32 = dev_upload(ctx, wf))) return B2O_ERR_CUDA;
    L.h_w_f32 = wf;
  } else {
    std::vector<__half> wk(static_cast<size_t>(cout) * taps * cin);
    std::vector<float> ws(static_cast<size_t>(taps) * cin * cout);
    for (int o = 0; o < cout; ++o)
      for (int ky = 0; ky < ksize; ++ky)
        for (int kx = 0; kx < ksize; ++kx)
          for (int c = 0; c < cin; ++c) {
            const __half hv = __float2half_rn(wget(o, c, ky, kx));
            const int tap = ky * ksize + kx;
            wk[(static_cast<size_t>(o) * taps + tap) * cin + c] = hv;
            ws[(static_cast<size_t>(tap) * cin + c) * cout + o] = __half2float(hv);
          }
    if (!(L.w_kmajor = dev_upload(ctx, wk))) return B2O_ERR_CUDA;
    if (!(L.w_simt = dev_upload(ctx, ws))) return B2O_ERR_CUDA;
    if (ws.size() <= 1024) L.h_w_simt = ws;
  }
  if (!(L.s1 = dev_upload(ctx, s1))) return B2O_ERR_CUDA;
  if (!(L.t1 = dev_upload(ctx, t1))) return B2O_ERR_CUDA;
  L.h_s1 = s1; L.h_t1 = t1;
  if (s2) { L.h_s2 = *s2; L.h_t2 = *t2; }
  if (s2) {
    if (!(L.s2 = dev_upload(ctx, *s2))) return B2O_ERR_CUDA;
    if (!(L.t2 = dev_upload(ctx, *t2))) return B2O_ERR_CUDA;
  }
  if (!keep_f32_stem) B2O_RETURN_IF(conv_tc_prepare(ctx, L));
  return B2O_OK;
}

struct CraftSpec { const char* name; int cin, cout, k, dil; const char* bn; int relu; };
const CraftSpec kCraft[] = {
    {"basenet.slice1.0", 3, 64, 3, 1, "basenet.slice1.1", 1},     {"basenet.slice1.3", 64, 64, 3, 1, "basenet.slice1.4", 1},
    {"basenet.slice1.7", 64, 128, 3, 1, "basenet.slice1.8", 1},   {"basenet.slice1.10", 128, 128, 3, 1, "basenet.slice1.11", 1},
    {"basenet.slice2.14", 128, 256, 3, 1, "basenet.slice2.15", 1}, {"basenet.slice2.17", 256, 256, 3, 1, "basenet.slice2.18", 1},
    {"basenet.slice3.20", 256, 256, 3, 1, "basenet.slice3.21", 1}, {"basenet.slice3.24", 256, 512, 3, 1, "basenet.slice3.25", 1},
    {"basenet.slice3.27", 512, 512, 3, 1, "basenet.slice3.28", 1}, {"basenet.slice4.30", 512, 512, 3, 1, "basenet.slice4.31", 1},
    {"basenet.slice4.34", 512, 512, 3, 1, "basenet.slice4.35", 1}, {"basenet.slice4.37", 512, 512, 3, 1, "basenet.slice4.38", 0},
    {"basenet.slice5.1", 512, 1024, 3, 6, nullptr, 0},             {"basenet.slice5.2", 1024, 1024, 1, 1, nullptr, 0},
    {"upconv1.conv.0", 1536, 512, 1, 1, "upconv1.conv.1", 1},      {"upconv1.conv.3", 512, 256, 3, 1, "upconv1.conv.4", 1},
    {"upconv2.conv.0", 768, 256, 1, 1, "upconv2.conv.1", 1},       {"upconv2.conv.3", 256, 128, 3, 1, "upconv2.conv.4", 1},
    {"upconv3.conv.0", 384, 128, 1, 1, "upconv3.conv.1", 1},       {"upconv3.conv.3", 128, 64, 3, 1, "upconv3.conv.4", 1},
    {"upconv4.conv.0", 192, 64, 1, 1, "upconv4.conv.1", 1},        {"upconv4.conv.3", 64, 32, 3, 1, "upconv4.conv.4", 1},
    {"conv_cls.0", 32, 32, 3, 1, nullptr, 1},                      {"conv_cls.2", 32, 32, 3, 1, nullptr, 1},
    {"conv_cls.4", 32, 16, 3, 1, nullptr, 1},                      {"conv_cls.6", 16, 16, 1, 1, nullptr, 1},
    {"conv_cls.8", 16, 2, 1, 1, nullptr, 0},
};

// The CRAFT forward's buffers (NHWC fp16), named as b2o_craft_tap names them.  The packer's stable sort breaks ties
// between equal sizes in this order, so reordering the table moves buffers in the workspace.
namespace cb {
enum Id : int8_t { x16, a, b, p1, c, cat4, p2, d, cat3, e, p3, f, cat2, g, p4, hh, cat1, mp, s5a, u1a, u1b, u2a, u2b, u3a,
                   u3b, u4a, u4b, h1, h2, h3, z2, z3, z4, count, none = -1 };
}
struct CraftBufSpec { const char* name; int level, c; };      // level: resolution divisor (1, 2, 4, 8, 16)
constexpr CraftBufSpec kCraftBufs[cb::count] = {
    {"x16", 1, 16},                                          // normalised input, 3 -> 16 channels, for the tensor-core stem
    {"a", 1, 64},     {"b", 1, 64},     {"p1", 2, 64},     {"c", 2, 128},     {"cat4", 2, 192},  {"p2", 4, 128},
    {"d", 4, 256},    {"cat3", 4, 384}, {"e", 4, 256},     {"p3", 8, 256},    {"f", 8, 512},     {"cat2", 8, 768},
    {"g", 8, 512},    {"p4", 16, 512},  {"hh", 16, 512},   {"cat1", 16, 1536}, {"mp", 16, 512},  {"s5a", 16, 1024},
    {"u1a", 16, 512}, {"u1b", 16, 256}, {"u2a", 8, 256},   {"u2b", 8, 128},   {"u3a", 4, 128},   {"u3b", 4, 64},
    {"u4a", 2, 64},   {"u4b", 2, 32},   {"h1", 2, 32},     {"h2", 2, 32},     {"h3", 2, 16},
    {"z2", 16, 256},  {"z3", 8, 128},   {"z4", 4, 64},       // low-resolution halves of upconv2/3/4.conv.0 (commuted)
};

// Channels [c0, c1) of a buffer; S(buf) is all of it.
struct Slice { cb::Id buf = cb::none; int c0 = 0, c1 = 0; };
constexpr Slice S(cb::Id buf, int c0 = 0, int c1 = -1) { return {buf, c0, c1 < 0 ? kCraftBufs[buf].c : c1}; }

// level_up / level_conv: the two steps of a decoder level, UpsampleLike(y) into the concat's decoder half and
// upconvN.conv.0 over the concat -- or, commuted, the decoder half z of that 1x1 conv at y's resolution and the skip half
// at full resolution adding z's upsampling in its epilogue.
enum class StepKind : int8_t { normalize, stem, conv, maxpool3, level_up, level_conv, tail };

// One launch of the forward (or none, where the engine folds the step into another).  Every slice any engine or switch
// setting may touch is listed: buffer lifetimes are derived from them.  A level step's y is src at level_up; at
// level_conv only z and skip (read by the commuted path) stand for it -- y is not read there.
struct CraftStep {
  StepKind kind;
  const char* layer;
  Slice src, out, pool, z, skip;
  int write_full = 1;         // a pooled conv stores its full-resolution output too (conv_run)
};
constexpr CraftStep kCraftSteps[] = {
    // encoder (detection.py:312-324); taps s1..s4 are written straight into the concat buffers
    {StepKind::normalize, nullptr, {}, S(cb::x16)},
    {StepKind::stem, "basenet.slice1.0", S(cb::x16), S(cb::a)},
    {StepKind::conv, "basenet.slice1.3", S(cb::a), S(cb::b), S(cb::p1), {}, {}, 0},
    {StepKind::conv, "basenet.slice1.7", S(cb::p1), S(cb::c)},
    {StepKind::conv, "basenet.slice1.10", S(cb::c), S(cb::cat4, 64, 192), S(cb::p2)},
    {StepKind::conv, "basenet.slice2.14", S(cb::p2), S(cb::d)},
    {StepKind::conv, "basenet.slice2.17", S(cb::d), S(cb::cat3, 128, 384)},
    {StepKind::conv, "basenet.slice3.20", S(cb::cat3, 128, 384), S(cb::e), S(cb::p3), {}, {}, 0},
    {StepKind::conv, "basenet.slice3.24", S(cb::p3), S(cb::f)},
    {StepKind::conv, "basenet.slice3.27", S(cb::f), S(cb::cat2, 256, 768)},
    {StepKind::conv, "basenet.slice4.30", S(cb::cat2, 256, 768), S(cb::g), S(cb::p4), {}, {}, 0},
    {StepKind::conv, "basenet.slice4.34", S(cb::p4), S(cb::hh)},
    {StepKind::conv, "basenet.slice4.37", S(cb::hh), S(cb::cat1, 1024, 1536)},      // BN only, no ReLU (333)
    // slice5 (365-378)
    {StepKind::maxpool3, nullptr, S(cb::cat1, 1024, 1536), S(cb::mp)},
    {StepKind::conv, "basenet.slice5.1", S(cb::mp), S(cb::s5a)},
    {StepKind::conv, "basenet.slice5.2", S(cb::s5a), S(cb::cat1, 0, 1024)},
    // decoder (380-390)
    {StepKind::conv, "upconv1.conv.0", S(cb::cat1), S(cb::u1a)},
    {StepKind::conv, "upconv1.conv.3", S(cb::u1a), S(cb::u1b)},
    {StepKind::level_up, "upconv2.conv.0", S(cb::u1b), S(cb::cat2, 0, 256), {}, S(cb::z2)},
    {StepKind::level_conv, "upconv2.conv.0", S(cb::cat2), S(cb::u2a), {}, S(cb::z2), S(cb::cat2, 256, 768)},
    {StepKind::conv, "upconv2.conv.3", S(cb::u2a), S(cb::u2b)},
    {StepKind::level_up, "upconv3.conv.0", S(cb::u2b), S(cb::cat3, 0, 128), {}, S(cb::z3)},
    {StepKind::level_conv, "upconv3.conv.0", S(cb::cat3), S(cb::u3a), {}, S(cb::z3), S(cb::cat3, 128, 384)},
    {StepKind::conv, "upconv3.conv.3", S(cb::u3a), S(cb::u3b)},
    {StepKind::level_up, "upconv4.conv.0", S(cb::u3b), S(cb::cat4, 0, 64), {}, S(cb::z4)},
    {StepKind::level_conv, "upconv4.conv.0", S(cb::cat4), S(cb::u4a), {}, S(cb::z4), S(cb::cat4, 64, 192)},
    {StepKind::conv, "upconv4.conv.3", S(cb::u4a), S(cb::u4b)},
    // head (392-410)
    {StepKind::conv, "conv_cls.0", S(cb::u4b), S(cb::h1)},
    {StepKind::conv, "conv_cls.2", S(cb::h1), S(cb::h2)},
    {StepKind::conv, "conv_cls.4", S(cb::h2), S(cb::h3)},          // the tail rides in its epilogue where tail_fused
    {StepKind::tail, nullptr, S(cb::h3)},                           // conv_cls.6 + conv_cls.8
};
static_assert(sizeof(kCraftSteps) / sizeof(kCraftSteps[0]) == B2O_CRAFT_LAST_STEP + 1, "one row per forward step");
static_assert(kCraftSteps[B2O_CRAFT_LAST_STEP].kind == StepKind::tail && kCraftSteps[B2O_CRAFT_LAST_STEP - 1].kind ==
              StepKind::conv, "the forward ends with conv_cls.4 and its tail");

// One buffer of the plan: placement, NHWC shape and lifetime in forward steps.
struct CraftBuf { size_t off, bytes; int h, w, first, last; };

// Buffer plan of the CRAFT forward pass, carved from one workspace.
struct CraftPlan {
  int n;
  size_t bytes;
  CraftBuf bufs[cb::count];
  TensorView view(void* ws, const Slice& s) const {
    if (s.buf == cb::none) return TensorView();
    const CraftBuf& b = bufs[s.buf];
    return make_view(reinterpret_cast<uint8_t*>(ws) + b.off, n, b.h, b.w, s.c1 - s.c0, kCraftBufs[s.buf].c, s.c0);
  }
};

// Liveness-based packing: every buffer lives from the first step that touches it (the one that writes it) to the last
// step that touches it (the forward pass is one stream-ordered chain of launches in kCraftSteps' order); buffers whose
// lifetimes do not overlap share memory.  Greedy by size: largest first, each at the lowest offset that is free for its
// whole lifetime.  32 x 1536 x 1536: 21.8 GB instead of 41 GB with every buffer live (the peak is the two
// full-resolution 64-channel maps around slice1.3), and 73 -> 39 GB at max_size 2048.
CraftPlan plan_craft(int n, int h, int w) {
  CraftPlan p;
  p.n = n;
  for (int i = 0; i < cb::count; ++i) {
    const CraftBufSpec& s = kCraftBufs[i];
    const int hh = h / s.level, ww = w / s.level;
    p.bufs[i] = {0, (static_cast<size_t>(n) * hh * ww * s.c * 2 + 255) / 256 * 256, hh, ww, B2O_CRAFT_LAST_STEP + 1, -1};
  }
  for (int k = 0; k <= B2O_CRAFT_LAST_STEP; ++k) {
    const CraftStep& s = kCraftSteps[k];
    for (const Slice* sl : {&s.src, &s.out, &s.pool, &s.z, &s.skip}) {
      if (sl->buf == cb::none) continue;
      CraftBuf& b = p.bufs[sl->buf];
      b.first = std::min(b.first, k);
      b.last = std::max(b.last, k);
    }
  }
  int order[cb::count];
  for (int i = 0; i < cb::count; ++i) order[i] = i;
  std::stable_sort(order, order + cb::count, [&](int a, int b) { return p.bufs[a].bytes > p.bufs[b].bytes; });
  std::vector<int> placed;
  size_t total = 0;
  for (int i : order) {
    CraftBuf& bi = p.bufs[i];
    // candidate offsets: 0 and the end of every placed buffer that is live at the same time
    std::vector<std::pair<size_t, size_t>> busy;      // [begin, end) of time-overlapping placed buffers
    for (int j : placed) {
      const CraftBuf& bj = p.bufs[j];
      if (bj.first <= bi.last && bi.first <= bj.last) busy.push_back({bj.off, bj.off + bj.bytes});
    }
    std::sort(busy.begin(), busy.end());
    size_t at = 0;
    for (const auto& b : busy) {
      if (at + bi.bytes <= b.first) break;
      if (b.second > at) at = b.second;
    }
    bi.off = at;
    placed.push_back(i);
    if (at + bi.bytes > total) total = at + bi.bytes;
  }
  p.bytes = total;
  return p;
}

// The CRNN's buffers, laid out one after the other (not liveness-packed: every tap stays readable after the forward).
// tap: b2o_crnn_tap reads the buffer under its name.
namespace rb {
enum Id : int8_t { x1, x2, x3, p3, x4, x5, p5, x6, features, sa, sb, d1, theta, warped, fc_9, xw1, hf, hb, l1, xw2, l2,
                   logits, count };
}
struct CrnnBufSpec { const char* name; size_t bytes; bool tap; };     // bytes per crop
constexpr CrnnBufSpec kCrnnBufs[rb::count] = {
    {"x1", 200 * 31 * 64 * 2, true},     {"x2", 200 * 31 * 128 * 2, true},  {"x3", 200 * 31 * 256 * 2, true},
    {"p3", 100 * 15 * 256 * 2, true},    {"x4", 100 * 15 * 256 * 2, true},  {"x5", 100 * 15 * 512 * 2, true},
    {"p5", 50 * 7 * 512 * 2, true},      {"x6", 50 * 7 * 512 * 2, true},    {"features", 50 * 7 * 512 * 2, true},
    {"sa", 50 * 7 * 16 * 2, false},      {"sb", 50 * 7 * 32 * 2, false},    {"d1", 64 * 2, false},
    {"theta", 6 * 4, true},              {"warped", 50 * 7 * 512 * 2, true}, {"fc_9", 50 * 128 * 2, true},
    {"xw1", 50 * 1024 * 4, false},       {"hf", 50 * 128 * 2, false},       {"hb", 50 * 128 * 2, false},
    {"l1", 50 * 128 * 2, true},          {"xw2", 50 * 1024 * 4, false},     {"l2", 50 * 256 * 2, true},
    {"logits", 48 * B2O_MAX_CLASSES * 4, true},   // sized for the largest alphabet so the plan is context-free
};

struct CrnnPlan {
  size_t off[rb::count], bytes;      // bytes: a multiple of 256
};

CrnnPlan plan_crnn(int b) {
  CrnnPlan p;
  size_t off = 0;
  for (int i = 0; i < rb::count; ++i) {
    p.off[i] = off;
    off += (static_cast<size_t>(b) * kCrnnBufs[i].bytes + 255) / 256 * 256;
  }
  p.bytes = off;
  return p;
}

// slot i of ws holds values of the context's last successful CRNN forward: plan_crnn(b) places the slots, so ws and b must
// be that forward's, and it must have written the slot
static_assert(rb::count <= 32, "b2o_ctx::crnn_written has one bit per slot");
bool crnn_wrote(const b2o_ctx* ctx, rb::Id i, const void* ws, int b) {
  return ws == ctx->crnn_ws && b == ctx->crnn_b && ((ctx->crnn_written >> i) & 1u);
}

// conv_cls.6 + conv_cls.8 (the tail) ride in conv_cls.4's epilogue on the auto engine's 16-column tile (same arithmetic
// as head_tail_kernel, bit for bit): one launch and the 16-channel map's round trip through HBM less.
bool tail_fused(const b2o_ctx* ctx, const ConvLayer& L4) {
  return ctx->conv_engine == B2O_CONV_AUTO && L4.block_n == 16 && !ctx->no_fused_tail;
}

// conv_cls.4 (L4: in -> out), with the tail (L6, L8) into scores where tail_fused; otherwise head_tail_run follows it.
int head_conv_run(b2o_ctx* ctx, const ConvLayer& L4, const ConvLayer& L6, const ConvLayer& L8, const TensorView& in,
                  const TensorView& out, float* scores, cudaStream_t st) {
  if (!tail_fused(ctx, L4)) return conv_run(ctx, L4, in, out, 0, st);
  ConvTail tail = {L6.w_simt, L6.t1, L8.w_simt, L8.t1, scores};
  if (L6.h_w_simt.size() == 256 && L8.h_w_simt.size() == 32) {
    tail.h_w6 = L6.h_w_simt.data(); tail.h_b6 = L6.h_t1.data(); tail.h_w8 = L8.h_w_simt.data(); tail.h_b8 = L8.h_t1.data();
  }
  return conv_tc_run(ctx, L4, in, out, 0, st, nullptr, 1, &tail);
}

std::vector<float> ones(int n) { return std::vector<float>(static_cast<size_t>(n), 1.0f); }
std::vector<float> tovec(const b2o_tensor* t, int n) { return std::vector<float>(t->data, t->data + n); }

}  // namespace

// ------------------------------------------------------------------------------------------------
extern "C" int b2o_version(void) { return 1; }

extern "C" int b2o_create(int device, b2o_ctx** out) {
  if (!out) return B2O_ERR_ARG;
  *out = nullptr;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count) return B2O_ERR_CUDA;
  DeviceGuard guard(device);                  // the caller's current device is restored on return
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return B2O_ERR_CUDA;
  if (prop.major != 9 || prop.minor != 0) {
    fprintf(stderr, "b2ocr: device %d is sm_%d%d; this library is built for sm_90a only\n", device, prop.major, prop.minor);
    return B2O_ERR_CUDA;
  }
  b2o_ctx* ctx = new b2o_ctx();
  ctx->device = device;
  ctx->sm_count = prop.multiProcessorCount;
  if (const char* e = getenv("B2O_UPCONV_COMMUTE")) ctx->no_commute = atoi(e) == 0;      // 1: commuted decoder upsampling (opt-in, see common.cuh)
  if (const char* e = getenv("B2O_TC_AFF")) ctx->tc_aff_const = std::string(e) != "smem";
  if (const char* e = getenv("B2O_GLUE")) ctx->glue_v1 = std::string(e) == "v1";
  if (const char* e = getenv("B2O_FUSED_TAIL")) ctx->no_fused_tail = atoi(e) == 0;      // 0: separate head_tail_kernel (A/B, tests)
  if (const char* e = getenv("B2O_TC_SWAP")) ctx->tc_swap = atoi(e) != 0;               // 0: 64-channel and streamed 128-channel layers as pixels x channels (A/B, tests)
  if (const char* e = getenv("B2O_TC_PAIR")) {        // default 0 = single-CTA tiles; 1 = pairs on halo tiles; 2 = generic tiles too
    ctx->tc_pair = atoi(e) != 0;
    ctx->tc_pair_generic = atoi(e) == 2;
  }
  *out = ctx;
  return B2O_OK;
}

extern "C" void b2o_destroy(b2o_ctx* ctx) {
  if (!ctx) return;
  {
    DeviceGuard guard(ctx->device);
    for (void* p : ctx->owned) cudaFree(p);
    for (cudaEvent_t e : ctx->prof_events) cudaEventDestroy(e);
    jpeg_release(ctx);
  }
  delete ctx;
}

extern "C" const char* b2o_last_error(const b2o_ctx* ctx) { return ctx ? ctx->error.c_str() : "null context"; }
extern "C" int64_t b2o_launch_count(const b2o_ctx* ctx) { return ctx ? ctx->launches : 0; }
extern "C" int64_t b2o_tc_tile256_launches(const b2o_ctx* ctx) { return ctx ? ctx->tc_tile256_launches : 0; }
extern "C" int64_t b2o_tc_coop_n_launches(const b2o_ctx* ctx) { return ctx ? ctx->tc_coop_n_launches : 0; }

extern "C" int b2o_profile_enable(b2o_ctx* ctx, int on) {
  if (!ctx) return B2O_ERR_ARG;
  for (cudaEvent_t e : ctx->prof_events) cudaEventDestroy(e);
  ctx->prof_events.clear();
  ctx->prof_flop = 0.0;
  ctx->profile = on != 0;
  return B2O_OK;
}

extern "C" int b2o_profile_read(b2o_ctx* ctx, double* tc_ms, double* tc_flop, int64_t* tc_launches) {
  if (!ctx || !tc_ms || !tc_flop || !tc_launches) return B2O_ERR_ARG;
  DeviceGuard guard(ctx->device);
  double ms = 0.0;
  for (size_t i = 0; i + 1 < ctx->prof_events.size(); i += 2) {
    B2O_CUDA_CHECK(ctx, cudaEventSynchronize(ctx->prof_events[i + 1]));
    float t = 0.f;
    B2O_CUDA_CHECK(ctx, cudaEventElapsedTime(&t, ctx->prof_events[i], ctx->prof_events[i + 1]));
    ms += t;
  }
  *tc_ms = ms;
  *tc_flop = ctx->prof_flop;
  *tc_launches = static_cast<int64_t>(ctx->prof_events.size() / 2);
  return B2O_OK;
}

extern "C" int b2o_set_conv_engine(b2o_ctx* ctx, int engine) {
  if (!ctx || (engine != B2O_CONV_AUTO && engine != B2O_CONV_SIMT && engine != B2O_CONV_TC_GENERIC)) return B2O_ERR_ARG;
  ctx->conv_engine = engine;
  return B2O_OK;
}

extern "C" int b2o_load_craft(b2o_ctx* ctx, const b2o_tensor* tensors, int n) {
  if (!ctx || !tensors) return B2O_ERR_ARG;
  DeviceGuard guard(ctx->device);
  TensorMap m;
  for (int i = 0; i < n; ++i) m[tensors[i].name] = &tensors[i];
  for (const CraftSpec& s : kCraft) {
    const int64_t wshape[4] = {s.cout, s.cin, s.k, s.k};
    const int64_t vshape[1] = {s.cout};
    const b2o_tensor* w = need(ctx, m, std::string(s.name) + ".weight", 4, wshape);
    const b2o_tensor* b = need(ctx, m, std::string(s.name) + ".bias", 1, vshape);
    if (!w || !b) return B2O_ERR_WEIGHTS;
    std::vector<float> s1 = ones(s.cout), t1 = tovec(b, s.cout);
    if (s.bn) {
      const b2o_tensor* g = need(ctx, m, std::string(s.bn) + ".weight", 1, vshape);
      const b2o_tensor* be = need(ctx, m, std::string(s.bn) + ".bias", 1, vshape);
      const b2o_tensor* mu = need(ctx, m, std::string(s.bn) + ".running_mean", 1, vshape);
      const b2o_tensor* var = need(ctx, m, std::string(s.bn) + ".running_var", 1, vshape);
      if (!g || !be || !mu || !var) return B2O_ERR_WEIGHTS;
      for (int o = 0; o < s.cout; ++o) {      // BN(eps=1e-5) folded around the conv bias (detection.py:95-97)
        const float sc = g->data[o] / sqrtf(var->data[o] + 1e-5f);
        s1[o] = sc;
        t1[o] = (b->data[o] - mu->data[o]) * sc + be->data[o];
      }
    }
    const float* wd = w->data;
    const int cin = s.cin, k = s.k;
    auto wget = [wd, cin, k](int o, int c, int ky, int kx) { return wd[((static_cast<size_t>(o) * cin + c) * k + ky) * k + kx]; };
    ConvLayer& L = ctx->craft[s.name];
    B2O_RETURN_IF(build_layer(ctx, L, s.name, s.cin, s.cout, s.k, s.dil, s.relu, wget, s1, t1, nullptr, nullptr, s.cin == 3));
    // decoder glue: upconvN.conv.0 reads Concatenate([upsampled decoder (cy channels), encoder tap]); the upsampling
    // commutes with this 1x1 convolution, so the layer is also kept as two halves -- ".y": the decoder columns, applied
    // at LOW resolution without bias / BN / ReLU; ".s": the tap columns at full resolution, whose epilogue adds the
    // upsampled ".y" result before the folded BN + ReLU (detection.py:65-84, 380-390)
    int cy = 0;
    if (std::string(s.name) == "upconv2.conv.0") cy = 256;
    if (std::string(s.name) == "upconv3.conv.0") cy = 128;
    if (std::string(s.name) == "upconv4.conv.0") cy = 64;
    if (cy) {
      auto wy = [wd, cin](int o, int c, int, int) { return wd[static_cast<size_t>(o) * cin + c]; };
      auto wsk = [wd, cin, cy](int o, int c, int, int) { return wd[static_cast<size_t>(o) * cin + cy + c]; };
      ConvLayer& Ly = ctx->craft[std::string(s.name) + ".y"];
      B2O_RETURN_IF(build_layer(ctx, Ly, std::string(s.name) + ".y", cy, s.cout, 1, 1, 0, wy, ones(s.cout),
                                std::vector<float>(s.cout, 0.0f), nullptr, nullptr, false));
      ConvLayer& Ls = ctx->craft[std::string(s.name) + ".s"];
      B2O_RETURN_IF(build_layer(ctx, Ls, std::string(s.name) + ".s", s.cin - cy, s.cout, 1, 1, s.relu, wsk, s1, t1, nullptr, nullptr, false));
    }
    if (s.cin == 3) {      // tensor-core stem: same filters over a 16-channel (zero-padded) input
      auto wget16 = [wd, cin, k](int o, int c, int ky, int kx) {
        return c < 3 ? wd[((static_cast<size_t>(o) * cin + c) * k + ky) * k + kx] : 0.0f;
      };
      ConvLayer& L16 = ctx->craft["stem16"];
      B2O_RETURN_IF(build_layer(ctx, L16, "stem16", 16, s.cout, s.k, 1, s.relu, wget16, s1, t1, nullptr, nullptr, false));
      L16.alg_cin = 3;
    }
  }
  ctx->craft_loaded = true;
  return B2O_OK;
}

extern "C" int b2o_load_crnn(b2o_ctx* ctx, const b2o_tensor* tensors, int n) {
  if (!ctx || !tensors) return B2O_ERR_ARG;
  DeviceGuard guard(ctx->device);
  TensorMap m;
  for (int i = 0; i < n; ++i) m[tensors[i].name] = &tensors[i];
  ctx->crnn_written = 0;      // a workspace written with other weights (other classes, no STN) has nothing to tap
  struct Spec { const char* name; int cin, cout, k; const char* bn; };
  const Spec convs[] = {{"conv_1", 1, 64, 3, nullptr},    {"conv_2", 64, 128, 3, nullptr}, {"conv_3", 128, 256, 3, "bn_3"},
                        {"conv_4", 256, 256, 3, nullptr}, {"conv_5", 256, 512, 3, "bn_5"}, {"conv_6", 512, 512, 3, nullptr},
                        {"conv_7", 512, 512, 3, "bn_7"},  {"stn.conv_a", 512, 16, 5, nullptr}, {"stn.conv_b", 16, 32, 5, nullptr}};
  // build_model(stn=False) (recognition.py:196, 243): a checkpoint without the localisation net's tensors is the
  // recognizer without the spatial transformer -- the conv features go straight to the reshape + fc_9
  const bool has_stn = m.count("stn.conv_a.kernel") != 0;
  ctx->crnn_stn = has_stn;
  // build_model(color=True) (recognition.py:214): conv_1 takes 3 input channels (RGB crops, no gray conversion)
  auto c1 = m.find("conv_1.kernel");
  const int in_ch = (c1 != m.end() && c1->second->ndim == 4 && c1->second->shape[2] == 3) ? 3 : 1;
  ctx->crnn_in_ch = in_ch;
  for (const Spec& s0 : convs) {
    Spec s = s0;
    if (std::string(s.name) == "conv_1") s.cin = in_ch;
    if (!has_stn && std::string(s.name).rfind("stn.", 0) == 0) continue;
    const int64_t wshape[4] = {s.k, s.k, s.cin, s.cout};
    const int64_t vshape[1] = {s.cout};
    const b2o_tensor* w = need(ctx, m, std::string(s.name) + ".kernel", 4, wshape);
    const b2o_tensor* b = need(ctx, m, std::string(s.name) + ".bias", 1, vshape);
    if (!w || !b) return B2O_ERR_WEIGHTS;
    std::vector<float> s1 = ones(s.cout), t1 = tovec(b, s.cout), s2, t2;
    if (s.bn) {                                // BatchNormalization AFTER the ReLU, Keras eps = 1e-3
      const b2o_tensor* g = need(ctx, m, std::string(s.bn) + ".gamma", 1, vshape);
      const b2o_tensor* be = need(ctx, m, std::string(s.bn) + ".beta", 1, vshape);
      const b2o_tensor* mu = need(ctx, m, std::string(s.bn) + ".moving_mean", 1, vshape);
      const b2o_tensor* var = need(ctx, m, std::string(s.bn) + ".moving_variance", 1, vshape);
      if (!g || !be || !mu || !var) return B2O_ERR_WEIGHTS;
      s2.resize(s.cout); t2.resize(s.cout);
      for (int o = 0; o < s.cout; ++o) {
        const float sc = g->data[o] / sqrtf(var->data[o] + 1e-3f);
        s2[o] = sc;
        t2[o] = be->data[o] - mu->data[o] * sc;
      }
    }
    const float* wd = w->data;
    const int cin = s.cin, cout = s.cout, k = s.k;
    auto wget = [wd, cin, cout, k](int o, int c, int ky, int kx) {
      return wd[((static_cast<size_t>(ky) * k + kx) * cin + c) * cout + o];
    };
    ConvLayer& L = ctx->crnn[s.name];
    B2O_RETURN_IF(build_layer(ctx, L, s.name, s.cin, s.cout, s.k, 1, 1, wget, s1, t1, s.bn ? &s2 : nullptr,
                              s.bn ? &t2 : nullptr, std::string(s.name) == "conv_1"));
    if (std::string(s.name) == "stn.conv_a") {
      // The 5x5, 512 -> 16 convolution as ONE 1x1 GEMM with N = 25 taps x 16 channels (400, padded to 512)
      // followed by a shift-and-add of the 25 column groups (stn_col2im): 16-column MMAs cost as much tensor
      // pipe time as 64-column ones, 256-column ones are ~5x cheaper per output.
      auto wgemm = [wd, cin, cout, k](int o, int c, int, int) {
        return o < k * k * cout ? wd[(static_cast<size_t>(o / cout) * cin + c) * cout + (o % cout)] : 0.0f;
      };
      ConvLayer& G = ctx->crnn["stn.conv_a_gemm"];
      B2O_RETURN_IF(build_layer(ctx, G, "stn.conv_a_gemm", s.cin, 512, 1, 1, 0, wgemm, ones(512),
                                std::vector<float>(512, 0.0f), nullptr, nullptr, false));
      G.alg_cout = k * k * cout;                 // 400 of the 512 columns are real
    }
  }
  // dense layers as 1x1 "convolutions" over a (1,1,rows,K) view
  struct Dense { const char* name; int k, n, relu; };
  const Dense dense[] = {{"stn.dense_a", 11200, 64, 1}, {"fc_9", 3584, 128, 1}};
  for (const Dense& d : dense) {
    if (!has_stn && std::string(d.name).rfind("stn.", 0) == 0) continue;
    const int64_t wshape[2] = {d.k, d.n};
    const int64_t vshape[1] = {d.n};
    const b2o_tensor* w = need(ctx, m, std::string(d.name) + ".kernel", 2, wshape);
    const b2o_tensor* b = need(ctx, m, std::string(d.name) + ".bias", 1, vshape);
    if (!w || !b) return B2O_ERR_WEIGHTS;
    const float* wd = w->data;
    const int nn = d.n;
    auto wget = [wd, nn](int o, int c, int, int) { return wd[static_cast<size_t>(c) * nn + o]; };
    ConvLayer& L = ctx->crnn[d.name];
    B2O_RETURN_IF(build_layer(ctx, L, d.name, d.k, d.n, 1, 1, d.relu, wget, ones(d.n), tovec(b, d.n), nullptr, nullptr, false));
  }
  if (has_stn) {
    const int64_t wshape[2] = {64, 6};
    const int64_t vshape[1] = {6};
    const b2o_tensor* w = need(ctx, m, "stn.dense_b.kernel", 2, wshape);
    const b2o_tensor* b = need(ctx, m, "stn.dense_b.bias", 1, vshape);
    if (!w || !b) return B2O_ERR_WEIGHTS;
    if (!(ctx->stn_d2_w = dev_upload(ctx, tovec(w, 64 * 6)))) return B2O_ERR_CUDA;
    if (!(ctx->stn_d2_b = dev_upload(ctx, tovec(b, 6)))) return B2O_ERR_CUDA;
  }
  // LSTM input projections: forward and go_backwards kernels side by side -> one GEMM per layer
  const char* lstm_names[4] = {"lstm_10", "lstm_10_back", "lstm_11", "lstm_11_back"};
  for (int layer = 0; layer < 2; ++layer) {
    const int64_t wshape[2] = {128, 512};
    const int64_t vshape[1] = {512};
    const b2o_tensor* wf = need(ctx, m, std::string(lstm_names[2 * layer]) + ".kernel", 2, wshape);
    const b2o_tensor* wb = need(ctx, m, std::string(lstm_names[2 * layer + 1]) + ".kernel", 2, wshape);
    const b2o_tensor* bf = need(ctx, m, std::string(lstm_names[2 * layer]) + ".bias", 1, vshape);
    const b2o_tensor* bb = need(ctx, m, std::string(lstm_names[2 * layer + 1]) + ".bias", 1, vshape);
    if (!wf || !wb || !bf || !bb) return B2O_ERR_WEIGHTS;
    const float* f = wf->data;
    const float* bk = wb->data;
    auto wget = [f, bk](int o, int c, int, int) { return o < 512 ? f[c * 512 + o] : bk[c * 512 + (o - 512)]; };
    std::vector<float> bias(1024);
    for (int i = 0; i < 512; ++i) { bias[i] = bf->data[i]; bias[512 + i] = bb->data[i]; }
    const std::string lname = layer == 0 ? "lstm_in_1" : "lstm_in_2";
    ConvLayer& L = ctx->crnn[lname];
    B2O_RETURN_IF(build_layer(ctx, L, lname, 128, 1024, 1, 1, 0, wget, ones(1024), bias, nullptr, nullptr, false));
    for (int dir = 0; dir < 2; ++dir) {
      const b2o_tensor* u = need(ctx, m, std::string(lstm_names[2 * layer + dir]) + ".recurrent_kernel", 2, wshape);
      if (!u) return B2O_ERR_WEIGHTS;
      std::vector<__half> uh(128 * 512);
      for (int i = 0; i < 128 * 512; ++i) uh[i] = __float2half_rn(u->data[i]);
      if (!(ctx->lstm_u[2 * layer + dir] = dev_upload(ctx, uh))) return B2O_ERR_CUDA;
    }
  }
  {
    // Dense(len(alphabet)+1) (recognition.py:322-327, 376-381): the class count comes from the tensor itself
    auto fc = m.find("fc_12.kernel");
    const int64_t K = fc != m.end() && fc->second->ndim == 2 ? fc->second->shape[1] : 0;
    if (K < 2 || K > B2O_MAX_CLASSES) { ctx->set_error("fc_12.kernel must be (256, K) with 2 <= K <= 1024"); return B2O_ERR_WEIGHTS; }
    const int64_t wshape[2] = {256, K};
    const int64_t vshape[1] = {K};
    const b2o_tensor* w = need(ctx, m, "fc_12.kernel", 2, wshape);
    const b2o_tensor* b = need(ctx, m, "fc_12.bias", 1, vshape);
    if (!w || !b) return B2O_ERR_WEIGHTS;
    if (!(ctx->fc12_w = dev_upload(ctx, tovec(w, 256 * K)))) return B2O_ERR_CUDA;
    if (!(ctx->fc12_b = dev_upload(ctx, tovec(b, K)))) return B2O_ERR_CUDA;
    ctx->n_classes = static_cast<int>(K);
  }
  ctx->crnn_loaded = true;
  return B2O_OK;
}

// ------------------------------------------------------------------------------------------------
extern "C" size_t b2o_craft_workspace_bytes(int n, int h, int w) {
  if (n <= 0 || h < 32 || w < 32) return 0;
  return plan_craft(n, h, w).bytes;
}

extern "C" int b2o_craft_forward_until(b2o_ctx* ctx, const uint8_t* img, int n, int h, int w, float* scores, void* ws,
                                       size_t ws_bytes, int last_step, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  if (!ctx->craft_loaded) { ctx->set_error("b2o_craft_forward: CRAFT weights not loaded"); return B2O_ERR_STATE; }
  DeviceGuard guard(ctx->device);
  if (!img || !scores || !ws || n <= 0 || h < 32 || w < 32 || last_step < 0 || last_step > B2O_CRAFT_LAST_STEP) {
    ctx->set_error("b2o_craft_forward: bad argument");
    return B2O_ERR_ARG;
  }
  // the glue kernels and the conv engine index inside one image's maps with 32-bit integers in places; the largest
  // per-image map is a full-resolution 64-channel one, h * w * 64 elements, which stays below 2^31 up to this bound
  if (static_cast<long long>(h) * w > B2O_CRAFT_MAX_PIXELS) {
    ctx->set_error("b2o_craft_forward: more than 2^25 pixels per image (h * w = " +
                   std::to_string(static_cast<long long>(h) * w) + "); detect a page this large over tiles (tile_size)");
    return B2O_ERR_ARG;
  }
  const CraftPlan p = plan_craft(n, h, w);
  if (ws_bytes < p.bytes) { ctx->set_error("b2o_craft_forward: workspace too small"); return B2O_ERR_WORKSPACE; }
  ctx->craft_step = -1;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  auto V = [&](const Slice& s) { return p.view(ws, s); };
  auto L = [&](const std::string& name) -> const ConvLayer& { return ctx->craft[name]; };
  const bool rgb_stem = ctx->conv_engine == B2O_CONV_SIMT || L("stem16").block_n == 0;     // fp32 CUDA-core stem
  // UpsampleLike + Concatenate + 1x1 conv (380-390).  Opt-in (B2O_UPCONV_COMMUTE=1): where the skip tensor is exactly
  // twice the decoder tensor the upsampling is commuted behind the convolution -- the decoder half of the 1x1 conv runs
  // at LOW resolution and the full-resolution half adds its bilinear upsampling in the epilogue, so no upsampled tensor
  // is written or read back.  Correct (tests) but not the default: the explicit UpsampleLike is what the reference graph runs.
  // z has the decoder tensor's resolution, `full` (a slice of the concat) the skip tensor's.
  auto commuted = [&](const CraftStep& s, const Slice& full) {
    const CraftBuf &y = p.bufs[s.z.buf], &skip = p.bufs[full.buf];
    const std::string base(s.layer);
    return ctx->conv_engine == B2O_CONV_AUTO && !ctx->no_commute && skip.h == 2 * y.h && skip.w == 2 * y.w &&
           L(base + ".y").block_n != 0 && L(base + ".s").kch == 64 && L(base + ".s").block_n >= 64;
  };
  for (int k = 0; k <= last_step; ++k) {
    const CraftStep& s = kCraftSteps[k];
    const TensorView src = V(s.src), out = V(s.out);
    switch (s.kind) {
      case StepKind::normalize:
        if (!rgb_stem) B2O_RETURN_IF(normalize16_run(ctx, img, n, h, w, out.ptr, st));
        break;
      case StepKind::stem:
        B2O_RETURN_IF(rgb_stem ? stem_rgb_run(ctx, L(s.layer), img, n, h, w, out, st)
                               : conv_run(ctx, L("stem16"), src, out, 0, st));
        break;
      case StepKind::conv:
        if (kCraftSteps[k + 1].kind == StepKind::tail) {
          B2O_RETURN_IF(head_conv_run(ctx, L(s.layer), L("conv_cls.6"), L("conv_cls.8"), src, out, scores, st));
        } else {
          const TensorView pool = V(s.pool);      // conv + fused 2x2 max pool
          B2O_RETURN_IF(conv_run(ctx, L(s.layer), src, out, 0, st, s.pool.buf == cb::none ? nullptr : &pool, s.write_full));
        }
        break;
      case StepKind::maxpool3:
        B2O_RETURN_IF(maxpool3s1_run(ctx, src, out, st));
        break;
      case StepKind::level_up:
        B2O_RETURN_IF(commuted(s, s.out) ? conv_run(ctx, L(std::string(s.layer) + ".y"), src, V(s.z), 0, st)
                                         : upsample_run(ctx, src, out, st));
        break;
      case StepKind::level_conv:
        if (commuted(s, s.skip)) {
          const TensorView z = V(s.z);
          B2O_RETURN_IF(conv_tc_run(ctx, L(std::string(s.layer) + ".s"), V(s.skip), out, 0, st, nullptr, 1, nullptr, &z));
        } else {
          B2O_RETURN_IF(conv_run(ctx, L(s.layer), src, out, 0, st));
        }
        break;
      case StepKind::tail:
        if (!tail_fused(ctx, L(kCraftSteps[k - 1].layer)))
          B2O_RETURN_IF(head_tail_run(ctx, L("conv_cls.6"), L("conv_cls.8"), src, scores, st));
        break;
    }
  }
  // the forward stops after step last_step (host side, between launches) and records it for b2o_craft_tap
  ctx->craft_step = last_step;
  ctx->craft_ws = ws; ctx->craft_n = n; ctx->craft_h = h; ctx->craft_w = w;
  return B2O_OK;
}

extern "C" int b2o_craft_forward(b2o_ctx* ctx, const uint8_t* img, int n, int h, int w, float* scores, void* ws,
                                 size_t ws_bytes, void* stream) {
  return b2o_craft_forward_until(ctx, img, n, h, w, scores, ws, ws_bytes, B2O_CRAFT_LAST_STEP, stream);
}

extern "C" int b2o_craft_tap(b2o_ctx* ctx, const char* name, const void* ws, int n, int h, int w, void* out,
                             size_t out_bytes, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  if (!name || !ws || !out || n <= 0 || h < 32 || w < 32) { ctx->set_error("b2o_craft_tap: bad argument"); return B2O_ERR_ARG; }
  // the plan's offsets are only those of the workspace the last forward wrote if the shape and workspace are its own
  if (ctx->craft_step < 0 || ws != ctx->craft_ws || n != ctx->craft_n || h != ctx->craft_h || w != ctx->craft_w) {
    ctx->set_error("b2o_craft_tap: ws, n, h, w are not those of the last successful forward of this context");
    return B2O_ERR_STATE;
  }
  DeviceGuard guard(ctx->device);
  const CraftPlan p = plan_craft(n, h, w);
  for (int i = 0; i < cb::count; ++i) {
    if (std::string(name) != kCraftBufs[i].name) continue;
    const CraftBuf& b = p.bufs[i];
    const size_t bytes = static_cast<size_t>(n) * b.h * b.w * kCraftBufs[i].c * 2;
    if (out_bytes < bytes) { ctx->set_error("b2o_craft_tap: output too small"); return B2O_ERR_ARG; }
    if (ctx->craft_step < b.first || ctx->craft_step > b.last) {
      ctx->set_error(std::string("b2o_craft_tap: ") + name + " is not live after the last forward's step");
      return B2O_ERR_STATE;
    }
    B2O_CUDA_CHECK(ctx, cudaMemcpyAsync(out, reinterpret_cast<const uint8_t*>(ws) + b.off, bytes, cudaMemcpyDeviceToDevice,
                                        reinterpret_cast<cudaStream_t>(stream)));
    return B2O_OK;
  }
  ctx->set_error(std::string("b2o_craft_tap: unknown buffer ") + name);
  return B2O_ERR_ARG;
}

// ------------------------------------------------------------------------------------------------
extern "C" size_t b2o_crnn_workspace_bytes(int b) { return b > 0 ? plan_crnn(b).bytes : 0; }

extern "C" int b2o_crnn_forward(b2o_ctx* ctx, const void* crnn_in, int b, int32_t* labels, void* ws, size_t ws_bytes,
                                void* stream) {
  return b2o_crnn_forward_scored(ctx, crnn_in, b, labels, nullptr, ws, ws_bytes, stream);
}

namespace {

// The CRNN through fc_12 + greedy CTC.  keep_logits: the fp32 logits always go to the workspace's logits slot (the beam
// search reads them there); otherwise only with the debug taps on.  features (b2o_crnn_features): the forward stops
// after the BiLSTM and copies its 48 kept steps (b, 48, 256) fp16 there instead of running fc_12 + CTC (labels unused).
// seq (b2o_crnn_sequence_features): the forward stops after fc_9 and copies it, (b, 50, 128) fp16, there.
int crnn_forward(b2o_ctx* ctx, const void* crnn_in, int b, int32_t* labels, float* logp, bool keep_logits, void* ws,
                 size_t ws_bytes, void* stream, __half* features = nullptr, __half* seq = nullptr) {
  if (!ctx) return B2O_ERR_ARG;
  if (!ctx->crnn_loaded) { ctx->set_error("b2o_crnn_forward: CRNN weights not loaded"); return B2O_ERR_STATE; }
  DeviceGuard guard(ctx->device);
  if (b == 0) return B2O_OK;
  if (!crnn_in || (!labels && !features && !seq) || !ws || b < 0) {
    ctx->set_error("b2o_crnn_forward: bad argument");
    return B2O_ERR_ARG;
  }
  const CrnnPlan p = plan_crnn(b);
  if (ws_bytes < p.bytes) { ctx->set_error("b2o_crnn_forward: workspace too small"); return B2O_ERR_WORKSPACE; }
  ctx->crnn_written = 0;      // from here on the slots hold neither the last forward's values nor this one's
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  uint8_t* base = reinterpret_cast<uint8_t*>(ws);
  auto at = [&](rb::Id i) { return base + p.off[i]; };
  auto V = [&](rb::Id i, int nn, int hh, int ww, int c) { return make_view(at(i), nn, hh, ww, c); };
  auto L = [&](const char* name) -> const ConvLayer& { return ctx->crnn[name]; };
  // the slots this forward writes, recorded on success for b2o_crnn_tap / b2o_crnn_align
  auto bit = [](rb::Id i) { return 1u << i; };
  const bool logits_kept = !features && !seq && (keep_logits || ctx->debug_taps);
  const uint32_t wrote = bit(rb::x1) | bit(rb::x2) | (conv_pool_fused(ctx, L("conv_3")) ? 0u : bit(rb::x3)) | bit(rb::p3) |
                         bit(rb::x4) | (conv_pool_fused(ctx, L("conv_5")) ? 0u : bit(rb::x5)) | bit(rb::p5) | bit(rb::x6) |
                         bit(rb::features) | (ctx->crnn_stn ? bit(rb::theta) | bit(rb::warped) : 0u) | bit(rb::fc_9) |
                         (seq ? 0u : bit(rb::l1) | bit(rb::l2)) | (logits_kept ? bit(rb::logits) : 0u);
  auto record = [&]() {
    ctx->crnn_ws = ws; ctx->crnn_b = b; ctx->crnn_written = wrote;
    return B2O_OK;
  };
  const TensorView x1 = V(rb::x1, b, 200, 31, 64), x2 = V(rb::x2, b, 200, 31, 128), x3 = V(rb::x3, b, 200, 31, 256);
  const TensorView p3 = V(rb::p3, b, 100, 15, 256), x4 = V(rb::x4, b, 100, 15, 256), x5 = V(rb::x5, b, 100, 15, 512);
  const TensorView p5 = V(rb::p5, b, 50, 7, 512), x6 = V(rb::x6, b, 50, 7, 512), x7 = V(rb::features, b, 50, 7, 512);
  const TensorView sa = V(rb::sa, b, 50, 7, 16), sb = V(rb::sb, b, 50, 7, 32);
  // conv stack (recognition.py:217-242)
  B2O_RETURN_IF(stem_crnn_run(ctx, L("conv_1"), reinterpret_cast<const __half*>(crnn_in), b, x1, st));
  B2O_RETURN_IF(conv_run(ctx, L("conv_2"), x1, x2, 0, st));
  B2O_RETURN_IF(conv_run(ctx, L("conv_3"), x2, x3, 0, st, &p3, 0));
  B2O_RETURN_IF(conv_run(ctx, L("conv_4"), p3, x4, 0, st));
  B2O_RETURN_IF(conv_run(ctx, L("conv_5"), x4, x5, 0, st, &p5, 0));
  B2O_RETURN_IF(conv_run(ctx, L("conv_6"), p5, x6, 0, st));
  B2O_RETURN_IF(conv_run(ctx, L("conv_7"), x6, x7, 0, st));
  __half* warped = reinterpret_cast<__half*>(at(rb::warped));
  if (!ctx->crnn_stn) {
    warped = x7.ptr;                                      // stn=False: Reshape consumes bn_7's output directly (282)
  } else {
  // spatial transformer (263-281)
  if (ctx->conv_engine == B2O_CONV_AUTO && L("stn.conv_a_gemm").block_n != 0) {
    const TensorView y = V(rb::warped, b, 50, 7, 512);   // the warp buffer is free until stn_sample
    B2O_RETURN_IF(conv_run(ctx, L("stn.conv_a_gemm"), x7, y, 0, st));
    B2O_RETURN_IF(stn_col2im_run(ctx, y.ptr, L("stn.conv_a").t1, b, sa.ptr, st));
  } else {
    B2O_RETURN_IF(conv_run(ctx, L("stn.conv_a"), x7, sa, 0, st));
  }
  B2O_RETURN_IF(conv_run(ctx, L("stn.conv_b"), sa, sb, 0, st));
  const TensorView sb_flat = V(rb::sb, 1, 1, b, 11200), d1 = V(rb::d1, 1, 1, b, 64);
  B2O_RETURN_IF(conv_run(ctx, L("stn.dense_a"), sb_flat, d1, 0, st));
  float* theta = reinterpret_cast<float*>(at(rb::theta));
  B2O_RETURN_IF(stn_theta_run(ctx, d1.ptr, b, theta, st));
  B2O_RETURN_IF(stn_sample_run(ctx, x7.ptr, theta, b, warped, st));
  }
  // reshape + fc_9 (282-290)
  const TensorView seq_in = make_view(warped, 1, 1, b * 50, 3584), fc9 = V(rb::fc_9, 1, 1, b * 50, 128);
  B2O_RETURN_IF(conv_run(ctx, L("fc_9"), seq_in, fc9, 0, st));
  if (seq) {
    B2O_CUDA_CHECK(ctx, cudaMemcpyAsync(seq, fc9.ptr, static_cast<size_t>(b) * 50 * 128 * sizeof(__half),
                                        cudaMemcpyDeviceToDevice, st));
    return record();
  }
  // BiLSTM (292-319)
  const TensorView xw1 = V(rb::xw1, 1, 1, b * 50, 1024);
  TensorView xw1v = xw1;      // fp32 output: the view's pointer arithmetic is done by the engine in floats
  B2O_RETURN_IF(conv_run(ctx, L("lstm_in_1"), fc9, xw1v, 1, st));
  __half* hf = reinterpret_cast<__half*>(at(rb::hf));
  __half* hb = reinterpret_cast<__half*>(at(rb::hb));
  __half* l1 = reinterpret_cast<__half*>(at(rb::l1));
  const float* xw1f = reinterpret_cast<const float*>(at(rb::xw1));
  B2O_RETURN_IF(lstm_run(ctx, xw1f, 1024, 0, ctx->lstm_u[0], b, 0, hf, 128, 0, st));
  B2O_RETURN_IF(lstm_run(ctx, xw1f, 1024, 512, ctx->lstm_u[1], b, 1, hb, 128, 0, st));
  B2O_RETURN_IF(add_run(ctx, hf, hb, l1, static_cast<long long>(b) * 50 * 128, st));
  const TensorView l1v = make_view(l1, 1, 1, b * 50, 128), xw2 = V(rb::xw2, 1, 1, b * 50, 1024);
  B2O_RETURN_IF(conv_run(ctx, L("lstm_in_2"), l1v, xw2, 1, st));
  const float* xw2f = reinterpret_cast<const float*>(at(rb::xw2));
  __half* l2 = reinterpret_cast<__half*>(at(rb::l2));
  B2O_RETURN_IF(lstm_run(ctx, xw2f, 1024, 0, ctx->lstm_u[2], b, 0, l2, 256, 0, st));
  B2O_RETURN_IF(lstm_run(ctx, xw2f, 1024, 512, ctx->lstm_u[3], b, 1, l2, 256, 128, st));
  if (features) {            // rnn_steps_to_discard = 2 (recognition.py:328): steps 2..49 of every crop
    B2O_CUDA_CHECK(ctx, cudaMemcpy2DAsync(features, 48 * 256 * sizeof(__half), l2 + 2 * 256, 50 * 256 * sizeof(__half),
                                          48 * 256 * sizeof(__half), b, cudaMemcpyDeviceToDevice, st));
    return record();
  }
  // fc_12 + discard + greedy CTC (321-333)
  B2O_RETURN_IF(fc_ctc_run(ctx, l2, b, logits_kept ? reinterpret_cast<float*>(at(rb::logits)) : nullptr, labels, logp, st));
  return record();
}

bool beam_args_ok(b2o_ctx* ctx, const char* fn, int k, int beam_width, int top_paths) {
  if (k < 2 || k > B2O_MAX_CLASSES) { ctx->set_error(std::string(fn) + ": k must be in [2, 1024]"); return false; }
  if (beam_width < 1 || beam_width > B2O_MAX_BEAM_WIDTH) {
    ctx->set_error(std::string(fn) + ": beam_width must be in [1, 128]");
    return false;
  }
  if (top_paths < 1 || top_paths > beam_width) {
    ctx->set_error(std::string(fn) + ": top_paths must be in [1, beam_width]");
    return false;
  }
  return true;
}

}  // namespace

extern "C" int b2o_crnn_forward_scored(b2o_ctx* ctx, const void* crnn_in, int b, int32_t* labels, float* logp, void* ws,
                                       size_t ws_bytes, void* stream) {
  return crnn_forward(ctx, crnn_in, b, labels, logp, false, ws, ws_bytes, stream);
}

extern "C" int b2o_crnn_forward_beam(b2o_ctx* ctx, const void* crnn_in, int b, int beam_width, int top_paths,
                                     int32_t* labels, float* logp, void* ws, size_t ws_bytes, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  if (!ctx->crnn_loaded) { ctx->set_error("b2o_crnn_forward_beam: CRNN weights not loaded"); return B2O_ERR_STATE; }
  if (!beam_args_ok(ctx, "b2o_crnn_forward_beam", ctx->n_classes, beam_width, top_paths)) return B2O_ERR_ARG;
  if (b == 0) return B2O_OK;
  // the greedy labels of fc_ctc_kernel go to the first b * 48 entries of `labels`, which the beam search then overwrites
  B2O_RETURN_IF(crnn_forward(ctx, crnn_in, b, labels, nullptr, true, ws, ws_bytes, stream));
  DeviceGuard guard(ctx->device);
  const float* logits = reinterpret_cast<const float*>(reinterpret_cast<uint8_t*>(ws) + plan_crnn(b).off[rb::logits]);
  return ctc_beam_run(ctx, logits, b, ctx->n_classes, beam_width, top_paths, labels, logp,
                      reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int b2o_ctc_beam_decode(b2o_ctx* ctx, const float* logits, int b, int k, int beam_width, int top_paths,
                                   int32_t* labels, float* logp, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  if (!beam_args_ok(ctx, "b2o_ctc_beam_decode", k, beam_width, top_paths)) return B2O_ERR_ARG;
  if (b < 0 || (b > 0 && (!logits || !labels))) { ctx->set_error("b2o_ctc_beam_decode: bad argument"); return B2O_ERR_ARG; }
  DeviceGuard guard(ctx->device);
  return ctc_beam_run(ctx, logits, b, k, beam_width, top_paths, labels, logp, reinterpret_cast<cudaStream_t>(stream));
}

namespace {

bool lm_args_ok(b2o_ctx* ctx, const char* fn, int k, int beam_width, int top_paths, const b2o_char_lm* lm) {
  if (!beam_args_ok(ctx, fn, k, beam_width, top_paths)) return false;
  if (k > B2O_MAX_LM_CLASSES) { ctx->set_error(std::string(fn) + ": k must be in [2, 127]"); return false; }
  if (!lm || !lm->keys_dev || !lm->rows_dev) { ctx->set_error(std::string(fn) + ": no language model"); return false; }
  if (lm->order < 2 || lm->order > B2O_MAX_LM_ORDER) {
    ctx->set_error(std::string(fn) + ": order must be in [2, 8]");
    return false;
  }
  if (lm->n_histories < 1 || lm->n_histories > B2O_MAX_LM_HISTORIES) {
    ctx->set_error(std::string(fn) + ": n_histories must be in [1, 2^20]");
    return false;
  }
  if (!std::isfinite(lm->alpha) || !std::isfinite(lm->beta)) {
    ctx->set_error(std::string(fn) + ": alpha and beta must be finite");
    return false;
  }
  return true;
}

}  // namespace

extern "C" int b2o_crnn_forward_beam_lm(b2o_ctx* ctx, const void* crnn_in, int b, int beam_width, int top_paths,
                                        const b2o_char_lm* lm, int32_t* labels, float* logp, float* fused, void* ws,
                                        size_t ws_bytes, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  if (!ctx->crnn_loaded) { ctx->set_error("b2o_crnn_forward_beam_lm: CRNN weights not loaded"); return B2O_ERR_STATE; }
  if (!lm_args_ok(ctx, "b2o_crnn_forward_beam_lm", ctx->n_classes, beam_width, top_paths, lm)) return B2O_ERR_ARG;
  if (b == 0) return B2O_OK;
  B2O_RETURN_IF(crnn_forward(ctx, crnn_in, b, labels, nullptr, true, ws, ws_bytes, stream));
  DeviceGuard guard(ctx->device);
  const float* logits = reinterpret_cast<const float*>(reinterpret_cast<uint8_t*>(ws) + plan_crnn(b).off[rb::logits]);
  return ctc_beam_lm_run(ctx, logits, b, ctx->n_classes, beam_width, top_paths, lm, labels, logp, fused,
                         reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int b2o_ctc_beam_lm_decode(b2o_ctx* ctx, const float* logits, int b, int k, int beam_width, int top_paths,
                                      const b2o_char_lm* lm, int32_t* labels, float* logp, float* fused, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  if (!lm_args_ok(ctx, "b2o_ctc_beam_lm_decode", k, beam_width, top_paths, lm)) return B2O_ERR_ARG;
  if (b < 0 || (b > 0 && (!logits || !labels))) {
    ctx->set_error("b2o_ctc_beam_lm_decode: bad argument");
    return B2O_ERR_ARG;
  }
  DeviceGuard guard(ctx->device);
  return ctc_beam_lm_run(ctx, logits, b, k, beam_width, top_paths, lm, labels, logp, fused,
                         reinterpret_cast<cudaStream_t>(stream));
}

namespace {

bool hotword_args_ok(b2o_ctx* ctx, const char* fn, int k, int beam_width, int top_paths, const b2o_char_lm* lm,
                     const b2o_hotwords* hw) {
  if (lm) {
    if (!lm_args_ok(ctx, fn, k, beam_width, top_paths, lm)) return false;
  } else {
    if (!beam_args_ok(ctx, fn, k, beam_width, top_paths)) return false;
    if (k > B2O_MAX_LM_CLASSES) { ctx->set_error(std::string(fn) + ": k must be in [2, 127]"); return false; }
  }
  if (!hw) { ctx->set_error(std::string(fn) + ": no hotwords"); return false; }
  if (hw->n_nodes < 1 || hw->n_nodes > B2O_MAX_HOTWORD_NODES || hw->n_edges != hw->n_nodes - 1) {
    ctx->set_error(std::string(fn) + ": n_nodes must be in [1, 2^24 + 1] and n_edges = n_nodes - 1");
    return false;
  }
  if (!hw->final_dev || (hw->n_edges > 0 && (!hw->keys_dev || !hw->child_dev))) {
    ctx->set_error(std::string(fn) + ": missing trie arrays");
    return false;
  }
  if (!std::isfinite(hw->weight) || hw->weight < 0.f) {
    ctx->set_error(std::string(fn) + ": weight must be finite and >= 0");
    return false;
  }
  return true;
}

// The model of b2o_ctc_beam_hotword_decode without one: order 2, one empty-history row of zeros, alpha = beta = 0,
// which makes the language-model search plain beam search bit for bit.  Uploaded once per context.
const b2o_char_lm* zero_lm(b2o_ctx* ctx) {
  if (!ctx->zero_lm.keys_dev) {
    const uint64_t* keys = dev_upload(ctx, std::vector<uint64_t>(1, 0));
    const float* rows = keys ? dev_upload(ctx, std::vector<float>(B2O_MAX_LM_CLASSES, 0.f)) : nullptr;
    if (!rows) return nullptr;
    ctx->zero_lm = b2o_char_lm{2, 1, keys, rows, 0.f, 0.f};
  }
  return &ctx->zero_lm;
}

}  // namespace

extern "C" int b2o_crnn_forward_beam_hotword(b2o_ctx* ctx, const void* crnn_in, int b, int beam_width, int top_paths,
                                             const b2o_char_lm* lm, const b2o_hotwords* hw, int32_t* labels,
                                             float* logp, float* fused, void* ws, size_t ws_bytes, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  if (!ctx->crnn_loaded) {
    ctx->set_error("b2o_crnn_forward_beam_hotword: CRNN weights not loaded");
    return B2O_ERR_STATE;
  }
  if (!hotword_args_ok(ctx, "b2o_crnn_forward_beam_hotword", ctx->n_classes, beam_width, top_paths, lm, hw))
    return B2O_ERR_ARG;
  if (b == 0) return B2O_OK;
  DeviceGuard guard(ctx->device);
  const b2o_char_lm* model = lm ? lm : zero_lm(ctx);
  if (!model) return B2O_ERR_CUDA;
  B2O_RETURN_IF(crnn_forward(ctx, crnn_in, b, labels, nullptr, true, ws, ws_bytes, stream));
  const float* logits = reinterpret_cast<const float*>(reinterpret_cast<uint8_t*>(ws) + plan_crnn(b).off[rb::logits]);
  return ctc_beam_hotword_run(ctx, logits, b, ctx->n_classes, beam_width, top_paths, model, hw, labels, logp, fused,
                              reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int b2o_ctc_beam_hotword_decode(b2o_ctx* ctx, const float* logits, int b, int k, int beam_width,
                                           int top_paths, const b2o_char_lm* lm, const b2o_hotwords* hw,
                                           int32_t* labels, float* logp, float* fused, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  if (!hotword_args_ok(ctx, "b2o_ctc_beam_hotword_decode", k, beam_width, top_paths, lm, hw)) return B2O_ERR_ARG;
  if (b < 0 || (b > 0 && (!logits || !labels))) {
    ctx->set_error("b2o_ctc_beam_hotword_decode: bad argument");
    return B2O_ERR_ARG;
  }
  if (b == 0) return B2O_OK;
  DeviceGuard guard(ctx->device);
  const b2o_char_lm* model = lm ? lm : zero_lm(ctx);
  if (!model) return B2O_ERR_CUDA;
  return ctc_beam_hotword_run(ctx, logits, b, k, beam_width, top_paths, model, hw, labels, logp, fused,
                              reinterpret_cast<cudaStream_t>(stream));
}

namespace {

bool pattern_args_ok(b2o_ctx* ctx, const char* fn, int k, int beam_width, int top_paths, const b2o_pattern* pat) {
  if (!beam_args_ok(ctx, fn, k, beam_width, top_paths)) return false;
  if (k > B2O_MAX_PATTERN_CLASSES) { ctx->set_error(std::string(fn) + ": k must be in [2, 127]"); return false; }
  if (!pat || !pat->trans_dev || !pat->dist_dev) { ctx->set_error(std::string(fn) + ": no pattern"); return false; }
  if (pat->n_states < 1 || pat->n_states > B2O_MAX_PATTERN_STATES) {
    ctx->set_error(std::string(fn) + ": n_states must be in [1, 4096]");
    return false;
  }
  if (pat->start < 0 || pat->start >= pat->n_states) {
    ctx->set_error(std::string(fn) + ": start must be in [0, n_states)");
    return false;
  }
  return true;
}

}  // namespace

extern "C" int b2o_crnn_forward_beam_pattern(b2o_ctx* ctx, const void* crnn_in, int b, int beam_width, int top_paths,
                                             const b2o_pattern* pattern, int32_t* labels, float* logp, void* ws,
                                             size_t ws_bytes, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  if (!ctx->crnn_loaded) {
    ctx->set_error("b2o_crnn_forward_beam_pattern: CRNN weights not loaded");
    return B2O_ERR_STATE;
  }
  if (!pattern_args_ok(ctx, "b2o_crnn_forward_beam_pattern", ctx->n_classes, beam_width, top_paths, pattern))
    return B2O_ERR_ARG;
  if (b == 0) return B2O_OK;
  B2O_RETURN_IF(crnn_forward(ctx, crnn_in, b, labels, nullptr, true, ws, ws_bytes, stream));
  DeviceGuard guard(ctx->device);
  const float* logits = reinterpret_cast<const float*>(reinterpret_cast<uint8_t*>(ws) + plan_crnn(b).off[rb::logits]);
  return ctc_beam_pattern_run(ctx, logits, b, ctx->n_classes, beam_width, top_paths, pattern, labels, logp,
                              reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int b2o_ctc_beam_pattern_decode(b2o_ctx* ctx, const float* logits, int b, int k, int beam_width,
                                           int top_paths, const b2o_pattern* pattern, int32_t* labels, float* logp,
                                           void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  if (!pattern_args_ok(ctx, "b2o_ctc_beam_pattern_decode", k, beam_width, top_paths, pattern)) return B2O_ERR_ARG;
  if (b < 0 || (b > 0 && (!logits || !labels))) {
    ctx->set_error("b2o_ctc_beam_pattern_decode: bad argument");
    return B2O_ERR_ARG;
  }
  DeviceGuard guard(ctx->device);
  return ctc_beam_pattern_run(ctx, logits, b, k, beam_width, top_paths, pattern, labels, logp,
                              reinterpret_cast<cudaStream_t>(stream));
}

namespace {

bool lexicon_args_ok(b2o_ctx* ctx, const char* fn, int k, int n_words, int top_paths) {
  if (k < 2 || k > B2O_MAX_CLASSES) { ctx->set_error(std::string(fn) + ": k must be in [2, 1024]"); return false; }
  if (n_words < 1 || n_words > B2O_MAX_LEXICON_WORDS) {
    ctx->set_error(std::string(fn) + ": n_words must be in [1, 2^20]");
    return false;
  }
  if (top_paths < 1 || top_paths > B2O_MAX_LEXICON_TOP_PATHS) {
    ctx->set_error(std::string(fn) + ": top_paths must be in [1, 128]");
    return false;
  }
  return true;
}

}  // namespace

extern "C" size_t b2o_lexicon_workspace_bytes(int b, int n_words, int top_paths) {
  if (b <= 0 || n_words < 1 || n_words > B2O_MAX_LEXICON_WORDS || top_paths < 1) return 0;
  return ctc_lexicon_workspace_bytes(b, n_words);
}

extern "C" int b2o_ctc_lexicon_decode(b2o_ctx* ctx, const float* logits, int b, int k, const int32_t* offsets,
                                      const int16_t* labels, int n_words, int top_paths, int32_t* labels_out,
                                      float* logp, void* ws, size_t ws_bytes, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  if (!lexicon_args_ok(ctx, "b2o_ctc_lexicon_decode", k, n_words, top_paths)) return B2O_ERR_ARG;
  if (b < 0 || (b > 0 && (!logits || !offsets || !labels || !labels_out || !ws))) {
    ctx->set_error("b2o_ctc_lexicon_decode: bad argument");
    return B2O_ERR_ARG;
  }
  if (b == 0) return B2O_OK;
  if (ws_bytes < ctc_lexicon_workspace_bytes(b, n_words)) {
    ctx->set_error("b2o_ctc_lexicon_decode: workspace too small");
    return B2O_ERR_WORKSPACE;
  }
  DeviceGuard guard(ctx->device);
  return ctc_lexicon_run(ctx, logits, b, k, offsets, labels, n_words, top_paths, labels_out, logp, ws,
                         reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int b2o_crnn_forward_lexicon(b2o_ctx* ctx, const void* crnn_in, int b, const int32_t* offsets,
                                        const int16_t* labels, int n_words, int top_paths, int32_t* labels_out,
                                        float* logp, void* ws, size_t ws_bytes, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  if (!ctx->crnn_loaded) { ctx->set_error("b2o_crnn_forward_lexicon: CRNN weights not loaded"); return B2O_ERR_STATE; }
  if (!lexicon_args_ok(ctx, "b2o_crnn_forward_lexicon", ctx->n_classes, n_words, top_paths)) return B2O_ERR_ARG;
  if (b < 0 || (b > 0 && (!crnn_in || !offsets || !labels || !labels_out || !ws))) {
    ctx->set_error("b2o_crnn_forward_lexicon: bad argument");
    return B2O_ERR_ARG;
  }
  if (b == 0) return B2O_OK;
  const CrnnPlan p = plan_crnn(b);
  const size_t scratch = p.bytes;           // the decoder's scratch follows the CRNN's buffers, 256-byte aligned
  if (ws_bytes < scratch + ctc_lexicon_workspace_bytes(b, n_words)) {
    ctx->set_error("b2o_crnn_forward_lexicon: workspace too small");
    return B2O_ERR_WORKSPACE;
  }
  // the greedy labels of fc_ctc_kernel go to the first b * 48 entries of `labels_out`, which the decoder then overwrites
  B2O_RETURN_IF(crnn_forward(ctx, crnn_in, b, labels_out, nullptr, true, ws, ws_bytes, stream));
  DeviceGuard guard(ctx->device);
  uint8_t* base = reinterpret_cast<uint8_t*>(ws);
  const float* logits = reinterpret_cast<const float*>(base + p.off[rb::logits]);
  return ctc_lexicon_run(ctx, logits, b, ctx->n_classes, offsets, labels, n_words, top_paths, labels_out, logp,
                         base + scratch, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int b2o_crnn_forward_logits(b2o_ctx* ctx, const void* crnn_in, int b, int32_t* labels, float* logp, void* ws,
                                       size_t ws_bytes, void* stream) {
  return crnn_forward(ctx, crnn_in, b, labels, logp, true, ws, ws_bytes, stream);
}

extern "C" int b2o_crnn_features(b2o_ctx* ctx, const void* crnn_in, int b, void* features, void* ws, size_t ws_bytes,
                                 void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  if (b > 0 && !features) { ctx->set_error("b2o_crnn_features: bad argument"); return B2O_ERR_ARG; }
  return crnn_forward(ctx, crnn_in, b, nullptr, nullptr, false, ws, ws_bytes, stream, reinterpret_cast<__half*>(features));
}

extern "C" size_t b2o_ctc_train_workspace_bytes(int b, int k) {
  if (b <= 0 || k < 2 || k > B2O_MAX_CLASSES) return 0;
  return ctc_train_workspace_bytes(b, k);
}

extern "C" int b2o_ctc_loss_grad(b2o_ctx* ctx, const void* features, int n_rows, const int32_t* index, int b, int k,
                                 const float* w, const float* bias, const int32_t* offsets, const int16_t* labels,
                                 float dropout, uint64_t seed, uint64_t step, float* loss, float* grad_w, float* grad_b,
                                 float* logits, void* ws, size_t ws_bytes, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  const char* fn = "b2o_ctc_loss_grad";
  if (k < 2 || k > B2O_MAX_CLASSES) { ctx->set_error(std::string(fn) + ": k must be in [2, 1024]"); return B2O_ERR_ARG; }
  if (!(dropout >= 0.f && dropout < 1.f)) { ctx->set_error(std::string(fn) + ": dropout must be in [0, 1)"); return B2O_ERR_ARG; }
  if (b < 0 || (b > 0 && (!features || n_rows <= 0 || !w || !bias || !offsets || !labels || !loss)) ||
      (!grad_w) != (!grad_b) || (reinterpret_cast<uintptr_t>(features) & 15)) {
    ctx->set_error(std::string(fn) + ": bad argument");
    return B2O_ERR_ARG;
  }
  if (b == 0) return B2O_OK;
  if (grad_w && (!ws || ws_bytes < ctc_train_workspace_bytes(b, k))) {
    ctx->set_error(std::string(fn) + ": workspace too small");
    return B2O_ERR_WORKSPACE;
  }
  DeviceGuard guard(ctx->device);
  return ctc_loss_grad_run(ctx, reinterpret_cast<const __half*>(features), 48 * 256, false, n_rows, index, b, k, w, bias,
                           offsets, labels, dropout, seed, step, loss, grad_w, grad_b, logits, ws,
                           reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int b2o_rmsprop_step(b2o_ctx* ctx, float* param, const float* grad, float* acc, int64_t n, float lr, float rho,
                                float eps, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  if (n < 0 || (n > 0 && (!param || !grad || !acc)) || !(lr >= 0.f) || !(rho >= 0.f && rho <= 1.f) || !(eps >= 0.f)) {
    ctx->set_error("b2o_rmsprop_step: bad argument");
    return B2O_ERR_ARG;
  }
  DeviceGuard guard(ctx->device);
  return rmsprop_run(ctx, param, grad, acc, n, lr, rho, eps, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int b2o_crnn_set_top(b2o_ctx* ctx, const float* w, const float* bias, int k, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  if (!ctx->crnn_loaded) { ctx->set_error("b2o_crnn_set_top: CRNN weights not loaded"); return B2O_ERR_STATE; }
  if (!w || !bias || k != ctx->n_classes) {
    ctx->set_error("b2o_crnn_set_top: w, bias must be given and k must equal the loaded class count");
    return B2O_ERR_ARG;
  }
  DeviceGuard guard(ctx->device);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  B2O_CUDA_CHECK(ctx, cudaMemcpyAsync(ctx->fc12_w, w, static_cast<size_t>(256) * k * sizeof(float), cudaMemcpyDeviceToDevice, st));
  B2O_CUDA_CHECK(ctx, cudaMemcpyAsync(ctx->fc12_b, bias, static_cast<size_t>(k) * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return B2O_OK;
}

extern "C" int b2o_crnn_sequence_features(b2o_ctx* ctx, const void* crnn_in, int b, void* out, void* ws, size_t ws_bytes,
                                          void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  if (b > 0 && !out) { ctx->set_error("b2o_crnn_sequence_features: bad argument"); return B2O_ERR_ARG; }
  return crnn_forward(ctx, crnn_in, b, nullptr, nullptr, false, ws, ws_bytes, stream, nullptr,
                      reinterpret_cast<__half*>(out));
}

extern "C" size_t b2o_rnn_train_workspace_bytes(int b, int k) {
  if (b <= 0 || k < 2 || k > B2O_MAX_CLASSES) return 0;
  return rnn_train_workspace_bytes(b, k);
}

extern "C" int b2o_rnn_loss_grad(b2o_ctx* ctx, const void* x, int n_rows, const int32_t* index, int b, int k,
                                 const float* params, const int32_t* offsets, const int16_t* labels, float dropout,
                                 uint64_t seed, uint64_t step, float* loss, float* grad, void* ws, size_t ws_bytes,
                                 void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  const char* fn = "b2o_rnn_loss_grad";
  if (k < 2 || k > B2O_MAX_CLASSES) { ctx->set_error(std::string(fn) + ": k must be in [2, 1024]"); return B2O_ERR_ARG; }
  if (!(dropout >= 0.f && dropout < 1.f)) { ctx->set_error(std::string(fn) + ": dropout must be in [0, 1)"); return B2O_ERR_ARG; }
  if (b < 0 || (b > 0 && (!x || n_rows <= 0 || !params || !offsets || !labels || !loss)) ||
      (reinterpret_cast<uintptr_t>(x) & 15)) {
    ctx->set_error(std::string(fn) + ": bad argument");
    return B2O_ERR_ARG;
  }
  if (b == 0) return B2O_OK;
  if (!ws || ws_bytes < rnn_train_workspace_bytes(b, k)) {
    ctx->set_error(std::string(fn) + ": workspace too small");
    return B2O_ERR_WORKSPACE;
  }
  DeviceGuard guard(ctx->device);
  return rnn_loss_grad_run(ctx, reinterpret_cast<const __half*>(x), n_rows, index, b, k, params, offsets, labels, dropout,
                           seed, step, loss, grad, ws, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int b2o_crnn_align(b2o_ctx* ctx, int b, const int32_t* labels_dev, int top_paths, int32_t* spans_dev,
                              float* logp_dev, float* theta_dev, const void* ws, size_t ws_bytes, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  if (!ctx->crnn_loaded) { ctx->set_error("b2o_crnn_align: CRNN weights not loaded"); return B2O_ERR_STATE; }
  if (top_paths < 1 || top_paths > B2O_MAX_ALIGN_PATHS || b < 0 || (b > 0 && (!labels_dev || !spans_dev || !ws))) {
    ctx->set_error("b2o_crnn_align: bad argument");
    return B2O_ERR_ARG;
  }
  if (b == 0) return B2O_OK;
  const CrnnPlan p = plan_crnn(b);
  if (ws_bytes < p.bytes) { ctx->set_error("b2o_crnn_align: workspace too small"); return B2O_ERR_WORKSPACE; }
  if (!crnn_wrote(ctx, rb::logits, ws, b)) {
    ctx->set_error("b2o_crnn_align: the last successful CRNN forward of this context did not keep its logits in this ws "
                   "with this b");
    return B2O_ERR_STATE;
  }
  DeviceGuard guard(ctx->device);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const uint8_t* base = reinterpret_cast<const uint8_t*>(ws);
  if (theta_dev && ctx->crnn_stn)
    B2O_CUDA_CHECK(ctx, cudaMemcpyAsync(theta_dev, base + p.off[rb::theta], static_cast<size_t>(b) * 6 * sizeof(float),
                                        cudaMemcpyDeviceToDevice, st));
  return ctc_align_run(ctx, reinterpret_cast<const float*>(base + p.off[rb::logits]), b, ctx->n_classes, labels_dev, top_paths,
                       spans_dev, logp_dev, st);
}

extern "C" int b2o_crnn_char_scores(b2o_ctx* ctx, int b, const int32_t* labels_dev, int top_paths, int alternatives,
                                    float* conf_dev, int32_t* alt_labels_dev, float* alt_post_dev, float* logp_dev,
                                    const void* ws, size_t ws_bytes, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  if (!ctx->crnn_loaded) { ctx->set_error("b2o_crnn_char_scores: CRNN weights not loaded"); return B2O_ERR_STATE; }
  if (!ctc_char_scores_args(ctx->n_classes, top_paths, alternatives) || b < 0 ||
      (b > 0 && (!labels_dev || !conf_dev || !ws || (alternatives > 0 && (!alt_labels_dev || !alt_post_dev))))) {
    ctx->set_error("b2o_crnn_char_scores: bad argument");
    return B2O_ERR_ARG;
  }
  if (b == 0) return B2O_OK;
  const CrnnPlan p = plan_crnn(b);
  if (ws_bytes < p.bytes) { ctx->set_error("b2o_crnn_char_scores: workspace too small"); return B2O_ERR_WORKSPACE; }
  if (!crnn_wrote(ctx, rb::logits, ws, b)) {
    ctx->set_error("b2o_crnn_char_scores: the last successful CRNN forward of this context did not keep its logits in "
                   "this ws with this b");
    return B2O_ERR_STATE;
  }
  DeviceGuard guard(ctx->device);
  const uint8_t* base = reinterpret_cast<const uint8_t*>(ws);
  return ctc_char_scores_run(ctx, reinterpret_cast<const float*>(base + p.off[rb::logits]), b, ctx->n_classes, labels_dev,
                             top_paths, alternatives, conf_dev, alternatives > 0 ? alt_labels_dev : nullptr,
                             alternatives > 0 ? alt_post_dev : nullptr, logp_dev, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int b2o_set_debug_taps(b2o_ctx* ctx, int on) {
  if (!ctx) return B2O_ERR_ARG;
  ctx->debug_taps = on != 0;
  return B2O_OK;
}

extern "C" int b2o_crnn_tap(b2o_ctx* ctx, const char* name, const void* ws, int b, void* out, size_t out_bytes, void* stream) {
  if (!ctx || !name || !ws || !out || b <= 0) return B2O_ERR_ARG;
  DeviceGuard guard(ctx->device);
  const std::string s(name);
  int i = 0;
  while (i < rb::count && !(kCrnnBufs[i].tap && s == kCrnnBufs[i].name)) ++i;
  if (i == rb::count) { ctx->set_error("b2o_crnn_tap: unknown tap " + s); return B2O_ERR_ARG; }
  if (!crnn_wrote(ctx, static_cast<rb::Id>(i), ws, b)) {
    ctx->set_error("b2o_crnn_tap: the last successful CRNN forward of this context did not write " + s +
                   " in this ws with this b" + ((i == rb::theta || i == rb::warped) && !ctx->crnn_stn
                                                    ? " (this recognizer has no spatial transformer)" : ""));
    return B2O_ERR_STATE;
  }
  // the logits slot is sized for B2O_MAX_CLASSES; the tap copies the context's classes
  const size_t bytes = static_cast<size_t>(b) * (i == rb::logits ? 48 * ctx->n_classes * 4 : kCrnnBufs[i].bytes);
  if (out_bytes < bytes) { ctx->set_error("b2o_crnn_tap: output too small"); return B2O_ERR_ARG; }
  B2O_CUDA_CHECK(ctx, cudaMemcpyAsync(out, reinterpret_cast<const uint8_t*>(ws) + plan_crnn(b).off[i], bytes,
                                      cudaMemcpyDeviceToDevice, reinterpret_cast<cudaStream_t>(stream)));
  return B2O_OK;
}

extern "C" int b2o_conv2d_test(b2o_ctx* ctx, const void* x, int n, int h, int w, int cin, const float* wgt, int cout,
                               int ksize, int dilation, const float* s1, const float* t1, int relu, const float* s2,
                               const float* t2, void* out, int engine, void* stream) {
  if (!ctx || !x || !wgt || !s1 || !t1 || !out) return B2O_ERR_ARG;
  DeviceGuard guard(ctx->device);
  const size_t owned_before = ctx->owned.size();
  ConvLayer L;
  auto wget = [wgt, cin, ksize](int o, int c, int ky, int kx) {
    return wgt[((static_cast<size_t>(o) * ksize + ky) * ksize + kx) * cin + c];
  };
  std::vector<float> vs1(s1, s1 + cout), vt1(t1, t1 + cout), vs2, vt2;
  if (s2 && t2) { vs2.assign(s2, s2 + cout); vt2.assign(t2, t2 + cout); }
  int rc = build_layer(ctx, L, "test", cin, cout, ksize, dilation, relu, wget, vs1, vt1, s2 ? &vs2 : nullptr,
                       s2 ? &vt2 : nullptr, false);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (rc == B2O_OK) {
    const TensorView in = make_view(const_cast<void*>(x), n, h, w, cin), o = make_view(out, n, h, w, cout);
    const int saved = ctx->conv_engine;
    ctx->conv_engine = engine;
    if (engine == B2O_CONV_SIMT) rc = conv_simt_run(ctx, L, in, o, 0, st);
    else rc = conv_tc_run(ctx, L, in, o, 0, st);
    ctx->conv_engine = saved;
  }
  cudaError_t e = cudaStreamSynchronize(st);
  if (rc == B2O_OK && e != cudaSuccess) { ctx->set_error(std::string("conv2d_test: ") + cudaGetErrorString(e)); rc = B2O_ERR_CUDA; }
  while (ctx->owned.size() > owned_before) { cudaFree(ctx->owned.back()); ctx->owned.pop_back(); }
  return rc;
}

namespace {

// The body of b2o_conv_test: builds the layer(s) like b2o_load_craft / b2o_load_crnn do and routes the launch like
// b2o_craft_forward / b2o_crnn_forward.  The caller frees what build_layer allocated.
int conv_test_run(b2o_ctx* ctx, const b2o_conv_test_desc& d, cudaStream_t st) {
  const int cin = d.cin, k = d.ksize;
  if (!d.x_dev || !d.wgt_host || !d.s1_host || !d.t1_host || !d.out_dev || d.n <= 0 || d.h <= 0 || d.w <= 0 ||
      cin <= 0 || d.cout <= 0 || k <= 0 || d.dilation <= 0 || d.x_ld < cin || d.out_ld < d.cout ||
      (d.pool_dev && d.pool_ld < d.cout) || (d.up_dev && d.up_ld < d.cout) || (!d.s2_host) != (!d.t2_host)) {
    ctx->set_error("b2o_conv_test: bad argument");
    return B2O_ERR_ARG;
  }
  // the vector loads and stores of every engine (and of maxpool2_kernel) need 16-byte aligned pixels
  auto misaligned = [](const void* p, int ld, int elems) { return (reinterpret_cast<uintptr_t>(p) & 15) || (ld % elems); };
  if (cin % 8 || misaligned(d.x_dev, d.x_ld, 8) || misaligned(d.out_dev, d.out_ld, d.out_f32 ? 4 : 8) ||
      (d.pool_dev && (d.cout % 8 || d.out_f32 || misaligned(d.pool_dev, d.pool_ld, 8)))) {
    ctx->set_error("b2o_conv_test: misaligned view");
    return B2O_ERR_ARG;
  }
  const bool tail = d.scores_dev != nullptr;
  if (tail && (!d.w6_host || !d.b6_host || !d.w8_host || !d.b8_host || d.cout != 16 || d.pool_dev || d.out_f32)) {
    ctx->set_error("b2o_conv_test: the tail needs a 16-channel fp16 layer without pool");
    return B2O_ERR_ARG;
  }
  if (d.up_dev && d.engine == B2O_CONV_SIMT) {
    ctx->set_error("b2o_conv_test: upsample-add runs on the tensor-core engine only");
    return B2O_ERR_ARG;
  }
  ConvLayer L;
  const float* wgt = d.wgt_host;
  auto wget = [wgt, cin, k](int o, int c, int ky, int kx) {
    return wgt[((static_cast<size_t>(o) * k + ky) * k + kx) * cin + c];
  };
  std::vector<float> s1(d.s1_host, d.s1_host + d.cout), t1(d.t1_host, d.t1_host + d.cout), s2, t2;
  if (d.s2_host) { s2.assign(d.s2_host, d.s2_host + d.cout); t2.assign(d.t2_host, d.t2_host + d.cout); }
  B2O_RETURN_IF(build_layer(ctx, L, "test", cin, d.cout, k, d.dilation, d.relu, wget, s1, t1, d.s2_host ? &s2 : nullptr,
                            d.s2_host ? &t2 : nullptr, false));
  const TensorView in = make_view(const_cast<void*>(d.x_dev), d.n, d.h, d.w, cin, d.x_ld);
  TensorView out = make_view(d.out_dev, d.n, d.h, d.w, d.cout, d.out_ld);
  ctx->conv_engine = d.engine;
  if (d.up_dev) {                         // conv_tc_run checks the layer and the views (tail / pool / fp32 are refused)
    const TensorView up = make_view(const_cast<void*>(d.up_dev), d.n, d.h / 2, d.w / 2, d.cout, d.up_ld);
    const TensorView pool = d.pool_dev ? make_view(d.pool_dev, d.n, d.h / 2, d.w / 2, d.cout, d.pool_ld) : TensorView();
    ConvTail none = {nullptr, nullptr, nullptr, nullptr, d.scores_dev};
    return conv_tc_run(ctx, L, in, out, d.out_f32, st, d.pool_dev ? &pool : nullptr, 1, tail ? &none : nullptr, &up);
  }
  if (tail) {
    // conv_cls.6 (16 -> 16, ReLU) and conv_cls.8 (16 -> 2) built as b2o_load_craft builds them; w6 / w8 are (in, out)
    ConvLayer L6, L8;
    const float *w6 = d.w6_host, *w8 = d.w8_host;
    auto g6 = [w6](int o, int c, int, int) { return w6[c * 16 + o]; };
    auto g8 = [w8](int o, int c, int, int) { return w8[c * 2 + o]; };
    B2O_RETURN_IF(build_layer(ctx, L6, "test.6", 16, 16, 1, 1, 1, g6, ones(16), std::vector<float>(d.b6_host, d.b6_host + 16),
                              nullptr, nullptr, false));
    B2O_RETURN_IF(build_layer(ctx, L8, "test.8", 16, 2, 1, 1, 0, g8, ones(2), std::vector<float>(d.b8_host, d.b8_host + 2),
                              nullptr, nullptr, false));
    B2O_RETURN_IF(head_conv_run(ctx, L, L6, L8, in, out, d.scores_dev, st));
    return tail_fused(ctx, L) ? B2O_OK : head_tail_run(ctx, L6, L8, out, d.scores_dev, st);
  }
  if (d.pool_dev) {
    const TensorView pool = make_view(d.pool_dev, d.n, d.h / 2, d.w / 2, d.cout, d.pool_ld);
    return conv_run(ctx, L, in, out, d.out_f32, st, &pool, d.write_full);
  }
  return conv_run(ctx, L, in, out, d.out_f32, st);
}

}  // namespace

extern "C" int b2o_conv_test(b2o_ctx* ctx, const b2o_conv_test_desc* desc, void* stream) {
  if (!ctx || !desc) return B2O_ERR_ARG;
  if (desc->engine != B2O_CONV_AUTO && desc->engine != B2O_CONV_SIMT && desc->engine != B2O_CONV_TC_GENERIC) {
    ctx->set_error("b2o_conv_test: unknown engine");
    return B2O_ERR_ARG;
  }
  DeviceGuard guard(ctx->device);
  const size_t owned_before = ctx->owned.size();
  const int saved = ctx->conv_engine;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int rc = conv_test_run(ctx, *desc, st);
  ctx->conv_engine = saved;
  cudaError_t e = cudaStreamSynchronize(st);
  if (rc == B2O_OK && e != cudaSuccess) { ctx->set_error(std::string("b2o_conv_test: ") + cudaGetErrorString(e)); rc = B2O_ERR_CUDA; }
  while (ctx->owned.size() > owned_before) { cudaFree(ctx->owned.back()); ctx->owned.pop_back(); }
  return rc;
}
