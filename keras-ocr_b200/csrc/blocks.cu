// blocks.cu -- text blocks in reading order (DESIGN.md section 1, "Text blocks"): one image's text lines, as
// b2o_group_lines outputs them, cut into blocks by recursive XY-cut, the blocks in depth-first order and one box per
// block.
//
//   blocks_kernel   one CTA per image: the page frame D from the line with the most words, every line's extents along
//                   D and N and its height, the scale s (lower median of the heights), then the cut rounds, then the
//                   CSR table
//
// The lines are kept as a permutation in which every node of the cut tree is a contiguous range [seg, seg + size).  One
// round splits every open node at once: a sort on (node start, b_lo, l), a segmented running max of b_hi, the gap flags
// and the children's starts by a running max; then the same along a, with a_lo / a_hi, for the open nodes that had no
// row cut.  A node that cuts neither way is a block; a node of one line is one at once.  Children replace their parent
// in place, in ascending b or a, so when no node is open the ranges are the leaves in depth-first order.
//
// Every quantity is fp64 with an explicit operation order (__dadd_rn / __dmul_rn / __dsqrt_rn / __ddiv_rn, no
// contraction), so tests/block_refs.py reproduces every output bit; everything else is a min, a max or a sort on a
// total order.
#include <limits.h>
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kThreads = 512;

struct LineGeo {                     // one line's corners projected on D (a) and N (b)
  double alo, ahi, blo, bhi;
};

// per-image workspace sections, each a multiple of 256 bytes
struct Layout {
  size_t geo, height, keys, seg, open, cand, cut, had, bound, run, per_image;
};

__host__ __device__ inline size_t align256(size_t b) { return (b + 255) & ~static_cast<size_t>(255); }

__host__ __device__ inline Layout layout(int max_boxes) {
  Layout l;
  int p = 1;
  while (p < max_boxes) p <<= 1;
  const size_t m = static_cast<size_t>(max_boxes), mi = align256(m * sizeof(int));
  l.geo = 0;
  l.height = l.geo + align256(m * sizeof(LineGeo));
  l.keys = l.height + align256(m * sizeof(double));
  l.seg = l.keys + align256(static_cast<size_t>(p) * sizeof(SortKey));
  l.open = l.seg + mi;
  l.cand = l.open + mi;
  l.cut = l.cand + mi;
  l.had = l.cut + mi;
  l.bound = l.had + mi;
  l.run = l.bound + mi;
  l.per_image = l.run + align256(m * sizeof(double));
  return l;
}

__device__ __forceinline__ double vmax(double a, double b) { return fmax(a, b); }
__device__ __forceinline__ int vmax(int a, int b) { return max(a, b); }

// out[k] = max of val(j) over j in [r, k], r the last restart at or before k (restart(0) must hold), by the whole CTA:
// each thread scans a contiguous chunk; the chunks' (restarted, max) pairs go through one block scan.  A max is exact,
// so the result does not depend on the order in which the values meet.
template <typename T, typename Val, typename Restart>
__device__ void running_max(int L, Val val, Restart restart, T* out, T lowest) {
  __shared__ int sf[32];
  __shared__ T sx[32];
  const int chunk = (L + blockDim.x - 1) / blockDim.x;
  const int k0 = min(L, static_cast<int>(threadIdx.x) * chunk), k1 = min(L, k0 + chunk);
  int f = 0;
  T x = lowest;
  for (int k = k0; k < k1; ++k) {
    if (restart(k)) { f = 1; x = val(k); } else { x = vmax(x, val(k)); }
  }
  // inclusive scan of the pairs across the warp, then across the warps' totals
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int o = 1; o < 32; o <<= 1) {
    const int fy = __shfl_up_sync(0xffffffffu, f, o);
    const T xy = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o && !f) { x = vmax(xy, x); f = fy; }
  }
  if (lane == 31) { sf[warp] = f; sx[warp] = x; }
  __syncthreads();
  if (warp == 0) {
    int g = lane < nw ? sf[lane] : 0;
    T y = lane < nw ? sx[lane] : lowest;
    for (int o = 1; o < 32; o <<= 1) {
      const int gy = __shfl_up_sync(0xffffffffu, g, o);
      const T yy = __shfl_up_sync(0xffffffffu, y, o);
      if (lane >= o && !g) { y = vmax(yy, y); g = gy; }
    }
    if (lane < nw) { sf[lane] = g; sx[lane] = y; }
  }
  __syncthreads();
  // exclusive prefix of this thread: the warps before it, then the lanes before it
  T px = warp ? sx[warp - 1] : lowest;
  const int lf = __shfl_up_sync(0xffffffffu, f, 1);
  const T lx = __shfl_up_sync(0xffffffffu, x, 1);
  if (lane) {
    if (lf) px = lx; else px = vmax(px, lx);
  }
  T run = px;
  for (int k = k0; k < k1; ++k) {
    run = restart(k) ? val(k) : vmax(run, val(k));
    out[k] = run;
  }
  __syncthreads();
}

// One cut of every candidate node along one axis (lo / hi = a or b extents, thr = gap * s).  On entry keys[k].p is the
// line at position k; on return the candidates' lines are sorted by (lo, l) inside their nodes, cut[k] = 1 where
// position k's node cut, and seg holds the children's starts (had is scratch).
template <typename Lo, typename Hi>
__device__ void cut_axis(int L, int p, SortKey* keys, int* seg, const int* cand, int* cut, int* had, int* bound,
                         double* run, Lo lo, Hi hi, double thr) {
  for (int k = threadIdx.x; k < L; k += blockDim.x) {
    const unsigned l = keys[k].p;
    SortKey s;
    s.a = static_cast<unsigned long long>(seg[k]);
    s.b = cand[k] ? dkey(lo(l)) : 0ull;
    s.c = s.p = l;
    keys[k] = s;
    had[k] = 0;
  }
  __syncthreads();
  block_sort(keys, p);
  running_max<double>(L, [&](int k) { return hi(keys[k].p); }, [&](int k) { return seg[k] == k; }, run, -INFINITY);
  for (int k = threadIdx.x; k < L; k += blockDim.x) {
    const bool c = cand[k] && k > seg[k] && __dsub_rn(lo(keys[k].p), run[k - 1]) >= thr;
    cut[k] = c;
    if (c) had[seg[k]] = 1;
  }
  __syncthreads();
  for (int k = threadIdx.x; k < L; k += blockDim.x) {
    bound[k] = (k == seg[k] || cut[k]) ? k : 0;
    cut[k] = had[seg[k]];
  }
  __syncthreads();
  running_max<int>(L, [&](int k) { return bound[k]; }, [](int) { return false; }, seg, INT_MIN);
}

__global__ void __launch_bounds__(kThreads) blocks_kernel(const int32_t* __restrict__ line_counts,
                                                          const int32_t* __restrict__ line_start,
                                                          const float* __restrict__ line_boxes, int max_boxes,
                                                          double row_gap, double col_gap,
                                                          unsigned char* __restrict__ ws, Layout lay,
                                                          int32_t* __restrict__ block_counts,
                                                          int32_t* __restrict__ line_order,
                                                          int32_t* __restrict__ block_start,
                                                          float* __restrict__ block_boxes) {
  const int img = blockIdx.x;
  const int c = line_counts[img];
  const int L = c < 0 ? 0 : (c > max_boxes ? max_boxes : c);
  __shared__ int scratch[33];
  __shared__ unsigned long long best;
  if (L == 0) {
    if (threadIdx.x == 0) { block_counts[img] = 0; block_start[static_cast<size_t>(img) * (max_boxes + 1)] = 0; }
    return;
  }
  unsigned char* base = ws + static_cast<size_t>(img) * lay.per_image;
  LineGeo* geo = reinterpret_cast<LineGeo*>(base + lay.geo);
  double* height = reinterpret_cast<double*>(base + lay.height);
  SortKey* keys = reinterpret_cast<SortKey*>(base + lay.keys);
  int* seg = reinterpret_cast<int*>(base + lay.seg);
  int* open = reinterpret_cast<int*>(base + lay.open);
  int* cand = reinterpret_cast<int*>(base + lay.cand);
  int* cut = reinterpret_cast<int*>(base + lay.cut);
  int* had = reinterpret_cast<int*>(base + lay.had);
  int* bound = reinterpret_cast<int*>(base + lay.bound);
  double* run = reinterpret_cast<double*>(base + lay.run);
  const int32_t* ls = line_start + static_cast<size_t>(img) * (max_boxes + 1);
  const float* q = line_boxes + static_cast<size_t>(img) * max_boxes * 8;
  int32_t* order_out = line_order + static_cast<size_t>(img) * max_boxes;
  int32_t* start_out = block_start + static_cast<size_t>(img) * (max_boxes + 1);
  float* box_out = block_boxes + static_cast<size_t>(img) * max_boxes * 8;
  int p = 1;
  while (p < L) p <<= 1;

  // 1. page frame: the line with the most words, ties to the smallest l
  if (threadIdx.x == 0) best = 0ull;
  __syncthreads();
  for (int l = threadIdx.x; l < L; l += blockDim.x)
    atomicMax(&best, (static_cast<unsigned long long>(static_cast<unsigned>(ls[l + 1] - ls[l])) << 32) |
                         (0xffffffffu - static_cast<unsigned>(l)));
  __syncthreads();
  const int dl = static_cast<int>(0xffffffffu - static_cast<unsigned>(best & 0xffffffffull));
  const double ex = __dsub_rn(q[dl * 8 + 2], q[dl * 8]), ey = __dsub_rn(q[dl * 8 + 3], q[dl * 8 + 1]);
  const double en = __dsqrt_rn(dot2(ex, ey, ex, ey));
  const double dx = en == 0.0 ? 1.0 : __ddiv_rn(ex, en), dy = en == 0.0 ? 0.0 : __ddiv_rn(ey, en);
  const double nx = -dy, ny = dx;
  // 2. extents along D and N and the height of every line; the heights sorted for the scale
  for (int l = threadIdx.x; l < L; l += blockDim.x) {
    const float* w = q + static_cast<size_t>(l) * 8;
    double amin = INFINITY, amax = -INFINITY, bmin = INFINITY, bmax = -INFINITY;
    for (int v = 0; v < 4; ++v) {
      const double px = w[2 * v], py = w[2 * v + 1];
      const double a = dot2(px, py, dx, dy), b = dot2(px, py, nx, ny);
      amin = fmin(amin, a);
      amax = fmax(amax, a);
      bmin = fmin(bmin, b);
      bmax = fmax(bmax, b);
    }
    geo[l] = LineGeo{amin, amax, bmin, bmax};
    const double fx = __dsub_rn(w[6], w[0]), fy = __dsub_rn(w[7], w[1]);
    const double g = __dsqrt_rn(dot2(fx, fy, fx, fy));
    height[l] = g;
    SortKey s;
    s.a = dkey(g);
    s.b = 0;
    s.c = s.p = static_cast<unsigned>(l);
    keys[l] = s;
    seg[l] = 0;
    open[l] = L > 1;
  }
  pad_keys(keys, L, p);
  __syncthreads();
  block_sort(keys, p);
  const double scale = height[keys[(L - 1) / 2].p];
  const double row_thr = __dmul_rn(row_gap, scale), col_thr = __dmul_rn(col_gap, scale);

  // 3. cut rounds until no node is open; keys[k].p is the line at position k (any order at first: one node)
  auto blo = [&](unsigned l) { return geo[l].blo; };
  auto bhi = [&](unsigned l) { return geo[l].bhi; };
  auto alo = [&](unsigned l) { return geo[l].alo; };
  auto ahi = [&](unsigned l) { return geo[l].ahi; };
  bool any_open = L > 1;
  while (any_open) {
    cut_axis(L, p, keys, seg, open, cut, had, bound, run, blo, bhi, row_thr);
    // a row cut's children are open; open nodes that did not cut rows try columns
    int any_cand = 0;
    for (int k = threadIdx.x; k < L; k += blockDim.x) {
      cand[k] = open[k] && !cut[k];
      open[k] = open[k] && cut[k];
      any_cand |= cand[k];
    }
    if (__syncthreads_or(any_cand)) {
      cut_axis(L, p, keys, seg, cand, cut, had, bound, run, alo, ahi, col_thr);
      for (int k = threadIdx.x; k < L; k += blockDim.x) open[k] |= cand[k] && cut[k];
      __syncthreads();
    }
    // a node of one line cannot cut
    int still = 0;
    for (int k = threadIdx.x; k < L; k += blockDim.x) {
      if (k == seg[k] && (k + 1 == L || seg[k + 1] == k + 1)) open[k] = 0;
      still |= open[k];
    }
    any_open = __syncthreads_or(still);
  }

  // 4. the CSR table: lines of every block in ascending l, blocks in ascending start (depth-first leaf order)
  for (int k = threadIdx.x; k < L; k += blockDim.x) {
    SortKey s;
    s.a = static_cast<unsigned long long>(seg[k]);
    s.b = 0;
    s.c = s.p = keys[k].p;
    keys[k] = s;
  }
  __syncthreads();
  block_sort(keys, p);
  int done = 0;
  for (int r0 = 0; r0 < L; r0 += blockDim.x) {
    const int k = r0 + threadIdx.x;
    const bool first = k < L && seg[k] == k;
    int total;
    const int j = done + block_exclusive_scan(first ? 1 : 0, scratch, &total);
    if (first) {
      start_out[j] = k;
      double amin = INFINITY, amax = -INFINITY, bmin = INFINITY, bmax = -INFINITY;
      for (int e = k; e < L && seg[e] == k; ++e) {
        const LineGeo& G = geo[keys[e].p];
        amin = fmin(amin, G.alo);
        amax = fmax(amax, G.ahi);
        bmin = fmin(bmin, G.blo);
        bmax = fmax(bmax, G.bhi);
      }
      const double ca[4] = {amin, amax, amax, amin}, cb[4] = {bmin, bmin, bmax, bmax};
      for (int v = 0; v < 4; ++v) {
        box_out[static_cast<size_t>(j) * 8 + 2 * v] = __double2float_rn(__dadd_rn(__dmul_rn(ca[v], dx), __dmul_rn(cb[v], nx)));
        box_out[static_cast<size_t>(j) * 8 + 2 * v + 1] =
            __double2float_rn(__dadd_rn(__dmul_rn(ca[v], dy), __dmul_rn(cb[v], ny)));
      }
    }
    done += total;
  }
  for (int k = threadIdx.x; k < L; k += blockDim.x) order_out[k] = static_cast<int32_t>(keys[k].p);
  if (threadIdx.x == 0) {
    start_out[done] = L;
    block_counts[img] = done;
  }
}

}  // namespace

extern "C" size_t b2o_blocks_workspace_bytes(int n, int max_boxes) {
  if (n <= 0 || max_boxes <= 0) return 0;
  return static_cast<size_t>(n) * layout(max_boxes).per_image;
}

extern "C" int b2o_group_blocks(b2o_ctx* ctx, const int32_t* line_counts, const int32_t* line_start,
                                const float* line_boxes, int n, int max_boxes, double row_gap, double col_gap,
                                int32_t* block_counts, int32_t* line_order, int32_t* block_start, float* block_boxes,
                                void* ws, size_t ws_bytes, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  DeviceGuard guard(ctx->device);
  if (n == 0) return B2O_OK;
  if (!line_counts || !line_start || !line_boxes || !block_counts || !line_order || !block_start || !block_boxes ||
      !ws || n < 0 || max_boxes <= 0 || max_boxes > (1 << 24) || !isfinite(row_gap) || !isfinite(col_gap) ||
      !(row_gap > 0.0) || !(col_gap > 0.0)) {
    ctx->set_error("b2o_group_blocks: bad argument");
    return B2O_ERR_ARG;
  }
  const Layout lay = layout(max_boxes);
  if (ws_bytes < static_cast<size_t>(n) * lay.per_image) {
    ctx->set_error("b2o_group_blocks: workspace too small");
    return B2O_ERR_WORKSPACE;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  blocks_kernel<<<n, kThreads, 0, st>>>(line_counts, line_start, line_boxes, max_boxes, row_gap, col_gap,
                                        static_cast<unsigned char*>(ws), lay, block_counts, line_order, block_start,
                                        block_boxes);
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}
