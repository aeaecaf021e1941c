// lines.cu -- text lines in reading order (DESIGN.md section 1, "Text lines"): one image's word boxes grouped into
// lines, the words of each line in reading order, one box per line and the lines in page order.
//
//   features_kernel   per word: u (reading direction), w, h, centre; union-find parent initialised
//   links_kernel      per (image, i-tile, j-tile >= i-tile): every pair i < j tested, linked pairs united
//                     (uf_unite: the root of a line is its lowest word index)
//   order_kernel      one CTA per image: roots -> line ids, members in ascending index, line direction U, the line
//                     boxes, word keys c . U, page direction D, line keys, then the CSR table
//
// Every quantity is fp64 with an explicit operation order (__dadd_rn / __dmul_rn / __dsqrt_rn / __ddiv_rn, no
// contraction), so tests/line_refs.py reproduces every output bit.  Sums that are order dependent (U) run sequentially
// in ascending word index; everything else is a min, a max or a sort on a total order.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kTile = 64;            // words per side of a link tile
constexpr int kLinkThreads = 256;
constexpr int kOrderThreads = 512;

struct WordFeat {                    // one word's geometry in fp64
  double ux, uy, w, h, cx, cy;
};

struct LineRec {                     // one line, indexed by line id (ascending root)
  double ux, uy, mx, my;             // U and the box centre m
  double amin, amax, bmin, bmax;     // the members' corners projected on U and N
  int start, size, low, out_start;   // slice of the sorted word keys, word count, lowest word index, first output slot
};

struct Params {
  double cos_tol, height_ratio, offset_ratio, gap_ratio;
};

// per-image workspace sections, each a multiple of 256 bytes
struct Layout {
  size_t feat, parent, line, keys, line_keys, lines, per_image;
};

__host__ __device__ inline size_t align256(size_t b) { return (b + 255) & ~static_cast<size_t>(255); }

__host__ __device__ inline Layout layout(int max_boxes) {
  Layout l;
  int p = 1;
  while (p < max_boxes) p <<= 1;
  const size_t m = static_cast<size_t>(max_boxes);
  l.feat = 0;
  l.parent = l.feat + align256(m * sizeof(WordFeat));
  l.line = l.parent + align256(m * sizeof(int));
  l.keys = l.line + align256(m * sizeof(int));
  l.line_keys = l.keys + align256(static_cast<size_t>(p) * sizeof(SortKey));
  l.lines = l.line_keys + align256(static_cast<size_t>(p) * sizeof(SortKey));
  l.per_image = l.lines + align256(m * sizeof(LineRec));
  return l;
}

__device__ __forceinline__ int image_count(const int32_t* counts, int img, int max_boxes) {
  const int c = counts[img];
  return c < 0 ? 0 : (c > max_boxes ? max_boxes : c);
}

__global__ void features_kernel(const float* __restrict__ boxes, const int32_t* __restrict__ counts, int n,
                                int max_boxes, unsigned char* __restrict__ ws, Layout lay) {
  const long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= static_cast<long long>(n) * max_boxes) return;
  const int img = static_cast<int>(t / max_boxes), i = static_cast<int>(t % max_boxes);
  if (i >= image_count(counts, img, max_boxes)) return;
  unsigned char* base = ws + static_cast<size_t>(img) * lay.per_image;
  const float* q = boxes + (static_cast<size_t>(img) * max_boxes + i) * 8;
  const double x0 = q[0], y0 = q[1], x1 = q[2], y1 = q[3], x2 = q[4], y2 = q[5], x3 = q[6], y3 = q[7];
  const double ex = __dsub_rn(x1, x0), ey = __dsub_rn(y1, y0);
  const double w = __dsqrt_rn(dot2(ex, ey, ex, ey));
  const double fx = __dsub_rn(x3, x0), fy = __dsub_rn(y3, y0);
  WordFeat f;
  f.w = w;
  f.h = __dsqrt_rn(dot2(fx, fy, fx, fy));
  f.ux = w == 0.0 ? 1.0 : __ddiv_rn(ex, w);
  f.uy = w == 0.0 ? 0.0 : __ddiv_rn(ey, w);
  f.cx = __dmul_rn(__dadd_rn(__dadd_rn(x0, x1), __dadd_rn(x2, x3)), 0.25);
  f.cy = __dmul_rn(__dadd_rn(__dadd_rn(y0, y1), __dadd_rn(y2, y3)), 0.25);
  reinterpret_cast<WordFeat*>(base + lay.feat)[i] = f;
  reinterpret_cast<int*>(base + lay.parent)[i] = i;
}

// The link relation of DESIGN.md section 1, for i < j.  Every condition is symmetric in (i, j) bit for bit: the dot
// products and min / max commute, and d for (j, i) is exactly -d.
__device__ __forceinline__ bool linked(const WordFeat& a, const WordFeat& b, const Params& P) {
  if (!(a.w > 0.0 && a.h > 0.0 && b.w > 0.0 && b.h > 0.0)) return false;
  if (!(dot2(a.ux, a.uy, b.ux, b.uy) >= P.cos_tol)) return false;
  const double hmin = fmin(a.h, b.h), hmax = fmax(a.h, b.h);
  if (!(hmin >= __dmul_rn(P.height_ratio, hmax))) return false;
  const double dx = __dsub_rn(b.cx, a.cx), dy = __dsub_rn(b.cy, a.cy);
  const double off = __dmul_rn(P.offset_ratio, hmin);
  if (!(fabs(dot2(dx, dy, -a.uy, a.ux)) <= off)) return false;
  if (!(fabs(dot2(dx, dy, -b.uy, b.ux)) <= off)) return false;
  const double half = __dmul_rn(__dadd_rn(a.w, b.w), 0.5);
  const double gap = __dmul_rn(P.gap_ratio, hmax);
  if (!(__dsub_rn(fabs(dot2(dx, dy, a.ux, a.uy)), half) <= gap)) return false;
  return __dsub_rn(fabs(dot2(dx, dy, b.ux, b.uy)), half) <= gap;
}

// grid.x = n * tiles * tiles, one CTA per (image, i-tile, j-tile); tiles below the diagonal exit at once
__global__ void __launch_bounds__(kLinkThreads) links_kernel(const int32_t* __restrict__ counts, int max_boxes,
                                                             int tiles, Params P, unsigned char* __restrict__ ws,
                                                             Layout lay) {
  const long long b = blockIdx.x;
  const int img = static_cast<int>(b / (static_cast<long long>(tiles) * tiles));
  const int rem = static_cast<int>(b % (static_cast<long long>(tiles) * tiles));
  const int ti = rem / tiles, tj = rem % tiles;
  if (tj < ti) return;
  const int c = image_count(counts, img, max_boxes);
  const int i0 = ti * kTile, j0 = tj * kTile;
  if (j0 >= c) return;
  unsigned char* base = ws + static_cast<size_t>(img) * lay.per_image;
  const WordFeat* feat = reinterpret_cast<const WordFeat*>(base + lay.feat);
  int* parent = reinterpret_cast<int*>(base + lay.parent);
  __shared__ WordFeat fi[kTile], fj[kTile];
  for (int k = threadIdx.x; k < kTile; k += blockDim.x) {
    if (i0 + k < c) fi[k] = feat[i0 + k];
    if (j0 + k < c) fj[k] = feat[j0 + k];
  }
  __syncthreads();
  for (int k = threadIdx.x; k < kTile * kTile; k += blockDim.x) {
    const int a = k / kTile, bb = k % kTile;
    const int i = i0 + a, j = j0 + bb;
    if (j <= i || j >= c) continue;
    if (linked(fi[a], fj[bb], P)) uf_unite(parent, i, j);
  }
}

__global__ void __launch_bounds__(kOrderThreads) order_kernel(const float* __restrict__ boxes,
                                                              const int32_t* __restrict__ counts, int max_boxes,
                                                              unsigned char* __restrict__ ws, Layout lay,
                                                              int32_t* __restrict__ line_counts,
                                                              int32_t* __restrict__ word_order,
                                                              int32_t* __restrict__ line_start,
                                                              float* __restrict__ line_boxes) {
  const int img = blockIdx.x;
  const int c = image_count(counts, img, max_boxes);
  __shared__ int scratch[33];
  __shared__ unsigned long long best;
  if (c == 0) {
    if (threadIdx.x == 0) { line_counts[img] = 0; line_start[static_cast<size_t>(img) * (max_boxes + 1)] = 0; }
    return;
  }
  unsigned char* base = ws + static_cast<size_t>(img) * lay.per_image;
  const WordFeat* feat = reinterpret_cast<const WordFeat*>(base + lay.feat);
  int* parent = reinterpret_cast<int*>(base + lay.parent);
  int* line = reinterpret_cast<int*>(base + lay.line);
  SortKey* keys = reinterpret_cast<SortKey*>(base + lay.keys);
  LineRec* lines = reinterpret_cast<LineRec*>(base + lay.lines);
  const float* q = boxes + static_cast<size_t>(img) * max_boxes * 8;
  int32_t* order_out = word_order + static_cast<size_t>(img) * max_boxes;
  int32_t* start_out = line_start + static_cast<size_t>(img) * (max_boxes + 1);
  float* box_out = line_boxes + static_cast<size_t>(img) * max_boxes * 8;
  int p = 1;
  while (p < c) p <<= 1;

  // 1. line id of every root: its rank among the roots (ascending root = ascending lowest word index)
  int n_lines = 0;
  for (int b0 = 0; b0 < c; b0 += blockDim.x) {
    const int i = b0 + threadIdx.x;
    const bool root = i < c && uf_find(parent, i) == i;
    int total;
    const int r = block_exclusive_scan(root ? 1 : 0, scratch, &total);
    if (root) line[i] = n_lines + r;
    n_lines += total;
  }
  __syncthreads();
  // 2. members of every line in ascending word index: sort by (line, index)
  for (int i = threadIdx.x; i < c; i += blockDim.x) {
    SortKey s;
    s.a = static_cast<unsigned long long>(line[uf_find(parent, i)]);
    s.b = 0;
    s.c = s.p = static_cast<unsigned>(i);
    keys[i] = s;
  }
  pad_keys(keys, c, p);
  __syncthreads();
  block_sort(keys, p);
  for (int k = threadIdx.x; k < c; k += blockDim.x) {
    const int l = static_cast<int>(keys[k].a);
    if (k == 0 || static_cast<int>(keys[k - 1].a) != l) { lines[l].start = k; lines[l].low = static_cast<int>(keys[k].p); }
    if (k == c - 1 || static_cast<int>(keys[k + 1].a) != l) lines[l].size = k + 1;     // end for now
  }
  __syncthreads();
  // 3. per line: U (sequential sum in ascending index, normalised), the extents of the members' corners, the centre
  for (int l = threadIdx.x; l < n_lines; l += blockDim.x) {
    LineRec& L = lines[l];
    const int s = L.start, e = L.size;
    double sx = 0.0, sy = 0.0;
    for (int k = s; k < e; ++k) {
      const WordFeat& f = feat[keys[k].p];
      sx = __dadd_rn(sx, f.ux);
      sy = __dadd_rn(sy, f.uy);
    }
    const double nrm = __dsqrt_rn(dot2(sx, sy, sx, sy));
    const double ux = nrm == 0.0 ? 1.0 : __ddiv_rn(sx, nrm), uy = nrm == 0.0 ? 0.0 : __ddiv_rn(sy, nrm);
    const double nx = -uy, ny = ux;
    double amin = INFINITY, amax = -INFINITY, bmin = INFINITY, bmax = -INFINITY;
    for (int k = s; k < e; ++k) {
      const float* w = q + static_cast<size_t>(keys[k].p) * 8;
      for (int v = 0; v < 4; ++v) {
        const double px = w[2 * v], py = w[2 * v + 1];
        const double a = dot2(px, py, ux, uy), b = dot2(px, py, nx, ny);
        amin = fmin(amin, a);
        amax = fmax(amax, a);
        bmin = fmin(bmin, b);
        bmax = fmax(bmax, b);
      }
    }
    const double am = __dmul_rn(__dadd_rn(amin, amax), 0.5), bm = __dmul_rn(__dadd_rn(bmin, bmax), 0.5);
    L.ux = ux;
    L.uy = uy;
    L.mx = __dadd_rn(__dmul_rn(am, ux), __dmul_rn(bm, nx));
    L.my = __dadd_rn(__dmul_rn(am, uy), __dmul_rn(bm, ny));
    L.amin = amin;
    L.amax = amax;
    L.bmin = bmin;
    L.bmax = bmax;
    L.size = e - s;
  }
  if (threadIdx.x == 0) best = 0ull;
  __syncthreads();
  // 4. words in reading order inside their line: sort by (line, c . U, index); a line keeps its slice [start, start+size)
  for (int k = threadIdx.x; k < c; k += blockDim.x) {
    const int l = static_cast<int>(keys[k].a), i = static_cast<int>(keys[k].p);
    keys[k].b = dkey(dot2(feat[i].cx, feat[i].cy, lines[l].ux, lines[l].uy));
  }
  // 5. page direction: the line with the most words, ties to the lowest line id (= the lowest word index)
  for (int l = threadIdx.x; l < n_lines; l += blockDim.x)
    atomicMax(&best, (static_cast<unsigned long long>(lines[l].size) << 32) | (0xffffffffu - static_cast<unsigned>(l)));
  __syncthreads();
  block_sort(keys, p);
  const int dl = static_cast<int>(0xffffffffu - static_cast<unsigned>(best & 0xffffffffull));
  const double dx = lines[dl].ux, dy = lines[dl].uy;
  // 6. lines in page order: sort by (m . N_D, m . D, lowest word index)
  SortKey* lkeys = reinterpret_cast<SortKey*>(base + lay.line_keys);
  int pl = 1;
  while (pl < n_lines) pl <<= 1;
  for (int l = threadIdx.x; l < n_lines; l += blockDim.x) {
    SortKey s;
    s.a = dkey(dot2(lines[l].mx, lines[l].my, -dy, dx));
    s.b = dkey(dot2(lines[l].mx, lines[l].my, dx, dy));
    s.c = static_cast<unsigned>(lines[l].low);
    s.p = static_cast<unsigned>(l);
    lkeys[l] = s;
  }
  pad_keys(lkeys, n_lines, pl);
  __syncthreads();
  block_sort(lkeys, pl);
  // 7. the CSR table: line starts in page order, line boxes (fp32, rounded once), then the words
  int done = 0;
  for (int r0 = 0; r0 < n_lines; r0 += blockDim.x) {
    const int r = r0 + threadIdx.x;
    const int l = r < n_lines ? static_cast<int>(lkeys[r].p) : 0;
    int total;
    const int off = block_exclusive_scan(r < n_lines ? lines[l].size : 0, scratch, &total);
    if (r < n_lines) {
      LineRec& L = lines[l];
      L.out_start = done + off;
      start_out[r] = done + off;
      const double nx = -L.uy, ny = L.ux;
      const double ca[4] = {L.amin, L.amax, L.amax, L.amin}, cb[4] = {L.bmin, L.bmin, L.bmax, L.bmax};
      for (int v = 0; v < 4; ++v) {
        box_out[static_cast<size_t>(r) * 8 + 2 * v] = __double2float_rn(__dadd_rn(__dmul_rn(ca[v], L.ux), __dmul_rn(cb[v], nx)));
        box_out[static_cast<size_t>(r) * 8 + 2 * v + 1] =
            __double2float_rn(__dadd_rn(__dmul_rn(ca[v], L.uy), __dmul_rn(cb[v], ny)));
      }
    }
    done += total;
  }
  __syncthreads();
  for (int k = threadIdx.x; k < c; k += blockDim.x) {
    const LineRec& L = lines[keys[k].a];
    order_out[L.out_start + (k - L.start)] = static_cast<int32_t>(keys[k].p);
  }
  if (threadIdx.x == 0) {
    start_out[n_lines] = c;
    line_counts[img] = n_lines;
  }
}

}  // namespace

extern "C" size_t b2o_lines_workspace_bytes(int n, int max_boxes) {
  if (n <= 0 || max_boxes <= 0) return 0;
  return static_cast<size_t>(n) * layout(max_boxes).per_image;
}

extern "C" int b2o_group_lines(b2o_ctx* ctx, const float* boxes, const int32_t* counts, int n, int max_boxes,
                               double cos_tol, double height_ratio, double offset_ratio, double gap_ratio,
                               int32_t* line_counts, int32_t* word_order, int32_t* line_start, float* line_boxes,
                               void* ws, size_t ws_bytes, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  DeviceGuard guard(ctx->device);
  if (n == 0) return B2O_OK;
  if (!boxes || !counts || !line_counts || !word_order || !line_start || !line_boxes || !ws || n < 0 ||
      max_boxes <= 0 || max_boxes > (1 << 24) || !isfinite(cos_tol) || !isfinite(height_ratio) ||
      !isfinite(offset_ratio) || !isfinite(gap_ratio)) {
    ctx->set_error("b2o_group_lines: bad argument");
    return B2O_ERR_ARG;
  }
  const Layout lay = layout(max_boxes);
  if (ws_bytes < static_cast<size_t>(n) * lay.per_image) {
    ctx->set_error("b2o_group_lines: workspace too small");
    return B2O_ERR_WORKSPACE;
  }
  const long long tiles = (max_boxes + kTile - 1) / kTile;
  if (static_cast<long long>(n) * tiles * tiles > 0x7fffffffll) {
    ctx->set_error("b2o_group_lines: n * tiles^2 exceeds the grid");
    return B2O_ERR_ARG;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  unsigned char* w = static_cast<unsigned char*>(ws);
  const long long words = static_cast<long long>(n) * max_boxes;
  features_kernel<<<static_cast<unsigned>((words + 255) / 256), 256, 0, st>>>(boxes, counts, n, max_boxes, w, lay);
  B2O_LAUNCH_CHECK(ctx);
  const Params P{cos_tol, height_ratio, offset_ratio, gap_ratio};
  links_kernel<<<static_cast<unsigned>(n * tiles * tiles), kLinkThreads, 0, st>>>(counts, max_boxes,
                                                                                  static_cast<int>(tiles), P, w, lay);
  B2O_LAUNCH_CHECK(ctx);
  order_kernel<<<n, kOrderThreads, 0, st>>>(boxes, counts, max_boxes, w, lay, line_counts, word_order, line_start,
                                            line_boxes);
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}
