// tiles.cu -- tiled detection (DESIGN.md section 1, "Tiles"): a page larger than one CRAFT tile is cut into overlapping
// square tiles, CRAFT runs on chunks of them as an ordinary batch, and each tile's core is copied into one page-sized
// score map.
//   b2o_tile_plan   : the grid, a pure host function (tests/tile_refs.py restates it).
//   cut_kernel      : 16 output bytes per thread; one 16-byte load where the bytes are one aligned run of the page.
//   stitch_kernel   : one CTA per (core row, tile), one float2 score per thread and column.
// Both are copies: the cut is bit-exact by construction, the stitch writes every page score from exactly one tile.
#include "common.cuh"

namespace {

// One axis of the grid: extent t, stride s, tile count k (the fewest whose tiles cover [0, L)).
void plan_axis(int L, int tile_size, int margin, int* t, int* s, int* k) {
  *t = L < tile_size ? L : tile_size;
  *s = *t - 2 * margin;
  *k = L <= tile_size ? 1 : 1 + (L - *t + *s - 1) / *s;
}

// [lo, hi) of tile k's core along an axis of length L, in score-map pixels (the detector-input range halved).
__device__ __forceinline__ void core_range(int k, int K, int s, int t, int margin, int L, int* lo, int* hi) {
  const int o = k * s;
  *lo = k == 0 ? 0 : (o + margin) / 2;
  *hi = k == K - 1 ? L / 2 : (o + t - margin) / 2;
}

__global__ void __launch_bounds__(256)
cut_kernel(const uint8_t* __restrict__ img, b2o_tiles p, int first_tile, long long total_bytes,
           uint8_t* __restrict__ tiles) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long b0 = 16 * i;
  if (b0 >= total_bytes) return;
  const int row_bytes = 3 * p.t_w;
  const long long tile_bytes = static_cast<long long>(row_bytes) * p.t_h;
  const int per_image = p.n_h * p.n_w;
  union { uint4 v; uint8_t b[16]; } out;
  // the 16 bytes in one tile row, inside the page and 16-byte aligned in it: one load
  {
    const long long j = b0 / tile_bytes, in_tile = b0 - j * tile_bytes;
    const int y = static_cast<int>(in_tile / row_bytes), xb = static_cast<int>(in_tile - static_cast<long long>(y) * row_bytes);
    const int g = first_tile + static_cast<int>(j);
    const int img_i = g / per_image, r = g - img_i * per_image, ty = r / p.n_w, tx = r - ty * p.n_w;
    const int py = ty * p.s_h + y;
    const long long pb = 3LL * (tx * p.s_w) + xb;                       // byte of the page row
    const long long src = (static_cast<long long>(img_i) * p.hp + py) * 3LL * p.wp + pb;
    if (xb + 16 <= row_bytes && py < p.hp && pb + 16 <= 3LL * p.wp && b0 + 16 <= total_bytes &&
        ((reinterpret_cast<uintptr_t>(img) + src) & 15) == 0) {
      out.v = __ldg(reinterpret_cast<const uint4*>(img + src));
      *reinterpret_cast<uint4*>(tiles + b0) = out.v;
      return;
    }
  }
  // otherwise byte by byte: a tile or row boundary inside the 16 bytes, the page's edge, or an unaligned page row
  const int nb = total_bytes - b0 < 16 ? static_cast<int>(total_bytes - b0) : 16;
  for (int e = 0; e < 16; ++e) {
    uint8_t v = 255;
    const long long b = b0 + e;
    if (e < nb) {
      const long long j = b / tile_bytes, in_tile = b - j * tile_bytes;
      const int y = static_cast<int>(in_tile / row_bytes), xb = static_cast<int>(in_tile - static_cast<long long>(y) * row_bytes);
      const int g = first_tile + static_cast<int>(j);
      const int img_i = g / per_image, r = g - img_i * per_image, ty = r / p.n_w, tx = r - ty * p.n_w;
      const int py = ty * p.s_h + y;
      const long long pb = 3LL * (tx * p.s_w) + xb;
      if (py < p.hp && pb < 3LL * p.wp) v = img[(static_cast<long long>(img_i) * p.hp + py) * 3LL * p.wp + pb];
    }
    out.b[e] = v;
  }
  if (nb == 16) {
    *reinterpret_cast<uint4*>(tiles + b0) = out.v;
  } else {
    for (int e = 0; e < nb; ++e) tiles[b0 + e] = out.b[e];
  }
}

__global__ void __launch_bounds__(256)
stitch_kernel(const float2* __restrict__ tile_scores, b2o_tiles p, int first_tile, int n_tiles,
              float2* __restrict__ scores) {
  const int th = p.t_h / 2, tw = p.t_w / 2, hs = p.hp / 2, ws = p.wp / 2;
  const int per_image = p.n_h * p.n_w;
  const int ly = blockIdx.x;                                 // row inside the tile's score map
  for (int j = blockIdx.y; j < n_tiles; j += gridDim.y) {
    const int g = first_tile + j;
    const int img_i = g / per_image, r = g - img_i * per_image, ty = r / p.n_w, tx = r - ty * p.n_w;
    int y0, y1, x0, x1;
    core_range(ty, p.n_h, p.s_h, p.t_h, p.margin, p.hp, &y0, &y1);
    core_range(tx, p.n_w, p.s_w, p.t_w, p.margin, p.wp, &x0, &x1);
    const int oy = ty * p.s_h / 2, ox = tx * p.s_w / 2;      // the tile's origin in the page's score map
    const int y = oy + ly;
    if (y < y0 || y >= y1) continue;
    const float2* src = tile_scores + (static_cast<size_t>(j) * th + ly) * tw;
    float2* dst = scores + (static_cast<size_t>(img_i) * hs + y) * ws;
    for (int x = x0 + static_cast<int>(threadIdx.x); x < x1; x += blockDim.x) dst[x] = src[x - ox];
  }
}

// plan is b2o_tile_plan's own for its parameters, and the chunk lies inside the batch's tiles
bool plan_ok(const b2o_tiles* plan, int n, int first_tile, int n_tiles) {
  b2o_tiles q;
  if (!plan || n <= 0 || b2o_tile_plan(plan->hp, plan->wp, plan->tile_size, plan->margin, &q) != B2O_OK) return false;
  if (q.t_h != plan->t_h || q.t_w != plan->t_w || q.s_h != plan->s_h || q.s_w != plan->s_w || q.n_h != plan->n_h ||
      q.n_w != plan->n_w)
    return false;
  return first_tile >= 0 && n_tiles >= 1 &&
         static_cast<long long>(first_tile) + n_tiles <= static_cast<long long>(n) * q.n_h * q.n_w;
}

}  // namespace

extern "C" int b2o_tile_plan(int hp, int wp, int tile_size, int margin, b2o_tiles* plan) {
  if (!plan || hp < 32 || wp < 32 || margin < 0 || margin % 16 != 0 || tile_size % 32 != 0 || tile_size > 2048 ||
      4 * margin > tile_size || tile_size < 32)
    return B2O_ERR_ARG;
  b2o_tiles p;
  p.hp = hp; p.wp = wp; p.tile_size = tile_size; p.margin = margin;
  plan_axis(hp, tile_size, margin, &p.t_h, &p.s_h, &p.n_h);
  plan_axis(wp, tile_size, margin, &p.t_w, &p.s_w, &p.n_w);
  *plan = p;
  return B2O_OK;
}

extern "C" int b2o_cut_tiles(b2o_ctx* ctx, const uint8_t* img, int n, const b2o_tiles* plan, int first_tile,
                             int n_tiles, uint8_t* tiles, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  DeviceGuard guard(ctx->device);
  if (!img || !tiles || (reinterpret_cast<uintptr_t>(tiles) & 15) || !plan_ok(plan, n, first_tile, n_tiles)) {
    ctx->set_error("b2o_cut_tiles: bad argument");
    return B2O_ERR_ARG;
  }
  const long long total = static_cast<long long>(n_tiles) * plan->t_h * plan->t_w * 3;
  const long long threads = (total + 15) / 16;
  cut_kernel<<<static_cast<unsigned>((threads + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      img, *plan, first_tile, total, tiles);
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}

extern "C" int b2o_stitch_tiles(b2o_ctx* ctx, const float* tile_scores, int n, const b2o_tiles* plan, int first_tile,
                                int n_tiles, float* scores, void* stream) {
  if (!ctx) return B2O_ERR_ARG;
  DeviceGuard guard(ctx->device);
  if (!tile_scores || !scores || (reinterpret_cast<uintptr_t>(tile_scores) & 7) ||
      (reinterpret_cast<uintptr_t>(scores) & 7) || !plan_ok(plan, n, first_tile, n_tiles)) {
    ctx->set_error("b2o_stitch_tiles: bad argument");
    return B2O_ERR_ARG;
  }
  const dim3 grid(static_cast<unsigned>(plan->t_h / 2), static_cast<unsigned>(n_tiles < 65535 ? n_tiles : 65535));
  stitch_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float2*>(tile_scores), *plan, first_tile, n_tiles, reinterpret_cast<float2*>(scores));
  B2O_LAUNCH_CHECK(ctx);
  return B2O_OK;
}
