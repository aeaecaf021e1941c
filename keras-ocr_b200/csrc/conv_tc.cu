// conv_tc.cu -- implicit-GEMM convolution / dense layer on the Hopper tensor cores (sm_90a: wgmma, TMA, mbarrier).
//
// Replaces the TensorFlow Conv2D / Dense kernels behind keras.Model.predict for CRAFT
// (reference detection.py:65-103, 365-410) and the CRNN (recognition.py:217-290, 292-327).
//
//   D[pixel, cout] = sum_{tap, c} X[pixel + offset(tap), c] * Wt[cout, tap, c]
//
// * M = 128 output pixels per tile = a box of the NHWC activation, so TMA fetches the A operand
//   straight from the feature map; out-of-bounds zero fill implements "same" padding / dilation.
//   - generic mode: one 4-D TMA box (KCH, BW, BH, BNI) per (tap, channel chunk), any k / dilation;
//   - halo mode (3x3, dilation 1): the tile is 8 (w) x 16 (h); ONE box of 8 x 18 rows per
//     (dx, channel chunk) serves the three dy taps, whose A descriptors are the same stage shifted
//     by whole 8-pixel rows (a multiple of the swizzle period) -- 3x less L2->SM traffic.
// * B = weights packed K-major [cout][tap*cin + c], 2-D TMA boxes (KCH x BLOCK_N); when the whole
//   filter bank fits in shared memory (small layers) it is loaded once per CTA and stays resident.
// * K chunk KCH = 64 / 32 / 16 channels (128B / 64B / 32B swizzle) so 32- and 16-channel layers
//   (CRAFT conv_cls.*, STN) also run on the tensor cores.
// * warp roles: thread 0 of warpgroup 0 = TMA producer (one ring of stages; a stage is the A box of one (tap group,
//   channel chunk) plus, unless the filter bank is resident, its B boxes, all on one mbarrier); warpgroups 1 and 2 =
//   ping-pong consumers, each owning whole tiles (the CTA's even / odd ones): two wgmma.mma_async m64 x BLOCK_N x k16
//   per k step (tile rows 0-63 and 64-127) with fp32 accumulators in registers, then the epilogue straight from those
//   registers: scale/shift/ReLU/affine -> fp16|fp32 NHWC stores (possibly into a channel slice of a concat buffer) and,
//   optionally, the fused 2x2 max-pool output or CRAFT tail.  The two warpgroups take turns on the main loop, so one
//   runs its epilogue while the other keeps the tensor cores busy.
// * persistent: grid = min(#tiles, #SMs); n-tiles of one pixel tile run back to back.
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace {

constexpr int WG_M = 64;                  // rows of one wgmma: half of a 128-pixel tile
constexpr int MMA_K = 16;
constexpr int NUM_THREADS = 384;          // warpgroup 0: producer; warpgroups 1, 2: MMA + epilogue
constexpr int TILE_WARPS = 4;             // the warps of the one consumer warpgroup that reads a stage
// setmaxnreg split of the 64K registers: the producer needs few, a consumer thread holds 2 x BLOCK_N / 2 accumulators
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;
constexpr int SMEM_TOTAL = 227 * 1024;    // dynamic shared memory per CTA (the sm_90 maximum, 232448 B)
constexpr int MAX_RING = 8;

struct TcParams {
  int N, H, W;
  int cin, cout, ksize, dil;
  int bw_log2, bh_log2, bn_log2;
  int tiles_w, tiles_h, tiles_n;          // M-tile grid
  int n_tiles;                            // cout / BLOCK_N
  int total_tiles;
  int halo, resident;
  int ns;                                 // ring depth (stages)
  int a_bytes, a_stride;                  // bytes one A box delivers / offset of a stage's B boxes
  int stage_bytes, stage_tx;              // bytes between stages / bytes a stage's barrier expects
  int off_res, off_bar;                   // shared-memory offsets: resident filter bank, barriers
  int aff_smem;                           // epilogue constants staged in shared memory behind the barriers (B2O_TC_AFF=smem)
  int aff_const;                          // epilogue constants read from the AffConst kernel parameter (default)
  const float *s1, *t1, *s2, *t2;
  int relu;
  void* out;
  int out_ld, out_f32, write_full;
  __half* pool_out;                       // fused 2x2/2 max-pool output (or null)
  int pool_ld, PH, PW;
  // decoder glue (UPADD instances): the accumulator gets the exact-2x bilinear upsampling (half-pixel centres, clamped
  // borders -- UpsampleLike, detection.py:290-309) of a low-resolution fp16 tensor (N, H/2, W/2, cout) added BEFORE
  // the affine/ReLU: relu(bn(W_y.up(y) + W_s.skip)) = relu(bn(up(W_y.y) + W_s.skip)), detection.py:380-390
  const __half* up_src;
  int up_ld, UH, UW;
  // fused CRAFT tail (16-channel layers only): conv_cls.6 (1x1 16->16 ReLU) + conv_cls.8 (1x1 16->2) applied to the
  // epilogue's 16 channels in registers, fp32 (text, link) scores out -- detection.py:404-410
  const float *tail_w6, *tail_b6, *tail_w8, *tail_b8;   // [16][16], [16], [16][2], [2]
  float* tail_out;                        // (N,H,W,2) fp32, or null
};
constexpr int TAIL_FLOATS = 256 + 16 + 32 + 2;

// ------------------------------------------------------------------------------------------ PTX
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a broken pipeline traps (surfacing as a CUDA error) instead of hanging the GPU.  No printf here: a
// function call in the consumer loop makes ptxas serialize every wgmma.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) __trap();
  }
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_4d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1,
                                            int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// ---- CTA pairs: clusters of two CTAs share every B tile.  Each CTA loads half of the tile's rows and multicasts them
// into the same shared-memory offset of both CTAs, signalling both CTAs' barriers at that offset.
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire;" ::: "memory");
}
__device__ __forceinline__ void tma_load_2d_multicast(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(static_cast<uint16_t>(3))
      : "memory");
}
// one arrival on the barrier at the same offset in CTA `cta` of the cluster
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
  asm volatile(
      "{\n\t.reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n\t}" ::"r"(smem_u32(bar)), "r"(cta)
      : "memory");
}
// K-major swizzled shared-memory matrix descriptor (wgmma): rows of KCH*2 bytes, 8-row atoms 16*KCH bytes apart.
// Every start address used is a whole number of 8-row atoms from a 1 KB-aligned stage, plus the 32-byte k-step
// inside a row, so the base-offset field stays 0.
template <int KCH>
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr) {
  constexpr uint64_t SBO = 16 * KCH;                       // 8 rows x (KCH*2) bytes
  constexpr uint64_t LAYOUT = KCH == 64 ? 1 : (KCH == 32 ? 2 : 3);   // SWIZZLE_128B / 64B / 32B
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);    // start address      bits [0,14)
  d |= static_cast<uint64_t>(1) << 16;                     // leading byte off.  bits [16,30) (unused: swizzled K-major)
  d |= (SBO >> 4) << 32;                                   // stride byte offset bits [32,46)
  d |= LAYOUT << 62;                                       // swizzle mode       bits [62,64)
  return d;
}
// named barriers between the two consumer warpgroups (id 0 is __syncthreads')
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(uint32_t id, uint32_t count) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory");
}
template <int REGS>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(REGS)); }
template <int REGS>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(REGS)); }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
__device__ __forceinline__ void reg_fence(float& r) { asm volatile("" : "+f"(r)::"memory"); }
// D[64 x N] (+)= A[64 x 16] * B[16 x N]^T, f16 inputs K-major in shared memory, f32 accumulators in registers
template <int N>
__device__ __forceinline__ void wgmma_f16(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate);
template <>
__device__ __forceinline__ void wgmma_f16<16>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_f16<32>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_f16<64>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_f16<128>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

// Walks the tiles first, first + step, ... keeping the mixed-radix coordinate (n_tile, tile_w, tile_h, tile_n)
// incrementally: no integer divisions in the per-tile path.  The radices are read from the kernel parameters rather
// than held in registers (the consumers need every register they can get for accumulators).
struct TileIter {
  int c0, c1, c2, c3;        // n_tile, tile_w, tile_h, tile_n
  int d0, d1, d2, d3;        // step in the same radix
  int tile, step;
  __device__ __forceinline__ TileIter(const TcParams& p, int first, int step_) {
    const int r0 = p.n_tiles, r1 = p.tiles_w, r2 = p.tiles_h;
    tile = first;
    step = step_;
    int t = first;
    c0 = t % r0; t /= r0; c1 = t % r1; t /= r1; c2 = t % r2; c3 = t / r2;
    t = step;
    d0 = t % r0; t /= r0; d1 = t % r1; t /= r1; d2 = t % r2; d3 = t / r2;
  }
  __device__ __forceinline__ bool valid(const TcParams& p) const { return tile < p.total_tiles; }
  __device__ __forceinline__ void next(const TcParams& p) {
    tile += step;
    c0 += d0; if (c0 >= p.n_tiles) { c0 -= p.n_tiles; ++c1; }
    c1 += d1; if (c1 >= p.tiles_w) { c1 -= p.tiles_w; ++c2; }
    c2 += d2; if (c2 >= p.tiles_h) { c2 -= p.tiles_h; ++c3; }
    c3 += d3;
  }
};

// Per-channel epilogue constants as a KERNEL PARAMETER (constant bank) for layers of <= AFF_MAX output channels.
// 16 KB of parameters need CUDA >= 12.1 (large kernel parameters).
constexpr int AFF_MAX = 1024;
struct AffConst {
  float s1[AFF_MAX], t1[AFF_MAX], s2[AFF_MAX], t2[AFF_MAX];
  float tail[320];          // fused CRAFT tail: [w6 transposed [out j][in c] 256 | b6 16 | w8 [j][2] 32 | b8 2]
};

// ------------------------------------------------------------------------------------------ kernel
// MODE: 0 = generic tiles, 1 = halo tiles (3x3, dilation 1), 2 = halo tiles + resident filter bank
// PAIR: clusters of two CTAs on horizontally adjacent pixel tiles of the same n-tile (rank = which).  Each CTA fetches
//       HALF of every B tile from L2 and multicasts it to both, so the filter bank crosses L2 -> SM once per 256 pixels
//       instead of once per 128; A boxes stay per CTA.  A stage may only be refilled when the consumers of BOTH CTAs have
//       released it, so every consumer warp arrives on the empty barriers of both CTAs.  The MMAs and their order are
//       those of the single-CTA tiles: results are bit-identical.
template <int BLOCK_N, int KCH, int MODE, bool PAIR, bool UPADD = false>
__global__ void __launch_bounds__(NUM_THREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap amap, const __grid_constant__ CUtensorMap bmap,
               const TcParams p, const __grid_constant__ AffConst ac) {
  constexpr bool HALO = MODE >= 1, RESIDENT = MODE == 2;
  constexpr int TAPS_PER_A = HALO ? 3 : 1;                 // dy taps served by one A stage
  constexpr int B_BYTES = BLOCK_N * KCH * 2;
  constexpr int B_HALF = B_BYTES / 2;                      // pair: the B rows one CTA fetches and multicasts
  const uint32_t rank = PAIR ? cluster_ctarank() : 0u;
  const int cta = PAIR ? static_cast<int>(blockIdx.x >> 1) : static_cast<int>(blockIdx.x);
  const int ncta = PAIR ? static_cast<int>(gridDim.x >> 1) : static_cast<int>(gridDim.x);
  const int pair_shift = PAIR ? 1 : 0;                     // tile column = (pair column << 1) + rank
  constexpr int KSTEPS = KCH / MMA_K;
  constexpr int NACC = BLOCK_N / 2;                        // fp32 accumulators per consumer thread and 64-row half
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + p.off_bar);
  uint64_t* empty = full + MAX_RING;
  uint64_t* res_full = empty + MAX_RING;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  float* aff = reinterpret_cast<float*>(smem + p.off_bar + 512);     // [s1 | t1 | s2 | t2] x cout
  if (p.aff_smem) {
    for (int i = threadIdx.x; i < p.cout; i += NUM_THREADS) {
      aff[i] = p.s1[i];
      aff[p.cout + i] = p.t1[i];
      if (p.s2 != nullptr) { aff[2 * p.cout + i] = p.s2[i]; aff[3 * p.cout + i] = p.t2[i]; }
    }
  }
  // fused tail constants behind the affine ones: [w6 transposed ([out j][in c]) | b6 | w8 | b8]
  float* const tail_s = aff + 4 * p.cout;
  if (BLOCK_N == 16 && p.tail_out != nullptr && !p.aff_const) {
    for (int i = threadIdx.x; i < TAIL_FLOATS; i += NUM_THREADS)
      tail_s[i] = i < 256 ? p.tail_w6[(i & 15) * 16 + (i >> 4)] : (i < 272 ? p.tail_b6[i - 256] : (i < 304 ? p.tail_w8[i - 272] : p.tail_b8[i - 304]));
  }
  if (threadIdx.x == 0) {
    for (int s = 0; s < MAX_RING; ++s) {
      mbar_init(&full[s], 1);                              // the producer's expect_tx arrival + the TMA bytes
      mbar_init(&empty[s], (PAIR ? 2 : 1) * TILE_WARPS);   // one arrival per warp of the stage's consumer warpgroup (of both CTAs of a pair) once its MMAs read it
    }
    mbar_init(res_full, 1);
    fence_barrier_init();
  }
  if (PAIR) cluster_sync_all();                            // the peer's barriers exist before anything signals them
  else __syncthreads();

  const int taps = p.ksize * p.ksize;
  const int kchunks = p.cin / KCH;
  const int groups = HALO ? 3 : taps;                      // dx positions (halo) or filter taps (generic)

  if (threadIdx.x < 128) {
    // ===================================================================== TMA producer
    setmaxnreg_dec<PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      tma_prefetch_desc(&amap);
      tma_prefetch_desc(&bmap);
      const int half_k = p.ksize >> 1;
      if (RESIDENT) {                                      // whole filter bank, once per CTA (pair: half of it from each CTA)
        mbar_expect_tx(res_full, static_cast<uint32_t>(taps * kchunks * B_BYTES));
        for (int tap = 0; tap < taps; ++tap)
          for (int kc = 0; kc < kchunks; ++kc) {
            uint8_t* const dst = smem + p.off_res + (tap * kchunks + kc) * B_BYTES;
            if (PAIR) tma_load_2d_multicast(&bmap, res_full, dst + rank * B_HALF, tap * p.cin + kc * KCH, static_cast<int>(rank) * (BLOCK_N / 2));
            else tma_load_2d(&bmap, res_full, dst, tap * p.cin + kc * KCH, 0);
          }
      }
      int s = 0;
      uint32_t ph = 0;
      for (TileIter ti(p, cta, ncta); ti.valid(p); ti.next(p)) {
        const int tw0 = ((ti.c1 << pair_shift) + static_cast<int>(rank)) << p.bw_log2, th0 = ti.c2 << p.bh_log2, tn0 = ti.c3 << p.bn_log2;
        int ky = 0, kx = 0;
        for (int g = 0; g < groups; ++g) {
          const int ax = HALO ? (tw0 + g - 1) : (tw0 + (kx - half_k) * p.dil);
          const int ay = HALO ? (th0 - 1) : (th0 + (ky - half_k) * p.dil);
          for (int kc = 0; kc < kchunks; ++kc) {
            mbar_wait(&empty[s], ph ^ 1);
            uint8_t* const st = smem + s * p.stage_bytes;
            mbar_expect_tx(&full[s], static_cast<uint32_t>(p.stage_tx));
            tma_load_4d(&amap, &full[s], st, kc * KCH, ax, ay, tn0);
            if (!RESIDENT) {
#pragma unroll
              for (int t = 0; t < TAPS_PER_A; ++t) {
                const int tap = HALO ? (t * 3 + g) : g;
                uint8_t* const dst = st + p.a_stride + t * B_BYTES;
                if (PAIR)
                  tma_load_2d_multicast(&bmap, &full[s], dst + rank * B_HALF, tap * p.cin + kc * KCH,
                                        ti.c0 * BLOCK_N + static_cast<int>(rank) * (BLOCK_N / 2));
                else
                  tma_load_2d(&bmap, &full[s], dst, tap * p.cin + kc * KCH, ti.c0 * BLOCK_N);
              }
            }
            if (++s == p.ns) { s = 0; ph ^= 1; }
          }
          if (++kx == p.ksize) { kx = 0; ++ky; }
        }
      }
    }
  } else {
    // ===================================================================== consumers (warpgroups 1, 2)
    // Ping-pong: warpgroup 1 takes the CTA's tiles 0, 2, 4, ... (TileIter order), warpgroup 2 tiles 1, 3, 5, ...  Both
    // CTAs of a pair give a tile to the same warpgroup, so the multicast B halves line up.  Every tile takes the same
    // number of ring stages, so a warpgroup steps over the other's tile by arithmetic on (s, ph).  The main loops take
    // turns: a warpgroup starts a tile only after the other has issued all MMAs of the tile before (named barrier 1 +
    // wg), which also keeps it from waiting on a stage more than one ring lap ahead of the one the producer fills.
    setmaxnreg_inc<CONSUMER_REGS>();
    const int wg = (threadIdx.x >> 7) - 1;
    const int q = lane & 3;
    // accumulator layout of wgmma m64: this thread holds rows r0 and r0 + 8 of each 64-row half, columns 8i + 2q, 8i + 2q + 1
    const int r0 = (warp & 3) * 16 + (lane >> 2);
    constexpr uint32_t TAP_BYTES = 8 * KCH * 2;              // halo: one dy tap = 8 pixel rows further into the stage
    constexpr uint32_t HALF_BYTES = WG_M * KCH * 2;          // tile rows 64-127: 64 rows (whole 8-row atoms) further
    const uint64_t desc_a0 = gmma_desc<KCH>(smem_u32(smem));
    const uint64_t desc_b0 = gmma_desc<KCH>(smem_u32(smem) + static_cast<uint32_t>(RESIDENT ? p.off_res : p.a_stride));
    const float* const e_s1 = p.aff_const ? ac.s1 : (p.aff_smem ? aff : p.s1);
    const float* const e_t1 = p.aff_const ? ac.t1 : (p.aff_smem ? aff + p.cout : p.t1);
    const float* const e_s2 = p.aff_const ? ac.s2 : (p.aff_smem ? aff + 2 * p.cout : p.s2);
    const float* const e_t2 = p.aff_const ? ac.t2 : (p.aff_smem ? aff + 3 * p.cout : p.t2);
    const float* const tail_c = p.aff_const ? ac.tail : tail_s;
    const int bw_mask = (1 << p.bw_log2) - 1, bh_mask = (1 << p.bh_log2) - 1;
    // a stage is free once the consumers of this CTA (and of the peer, whose B halves it also holds) are done with it
    auto release = [&](int stage) {
      if (PAIR) { mbar_arrive_cluster(&empty[stage], 0u); mbar_arrive_cluster(&empty[stage], 1u); }
      else mbar_arrive(&empty[stage]);
    };

    int s = 0;
    uint32_t ph = 0;
    const int tile_stages = groups * kchunks;
    auto skip_tile = [&]() {                                 // the other warpgroup's tile
      s += tile_stages;
      const int laps = s / p.ns;
      s -= laps * p.ns;
      ph ^= static_cast<uint32_t>(laps & 1);
    };
    TileIter ti(p, cta + wg * ncta, 2 * ncta);              // the CTA's tiles wg, wg + 2, ...
    if (wg == 1) skip_tile();
    if (RESIDENT && ti.valid(p)) mbar_wait(res_full, 0);
    float acc[2 * NACC];                                     // [rows 0-63 | rows 64-127]
  #pragma unroll
    for (int i = 0; i < 2 * NACC; ++i) acc[i] = 0.0f;
    for (bool after_other = wg == 1; ti.valid(p); ti.next(p), after_other = true) {
      if (after_other) named_bar_sync(1 + wg, 2 * 128);      // the other warpgroup has issued the previous tile
      // ---- main loop: every stage of the tile, MMAs in (dx | tap, chunk, dy, k) order, both halves per k step
      int prev = -1;
      uint32_t accumulate = 0;
      for (int g = 0; g < groups; ++g) {
        for (int kc = 0; kc < kchunks; ++kc) {
          mbar_wait(&full[s], ph);
          const uint64_t adesc = desc_a0 + static_cast<uint64_t>(static_cast<uint32_t>(s * p.stage_bytes) >> 4);
  #pragma unroll
          for (int i = 0; i < 2 * NACC; ++i) reg_fence(acc[i]);
          wgmma_fence();
  #pragma unroll
          for (int t = 0; t < TAPS_PER_A; ++t) {
            const uint32_t boff = RESIDENT ? static_cast<uint32_t>(((t * 3 + g) * kchunks + kc) * B_BYTES)
                                           : static_cast<uint32_t>(s * p.stage_bytes + t * B_BYTES);
            const uint64_t bdesc = desc_b0 + static_cast<uint64_t>(boff >> 4);
  #pragma unroll
            for (int k = 0; k < KSTEPS; ++k) {
  #pragma unroll
              for (int mh = 0; mh < 2; ++mh)
                wgmma_f16<BLOCK_N>(acc + mh * NACC, adesc + static_cast<uint64_t>((mh * HALF_BYTES + t * TAP_BYTES + k * 32) >> 4),
                                   bdesc + static_cast<uint64_t>((k * 32) >> 4), accumulate);
              accumulate = 1;
            }
          }
          wgmma_commit();
          wgmma_wait<1>();                                   // the previous stage's MMAs are done: release it
          if (prev >= 0) {
            __syncwarp();
            if (lane == 0) release(prev);
          }
          prev = s;
          if (++s == p.ns) { s = 0; ph ^= 1; }
        }
      }
      if (ti.tile + ncta < p.total_tiles) named_bar_arrive(1 + (wg ^ 1), 2 * 128);   // the CTA's next tile may start
      skip_tile();
      wgmma_wait<0>();
  #pragma unroll
      for (int i = 0; i < 2 * NACC; ++i) reg_fence(acc[i]);
      __syncwarp();
      if (lane == 0) release(prev);

      // ---- epilogue from the registers, one 64-row half after the other
      const int c_base = ti.c0 * BLOCK_N;
  #pragma unroll
      for (int mh = 0; mh < 2; ++mh) {
        float* const acc_h = acc + mh * NACC;
        bool valid[2];
        size_t pix[2];
        int px_w[2], px_h[2], px_n[2];
  #pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int row = mh * WG_M + r0 + 8 * hh;
          px_w[hh] = (((ti.c1 << pair_shift) + static_cast<int>(rank)) << p.bw_log2) + (row & bw_mask);
          px_h[hh] = (ti.c2 << p.bh_log2) + ((row >> p.bw_log2) & bh_mask);
          px_n[hh] = (ti.c3 << p.bn_log2) + (row >> (p.bw_log2 + p.bh_log2));
          valid[hh] = (px_w[hh] < p.W) && (px_h[hh] < p.H) && (px_n[hh] < p.N);
          pix[hh] = (static_cast<size_t>(px_n[hh]) * p.H + px_h[hh]) * p.W + px_w[hh];
        }
        if (UPADD) {
          // acc += hy * (hx * A + lx * B) + ly * (hx * C + lx * D), the expression of upsample2x_kernel, in fp32
  #pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            if (!valid[hh]) continue;
            const int h = px_h[hh], w = px_w[hh];
            const int qy = (h + 1) >> 1, qx = (w + 1) >> 1;
            const int ya = max(qy - 1, 0), yb = min(qy, p.UH - 1), xa = max(qx - 1, 0), xb = min(qx, p.UW - 1);
            const float ly = ((h + 1) & 1) ? ((qy == 0) ? 0.0f : 0.75f) : 0.25f;
            const float lx = ((w + 1) & 1) ? ((qx == 0) ? 0.0f : 0.75f) : 0.25f;
            const float hy = 1.0f - ly, hx = 1.0f - lx;
            const size_t nb = static_cast<size_t>(px_n[hh]) * p.UH;
            const __half* const ua = p.up_src + ((nb + ya) * p.UW + xa) * p.up_ld + c_base + 2 * q;
            const __half* const ub = p.up_src + ((nb + ya) * p.UW + xb) * p.up_ld + c_base + 2 * q;
            const __half* const uc = p.up_src + ((nb + yb) * p.UW + xa) * p.up_ld + c_base + 2 * q;
            const __half* const ud = p.up_src + ((nb + yb) * p.UW + xb) * p.up_ld + c_base + 2 * q;
  #pragma unroll
            for (int i = 0; i < BLOCK_N / 8; ++i) {
              const float2 fa = __half22float2(*reinterpret_cast<const __half2*>(ua + 8 * i));
              const float2 fb = __half22float2(*reinterpret_cast<const __half2*>(ub + 8 * i));
              const float2 fc = __half22float2(*reinterpret_cast<const __half2*>(uc + 8 * i));
              const float2 fd = __half22float2(*reinterpret_cast<const __half2*>(ud + 8 * i));
              acc_h[4 * i + 2 * hh] += hy * (hx * fa.x + lx * fb.x) + ly * (hx * fc.x + lx * fd.x);
              acc_h[4 * i + 2 * hh + 1] += hy * (hx * fa.y + lx * fb.y) + ly * (hx * fc.y + lx * fd.y);
            }
          }
        }
        // y = relu?(acc * s1 + t1) [* s2 + t2], in place
  #pragma unroll
        for (int i = 0; i < BLOCK_N / 8; ++i) {
          const int c = c_base + 8 * i + 2 * q;
          const float2 a1 = *reinterpret_cast<const float2*>(e_s1 + c);
          const float2 b1 = *reinterpret_cast<const float2*>(e_t1 + c);
  #pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            float& y0 = acc_h[4 * i + 2 * hh];
            float& y1 = acc_h[4 * i + 2 * hh + 1];
            y0 = fmaf(y0, a1.x, b1.x);
            y1 = fmaf(y1, a1.y, b1.y);
            if (p.relu) { y0 = fmaxf(y0, 0.0f); y1 = fmaxf(y1, 0.0f); }
          }
          if (p.s2 != nullptr) {
            const float2 a2 = *reinterpret_cast<const float2*>(e_s2 + c);
            const float2 b2 = *reinterpret_cast<const float2*>(e_t2 + c);
  #pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              acc_h[4 * i + 2 * hh] = fmaf(acc_h[4 * i + 2 * hh], a2.x, b2.x);
              acc_h[4 * i + 2 * hh + 1] = fmaf(acc_h[4 * i + 2 * hh + 1], a2.y, b2.y);
            }
          }
        }
        if (BLOCK_N == 16 && p.tail_out != nullptr) {          // block-uniform; only the 16-channel instances carry it
          // The unfused path stores these 16 channels as fp16 and head_tail_kernel reads them back: round the same way
          // and run the same fmaf chains, so the scores are bit-identical to conv_cls.4 -> head_tail_kernel.
          // The quad's four lanes hold a pixel's 16 channels between them: gather them, lane q & 1 takes pixel row
          // r0 + 8 * (q & 1) (lanes 2, 3 compute the same pixels again and do not store).
          uint32_t hv[2][2];                                   // [column group i][row hh]
  #pragma unroll
          for (int i = 0; i < 2; ++i)
  #pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              const __half2 h2 = __floats2half2_rn(acc_h[4 * i + 2 * hh], acc_h[4 * i + 2 * hh + 1]);
              hv[i][hh] = *reinterpret_cast<const uint32_t*>(&h2);
            }
          const int mine = q & 1;
          float x[16];
  #pragma unroll
          for (int src = 0; src < 4; ++src)
  #pragma unroll
            for (int i = 0; i < 2; ++i) {
              const uint32_t v0 = __shfl_sync(0xffffffffu, hv[i][0], (lane & ~3) | src);
              const uint32_t v1 = __shfl_sync(0xffffffffu, hv[i][1], (lane & ~3) | src);
              const uint32_t v = mine ? v1 : v0;
              const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&v));
              x[8 * i + 2 * src] = f.x;
              x[8 * i + 2 * src + 1] = f.y;
            }
          float o0 = tail_c[304], o1 = tail_c[305];
  #pragma unroll
          for (int j = 0; j < 16; ++j) {
            float a = tail_c[256 + j];
  #pragma unroll
            for (int c = 0; c < 16; ++c) a = fmaf(x[c], tail_c[j * 16 + c], a);
            a = fmaxf(a, 0.0f);
            o0 = fmaf(a, tail_c[272 + j * 2 + 0], o0);
            o1 = fmaf(a, tail_c[272 + j * 2 + 1], o1);
          }
          if (q < 2 && valid[mine]) reinterpret_cast<float2*>(p.tail_out)[pix[mine]] = make_float2(o0, o1);
          continue;
        }
        if (p.out_f32) {
  #pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            if (!valid[hh]) continue;
            float* const o = reinterpret_cast<float*>(p.out) + pix[hh] * p.out_ld + c_base + 2 * q;
  #pragma unroll
            for (int i = 0; i < BLOCK_N / 8; ++i)
              *reinterpret_cast<float2*>(o + 8 * i) = make_float2(acc_h[4 * i + 2 * hh], acc_h[4 * i + 2 * hh + 1]);
          }
          continue;
        }
        // fp16 out; fused 2x2/2 max pool on halo tiles: rows r0 / r0 + 8 are vertical neighbours (h even, h + 1), the w
        // neighbour is lane ^ 4
        const bool pool_writer = p.pool_out != nullptr && !(px_w[0] & 1) && !(px_h[0] & 1) && (px_w[0] >> 1) < p.PW &&
                                 (px_h[0] >> 1) < p.PH && px_n[0] < p.N;
        const size_t ppix = (static_cast<size_t>(px_n[0]) * p.PH + (px_h[0] >> 1)) * p.PW + (px_w[0] >> 1);
        __half* const o0 = reinterpret_cast<__half*>(p.out) + pix[0] * p.out_ld + c_base + 2 * q;
        __half* const o1 = reinterpret_cast<__half*>(p.out) + pix[1] * p.out_ld + c_base + 2 * q;
  #pragma unroll
        for (int i = 0; i < BLOCK_N / 8; ++i) {
          const __half2 h0 = __floats2half2_rn(acc_h[4 * i], acc_h[4 * i + 1]);
          const __half2 h1 = __floats2half2_rn(acc_h[4 * i + 2], acc_h[4 * i + 3]);
          if (p.write_full) {
            if (valid[0]) *reinterpret_cast<__half2*>(o0 + 8 * i) = h0;
            if (valid[1]) *reinterpret_cast<__half2*>(o1 + 8 * i) = h1;
          }
          if (p.pool_out != nullptr) {                         // block-uniform branch
            __half2 m = __hmax2(h0, h1);
            const uint32_t mu = *reinterpret_cast<const uint32_t*>(&m);
            const uint32_t ou = __shfl_xor_sync(0xffffffffu, mu, 4);
            m = __hmax2(m, *reinterpret_cast<const __half2*>(&ou));
            if (pool_writer) *reinterpret_cast<__half2*>(p.pool_out + ppix * p.pool_ld + c_base + 8 * i + 2 * q) = m;
          }
        }
      }
    }
  }
  // neither CTA of a pair leaves while the other may still signal its barriers
  if (PAIR) cluster_sync_all();
}

// ------------------------------------------------------------------------------------------ host
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
      q != cudaDriverEntryPointSuccess)
    return nullptr;
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

CUtensorMapSwizzle swizzle_for(int kch) {
  return kch == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : (kch == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
}

// Pick the (bw, bh, bn) power-of-two box with bw*bh*bn = 128 that wastes the fewest pixels.
double pick_box(int N, int H, int W, int* bw_l, int* bh_l, int* bn_l) {
  double best = 1e30, best_cover = 0;
  int b_w = 7, b_h = 0, b_n = 0;
  for (int lw = 0; lw <= 7; ++lw)
    for (int lh = 0; lw + lh <= 7; ++lh) {
      const int ln = 7 - lw - lh;
      const int bw = 1 << lw, bh = 1 << lh, bn = 1 << ln;
      if (ln > 0 && (bn > 2 * N)) continue;
      const double cover = double((W + bw - 1) / bw * bw) * double((H + bh - 1) / bh * bh) *
                           double((N + bn - 1) / bn * bn);
      // prefer wide rows (coalesced stores / fewer TMA rows) on ties; keep bw >= 8 when W allows
      const double score = cover * (1.0 + 0.001 * (7 - lw)) * ((bw < 8 && W >= 8) ? 1.05 : 1.0);
      if (score < best) { best = score; best_cover = cover; b_w = lw; b_h = lh; b_n = ln; }
    }
  *bw_l = b_w; *bh_l = b_h; *bn_l = b_n;
  return best_cover;
}

thread_local const float* g_tail_host = nullptr;     // the fused tail's constants in AffConst::tail order (set by conv_tc_run)

template <int BLOCK_N, int KCH, int MODE, bool PAIR, bool UPADD = false>
int launch(b2o_ctx* ctx, const CUtensorMap& amap, const ConvLayer& L, const TcParams& p, int smem_bytes,
           cudaStream_t st) {
  static thread_local AffConst ac;                         // 16 KB: filled per launch from the layer's host copies
  if (p.aff_const) {
    const size_t nb = static_cast<size_t>(L.cout) * sizeof(float);
    memcpy(ac.s1, L.h_s1.data(), nb);
    memcpy(ac.t1, L.h_t1.data(), nb);
    if (!L.h_s2.empty()) { memcpy(ac.s2, L.h_s2.data(), nb); memcpy(ac.t2, L.h_t2.data(), nb); }
    if (p.tail_out != nullptr && g_tail_host != nullptr) memcpy(ac.tail, g_tail_host, TAIL_FLOATS * sizeof(float));
  }
  const void* fn = reinterpret_cast<const void*>(&conv_tc_kernel<BLOCK_N, KCH, MODE, PAIR, UPADD>);
  if (!ctx->configured.count(fn)) {                        // a per-device attribute: remembered per context
    B2O_CUDA_CHECK(ctx, cudaFuncSetAttribute(conv_tc_kernel<BLOCK_N, KCH, MODE, PAIR, UPADD>,
                                             cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_TOTAL));
    ctx->configured.insert(fn);
  }
  // persistent: one CTA per SM; pairs: one cluster of two CTAs per two SMs
  const int units = PAIR ? ctx->sm_count / 2 : ctx->sm_count;
  const int grid = (p.total_tiles < units ? p.total_tiles : units) * (PAIR ? 2 : 1);
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  if (ctx->profile) {
    B2O_CUDA_CHECK(ctx, cudaEventCreate(&e0));
    B2O_CUDA_CHECK(ctx, cudaEventCreate(&e1));
    B2O_CUDA_CHECK(ctx, cudaEventRecord(e0, st));
  }
  if (PAIR) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(NUM_THREADS);
    cfg.dynamicSmemBytes = static_cast<size_t>(smem_bytes);
    cfg.stream = st;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = 2; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    B2O_CUDA_CHECK(ctx, cudaLaunchKernelEx(&cfg, conv_tc_kernel<BLOCK_N, KCH, MODE, PAIR, UPADD>, amap, L.wmap_pair, p, ac));
  } else {
    conv_tc_kernel<BLOCK_N, KCH, MODE, PAIR, UPADD><<<grid, NUM_THREADS, smem_bytes, st>>>(amap, L.wmap, p, ac);
  }
  B2O_LAUNCH_CHECK(ctx);
  if (ctx->profile) {
    B2O_CUDA_CHECK(ctx, cudaEventRecord(e1, st));
    ctx->prof_events.push_back(e0);
    ctx->prof_events.push_back(e1);
    // algorithmic FLOPs of this launch: 2 * pixels * (taps * cin) * cout with the REFERENCE layer's channel counts
    // (SURVEY.md 8(d)): the zero-padded channels of the stem (3 -> 16) and of the STN GEMM (400 -> 512) do not count
    ctx->prof_flop += 2.0 * double(p.N) * p.H * p.W * double(p.ksize * p.ksize) * (L.alg_cin ? L.alg_cin : p.cin) *
                      (L.alg_cout ? L.alg_cout : p.cout);
  }
  return B2O_OK;
}

}  // namespace

int conv_tc_prepare(b2o_ctx* ctx, ConvLayer& L) {
  L.block_n = 0;
  L.kch = L.cin % 64 == 0 ? 64 : (L.cin % 32 == 0 ? 32 : (L.cin % 16 == 0 ? 16 : 0));
  if (L.kch == 0 || L.cout % 16 != 0) return B2O_OK;      // handled by the SIMT engine
  // N tile <= 128: a consumer thread holds BLOCK_N / 2 fp32 accumulators in registers
  int bn = 128;
  while (bn > 16 && (L.cout % bn != 0)) bn >>= 1;
  if (L.cout % bn != 0) return B2O_OK;
  if (L.kch == 32 && bn > 32) return B2O_OK;               // instantiated combinations only
  if (L.kch == 16 && bn != 32 && bn != 64) return B2O_OK;
  EncodeTiledFn enc = get_encode();
  if (!enc) { ctx->set_error("cuTensorMapEncodeTiled entry point not available"); return B2O_ERR_CUDA; }
  const cuuint64_t ktot = static_cast<cuuint64_t>(L.ksize) * L.ksize * L.cin;
  cuuint64_t dims[2] = {ktot, static_cast<cuuint64_t>(L.cout)};
  cuuint64_t strides[1] = {ktot * 2};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(L.kch), static_cast<cuuint32_t>(bn)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(&L.wmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, L.w_kmajor, dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_for(L.kch), CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    ctx->set_error("cuTensorMapEncodeTiled(weights " + L.name + ") failed: " + std::to_string(static_cast<int>(r)));
    return B2O_ERR_CUDA;
  }
  L.block_n = bn;
  // CTA pairs: each CTA fetches bn / 2 filter rows of an n-tile (instantiated for 64-channel chunks, bn >= 64)
  L.pair_ok = false;
  if (L.kch == 64 && bn >= 64) {
    cuuint32_t half_box[2] = {static_cast<cuuint32_t>(L.kch), static_cast<cuuint32_t>(bn / 2)};
    r = enc(&L.wmap_pair, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, L.w_kmajor, dims, strides, half_box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_for(L.kch), CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      ctx->set_error("cuTensorMapEncodeTiled(pair weights " + L.name + ") failed: " + std::to_string(static_cast<int>(r)));
      return B2O_ERR_CUDA;
    }
    L.pair_ok = true;
  }
  return B2O_OK;
}

int conv_tc_run(b2o_ctx* ctx, const ConvLayer& L, const TensorView& in, const TensorView& out, int out_f32,
                cudaStream_t st, const TensorView* pool_out, int write_full, const ConvTail* tail, const TensorView* up_add) {
  if (up_add != nullptr && (L.ksize != 1 || L.kch != 64 || L.block_n < 64 || out_f32 || pool_out != nullptr || tail != nullptr ||
                            up_add->c != L.cout || up_add->n != in.n || 2 * up_add->h != in.h || 2 * up_add->w != in.w ||
                            (up_add->ld % 8) || (reinterpret_cast<uintptr_t>(up_add->ptr) & 15))) {
    ctx->set_error("conv_tc_run: up_add needs a 1x1 layer with 64-channel chunks and an exactly half-size fp16 tensor (" + L.name + ")");
    return B2O_ERR_ARG;
  }
  if (tail != nullptr && (L.block_n != 16 || L.cout != 16 || pool_out != nullptr)) {
    ctx->set_error("conv_tc_run: the fused tail needs a 16-channel layer (" + L.name + ")");
    return B2O_ERR_ARG;
  }
  if (L.block_n == 0) { ctx->set_error("conv_tc_run: layer " + L.name + " not eligible"); return B2O_ERR_ARG; }
  if (in.c != L.cin || out.c != L.cout || in.n != out.n || in.h != out.h || in.w != out.w) {
    ctx->set_error("conv_tc_run: shape mismatch in " + L.name);
    return B2O_ERR_ARG;
  }
  if ((reinterpret_cast<uintptr_t>(in.ptr) & 15) || (in.ld % 8) || (reinterpret_cast<uintptr_t>(out.ptr) & 15) ||
      (out.ld % (out_f32 ? 4 : 8))) {
    ctx->set_error("conv_tc_run: misaligned view in " + L.name);
    return B2O_ERR_ARG;
  }
  EncodeTiledFn enc = get_encode();
  if (!enc) { ctx->set_error("cuTensorMapEncodeTiled entry point not available"); return B2O_ERR_CUDA; }
  const int kch = L.kch, bn = L.block_n;
  const int taps = L.ksize * L.ksize, kchunks = L.cin / kch;
  const int b_bytes = bn * kch * 2;

  TcParams p;
  memset(&p, 0, sizeof(p));
  p.N = in.n; p.H = in.h; p.W = in.w;
  p.cin = L.cin; p.cout = L.cout; p.ksize = L.ksize; p.dil = L.dil;
  pick_box(in.n, in.h, in.w, &p.bw_log2, &p.bh_log2, &p.bn_log2);
  // halo mode: 3x3, dilation 1, fixed 8 x 16 tile; skip it when that tile wastes >15 % more pixels.  The two
  // modes add the taps in different orders, so the choice must not depend on the batch size (a crop's result
  // may not change with the batch it travels in): both covers are taken per image, as if N were unbounded.
  int dw, dh, dn;
  const double big_n = 1 << 20;
  const double generic_cover = pick_box(1 << 20, in.h, in.w, &dw, &dh, &dn) / big_n;
  const double halo_cover = double((in.w + 7) / 8 * 8) * double((in.h + 15) / 16 * 16);
  const bool want_pool = pool_out != nullptr;
  p.halo = (L.ksize == 3 && L.dil == 1 && ctx->conv_engine != B2O_CONV_TC_GENERIC &&
            (halo_cover <= 1.15 * generic_cover || want_pool)) ? 1 : 0;
  if (want_pool && !p.halo) { ctx->set_error("conv_tc_run: fused pool needs the halo tile (" + L.name + ")"); return B2O_ERR_ARG; }
  if (p.halo) { p.bw_log2 = 3; p.bh_log2 = 4; p.bn_log2 = 0; }
  // CTA pairs (opt-in): halo tiles with B2O_TC_PAIR=1, generic tiles too with B2O_TC_PAIR=2; a pair covers
  // two horizontally adjacent tiles.  Same MMAs in the same order per output: bit-identical results.
  const bool pair = ctx->tc_pair && (p.halo || ctx->tc_pair_generic) && L.pair_ok && ctx->conv_engine == B2O_CONV_AUTO &&
                    up_add == nullptr;
  p.tiles_w = (in.w + (1 << p.bw_log2) - 1) >> p.bw_log2;
  if (pair) p.tiles_w = (p.tiles_w + 1) / 2;                // pair columns
  p.tiles_h = (in.h + (1 << p.bh_log2) - 1) >> p.bh_log2;
  p.tiles_n = (in.n + (1 << p.bn_log2) - 1) >> p.bn_log2;
  p.n_tiles = L.cout / bn;
  const long long total = static_cast<long long>(p.tiles_w) * p.tiles_h * p.tiles_n * p.n_tiles;
  if (total > 0x7fffffffLL) { ctx->set_error("conv_tc_run: too many tiles"); return B2O_ERR_ARG; }
  p.total_tiles = static_cast<int>(total);

  // shared-memory plan: [ring of stages: A box | B boxes][resident filter bank][barriers][epilogue constants]
  p.aff_const = (ctx->tc_aff_const && L.cout <= 256 && static_cast<int>(L.h_s1.size()) == L.cout) ? 1 : 0;
  p.aff_smem = (!p.aff_const && L.cout <= 256) ? 1 : 0;
  const int aff_bytes = (p.aff_smem ? 4 * L.cout * 4 : 0) + (tail ? TAIL_FLOATS * 4 : 0);
  const int budget = SMEM_TOTAL - 1024 /*alignment slack*/ - 512 /*barriers*/ - aff_bytes;
  p.a_bytes = p.halo ? 18 * 8 * kch * 2 : 128 * kch * 2;
  p.a_stride = (p.a_bytes + 1023) / 1024 * 1024;
  const long long res_bytes = static_cast<long long>(taps) * kchunks * b_bytes;
  // (the mbarrier tx-count holds 2^20 - 1 bytes)
  p.resident = (p.halo && p.n_tiles == 1 && res_bytes + 2LL * p.a_stride <= budget && res_bytes <= (1 << 20) - 1) ? 1 : 0;
  const int b_per_stage = p.resident ? 0 : (p.halo ? 3 : 1);
  p.stage_bytes = p.a_stride + b_per_stage * b_bytes;
  p.stage_tx = p.a_bytes + b_per_stage * b_bytes;
  p.ns = static_cast<int>((budget - (p.resident ? res_bytes : 0)) / p.stage_bytes);
  if (p.ns > MAX_RING) p.ns = MAX_RING;
  if (p.ns < 2) { ctx->set_error("conv_tc_run: shared-memory plan failed for " + L.name); return B2O_ERR_ARG; }
  p.off_res = p.ns * p.stage_bytes;
  p.off_bar = p.off_res + (p.resident ? static_cast<int>((res_bytes + 1023) / 1024 * 1024) : 0);
  int smem_bytes = p.off_bar + 512 + aff_bytes + 1024;
  // the grid is one persistent CTA per SM: a request above half of the SM's 228 KB keeps a second CTA of a small layer
  // from landing on an SM that already runs one while other SMs sit idle
  if (smem_bytes < 116 * 1024) smem_bytes = 116 * 1024;

  p.s1 = L.s1; p.t1 = L.t1; p.s2 = L.s2; p.t2 = L.t2; p.relu = L.relu;
  if (up_add) { p.up_src = up_add->ptr; p.up_ld = up_add->ld; p.UH = up_add->h; p.UW = up_add->w; }
  float tail_host[TAIL_FLOATS];
  g_tail_host = nullptr;
  if (tail && tail->h_w6 != nullptr) {                      // [w6 transposed | b6 | w8 | b8]
    for (int j = 0; j < 16; ++j)
      for (int c = 0; c < 16; ++c) tail_host[j * 16 + c] = tail->h_w6[c * 16 + j];
    memcpy(tail_host + 256, tail->h_b6, 16 * sizeof(float));
    memcpy(tail_host + 272, tail->h_w8, 32 * sizeof(float));
    memcpy(tail_host + 304, tail->h_b8, 2 * sizeof(float));
    g_tail_host = tail_host;
  }
  if (tail) { p.tail_w6 = tail->w6; p.tail_b6 = tail->b6; p.tail_w8 = tail->w8; p.tail_b8 = tail->b8; p.tail_out = tail->scores; }
  p.out = out.ptr; p.out_ld = out.ld; p.out_f32 = out_f32; p.write_full = write_full;
  if (want_pool) {
    if (out_f32 || pool_out->c != L.cout || pool_out->h != in.h / 2 || pool_out->w != in.w / 2 || (pool_out->ld % 8)) {
      ctx->set_error("conv_tc_run: bad pool view for " + L.name);
      return B2O_ERR_ARG;
    }
    p.pool_out = pool_out->ptr; p.pool_ld = pool_out->ld; p.PH = pool_out->h; p.PW = pool_out->w;
  }

  CUtensorMap amap;
  cuuint64_t dims[4] = {static_cast<cuuint64_t>(in.c), static_cast<cuuint64_t>(in.w), static_cast<cuuint64_t>(in.h),
                        static_cast<cuuint64_t>(in.n)};
  cuuint64_t strides[3] = {static_cast<cuuint64_t>(in.ld) * 2, static_cast<cuuint64_t>(in.ld) * 2 * in.w,
                           static_cast<cuuint64_t>(in.ld) * 2 * in.w * in.h};
  cuuint32_t box[4] = {static_cast<cuuint32_t>(kch), 1u << p.bw_log2, 1u << p.bh_log2, 1u << p.bn_log2};
  if (p.halo) { box[1] = 8; box[2] = 18; box[3] = 1; }
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(&amap, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, in.ptr, dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_for(kch), CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    ctx->set_error("cuTensorMapEncodeTiled(activation for " + L.name + ") failed: " +
                   std::to_string(static_cast<int>(r)));
    return B2O_ERR_CUDA;
  }
  if (up_add != nullptr) {                                 // generic 1x1 tiles
    if (bn == 64) return launch<64, 64, 0, false, true>(ctx, amap, L, p, smem_bytes, st);
    if (bn == 128) return launch<128, 64, 0, false, true>(ctx, amap, L, p, smem_bytes, st);
  }
#define B2O_TC_PAIR_CASE(BN)                                                           \
  if (pair && bn == BN) {                                                              \
    if (p.resident) return launch<BN, 64, 2, true>(ctx, amap, L, p, smem_bytes, st);   \
    if (p.halo) return launch<BN, 64, 1, true>(ctx, amap, L, p, smem_bytes, st);       \
    return launch<BN, 64, 0, true>(ctx, amap, L, p, smem_bytes, st);                   \
  }
  B2O_TC_PAIR_CASE(64); B2O_TC_PAIR_CASE(128);
#undef B2O_TC_PAIR_CASE
#define B2O_TC_CASE(BN, KC)                                                            \
  if (bn == BN && kch == KC) {                                                         \
    if (p.resident) return launch<BN, KC, 2, false>(ctx, amap, L, p, smem_bytes, st);  \
    if (p.halo) return launch<BN, KC, 1, false>(ctx, amap, L, p, smem_bytes, st);      \
    return launch<BN, KC, 0, false>(ctx, amap, L, p, smem_bytes, st);                  \
  }
  B2O_TC_CASE(16, 64); B2O_TC_CASE(32, 64); B2O_TC_CASE(64, 64); B2O_TC_CASE(128, 64);
  B2O_TC_CASE(16, 32); B2O_TC_CASE(32, 32);
  B2O_TC_CASE(32, 16); B2O_TC_CASE(64, 16);
#undef B2O_TC_CASE
  ctx->set_error("conv_tc_run: no kernel instance for " + L.name);
  return B2O_ERR_ARG;
}
