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
//   runs its epilogue while the other keeps the tensor cores busy.  64-channel fp16 layers run transposed (p.ct,
//   see conv_tc_body): one m64 (channels) x n128 (pixels) x k16 wgmma per k step and TMA-stored outputs;
//   the streamed 128-channel halo layers run transposed on 16 x 16-pixel tiles (p.tile256): both warpgroups read every
//   stage, one m64 (their 64 channels) x n256 (pixels) x k16 wgmma each per k step; the generic 128-channel tiles of
//   layers with cout % 256 == 0 run paired n-tiles (p.coop_n): both warpgroups share each activation box, one n-tile each.
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
  int ct;                                 // channels by pixels (64-channel fp16 layers, see conv_tc_body)
  int tile256;                            // channels by pixels on 16 x 16-pixel tiles (streamed 128-channel halo layers)
  int off_out;                            // ct, tile256: the two warpgroups' output tiles (+ pooled tiles)
  int aff_smem;                           // epilogue constants staged in shared memory behind the barriers (B2O_TC_AFF=smem)
  int aff_const;                          // epilogue constants read from the AffConst kernel parameter (default)
  int coop_n;                             // paired n-tiles: both warpgroups share every activation box (generic tiles)
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
// ---- epilogue stores of the channels-by-pixels body: shared-memory tile -> global through TMA (bulk groups)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
          reinterpret_cast<uint64_t>(m)),
      "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// four transposed 8x8 b16 matrices: register j of a lane holds row lane / 4, columns 2 (lane % 4) + {0, 1} of matrix j;
// lanes 8j .. 8j + 7 give the addresses of the 8 stored rows (= the matrix's columns) of matrix j
__device__ __forceinline__ void stmatrix_x4_trans(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r0), "r"(r1),
               "r"(r2), "r"(r3)
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
template <>
__device__ __forceinline__ void wgmma_f16<256>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
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
// CT:   channels by pixels (p.ct), for 64-channel fp16 layers: D^T[cout, pixel] = W . X^T, the filter stage (K-major, 64 rows)
//       as the wgmma A operand and the pixel stage (K-major, 128 rows) as B -- one m64 x n128 x k16 per k step instead
//       of two m64 x n64 x k16 that both read the same B tile, so a k step reads 6 KB of shared memory instead of 8 KB.
//       Every output sums the same products in the same order: results are bit-identical to the pixels-by-channels
//       body.  A thread then holds 2 channels x 32 pixels, so the epilogue goes through a 16 KB shared-memory
//       tile per warpgroup (stmatrix .trans) and TMA stores (omap, and pmap for the fused pool), which clip at the
//       image edges.
// WIDE: channels by pixels on 16 (w) x 16 (h)-pixel halo tiles (p.tile256), for the 128-channel layers whose filter bank
//       streams through the ring.  A stage is one (64, 16, 18) activation box plus the three dy taps' 128 filter rows,
//       so each filter stage serves 256 pixels: a third less L2 -> shared-memory traffic per MMA than on 8 x 16 tiles.
//       The two consumer warpgroups work cooperatively (no ping-pong): both read every stage, warpgroup wg computes
//       output channels 64 wg .. 64 wg + 63 of all 256 pixels with one m64 x n256 x k16 per (dy, k step), A = its 64
//       filter rows of the tap, B = pixel rows 16 dy .. 16 dy + 255 of the stage.  The sums are those of the 8 x 16
//       tiles, in the same order: bit-identical results.  The epilogue is the CT one, once per 128-pixel half of the
//       tile (tile rows 0-7, then 8-15), each a (64, 16, 8) TMA store at the warpgroup's channels.  Only two 84 KB stages
//       fit, so a slot lands in three parts (halo box + dy = 0's rows on full[s], dy = 1, 2 on tap_full) and the MMAs
//       of each dy start as soon as their part is in.
// COOP: paired n-tiles (p.coop_n) on generic 128-channel tiles: a work unit is tiles 2u and 2u + 1, i.e. n-tiles 2j and
//       2j + 1 of one pixel tile, and warpgroup wg computes n-tile 2j + wg.  Per (tap, chunk) the producer fills a pair
//       of ring slots: slot s gets the activation box and n-tile 2j's filter rows, slot s + 1 only n-tile 2j + 1's
//       filter rows (in its B part), so the activation box is fetched once for both n-tiles: 24 instead of 32 KB per
//       128 x 128 x 64 block.  Both warpgroups wait on both slots and release both (no ping-pong); each issues the
//       two m64 x n128 x k16 of the pixels-by-channels body per k step, A from slot s, B from slot s + wg, and runs the
//       same epilogue at its n-tile: every output gets the same products in the same order, bit-identical results.
template <int BLOCK_N, int KCH, int MODE, bool PAIR, bool UPADD, bool CT, bool WIDE = false, bool COOP = false>
__device__ __forceinline__ void conv_tc_body(const CUtensorMap& amap, const CUtensorMap& bmap, const CUtensorMap& omap,
                                             const CUtensorMap& pmap, const TcParams& p, const AffConst& ac) {
  static_assert(!CT || (!PAIR && !UPADD && (WIDE ? (BLOCK_N == 128 && KCH == 64 && MODE == 1) : BLOCK_N == 64)),
                "channels by pixels: 64-channel single-CTA tiles, or 128-channel streamed halo tiles (WIDE)");
  static_assert(!WIDE || CT, "the 16 x 16 tiles run channels by pixels");
  static_assert(!COOP || (BLOCK_N == 128 && KCH == 64 && MODE == 0 && !PAIR && !UPADD && !CT),
                "paired n-tiles: generic single-CTA 128-channel tiles, pixels by channels");
  constexpr bool HALO = MODE >= 1, RESIDENT = MODE == 2;
  constexpr bool SHARED = WIDE || COOP;                    // both consumer warpgroups read every stage (no ping-pong)
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
  uint64_t* tap_full = res_full + 1;                       // WIDE: filter rows of tap dy = 1, 2 of slot s at [(dy - 1) MAX_RING + s]

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
      // one arrival per warp of the stage's consumer warpgroup (of both CTAs of a pair; of both warpgroups on 16 x 16
      // tiles and paired n-tiles) once its MMAs read it
      mbar_init(&empty[s], (PAIR ? 2 : 1) * ((COOP || p.tile256) ? 2 : 1) * TILE_WARPS);
    }
    mbar_init(res_full, 1);
    for (int i = 0; i < 2 * MAX_RING; ++i) mbar_init(&tap_full[i], 1);
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
      // COOP: the CTA's units u = cta, cta + ncta, ... as their first tiles 2u (n-tile c0 = 2j, n_tiles being even)
      for (TileIter ti(p, COOP ? 2 * cta : cta, COOP ? 2 * ncta : ncta); ti.valid(p); ti.next(p)) {
        const int tw0 = ((ti.c1 << pair_shift) + static_cast<int>(rank)) << p.bw_log2, th0 = ti.c2 << p.bh_log2, tn0 = ti.c3 << p.bn_log2;
        int ky = 0, kx = 0;
        for (int g = 0; g < groups; ++g) {
          const int ax = HALO ? (tw0 + g - 1) : (tw0 + (kx - half_k) * p.dil);
          const int ay = HALO ? (th0 - 1) : (th0 + (ky - half_k) * p.dil);
          for (int kc = 0; kc < kchunks; ++kc) {
            mbar_wait(&empty[s], ph ^ 1);
            uint8_t* const st = smem + s * p.stage_bytes;
            // WIDE: full[s] covers the halo box and tap dy = 0's filter rows, taps 1 and 2 land on their own barriers, so
            // the consumers start on dy = 0 before the whole 84 KB slot is in
            mbar_expect_tx(&full[s], static_cast<uint32_t>(WIDE ? p.a_bytes + B_BYTES : p.stage_tx));
            tma_load_4d(&amap, &full[s], st, kc * KCH, ax, ay, tn0);
            if (!RESIDENT) {
#pragma unroll
              for (int t = 0; t < TAPS_PER_A; ++t) {
                const int tap = HALO ? (t * 3 + g) : g;
                uint8_t* const dst = st + p.a_stride + t * B_BYTES;
                uint64_t* const bar = (WIDE && t > 0) ? &tap_full[(t - 1) * MAX_RING + s] : &full[s];
                if (WIDE && t > 0) mbar_expect_tx(bar, static_cast<uint32_t>(B_BYTES));
                if (PAIR)
                  tma_load_2d_multicast(&bmap, bar, dst + rank * B_HALF, tap * p.cin + kc * KCH,
                                        ti.c0 * BLOCK_N + static_cast<int>(rank) * (BLOCK_N / 2));
                else
                  tma_load_2d(&bmap, bar, dst, tap * p.cin + kc * KCH, ti.c0 * BLOCK_N);
              }
            }
            if (COOP) {                                    // slot s + 1: the second n-tile's filter rows only
              mbar_wait(&empty[s + 1], ph ^ 1);
              mbar_expect_tx(&full[s + 1], static_cast<uint32_t>(B_BYTES));
              tma_load_2d(&bmap, &full[s + 1], st + p.stage_bytes + p.a_stride, g * p.cin + kc * KCH,
                          (ti.c0 + 1) * BLOCK_N);
            }
            if (COOP ? (s += 2) == (p.ns & ~1) : ++s == p.ns) { s = 0; ph ^= 1; }   // COOP: the ring as slot pairs
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
    constexpr uint32_t TAP_BYTES = (WIDE ? 16 : 8) * KCH * 2;   // halo: one dy tap = one tile row (8 | 16 pixels) further
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
    // the CTA's tiles wg, wg + 2, ... (WIDE: both warpgroups take every tile; COOP: every unit, n-tile c0 + wg of it)
    TileIter ti(p, COOP ? 2 * cta : cta + (WIDE ? 0 : wg * ncta), (COOP ? 2 : (WIDE ? 1 : 2)) * ncta);
    if (!SHARED && wg == 1) skip_tile();
    if (RESIDENT && ti.valid(p)) mbar_wait(res_full, 0);
    float acc[2 * NACC];                                     // [rows 0-63 | rows 64-127] (WIDE: pixels 0-127 | 128-255)
  #pragma unroll
    for (int i = 0; i < 2 * NACC; ++i) acc[i] = 0.0f;
    for (bool after_other = !SHARED && wg == 1; ti.valid(p); ti.next(p), after_other = !SHARED) {
      if (after_other) named_bar_sync(1 + wg, 2 * 128);      // the other warpgroup has issued the previous tile
      // ---- main loop: every stage of the tile, MMAs in (dx | tap, chunk, dy, k) order, both halves per k step
      int prev = -1;
      uint32_t accumulate = 0;
      for (int g = 0; g < groups; ++g) {
        for (int kc = 0; kc < kchunks; ++kc) {
          mbar_wait(&full[s], ph);
          if (COOP) mbar_wait(&full[s + 1], ph);
          const uint64_t adesc = desc_a0 + static_cast<uint64_t>(static_cast<uint32_t>(s * p.stage_bytes) >> 4);
          const int bs = COOP ? s + wg : s;                  // the slot holding this warpgroup's filter rows
  #pragma unroll
          for (int i = 0; i < 2 * NACC; ++i) reg_fence(acc[i]);
          wgmma_fence();
  #pragma unroll
          for (int t = 0; t < TAPS_PER_A; ++t) {
            if (WIDE && t > 0) {                             // this tap's filter rows (full[s]: halo box + dy = 0)
              mbar_wait(&tap_full[(t - 1) * MAX_RING + s], ph);
              wgmma_fence();
            }
            const uint32_t boff = RESIDENT ? static_cast<uint32_t>(((t * 3 + g) * kchunks + kc) * B_BYTES)
                                           : static_cast<uint32_t>(bs * p.stage_bytes + t * B_BYTES);
            const uint64_t bdesc = desc_b0 + static_cast<uint64_t>(boff >> 4);
  #pragma unroll
            for (int k = 0; k < KSTEPS; ++k) {
              if constexpr (WIDE) {
                wgmma_f16<256>(acc, bdesc + static_cast<uint64_t>((wg * HALF_BYTES + k * 32) >> 4),
                               adesc + static_cast<uint64_t>((t * TAP_BYTES + k * 32) >> 4), accumulate);
              } else if constexpr (CT) {
                wgmma_f16<128>(acc, bdesc + static_cast<uint64_t>((k * 32) >> 4),
                               adesc + static_cast<uint64_t>((t * TAP_BYTES + k * 32) >> 4), accumulate);
              } else {
  #pragma unroll
                for (int mh = 0; mh < 2; ++mh)
                  wgmma_f16<BLOCK_N>(acc + mh * NACC, adesc + static_cast<uint64_t>((mh * HALF_BYTES + t * TAP_BYTES + k * 32) >> 4),
                                     bdesc + static_cast<uint64_t>((k * 32) >> 4), accumulate);
              }
              accumulate = 1;
            }
            if (WIDE) {
              // one commit group per tap: once dy = 0's MMAs are issued, the previous stage's are waited for and
              // the stage released, before this stage's dy = 1, 2 rows have to be in
              wgmma_commit();
              if (t == 0) {
                wgmma_wait<1>();
                if (prev >= 0) {
                  __syncwarp();
                  if (lane == 0) release(prev);
                }
              }
            }
          }
          if (!WIDE) {
            wgmma_commit();
            wgmma_wait<1>();                                 // the previous stage's MMAs are done: release it
            if (prev >= 0) {
              __syncwarp();
              if (lane == 0) {
                release(prev);
                if (COOP) release(prev + 1);
              }
            }
          }
          prev = s;
          if (COOP ? (s += 2) == (p.ns & ~1) : ++s == p.ns) { s = 0; ph ^= 1; }
        }
      }
      if (!SHARED) {
        if (ti.tile + ncta < p.total_tiles) named_bar_arrive(1 + (wg ^ 1), 2 * 128);   // the CTA's next tile may start
        skip_tile();
      }
      wgmma_wait<0>();
  #pragma unroll
      for (int i = 0; i < 2 * NACC; ++i) reg_fence(acc[i]);
      __syncwarp();
      if (lane == 0) {
        release(prev);
        if (COOP) release(prev + 1);
      }

      // ---- epilogue from the registers, one 64-row half after the other
      const int c_base = (COOP ? ti.c0 + wg : ti.c0) * BLOCK_N;
      if constexpr (CT) {
        // this thread holds channels r0, r0 + 8 (hh = 0, 1) x pixels 8i + 2q, 8i + 2q + 1 in acc[4i + 2hh + 0, 1]
        // (i < 16; WIDE: i < 32, two 128-pixel halves = tile rows 0-7 and 8-15, each stored on its own): the same
        // per-element fmaf / ReLU / fmaf and fp16 rounding as below, with per-channel scalars
        constexpr int BW = WIDE ? 16 : 8;                      // halo tile width (the fused pool runs on halo tiles only)
        constexpr int OUT_TILE = 128 * 64 * 2, POOL_TILE = 32 * 64 * 2;
        uint8_t* const otile = smem + p.off_out + wg * OUT_TILE;
        uint8_t* const ptile = smem + p.off_out + 2 * OUT_TILE + wg * POOL_TILE;
        const int et = threadIdx.x & 127;
        const int c_wg = c_base + (WIDE ? WG_M * wg : 0);      // WIDE: this warpgroup's 64 of the tile's 128 channels
  #pragma unroll
        for (int half = 0; half < (WIDE ? 2 : 1); ++half) {
          // keeps the second half's arithmetic behind the first half's stores (registers: 128 accumulators live)
  #pragma unroll
          for (int i = 64 * half; i < 64 * half + 64; ++i) reg_fence(acc[i]);
          float a1[2], b1[2], a2[2], b2[2];
  #pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int c = c_wg + r0 + 8 * hh;
            if constexpr (WIDE) {                            // read from p here: no pointers held across the main loop
              a1[hh] = p.aff_const ? ac.s1[c] : p.s1[c]; b1[hh] = p.aff_const ? ac.t1[c] : p.t1[c];
              a2[hh] = p.s2 == nullptr ? 0.0f : (p.aff_const ? ac.s2[c] : p.s2[c]);
              b2[hh] = p.s2 == nullptr ? 0.0f : (p.aff_const ? ac.t2[c] : p.t2[c]);
            } else {
              a1[hh] = e_s1[c]; b1[hh] = e_t1[c];
              a2[hh] = p.s2 != nullptr ? e_s2[c] : 0.0f; b2[hh] = p.s2 != nullptr ? e_t2[c] : 0.0f;
            }
          }
          // pixels 8i + 2q, 8i + 2q + 1 of channel r0 + 8hh, as fp16.  The 64-channel body converts all 32 pairs before
          // the stores; WIDE converts each right before its stmatrix, so only four are live beside the other half's
          // 64 accumulators
          auto h2 = [&](int i, int hh) {
            float y0 = fmaf(acc[64 * half + 4 * i + 2 * hh], a1[hh], b1[hh]);
            float y1 = fmaf(acc[64 * half + 4 * i + 2 * hh + 1], a1[hh], b1[hh]);
            if (p.relu) { y0 = fmaxf(y0, 0.0f); y1 = fmaxf(y1, 0.0f); }
            if (p.s2 != nullptr) { y0 = fmaf(y0, a2[hh], b2[hh]); y1 = fmaf(y1, a2[hh], b2[hh]); }
            const __half2 h = __floats2half2_rn(y0, y1);
            return *reinterpret_cast<const uint32_t*>(&h);
          };
          uint32_t hv[16][2];
          if constexpr (!WIDE) {
  #pragma unroll
            for (int i = 0; i < 16; ++i) { hv[i][0] = h2(i, 0); hv[i][1] = h2(i, 1); }
          }
          auto hval = [&](int i, int hh) {
            if constexpr (WIDE) return h2(i, hh);
            else return hv[i][hh];
          };
          // NHWC tile [128 pixel rows][64 channels] with the 128B swizzle of omap / pmap: 16-byte chunk j of row r sits
          // at chunk j ^ (r & 7).  An 8x8 block (8 channels x 8 pixels) stored transposed = 8 pixel rows of one chunk.
          if (et == 0) bulk_wait_read_all();                 // the previous half's / tile's stores have read the tile
          named_bar_sync(3 + wg, 128);
          {
            const int m = lane >> 3, r = lane & 7;             // this lane addresses row r of matrix m = (i & 1, hh)
            const uint32_t row = smem_u32(otile) + static_cast<uint32_t>(r * 128 + (((2 * (warp & 3) + (m & 1)) ^ r) << 4));
  #pragma unroll
            for (int i0 = 0; i0 < 16; i0 += 2)
              stmatrix_x4_trans(row + static_cast<uint32_t>((8 * (i0 + (m >> 1))) * 128), hval(i0, 0), hval(i0, 1),
                                hval(i0 + 1, 0), hval(i0 + 1, 1));
          }
          fence_proxy_async_smem();
          named_bar_sync(3 + wg, 128);
          if (p.pool_out != nullptr) {   // halo half-tile BW x 128/BW -> pooled BW/2 x 64/BW, max(max(v00, v10), max(v01, v11))
  #pragma unroll (WIDE ? 1 : 2)                            // WIDE: rolled, for registers
            for (int j = 0; j < 2; ++j) {
              const int item = et + 128 * j, pr = item >> 3, ch = item & 7;
              const int r00 = 2 * (pr % (BW / 2)) + 2 * BW * (pr / (BW / 2));   // (2 pw, 2 ph) in the BW-wide tile
              auto ld = [&](int rr) { return *reinterpret_cast<const uint4*>(otile + rr * 128 + ((ch ^ (rr & 7)) << 4)); };
              const uint4 v00 = ld(r00), v10 = ld(r00 + BW), v01 = ld(r00 + 1), v11 = ld(r00 + BW + 1);
              uint4 o;
              const __half2* a = reinterpret_cast<const __half2*>(&v00);
              const __half2* b = reinterpret_cast<const __half2*>(&v10);
              const __half2* c = reinterpret_cast<const __half2*>(&v01);
              const __half2* d = reinterpret_cast<const __half2*>(&v11);
              __half2* op = reinterpret_cast<__half2*>(&o);
  #pragma unroll
              for (int e = 0; e < 4; ++e) op[e] = __hmax2(__hmax2(a[e], b[e]), __hmax2(c[e], d[e]));
              *reinterpret_cast<uint4*>(ptile + pr * 128 + ((ch ^ (pr & 7)) << 4)) = o;
            }
            fence_proxy_async_smem();
            named_bar_sync(3 + wg, 128);
          }
          if (et == 0) {
            const int tw0 = ti.c1 << p.bw_log2, th0 = (ti.c2 << p.bh_log2) + 8 * half, tn0 = ti.c3 << p.bn_log2;
            if (p.write_full) tma_store_4d(&omap, otile, c_wg, tw0, th0, tn0);
            if (p.pool_out != nullptr) tma_store_4d(&pmap, ptile, c_wg, tw0 >> 1, th0 >> 1, tn0);
            bulk_commit();
          }
        }
      }
  #pragma unroll
      for (int mh = 0; mh < (CT ? 0 : 2); ++mh) {
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
    if (CT && (threadIdx.x & 127) == 0) bulk_wait_all();    // the output tiles stay until the last stores are done
  }
  // neither CTA of a pair leaves while the other may still signal its barriers
  if (PAIR) cluster_sync_all();
}

// The 64-channel single-CTA instances carry both bodies and take the channels-by-pixels one when p.ct is set; the
// streamed 128-channel halo instance takes the 16 x 16-tile channels-by-pixels body when p.tile256 is set, and the
// generic 128-channel instance the paired n-tiles when p.coop_n is set.
template <int BLOCK_N, int KCH, int MODE, bool PAIR, bool UPADD = false>
__global__ void __launch_bounds__(NUM_THREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap amap, const __grid_constant__ CUtensorMap bmap,
               const __grid_constant__ CUtensorMap omap, const __grid_constant__ CUtensorMap pmap,
               const TcParams p, const __grid_constant__ AffConst ac) {
  if constexpr (BLOCK_N == 64 && !PAIR && !UPADD) {
    if (p.ct) {
      conv_tc_body<BLOCK_N, KCH, MODE, PAIR, UPADD, true>(amap, bmap, omap, pmap, p, ac);
      return;
    }
  }
  if constexpr (BLOCK_N == 128 && KCH == 64 && MODE == 1 && !PAIR && !UPADD) {
    if (p.tile256) {
      conv_tc_body<BLOCK_N, KCH, MODE, PAIR, UPADD, true, true>(amap, bmap, omap, pmap, p, ac);
      return;
    }
  }
  if constexpr (BLOCK_N == 128 && KCH == 64 && MODE == 0 && !PAIR && !UPADD) {
    if (p.coop_n) {
      conv_tc_body<BLOCK_N, KCH, MODE, PAIR, UPADD, false, false, true>(amap, bmap, omap, pmap, p, ac);
      return;
    }
  }
  conv_tc_body<BLOCK_N, KCH, MODE, PAIR, UPADD, false>(amap, bmap, omap, pmap, p, ac);
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

// The tensor-core tiling of a layer: K chunk kch (channels per stage) and N tile block_n; block_n = 0 leaves the layer to
// the SIMT engine.  pair_ok: CTA pairs can run it (each CTA fetches block_n / 2 filter rows of a 64-channel chunk).
struct TcTiling {
  int kch, block_n;
  bool pair_ok;
};
TcTiling plan_tc_tiling(int cin, int cout) {
  TcTiling t = {cin % 64 == 0 ? 64 : (cin % 32 == 0 ? 32 : (cin % 16 == 0 ? 16 : 0)), 0, false};
  if (t.kch == 0 || cout % 16 != 0) return t;
  // N tile <= 128: a consumer thread holds BLOCK_N / 2 fp32 accumulators in registers
  int bn = 128;
  while (bn > 16 && (cout % bn != 0)) bn >>= 1;
  if (cout % bn != 0) return t;
  if (t.kch == 32 && bn > 32) return t;                    // instantiated combinations only
  if (t.kch == 16 && bn != 32 && bn != 64) return t;
  t.block_n = bn;
  t.pair_ok = t.kch == 64 && bn >= 64;
  return t;
}

// The context's switches a plan depends on (the b2o_ctx fields of the same names).
struct TcOptions {
  int conv_engine;
  bool tc_swap, tc_pair, tc_pair_generic, tc_aff_const;
  int sm_count;
};

// What a plan reads of a layer (the ConvLayer fields of the same names).  host_aff: the epilogue constants, and the
// fused tail's when there is one, have host copies, so they can travel in the AffConst kernel parameter.
struct TcLayerShape {
  const char* name;
  int cin, cout, ksize, dil, kch, block_n;
  bool pair_ok, host_aff;
};

// A conv_tc_kernel<BLOCK_N, KCH, MODE, PAIR, UPADD> instance.
struct TcInstance {
  int block_n, kch, mode;
  bool pair, upadd;
};

// How one convolution runs: the kernel's parameters without the pointer fields and the strides and epilogue switches
// that go with them, the instance, the launch shape and the TMA boxes of the activation map, the channels-by-pixels
// output map and its pooled map.
struct TcPlan {
  TcParams p;
  TcInstance inst;
  int smem_bytes, grid;
  cuuint32_t abox[4], obox[4], pbox[4];
};

template <int BLOCK_N, int KCH, int MODE, bool PAIR, bool UPADD>
int launch(b2o_ctx* ctx, const ConvLayer& L, const TcPlan& plan, const CUtensorMap& amap, const CUtensorMap& omap,
           const CUtensorMap& pmap, const AffConst& ac, cudaStream_t st) {
  const void* fn = reinterpret_cast<const void*>(&conv_tc_kernel<BLOCK_N, KCH, MODE, PAIR, UPADD>);
  if (!ctx->configured.count(fn)) {                        // a per-device attribute: remembered per context
    B2O_CUDA_CHECK(ctx, cudaFuncSetAttribute(conv_tc_kernel<BLOCK_N, KCH, MODE, PAIR, UPADD>,
                                             cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_TOTAL));
    ctx->configured.insert(fn);
  }
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  if (ctx->profile) {
    B2O_CUDA_CHECK(ctx, cudaEventCreate(&e0));
    B2O_CUDA_CHECK(ctx, cudaEventCreate(&e1));
    B2O_CUDA_CHECK(ctx, cudaEventRecord(e0, st));
  }
  const TcParams& p = plan.p;
  if (PAIR) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(plan.grid);
    cfg.blockDim = dim3(NUM_THREADS);
    cfg.dynamicSmemBytes = static_cast<size_t>(plan.smem_bytes);
    cfg.stream = st;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = 2; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    B2O_CUDA_CHECK(ctx, cudaLaunchKernelEx(&cfg, conv_tc_kernel<BLOCK_N, KCH, MODE, PAIR, UPADD>, amap, L.wmap_pair, omap, pmap, p, ac));
  } else {
    conv_tc_kernel<BLOCK_N, KCH, MODE, PAIR, UPADD><<<plan.grid, NUM_THREADS, plan.smem_bytes, st>>>(amap, L.wmap, omap, pmap, p, ac);
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

// Every compiled instance: MODE 0 = generic tiles, 1 = halo tiles (3x3, dilation 1), 2 = halo tiles + resident filter
// bank; CTA pairs for 64-channel chunks with BLOCK_N >= 64; the decoder's upsample-add on generic 1x1 tiles.
typedef int (*LaunchFn)(b2o_ctx*, const ConvLayer&, const TcPlan&, const CUtensorMap&, const CUtensorMap&,
                        const CUtensorMap&, const AffConst&, cudaStream_t);
struct TcKernel {
  TcInstance inst;
  LaunchFn launch;
};
const TcKernel kTcKernels[] = {
    {{16, 64, 0, false, false}, launch<16, 64, 0, false, false>},   {{16, 64, 1, false, false}, launch<16, 64, 1, false, false>},
    {{16, 64, 2, false, false}, launch<16, 64, 2, false, false>},   {{32, 64, 0, false, false}, launch<32, 64, 0, false, false>},
    {{32, 64, 1, false, false}, launch<32, 64, 1, false, false>},   {{32, 64, 2, false, false}, launch<32, 64, 2, false, false>},
    {{64, 64, 0, false, false}, launch<64, 64, 0, false, false>},   {{64, 64, 1, false, false}, launch<64, 64, 1, false, false>},
    {{64, 64, 2, false, false}, launch<64, 64, 2, false, false>},   {{128, 64, 0, false, false}, launch<128, 64, 0, false, false>},
    {{128, 64, 1, false, false}, launch<128, 64, 1, false, false>}, {{128, 64, 2, false, false}, launch<128, 64, 2, false, false>},
    {{16, 32, 0, false, false}, launch<16, 32, 0, false, false>},   {{16, 32, 1, false, false}, launch<16, 32, 1, false, false>},
    {{16, 32, 2, false, false}, launch<16, 32, 2, false, false>},   {{32, 32, 0, false, false}, launch<32, 32, 0, false, false>},
    {{32, 32, 1, false, false}, launch<32, 32, 1, false, false>},   {{32, 32, 2, false, false}, launch<32, 32, 2, false, false>},
    {{32, 16, 0, false, false}, launch<32, 16, 0, false, false>},   {{32, 16, 1, false, false}, launch<32, 16, 1, false, false>},
    {{32, 16, 2, false, false}, launch<32, 16, 2, false, false>},   {{64, 16, 0, false, false}, launch<64, 16, 0, false, false>},
    {{64, 16, 1, false, false}, launch<64, 16, 1, false, false>},   {{64, 16, 2, false, false}, launch<64, 16, 2, false, false>},
    {{64, 64, 0, true, false}, launch<64, 64, 0, true, false>},     {{64, 64, 1, true, false}, launch<64, 64, 1, true, false>},
    {{64, 64, 2, true, false}, launch<64, 64, 2, true, false>},     {{128, 64, 0, true, false}, launch<128, 64, 0, true, false>},
    {{128, 64, 1, true, false}, launch<128, 64, 1, true, false>},   {{128, 64, 2, true, false}, launch<128, 64, 2, true, false>},
    {{64, 64, 0, false, true}, launch<64, 64, 0, false, true>},     {{128, 64, 0, false, true}, launch<128, 64, 0, false, true>},
};

LaunchFn find_kernel(const TcInstance& k) {
  for (const TcKernel& e : kTcKernels)
    if (e.inst.block_n == k.block_n && e.inst.kch == k.kch && e.inst.mode == k.mode && e.inst.pair == k.pair &&
        e.inst.upadd == k.upadd)
      return e.launch;
  return nullptr;
}

// Every decision about how a convolution of L over `in` runs on the tensor cores, with no CUDA call: an empty string
// and *plan, or the reason the engine cannot run it.  pool_out and up_add are only read for their shapes (and up_add
// for its alignment).
std::string plan_conv_tc(const TcOptions& o, const TcLayerShape& L, const TensorView& in, int out_f32,
                         const TensorView* pool_out, bool tail, const TensorView* up_add, TcPlan* plan) {
  auto refuse = [&](const char* what, const char* after) { return std::string(what) + L.name + after; };
  if (up_add != nullptr && (L.ksize != 1 || L.kch != 64 || L.block_n < 64 || out_f32 || pool_out != nullptr || tail ||
                            up_add->c != L.cout || up_add->n != in.n || 2 * up_add->h != in.h || 2 * up_add->w != in.w ||
                            (up_add->ld % 8) || (reinterpret_cast<uintptr_t>(up_add->ptr) & 15)))
    return refuse("conv_tc_run: up_add needs a 1x1 layer with 64-channel chunks and an exactly half-size fp16 tensor (", ")");
  if (tail && (L.block_n != 16 || L.cout != 16 || pool_out != nullptr))
    return refuse("conv_tc_run: the fused tail needs a 16-channel layer (", ")");
  if (L.block_n == 0) return refuse("conv_tc_run: layer ", " not eligible");
  const int kch = L.kch, bn = L.block_n;
  const int taps = L.ksize * L.ksize, kchunks = L.cin / kch;
  const int b_bytes = bn * kch * 2;

  memset(plan, 0, sizeof(*plan));
  TcParams& p = plan->p;
  p.N = in.n; p.H = in.h; p.W = in.w;
  p.cin = L.cin; p.cout = L.cout; p.ksize = L.ksize; p.dil = L.dil;
  p.out_f32 = out_f32;
  pick_box(in.n, in.h, in.w, &p.bw_log2, &p.bh_log2, &p.bn_log2);
  // halo mode: 3x3, dilation 1, fixed 8 x 16 tile; skip it when that tile wastes >15 % more pixels.  The two
  // modes add the taps in different orders, so the choice must not depend on the batch size (a crop's result
  // may not change with the batch it travels in): both covers are taken per image, as if N were unbounded.
  int dw, dh, dn;
  const double big_n = 1 << 20;
  const double generic_cover = pick_box(1 << 20, in.h, in.w, &dw, &dh, &dn) / big_n;
  const double halo_cover = double((in.w + 7) / 8 * 8) * double((in.h + 15) / 16 * 16);
  const bool want_pool = pool_out != nullptr;
  p.halo = (L.ksize == 3 && L.dil == 1 && o.conv_engine != B2O_CONV_TC_GENERIC &&
            (halo_cover <= 1.15 * generic_cover || want_pool)) ? 1 : 0;
  if (want_pool && !p.halo) return refuse("conv_tc_run: fused pool needs the halo tile (", ")");
  if (want_pool) {
    if (out_f32 || pool_out->c != L.cout || pool_out->h != in.h / 2 || pool_out->w != in.w / 2 || (pool_out->ld % 8))
      return refuse("conv_tc_run: bad pool view for ", "");
    p.PH = pool_out->h; p.PW = pool_out->w;
  }
  if (up_add) { p.UH = up_add->h; p.UW = up_add->w; }
  if (p.halo) { p.bw_log2 = 3; p.bh_log2 = 4; p.bn_log2 = 0; }
  // CTA pairs (opt-in): halo tiles with B2O_TC_PAIR=1, generic tiles too with B2O_TC_PAIR=2; a pair covers
  // two horizontally adjacent tiles.  Same MMAs in the same order per output: bit-identical results.
  const bool pair = o.tc_pair && (p.halo || o.tc_pair_generic) && L.pair_ok && o.conv_engine == B2O_CONV_AUTO &&
                    up_add == nullptr;
  p.tiles_w = (in.w + (1 << p.bw_log2) - 1) >> p.bw_log2;
  if (pair) p.tiles_w = (p.tiles_w + 1) / 2;                // pair columns
  p.tiles_h = (in.h + (1 << p.bh_log2) - 1) >> p.bh_log2;
  p.tiles_n = (in.n + (1 << p.bn_log2) - 1) >> p.bn_log2;
  p.n_tiles = L.cout / bn;
  const long long total = static_cast<long long>(p.tiles_w) * p.tiles_h * p.tiles_n * p.n_tiles;
  if (total > 0x7fffffffLL) return "conv_tc_run: too many tiles";
  p.total_tiles = static_cast<int>(total);
  // channels by pixels for the 64-channel fp16 layers; a pool whose output has no pixel keeps the old path
  const bool ct = o.tc_swap && L.cout == 64 && bn == 64 && !out_f32 && up_add == nullptr && !tail && !pair &&
                  (!want_pool || (in.h >= 2 && in.w >= 2));
  p.ct = ct ? 1 : 0;

  // shared-memory plan: [ring of stages: A box | B boxes][resident filter bank][ct output tiles][barriers][epilogue constants]
  p.aff_const = (o.tc_aff_const && L.cout <= 256 && L.host_aff) ? 1 : 0;
  p.aff_smem = (!p.aff_const && L.cout <= 256) ? 1 : 0;
  const int aff_bytes = (p.aff_smem ? 4 * L.cout * 4 : 0) + (tail ? TAIL_FLOATS * 4 : 0);
  const int tma_out_tiles = 2 * 128 * 64 * 2 + (want_pool ? 2 * 32 * 64 * 2 : 0);   // per warpgroup: 16 KB (+ 4 KB pooled)
  int out_tiles = ct ? tma_out_tiles : 0;
  int budget = SMEM_TOTAL - 1024 /*alignment slack*/ - 512 /*barriers*/ - aff_bytes - out_tiles;
  p.a_bytes = p.halo ? 18 * 8 * kch * 2 : 128 * kch * 2;
  p.a_stride = (p.a_bytes + 1023) / 1024 * 1024;
  const long long res_bytes = static_cast<long long>(taps) * kchunks * b_bytes;
  // (the mbarrier tx-count holds 2^20 - 1 bytes)
  p.resident = (p.halo && p.n_tiles == 1 && res_bytes + 2LL * p.a_stride <= budget && res_bytes <= (1 << 20) - 1) ? 1 : 0;
  // channels by pixels on 16 x 16 tiles for the streamed 128-channel fp16 halo layers (conv_tc_body, WIDE): one filter
  // stage serves 256 pixels.  Only where the 16-wide tile covers the same columns of an image as the 8-wide one, so the
  // choice depends on the layer and the image shape alone, never on the batch.
  const bool tile256 = o.tc_swap && p.halo && !p.resident && kch == 64 && bn == 128 && !pair && !out_f32 &&
                       up_add == nullptr && !tail && (in.w + 15) / 16 * 16 == (in.w + 7) / 8 * 8 &&
                       (!want_pool || (in.h >= 2 && in.w >= 2));
  if (tile256) {
    p.tile256 = 1;
    p.bw_log2 = 4;
    p.tiles_w = (in.w + 15) >> 4;
    p.total_tiles = p.tiles_w * p.tiles_h * p.tiles_n * p.n_tiles;     // half of the 8 x 16 tiles' count
    p.a_bytes = p.a_stride = 18 * 16 * kch * 2;                          // 36 KB: (64, 16, 18, 1)
    out_tiles = tma_out_tiles;
    budget -= out_tiles;
  }
  const int b_per_stage = p.resident ? 0 : (p.halo ? 3 : 1);
  p.stage_bytes = p.a_stride + b_per_stage * b_bytes;
  p.stage_tx = p.a_bytes + b_per_stage * b_bytes;
  p.ns = static_cast<int>((budget - (p.resident ? res_bytes : 0)) / p.stage_bytes);
  if (p.ns > MAX_RING) p.ns = MAX_RING;
  if (p.ns < 2) return refuse("conv_tc_run: shared-memory plan failed for ", "");
  // paired n-tiles (conv_tc_body, COOP) on the generic 128-channel tiles of layers with an even number of n-tiles: one
  // activation box per two n-tiles.  Tiles, boxes, stages and grid stay as above; the rule reads the shapes, never the
  // batch.  Short-K layers (down to lstm_in's 2 stages per tile) measured no slower than on the ping-pong schedule,
  // whose epilogue overlap they give up, so there is no threshold on the stage count.  The ring needs two slot pairs
  // (a pair is released once the next pair's MMAs are issued); these 32 KB stages always leave room for three.
  p.coop_n = (!p.halo && kch == 64 && bn == 128 && L.cout % 256 == 0 && !pair && up_add == nullptr && !tail &&
              p.ns >= 4) ? 1 : 0;
  p.off_res = p.ns * p.stage_bytes;
  p.off_out = p.off_res + (p.resident ? static_cast<int>((res_bytes + 1023) / 1024 * 1024) : 0);
  p.off_bar = p.off_out + out_tiles;
  plan->smem_bytes = p.off_bar + 512 + aff_bytes + 1024;
  // the grid is one persistent CTA per SM: a request above half of the SM's 228 KB keeps a second CTA of a small layer
  // from landing on an SM that already runs one while other SMs sit idle
  if (plan->smem_bytes < 116 * 1024) plan->smem_bytes = 116 * 1024;
  // persistent: one CTA per SM; pairs: one cluster of two CTAs per two SMs
  const int units = pair ? o.sm_count / 2 : o.sm_count;
  plan->grid = (p.total_tiles < units ? p.total_tiles : units) * (pair ? 2 : 1);

  // the activation box: one tile, or on halo tiles 8 (tile256: 16) x 18 rows; channels-by-pixels output boxes: 64
  // channels x one tile (tile256: one 16 x 8 half-tile), pooled: the 2x2 max of one 8 x 16 tile or 16 x 8 half-tile
  const cuuint32_t bw = 1u << p.bw_log2, bh = 1u << p.bh_log2, bnn = 1u << p.bn_log2;
  const cuuint32_t abox[4] = {static_cast<cuuint32_t>(kch), bw, p.halo ? 18u : bh, p.halo ? 1u : bnn};
  const cuuint32_t obox[4] = {64, bw, tile256 ? 8u : bh, bnn};
  const cuuint32_t pbox[4] = {64, tile256 ? 8u : 4u, tile256 ? 4u : 8u, 1};
  memcpy(plan->abox, abox, sizeof(abox));
  memcpy(plan->obox, obox, sizeof(obox));
  memcpy(plan->pbox, pbox, sizeof(pbox));
  plan->inst = {bn, kch, p.resident ? 2 : (p.halo ? 1 : 0), pair, up_add != nullptr};
  if (find_kernel(plan->inst) == nullptr) return refuse("conv_tc_run: no kernel instance for ", "");
  return std::string();
}

}  // namespace

int conv_tc_prepare(b2o_ctx* ctx, ConvLayer& L) {
  const TcTiling t = plan_tc_tiling(L.cin, L.cout);
  L.kch = t.kch;
  L.block_n = 0;
  L.pair_ok = false;
  if (t.block_n == 0) return B2O_OK;                       // handled by the SIMT engine
  EncodeTiledFn enc = get_encode();
  if (!enc) { ctx->set_error("cuTensorMapEncodeTiled entry point not available"); return B2O_ERR_CUDA; }
  const cuuint64_t ktot = static_cast<cuuint64_t>(L.ksize) * L.ksize * L.cin;
  cuuint64_t dims[2] = {ktot, static_cast<cuuint64_t>(L.cout)};
  cuuint64_t strides[1] = {ktot * 2};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(L.kch), static_cast<cuuint32_t>(t.block_n)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(&L.wmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, L.w_kmajor, dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_for(L.kch), CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    ctx->set_error("cuTensorMapEncodeTiled(weights " + L.name + ") failed: " + std::to_string(static_cast<int>(r)));
    return B2O_ERR_CUDA;
  }
  L.block_n = t.block_n;
  if (t.pair_ok) {
    cuuint32_t half_box[2] = {static_cast<cuuint32_t>(L.kch), static_cast<cuuint32_t>(t.block_n / 2)};
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
  if (in.c != L.cin || out.c != L.cout || in.n != out.n || in.h != out.h || in.w != out.w) {
    ctx->set_error("conv_tc_run: shape mismatch in " + L.name);
    return B2O_ERR_ARG;
  }
  if ((reinterpret_cast<uintptr_t>(in.ptr) & 15) || (in.ld % 8) || (reinterpret_cast<uintptr_t>(out.ptr) & 15) ||
      (out.ld % (out_f32 ? 4 : 8))) {
    ctx->set_error("conv_tc_run: misaligned view in " + L.name);
    return B2O_ERR_ARG;
  }
  const TcOptions opt = {ctx->conv_engine, ctx->tc_swap, ctx->tc_pair, ctx->tc_pair_generic, ctx->tc_aff_const,
                         ctx->sm_count};
  const int cout = L.cout;
  const bool host_aff = static_cast<int>(L.h_s1.size()) == cout &&
                        (L.s2 == nullptr || static_cast<int>(L.h_s2.size()) == cout) &&
                        (tail == nullptr || tail->h_w6 != nullptr);
  const TcLayerShape shape = {L.name.c_str(), L.cin, cout, L.ksize, L.dil, L.kch, L.block_n, L.pair_ok, host_aff};
  TcPlan plan;
  const std::string err = plan_conv_tc(opt, shape, in, out_f32, pool_out, tail != nullptr, up_add, &plan);
  if (!err.empty()) { ctx->set_error(err); return B2O_ERR_ARG; }

  TcParams& p = plan.p;
  p.s1 = L.s1; p.t1 = L.t1; p.s2 = L.s2; p.t2 = L.t2; p.relu = L.relu;
  p.out = out.ptr; p.out_ld = out.ld; p.write_full = write_full;
  if (pool_out) { p.pool_out = pool_out->ptr; p.pool_ld = pool_out->ld; }
  if (up_add) { p.up_src = up_add->ptr; p.up_ld = up_add->ld; }
  if (tail) { p.tail_w6 = tail->w6; p.tail_b6 = tail->b6; p.tail_w8 = tail->w8; p.tail_b8 = tail->b8; p.tail_out = tail->scores; }
  AffConst ac;                                             // the epilogue constants as a kernel parameter (16 KB)
  if (p.aff_const) {
    const size_t nb = static_cast<size_t>(cout) * sizeof(float);
    memcpy(ac.s1, L.h_s1.data(), nb);
    memcpy(ac.t1, L.h_t1.data(), nb);
    if (L.s2 != nullptr) { memcpy(ac.s2, L.h_s2.data(), nb); memcpy(ac.t2, L.h_t2.data(), nb); }
    if (tail) {                                            // [w6 transposed | b6 | w8 | b8]
      for (int j = 0; j < 16; ++j)
        for (int c = 0; c < 16; ++c) ac.tail[j * 16 + c] = tail->h_w6[c * 16 + j];
      memcpy(ac.tail + 256, tail->h_b6, 16 * sizeof(float));
      memcpy(ac.tail + 272, tail->h_w8, 32 * sizeof(float));
      memcpy(ac.tail + 304, tail->h_b8, 2 * sizeof(float));
    }
  }

  EncodeTiledFn enc = get_encode();
  if (!enc) { ctx->set_error("cuTensorMapEncodeTiled entry point not available"); return B2O_ERR_CUDA; }
  CUtensorMap amap;
  cuuint64_t dims[4] = {static_cast<cuuint64_t>(in.c), static_cast<cuuint64_t>(in.w), static_cast<cuuint64_t>(in.h),
                        static_cast<cuuint64_t>(in.n)};
  cuuint64_t strides[3] = {static_cast<cuuint64_t>(in.ld) * 2, static_cast<cuuint64_t>(in.ld) * 2 * in.w,
                           static_cast<cuuint64_t>(in.ld) * 2 * in.w * in.h};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(&amap, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, in.ptr, dims, strides, plan.abox, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_for(L.kch), CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    ctx->set_error("cuTensorMapEncodeTiled(activation for " + L.name + ") failed: " +
                   std::to_string(static_cast<int>(r)));
    return B2O_ERR_CUDA;
  }
  // channels-by-pixels output maps: 4-D (c, w, h, n) over the layer's cout-channel view (a channel slice: base pointer +
  // ld)
  CUtensorMap omap, pmap;
  memset(&omap, 0, sizeof(omap));
  memset(&pmap, 0, sizeof(pmap));
  auto encode_out = [&](CUtensorMap* m, void* ptr, int ld, int n, int h, int w, const cuuint32_t* obox) {
    cuuint64_t odims[4] = {static_cast<cuuint64_t>(cout), static_cast<cuuint64_t>(w), static_cast<cuuint64_t>(h),
                           static_cast<cuuint64_t>(n)};
    cuuint64_t ostr[3] = {static_cast<cuuint64_t>(ld) * 2, static_cast<cuuint64_t>(ld) * 2 * w,
                          static_cast<cuuint64_t>(ld) * 2 * w * h};
    return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, ptr, odims, ostr, obox, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  };
  const bool tma_out = p.ct || p.tile256;
  if (tma_out && write_full) r = encode_out(&omap, out.ptr, out.ld, in.n, in.h, in.w, plan.obox);
  if (tma_out && pool_out && r == CUDA_SUCCESS) r = encode_out(&pmap, pool_out->ptr, pool_out->ld, in.n, p.PH, p.PW, plan.pbox);
  if (r != CUDA_SUCCESS) {
    ctx->set_error("cuTensorMapEncodeTiled(output of " + L.name + ") failed: " + std::to_string(static_cast<int>(r)));
    return B2O_ERR_CUDA;
  }
  if (p.tile256) ++ctx->tc_tile256_launches;
  if (p.coop_n) ++ctx->tc_coop_n_launches;
  return find_kernel(plan.inst)(ctx, L, plan, amap, omap, pmap, ac, st);
}

extern "C" int b2o_conv_plan_test(const b2o_conv_plan_desc* d, b2o_conv_plan* out) {
  if (!d || !out || d->n <= 0 || d->h <= 0 || d->w <= 0 || d->cin <= 0 || d->cout <= 0 || d->ksize <= 0 ||
      d->dilation <= 0 || d->sm_count <= 0 || (d->engine != B2O_CONV_AUTO && d->engine != B2O_CONV_TC_GENERIC))
    return B2O_ERR_ARG;
  const TcOptions opt = {d->engine, d->swap != 0, false, false, true, d->sm_count};
  const TcTiling t = plan_tc_tiling(d->cin, d->cout);
  const TcLayerShape L = {"test", d->cin, d->cout, d->ksize, d->dilation, t.kch, t.block_n, t.pair_ok, true};
  const TensorView in = make_view(nullptr, d->n, d->h, d->w, d->cin);
  const TensorView half = make_view(nullptr, d->n, d->h / 2, d->w / 2, d->cout);     // pooled output, low-res summand
  TcPlan plan;
  if (!plan_conv_tc(opt, L, in, d->out_f32, d->pool ? &half : nullptr, d->tail != 0, d->up_add ? &half : nullptr, &plan).empty())
    return B2O_ERR_ARG;
  const TcParams& p = plan.p;
  out->block_n = plan.inst.block_n; out->kch = plan.inst.kch; out->mode = plan.inst.mode;
  out->pair = plan.inst.pair; out->upadd = plan.inst.upadd;
  out->body = p.tile256 ? 2 : p.ct;
  out->tile_w = 1 << p.bw_log2; out->tile_h = 1 << p.bh_log2; out->tile_n = 1 << p.bn_log2;
  out->tiles = p.total_tiles;
  out->stages = p.ns; out->stage_bytes = p.stage_bytes; out->stage_tx = p.stage_tx;
  out->resident_bytes = p.resident ? d->ksize * d->ksize * d->cin * plan.inst.block_n * 2 : 0;
  out->smem_bytes = plan.smem_bytes; out->grid = plan.grid;
  out->coop_n = p.coop_n;
  return B2O_OK;
}
