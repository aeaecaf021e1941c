/*
 * b2ocr.h -- C-ABI of the H100-native drop-in for keras_ocr.pipeline.Pipeline.recognize().
 *
 * The reference (faustomorales/keras-ocr @ 9661d6f) is pure Python and has no FFI of its own:
 * its "device boundary" is two keras.Model.predict() calls (detection.py:779, recognition.py:535)
 * plus OpenCV calls.  Each entry point below replaces one of those call sites; the reference
 * line(s) it stands in for are cited.  INTEGRATION.md shows the ctypes binding a keras-ocr
 * maintainer would add.
 *
 * Conventions
 *   - plain C: pointers + sizes, no torch / C++ types.  Every function returns 0 on success or a
 *     negative b2o_status; b2o_last_error() gives the message.  No C++ exception crosses the ABI.
 *   - "dev" pointers are CUDA device pointers on the context's device, "host" pointers are host
 *     memory.  All work is enqueued on `stream` (a cudaStream_t passed as void*) and is
 *     asynchronous unless stated.  The caller owns every I/O and workspace buffer; the library
 *     owns only the packed weights inside the context.
 *   - images are NHWC uint8 RGB; activations NHWC fp16; score maps NHWC fp32 (text, link).
 *   - there is NO CPU fallback: without a CUDA device every call fails with B2O_ERR_CUDA.
 */
#ifndef B2OCR_H
#define B2OCR_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b2o_ctx b2o_ctx;

typedef enum {
  B2O_OK = 0,
  B2O_ERR_CUDA = -1,       /* CUDA runtime / driver error (message has the detail)            */
  B2O_ERR_ARG = -2,        /* bad argument (NULL, shape, alignment)                           */
  B2O_ERR_WEIGHTS = -3,    /* missing / mis-shaped tensor in b2o_load_*                       */
  B2O_ERR_WORKSPACE = -4,  /* workspace too small                                             */
  B2O_ERR_STATE = -5       /* call needs weights that were not loaded                         */
} b2o_status;

/* Largest CTC class count (len(alphabet) + 1, recognition.py:376-381) the recognizer accepts; the class
 * count itself is read from the shape of "fc_12.kernel" (256, K) at b2o_load_crnn.                */
#define B2O_MAX_CLASSES 1024

/* One named float32 host tensor (row-major) of a checkpoint, in the reference's naming:
 * CRAFT: PyTorch keys of craft_mlt_25k.pth without the "module." prefix (detection.py:428-468);
 * CRNN : Keras layer names of build_model (recognition.py:214-329), Keras layouts.            */
typedef struct {
  const char* name;
  const float* data;
  int32_t ndim;
  int64_t shape[4];
} b2o_tensor;

/* Which convolution engine to use: B2O_CONV_AUTO = tensor cores (wgmma) wherever the shape allows (the product
 * path), B2O_CONV_SIMT = CUDA-core debug engine used to cross-check the tensor-core kernels. */
enum { B2O_CONV_AUTO = 0, B2O_CONV_SIMT = 1, B2O_CONV_TC_GENERIC = 2 /* tensor cores without halo tiles / fused pool */ };

int b2o_version(void);
int b2o_create(int device, b2o_ctx** out);
void b2o_destroy(b2o_ctx* ctx);
const char* b2o_last_error(const b2o_ctx* ctx);
int b2o_set_conv_engine(b2o_ctx* ctx, int engine);
/* number of kernels this library has launched since creation (bench.py's gpu_launches) */
int64_t b2o_launch_count(const b2o_ctx* ctx);
/* number of tensor-core conv launches since creation that ran channels by pixels on 16 x 16-pixel tiles (the streamed
 * 128-channel 3x3 layers; B2O_TC_SWAP=0 turns that body off): lets tests see which body computed a result */
int64_t b2o_tc_tile256_launches(const b2o_ctx* ctx);
/* number of tensor-core conv launches since creation that ran paired n-tiles (generic 128-channel tiles of layers with
 * cout % 256 == 0: both consumer warpgroups share every activation box) */
int64_t b2o_tc_coop_n_launches(const b2o_ctx* ctx);

/* Measurement hook (bench.py's roofline leg): when enabled, every launch of the tensor-core conv
 * kernel is bracketed by CUDA events on its stream; b2o_profile_read sums the kernel time (ms), the
 * algorithmic FLOPs (2*pixels*taps*cin*cout) and the launch count since b2o_profile_enable(1). */
int b2o_profile_enable(b2o_ctx* ctx, int on);
int b2o_profile_read(b2o_ctx* ctx, double* tc_ms, double* tc_flop, int64_t* tc_launches);

/* Detector() / Recognizer() weight loading (detection.py:686-696, recognition.py:382-404).
 * Folds batch-norm, converts to fp16 and packs into the kernels' layouts on the device.      */
int b2o_load_craft(b2o_ctx* ctx, const b2o_tensor* tensors, int n);
int b2o_load_crnn(b2o_ctx* ctx, const b2o_tensor* tensors, int n);

/* tools.resize_image + tools.pad (tools.py:378-398, 356-375; pipeline.py:44-57), one image:
 * bilinear (OpenCV fixed-point INTER_LINEAR) resize of src (hs x ws x 3) to (hr x wr), written into
 * the top-left of dst image `index` of a (n, hp, wp, 3) batch; the rest is filled with 255.   */
int b2o_resize_pad(b2o_ctx* ctx, const uint8_t* src_dev, int hs, int ws, int hr, int wr,
                   uint8_t* dst_dev, int index, int hp, int wp, void* stream);

/* The same for a batch of n equally sized sources (n,hs,ws,3) in ONE launch (the 4-D ndarray input of
 * pipeline.py:41-42).  gray, when not NULL, also receives cv2.cvtColor(RGB2GRAY) of the padded batch
 * (n,hp,wp) -- recognition.py:510 -- so that the recognizer need not read the batch again.       */
int b2o_resize_pad_batch(b2o_ctx* ctx, const uint8_t* src_dev, int n, int hs, int ws, int hr, int wr,
                         uint8_t* dst_dev, int hp, int wp, uint8_t* gray_dev, void* stream);

/* tools.read for JPEG input (tools.py:19-38: cv2.imread / cv2.imdecode + BGR->RGB) decoded on the GPU by nvJPEG, so
 * that only the compressed file crosses PCIe.  b2o_jpeg_info parses the header (host only); b2o_decode_jpeg writes
 * (height, width, 3) uint8 interleaved RGB at rgb_dev (gray files are expanded to three equal channels, as
 * cv2.imread's default flag does).  nvJPEG is opened with dlopen on first use: B2O_ERR_STATE if the box has none,
 * B2O_ERR_ARG for a stream it refuses (the caller then decodes that file on the host).  Pixels can differ from
 * libjpeg-turbo's (IDCT rounding: <= 4 levels; 4:2:0 chroma upsampling: up to ~25 levels at sharp colour edges, mean < 0.5);
 * tests/test_gpu_parity.py::test_gpu_jpeg_decode states the bounds.                                             */
int b2o_jpeg_info(b2o_ctx* ctx, const uint8_t* data_host, size_t size, int* height, int* width, int* components);
int b2o_decode_jpeg(b2o_ctx* ctx, const uint8_t* data_host, size_t size, uint8_t* rgb_dev, int height, int width,
                    void* stream);

/* cv2.cvtColor(RGB2GRAY) (recognition.py:510) for a whole (n,h,w,3) batch -> (n,h,w).         */
int b2o_rgb_to_gray(b2o_ctx* ctx, const uint8_t* img_dev, int n, int h, int w, uint8_t* gray_dev,
                    void* stream);

/* compute_input + model.predict of Detector.detect (detection.py:34-42, 777-779): CRAFT forward.
 * img: (n,h,w,3) uint8 RGB.  scores: (n, h/2, w/2, 2) float32.                                */
size_t b2o_craft_workspace_bytes(int n, int h, int w);
int b2o_craft_forward(b2o_ctx* ctx, const uint8_t* img_dev, int n, int h, int w, float* scores_dev,
                      void* ws_dev, size_t ws_bytes, void* stream);

/* Test hooks into the CRAFT forward (not on the product path).  The forward is a chain of steps, 0 normalize16,
 * 1 stem, 2 slice1.3, ..., 12 slice4.37, 13 maxpool3, 14 slice5.1, 15 slice5.2, 16 upconv1.0, 17 upconv1.3,
 * 18 / 21 / 24 the decoder upsampling (or the low-resolution half of upconvN.conv.0 when it is commuted),
 * 19 / 22 / 25 upconv2/3/4.conv.0, 20 / 23 / 26 upconv2/3/4.conv.3, 27 conv_cls.0, 28 conv_cls.2, 29 conv_cls.4 (with
 * the fused tail when it runs), 30 the separate head tail; a step with nothing to launch on the selected path is empty.
 * b2o_craft_forward_until runs steps 0..last_step (0 <= last_step <= B2O_CRAFT_LAST_STEP) and returns; b2o_craft_forward
 * is b2o_craft_forward_until(B2O_CRAFT_LAST_STEP).
 * b2o_craft_tap copies one workspace buffer of the most recent forward of this context (n, h, w and ws_dev as passed to
 * it), NHWC fp16 in its full channel stride: "x16" (h,w,16), "a", "b" (h,w,64), "p1" (h/2,w/2,64), "c" (128),
 * "cat4" (192 = [upsampled | s1]), "p2" (h/4,w/4,128), "d" (256), "cat3" (384), "e" (256), "p3" (h/8,w/8,256),
 * "f" (512), "cat2" (768), "g" (512), "p4" (h/16,w/16,512), "hh" (512), "cat1" (1536 = [s5 | s4]), "mp" (512),
 * "s5a" (1024), "u1a" (512), "u1b" (256), "u2a" (h/8: 256), "u2b" (128), "u3a" (h/4: 128), "u3b" (64),
 * "u4a" (h/2: 64), "u4b" (32), "h1", "h2" (32), "h3" (16), "z2" (h/16: 256), "z3" (h/8: 128), "z4" (h/4: 64)
 * (sizes floor-halved per level).  Buffers whose lifetimes do not overlap share memory, so a buffer is only readable
 * while its lifetime includes the forward's last step: otherwise B2O_ERR_STATE, as for ws_dev, n, h, w other than those
 * of the context's last successful forward.  Unknown name or out_bytes smaller than n * h_buf * w_buf * c_buf * 2:
 * B2O_ERR_ARG.                                                                                                 */
#define B2O_CRAFT_LAST_STEP 30
int b2o_craft_forward_until(b2o_ctx* ctx, const uint8_t* img_dev, int n, int h, int w, float* scores_dev,
                            void* ws_dev, size_t ws_bytes, int last_step, void* stream);
int b2o_craft_tap(b2o_ctx* ctx, const char* name, const void* ws_dev, int n, int h, int w, void* out_dev,
                  size_t out_bytes, void* stream);
/* b2o_craft_forward refuses (B2O_ERR_ARG) an image of more than B2O_CRAFT_MAX_PIXELS pixels (h * w): its 64-channel
 * full-resolution maps would pass 2^31 elements per image.  Larger pages run over tiles (below).               */
#define B2O_CRAFT_MAX_PIXELS (1 << 25)

/* Tiled detection (DESIGN.md section 1, "Tiles"): CRAFT over overlapping square tiles of a padded (n, hp, wp, 3)
 * batch, whose cores are stitched into one (n, hp/2, wp/2, 2) score map.  One grid serves every image; per axis of
 * length L: tile extent t = min(tile_size, L), stride s = t - 2 margin, origins o_k = k s (multiples of 32), the fewest
 * tiles that cover L.  The core of tile k is [o_k + margin, o_k + t - margin), except that the first starts at 0 and
 * the last ends at L: the cores partition [0, L).  In the score map every range is halved (floor).
 * b2o_tile_plan: pure host function (no context, no GPU).  tile_size a multiple of 32 with 4 margin <= tile_size <= 2048,
 * margin >= 0 a multiple of 16, hp, wp >= 32, otherwise B2O_ERR_ARG and *plan is not written.                  */
typedef struct {
  int hp, wp, tile_size, margin;
  int t_h, t_w;            /* tile extent per axis: min(tile_size, hp), min(tile_size, wp) */
  int s_h, s_w;            /* stride per axis: t - 2 margin */
  int n_h, n_w;            /* tiles per axis; tiles per image = n_h * n_w */
} b2o_tiles;
int b2o_tile_plan(int hp, int wp, int tile_size, int margin, b2o_tiles* plan);
/* b2o_cut_tiles: tiles [first_tile, first_tile + n_tiles) of img_dev (n, plan->hp, plan->wp, 3) uint8, numbered image by
 * image, then tile row, then tile column, into tiles_dev (n_tiles, t_h, t_w, 3) uint8 (16-byte aligned); pixels past the
 * page are 255, as b2o_resize_pad pads.  b2o_stitch_tiles: the cores of those tiles' scores, tile_scores_dev (n_tiles,
 * t_h/2, t_w/2, 2) float32, copied bit for bit into scores_dev (n, hp/2, wp/2, 2) float32; over the chunks of one batch
 * every score is written exactly once and nothing else is.  Both: plan must be b2o_tile_plan's for its own hp, wp,
 * tile_size, margin, and 0 <= first_tile, n_tiles >= 1, first_tile + n_tiles <= n * n_h * n_w, otherwise B2O_ERR_ARG
 * and nothing is enqueued.                                                                                     */
int b2o_cut_tiles(b2o_ctx* ctx, const uint8_t* img_dev, int n, const b2o_tiles* plan, int first_tile, int n_tiles,
                  uint8_t* tiles_dev, void* stream);
int b2o_stitch_tiles(b2o_ctx* ctx, const float* tile_scores_dev, int n, const b2o_tiles* plan, int first_tile,
                     int n_tiles, float* scores_dev, void* stream);

/* getBoxes (detection.py:207-287).  scores: (n,hs,ws,2) float32.  Writes, per image i,
 * counts[i] = number of boxes found (may exceed max_boxes: then only the first max_boxes are
 * stored and the caller retries with a larger buffer) and boxes[i][k][4][2] float32 in
 * detector-input pixels, in connected-component label order (= reference order).  Slots k >= min(counts[i], max_boxes)
 * of boxes (and of box_scores below) are left as they were.  Every byte of the workspace the result depends on is
 * written by the call itself: the result does not depend on what the workspace held.                          */
size_t b2o_boxes_workspace_bytes(int n, int hs, int ws, int max_boxes);
int b2o_get_boxes(b2o_ctx* ctx, const float* scores_dev, int n, int hs, int ws,
                  float detection_threshold, float text_threshold, float link_threshold,
                  int size_threshold, float* boxes_dev, int32_t* counts_dev, int max_boxes,
                  void* ws_dev, size_t ws_bytes, void* stream);
/* The same, and box_scores_dev (n, max_boxes) float32 receives each stored box's detection score, in box order: the
 * largest text-channel value (channel 0 of scores) over the box's connected component -- the value compared with
 * detection_threshold (detection.py:240-241), so every kept box scores >= detection_threshold.  It is a max over the
 * map's own floats, hence exact.  box_scores_dev == NULL behaves as b2o_get_boxes.                            */
int b2o_get_boxes_scored(b2o_ctx* ctx, const float* scores_dev, int n, int hs, int ws,
                         float detection_threshold, float text_threshold, float link_threshold,
                         int size_threshold, float* boxes_dev, int32_t* counts_dev, float* box_scores_dev,
                         int max_boxes, void* ws_dev, size_t ws_bytes, void* stream);

/* Polygons for curved words (DESIGN.md section 1): b2o_get_boxes_scored, and per kept component a polygon that follows
 * the word's centre line.  boxes, counts and box_scores (may be NULL) are bit-identical to b2o_get_boxes_scored's.
 * polys_dev (n, max_boxes, 2 * (B2O_MAX_POLY_SEGMENTS + 1), 2) float32 and points_dev (n, max_boxes) int32: a word kept
 * as its rectangle has 4 points, the box itself; a polygon of s segments has 2 (s + 1) points, the top edge t_0 .. t_s
 * left to right, then the bottom edge b_s .. b_0, clockwise from the top-left (s = 1 would be the box).  Points past
 * points[k] are NaN.  Slots k >= min(counts[i], max_boxes) are left as they were.  The polygon is a function of the
 * component's filled blob and its box, computed in fp64 with order-independent reductions: bit-identical in any batch
 * and on every run.  Workspace: b2o_boxes_workspace_bytes.                                                       */
#define B2O_MAX_POLY_SEGMENTS 8
int b2o_get_boxes_poly(b2o_ctx* ctx, const float* scores_dev, int n, int hs, int ws,
                       float detection_threshold, float text_threshold, float link_threshold,
                       int size_threshold, float* boxes_dev, int32_t* counts_dev, float* box_scores_dev,
                       float* polys_dev, int32_t* points_dev, int max_boxes, void* ws_dev, size_t ws_bytes,
                       void* stream);

/* b2o_compact_boxes for the polygons of b2o_get_boxes_poly: flat_polys (sum_i min(counts[i], max_boxes),
 * 2 * (B2O_MAX_POLY_SEGMENTS + 1), 2), flat_points and image_index, each sized for n * max_boxes entries.        */
int b2o_compact_polys(b2o_ctx* ctx, const float* polys_dev, const int32_t* points_dev, const int32_t* counts_dev, int n,
                      int max_boxes, float* flat_polys_dev, int32_t* flat_points_dev, int32_t* image_index_dev,
                      void* stream);

/* The box bookkeeping of recognize_from_boxes (recognition.py:511-521: crops are appended image after
 * image, start_end = running offsets) on the device: the (n,max_boxes,4,2) table of b2o_get_boxes becomes
 * the dense list flat (sum_i min(counts[i],max_boxes), 4, 2) with image_index[k] = image of box k, both
 * sized for n*max_boxes entries by the caller.  Runs without the host knowing the counts, i.e. BEFORE
 * the one synchronisation of the path.                                                          */
int b2o_compact_boxes(b2o_ctx* ctx, const float* boxes_dev, const int32_t* counts_dev, int n, int max_boxes,
                      float* flat_dev, int32_t* image_index_dev, void* stream);

/* Text lines in reading order (DESIGN.md section 1, "Text lines").  boxes (n, max_boxes, 4, 2) float32 as b2o_get_boxes
 * writes them (box[0] -> box[1] the reading direction), c_i = min(counts[i], max_boxes) words in image i; only those
 * are read.  Words are linked when their directions agree within cos_tol (= cos(angle tolerance), computed by the
 * caller), their heights within height_ratio, their centres lie within offset_ratio * the smaller height of each
 * other's centre line and the gap between them is at most gap_ratio * the larger height; lines are the connected
 * components.  Outputs, a CSR table per image: line_counts[i] = L_i lines; the words of line l in reading order are
 * word_order[i, line_start[i, l] : line_start[i, l + 1]] (word indices into boxes[i]); line_boxes[i, l] the line's
 * (4, 2) box, box[0] -> box[1] its reading direction; lines in page order.  Written: line_counts (n) all,
 * word_order[i, :c_i], line_start[i, :L_i + 1], line_boxes[i, :L_i]; every other slot is left as it was.
 * word_order is (n, max_boxes), line_start (n, max_boxes + 1), line_boxes (n, max_boxes, 4, 2).  Every value is fp64
 * with a fixed operation order: bit-identical in any batch and on every run.  n = 0 does nothing.             */
size_t b2o_lines_workspace_bytes(int n, int max_boxes);
int b2o_group_lines(b2o_ctx* ctx, const float* boxes_dev, const int32_t* counts_dev, int n, int max_boxes,
                    double cos_tol, double height_ratio, double offset_ratio, double gap_ratio,
                    int32_t* line_counts_dev, int32_t* word_order_dev, int32_t* line_start_dev,
                    float* line_boxes_dev, void* ws_dev, size_t ws_bytes, void* stream);

/* Text blocks in reading order (DESIGN.md section 1, "Text blocks"): recursive XY-cut over the lines of each image.
 * Inputs are b2o_group_lines' outputs (or any lines in that layout): L_i = min(line_counts[i], max_boxes) lines of
 * image i, line l's word count line_start[i, l + 1] - line_start[i, l] (line_start nondecreasing) and its (4, 2) box
 * line_boxes[i, l] (finite corners); only those are read.  The page frame D is box[1] - box[0] of the line with the
 * most words; a node of lines is cut into rows wherever the gap along N between a line and the running max of those
 * before it reaches row_gap * s, else into columns along D with col_gap * s (s the lower median of the lines'
 * heights), recursively; a node that cuts neither way is a block.  Outputs, a CSR table per image: block_counts[i] =
 * B_i blocks in depth-first order; the lines of block b in ascending line index are
 * line_order[i, block_start[i, b] : block_start[i, b + 1]]; block_boxes[i, b] the block's (4, 2) box aligned to D,
 * box[0] -> box[1] the page's reading direction.  Written: block_counts (n) all, line_order[i, :L_i],
 * block_start[i, :B_i + 1], block_boxes[i, :B_i]; every other slot is left as it was.  line_order is (n, max_boxes),
 * block_start (n, max_boxes + 1), block_boxes (n, max_boxes, 4, 2).  row_gap and col_gap must be finite and > 0.
 * Every value is fp64 with a fixed operation order: bit-identical in any batch and on every run.  n = 0 does nothing. */
size_t b2o_blocks_workspace_bytes(int n, int max_boxes);
int b2o_group_blocks(b2o_ctx* ctx, const int32_t* line_counts_dev, const int32_t* line_start_dev,
                     const float* line_boxes_dev, int n, int max_boxes, double row_gap, double col_gap,
                     int32_t* block_counts_dev, int32_t* line_order_dev, int32_t* block_start_dev,
                     float* block_boxes_dev, void* ws_dev, size_t ws_bytes, void* stream);

/* Wide words (DESIGN.md section 1, "Wide words"): a box wider than the 200 x 31 crop at full height is read in up to
 * M = max_windows overlapping windows (1 <= M <= B2O_MAX_WINDOWS).  In warp_extent's turn-0 frame of the box (w, h
 * from get_rotated_width_height): scale = min(T / w, 31 / h), T = 200 + (M - 1) S, S = B2O_WINDOW_STRIDE; wc = scale w,
 * sh = scale h.  A word with wc <= 200 has K = 1 and reads as b2o_warp_boxes reads it; otherwise K = 1 + ceil((wc - 200)
 * / S), at most M, windows start at a_k = k S (k < K - 1) and a_{K-1} = wc - 200, and window k is the homography of
 * the ordered box onto (-a_k, 0), (wc - a_k, 0), (wc - a_k, sh), (-a_k, sh) (float32 corners), dsize (200, int(sh)).
 * A box where warpBox raises ZeroDivisionError has K = 1.
 *
 * b2o_window_counts: K of every box of a table, boxes_dev (n, max_boxes, 4, 2), windows_dev (n, max_boxes) int32;
 * counts_dev (n) int32 limits image i to its first counts[i] boxes (NULL: every slot); slots past it are not written.
 *
 * The wide words are then listed as words_dev (n_words) int32, indices into a dense box list boxes_dev (., 4, 2) with
 * image_index_dev, and a CSR win_start_dev (n_words + 1) int32 of their windows: word i owns windows win_start[i] ..
 * win_start[i+1] - 1, whose count must be its K.  b2o_warp_windows cuts windows first .. first + count - 1 into slots
 * 0 .. count - 1 of crops_dev (count, 31, 200[, 3]) uint8 and / or crnn_in_dev (count, 200, 31[, 3]) fp16, as
 * b2o_warp_boxes lays them out (channels 1: gray image, 3: RGB for a color recognizer).
 *
 * b2o_stitch_windows reads every window's fc_12 logits, logits_dev (win_start[n_words], 48, k) float32, and its STN
 * theta, theta_dev (win_start[n_words], 6) float32 (NULL: no STN), and writes word i's reading to row words[i] of
 * labels_dev (., 48 M) int32, -1 padded, and its log-probability S to logp_dev[words[i]] (NULL: not written); no other
 * row is written.  Step t of window k lies at P = a_k + x in the word, x = stn_crop_x of grid row t + 2 (the map of
 * b2o_char_cells) clamped to [0, 200] and made non-decreasing.  The cut between windows k and k+1 is the position p
 * of a step of window k+1 inside the overlap [a_{k+1}, a_k + 200] shrunk by B2O_WINDOW_SHRINK at each end, nearest to
 * the overlap's centre (lower step on a tie), where that step and window k's step nearest to p (lower step on a tie)
 * both emit the blank; without such a step, the centre; a cut below the previous cut is raised to it.  Window k keeps
 * the steps with cut_{k-1} <= P < cut_k in order; greedy CTC (first maximum, merge repeats, drop blanks) over all kept
 * steps gives the labels, and S is the sum
 * over them of log(max p + 1e-7), max p = 1 / sum_c exp(l_c - l_max) summed in ascending c.
 *
 * b2o_window_plan_test (test hook): the plan of every window slot, plans_dev (n, M): record k of box i is window k's
 * plan, m the inverse homography, dw, dh the dsize (for K = 1, warpBox's), a = a_k; k = the box's K in every record,
 * valid = 0 for slots k >= K and where the system is singular (b2o_warp_windows cuts an all-zero crop there).      */
#define B2O_MAX_WINDOWS 16
#define B2O_WINDOW_STRIDE 136
#define B2O_WINDOW_SHRINK 8
typedef struct {
  double m[9];
  double a, wc, sh;
  int32_t k, dw, dh, valid;
} b2o_window_plan;
int b2o_window_counts(b2o_ctx* ctx, const float* boxes_dev, const int32_t* counts_dev, int n, int max_boxes,
                      int max_windows, int32_t* windows_dev, void* stream);
int b2o_warp_windows(b2o_ctx* ctx, const uint8_t* img_dev, int channels, int n, int h, int w, const float* boxes_dev,
                     const int32_t* image_index_dev, const int32_t* words_dev, const int32_t* win_start_dev,
                     int n_words, int max_windows, int first, int count, uint8_t* crops_dev, void* crnn_in_dev,
                     void* stream);
int b2o_stitch_windows(b2o_ctx* ctx, const float* logits_dev, int k, const float* theta_dev, const float* boxes_dev,
                       const int32_t* words_dev, const int32_t* win_start_dev, int n_words, int max_windows,
                       int32_t* labels_dev, float* logp_dev, void* stream);
int b2o_window_plan_test(b2o_ctx* ctx, const float* boxes_dev, int n, int max_windows, b2o_window_plan* plans_dev,
                         void* stream);

/* tools.warpBox over box groups (recognition.py:506-519; tools.py:61-117).  boxes: (n_boxes,4,2)
 * float32; image_index[k] selects the gray image of box k.  crops: (n_boxes,31,200) uint8
 * (exactly warpBox's output) and, when crnn_in != NULL, the CRNN input (n_boxes,200,31) fp16 =
 * crop/255 after Permute((2,1,3)) and the axis flip of recognition.py:215-216.                */
int b2o_warp_boxes(b2o_ctx* ctx, const uint8_t* gray_dev, int n, int h, int w,
                   const float* boxes_dev, const int32_t* image_index_dev, int n_boxes,
                   uint8_t* crops_dev, void* crnn_in_dev, void* stream);

/* The same for a recognizer built with color=True (recognition.py:214, 508-510: crops are cut from the RGB image, no
 * gray conversion): rgb (n,h,w,3) uint8, crops (n_boxes,31,200,3) uint8, crnn_in (n_boxes,200,31,3) fp16.            */
int b2o_warp_boxes_color(b2o_ctx* ctx, const uint8_t* rgb_dev, int n, int h, int w,
                         const float* boxes_dev, const int32_t* image_index_dev, int n_boxes,
                         uint8_t* crops_dev, void* crnn_in_dev, void* stream);

/* The crops of b2o_warp_boxes (channels = 1) or b2o_warp_boxes_color (channels = 3) cut in quarter turn `turn` (0..3).
 * With c = (tl, tr, br, bl) the corner order warpBox cuts with (get_rotated_box, tools.py:533-581), the crop in turn r is
 * warpBox(image, np.roll(c, -r, axis=0), 31, 200, skip_rotate=True): its top-left is c[r], and width and height are
 * measured after the roll, so odd turns swap them.  A word on a page turned by np.rot90(page, k) reads upright in turn
 * (4 - k) % 4.  Turn 0 is bit-identical to b2o_warp_boxes / b2o_warp_boxes_color; the kernel is the same one.        */
int b2o_warp_boxes_turned(b2o_ctx* ctx, const uint8_t* img_dev, int channels, int n, int h, int w,
                          const float* boxes_dev, const int32_t* image_index_dev, int n_boxes, int turn,
                          uint8_t* crops_dev, void* crnn_in_dev, void* stream);

/* warpBox along a polygon (the piecewise form of b2o_warp_boxes): polys (n_polys, 2 * (B2O_MAX_POLY_SEGMENTS + 1), 2)
 * float32 laid out as b2o_get_boxes_poly writes them, points (n_polys) int32, image_index (n_polys) int32; channels 1
 * (gray image (n,h,w)) or 3 (RGB (n,h,w,3)).  Crops and CRNN input as b2o_warp_boxes(_color) writes them.
 * A 4-point entry is cut exactly as b2o_warp_boxes cuts it.  An entry of s >= 2 segments (t_i the top edge, b_i the
 * bottom edge): w = int(sum_i (|t_i t_i+1| + |b_i b_i+1|) / 2), h = int(mean_j |t_j b_j|), scale = min(200 / w, 31 / h),
 * dsize = (int(scale w), int(scale h)); segment i maps (t_i, t_i+1, b_i+1, b_i) onto x in [X_i, X_i+1], y in
 * [0, scale h], X_i = float32(scale w * cum_i / cum_s) with cum_i the running sum of (|t t| + |b b|) / 2 (fp64
 * cv2.getPerspectiveTransform), and crop column x takes the last segment with X_i <= x, sampled as
 * cv2.warpPerspective samples it over the full dsize.  An entry whose w or h is 0, or whose point count is not 4
 * or an even number in [6, 2 (B2O_MAX_POLY_SEGMENTS + 1)], gets an all-zero crop; a singular segment zero columns. */
int b2o_warp_polys(b2o_ctx* ctx, const uint8_t* img_dev, int channels, int n, int h, int w, const float* polys_dev,
                   const int32_t* points_dev, const int32_t* image_index_dev, int n_polys, uint8_t* crops_dev,
                   void* crnn_in_dev, void* stream);

/* Choosing between the readings of several quarter turns.  Inputs: the results of n_turns runs of
 * b2o_warp_boxes_turned + a decoder (b2o_crnn_forward_scored, _beam or _lexicon), stacked in the order of turns_host
 * (host, n_turns distinct values in 0..3, 1 <= n_turns <= 4): labels_dev (n_turns, b, top_paths, 48) int32 and
 * logp_dev (n_turns, b, top_paths) float32, best reading first.  image_index_dev (b) int32 is non-decreasing with values
 * in [0, n_images), as b2o_compact_boxes writes it.
 * The vote compares each turn's best reading, logp[j, k, 0]:
 *   B2O_ROTATION_VOTE_WORD: every word keeps the turn with the largest score;
 *   B2O_ROTATION_VOTE_PAGE: every image keeps one turn for all its words, the one with the largest float32 sum of its
 *                           words' scores, added in word order by one thread (the sum does not depend on the batch).
 * Ties, and words or images whose scores are all -inf, keep the turn listed first.
 * Outputs: labels_out_dev (b, top_paths, 48) and logp_out_dev (b, top_paths), the chosen turn's readings (a (b, 1, 48)
 * result has the (b, 48) layout b2o_pack_records(_scored) takes), and turn_out_dev (b) int32 the chosen turn r.
 * boxes_dev (b,4,2) float32, when not NULL, is rewritten in place as np.roll(c, -r, axis=0): box[0] is then the corner the
 * crop started at, the text's own top-left, still clockwise.  table_dev (n_images, max_boxes, 4, 2), when not NULL, is
 * the b2o_get_boxes table that b2o_compact_boxes made boxes_dev from, and receives the same rolled boxes (word k of
 * image i at slot k - (first word of i)), so the host copy and b2o_pack_records(_scored) read them unchanged.
 * The corner order is the one b2o_warp_boxes_turned uses.  A word's result is bit-identical in any batch.          */
#define B2O_ROTATION_VOTE_WORD 0
#define B2O_ROTATION_VOTE_PAGE 1
int b2o_select_rotation(b2o_ctx* ctx, const int32_t* labels_dev, const float* logp_dev, const int32_t* image_index_dev,
                        int n_images, int b, int top_paths, const int32_t* turns_host, int n_turns, int vote,
                        int32_t* labels_out_dev, float* logp_out_dev, int32_t* turn_out_dev, float* boxes_dev,
                        float* table_dev, int max_boxes, void* stream);

/* prediction_model.predict (recognition.py:535; graph 214-333): CRNN + STN + BiLSTM + greedy CTC (beam search:
 * b2o_crnn_forward_beam below; a caller's word list: b2o_crnn_forward_lexicon).
 * crnn_in: (b,200,31) fp16 from b2o_warp_boxes (or b2o_crops_to_input).  labels: (b,48) int32,
 * merged + blank-free, padded with -1 -- the tensor recognize_from_boxes iterates (527-534).  */
size_t b2o_crnn_workspace_bytes(int b);
int b2o_crops_to_input(b2o_ctx* ctx, const uint8_t* crops_dev, int b, void* crnn_in_dev, void* stream);
/* crops (b,31,200,3) uint8 -> (b,200,31,3) fp16 for a color=True recognizer (conv_1.kernel of shape (3,3,3,64));
 * b2o_crnn_forward then takes that 3-channel input.                                                              */
int b2o_crops_to_input_color(b2o_ctx* ctx, const uint8_t* crops_dev, int b, void* crnn_in_dev, void* stream);
int b2o_crnn_forward(b2o_ctx* ctx, const void* crnn_in_dev, int b, int32_t* labels_dev,
                     void* ws_dev, size_t ws_bytes, void* stream);
/* The same labels, and logp_dev (b) float32 receives each crop's greedy-path log-probability
 * S = sum over the 48 kept steps t of log(max_c p[t,c] + 1e-7), p = softmax of fc_12 (recognition.py:322-328).
 * exp(S) in (0, 1] is the word's confidence; per TensorFlow's documentation S is minus the second output of
 * keras.backend.ctc_decode(greedy=True), which CTCDecoder drops (recognition.py:175) -- that link is not pinned
 * against TensorFlow.  S of a crop is bit-reproducible and does not depend on the batch it runs in.  logp_dev == NULL
 * behaves as b2o_crnn_forward.                                                                                */
int b2o_crnn_forward_scored(b2o_ctx* ctx, const void* crnn_in_dev, int b, int32_t* labels_dev, float* logp_dev,
                            void* ws_dev, size_t ws_bytes, void* stream);

/* CTC prefix beam search, the greedy=False form of keras.backend.ctc_decode (which CTCDecoder does not use,
 * recognition.py:169-184).  Per kept step t and class c the input is lp[t,c] = log(softmax(logits_t)_c + 1e-7), blank =
 * k-1; a beam is a label prefix with the log-probabilities of ending in blank and in a label, scored by their logaddexp;
 * each step every beam continues via blank, via its last label and by every label (a repeated label only after a
 * blank), equal prefixes merge and the beam_width best survive.  Equal scores rank by label sequence, ascending, a
 * prefix before its extensions.  Repeated letters are kept as the prefix search yields them (no merge_repeated pass).
 * 1 <= beam_width <= B2O_MAX_BEAM_WIDTH, 1 <= top_paths <= beam_width, otherwise B2O_ERR_ARG.
 * labels_dev (b, top_paths, 48) int32, best first, -1 padded; logp_dev (b, top_paths) float32, the beam scores,
 * non-increasing (NULL: not written).  Paths beyond the number of distinct prefixes (tiny k) are all -1 with logp -inf.
 * A crop's result is bit-identical in any batch and on every run.  A (b, 1, 48) result has the (b, 48) layout that
 * b2o_pack_records(_scored) takes.
 * b2o_ctc_beam_decode: the search alone on caller-supplied (b, 48, k) float32 logits, 2 <= k <= B2O_MAX_CLASSES.
 * b2o_crnn_forward_beam: the CRNN of b2o_crnn_forward, its fc_12 logits into the workspace, then the search.       */
#define B2O_MAX_BEAM_WIDTH 128
int b2o_ctc_beam_decode(b2o_ctx* ctx, const float* logits_dev, int b, int k, int beam_width, int top_paths,
                        int32_t* labels_dev, float* logp_dev, void* stream);
int b2o_crnn_forward_beam(b2o_ctx* ctx, const void* crnn_in_dev, int b, int beam_width, int top_paths,
                          int32_t* labels_dev, float* logp_dev, void* ws_dev, size_t ws_bytes, void* stream);

/* CTC prefix beam search ranked by a character n-gram language model (DESIGN.md section 1, "Language model").
 * The device model, built on the host (recognition.CharLM.device_arrays): n_histories listed histories, each of
 * length 0 .. order-1, as a sorted uint64 key array keys_dev, key = (length << 56) | the symbols packed 8 bits each,
 * oldest in the highest byte, a label c as c and <s> as 127 (keys_dev[0] = 0, the empty history); rows_dev
 * (n_histories, k) float32: column c < k-1 is log P(c | h) with the backoff folded in, column k-1 log P(</s> | h).
 * A beam also carries G in float32: G(empty) = 0, G(a + c) = G(a) + (alpha * l(c | hist(a)) + beta), l the row value
 * of the longest listed suffix of hist(a), the last order-1 symbols of "<s> a".  Candidates rank by F = A + G (one
 * float32 rounding), A = the acoustic beam score of b2o_ctc_beam_decode; equal F by label sequence as there.  Each
 * step a beam extends by its own shortlist, the min(beam_width + 1, k - 1) labels with the largest
 * lp[t,c] + alpha * l(c | hist) (ties: smaller label).  The top_paths readings rank by F_end = F + alpha * l(</s> | hist).
 * labels_dev (b, top_paths, 48) as b2o_ctc_beam_decode writes them; logp_dev (b, top_paths) float32 the acoustic A of
 * each reading and fused_dev (b, top_paths) float32 its F_end (either NULL: not written).  With alpha = beta = 0 labels
 * and logp equal b2o_ctc_beam_decode's bit for bit.  A crop's result is a function of its logits and the model alone.
 * 2 <= order <= B2O_MAX_LM_ORDER, 1 <= n_histories <= B2O_MAX_LM_HISTORIES, finite alpha and beta, keys and rows not
 * NULL, 2 <= k <= B2O_MAX_LM_CLASSES and the beam_width / top_paths rules of beam search, otherwise B2O_ERR_ARG.
 * b2o_ctc_beam_lm_decode: the search alone on caller-supplied (b, 48, k) float32 logits.
 * b2o_crnn_forward_beam_lm: the CRNN of b2o_crnn_forward, its fc_12 logits into the workspace, then the search.    */
#define B2O_MAX_LM_ORDER 8
#define B2O_MAX_LM_HISTORIES (1 << 20)
#define B2O_MAX_LM_CLASSES 127
typedef struct {
  int order;
  int n_histories;
  const uint64_t* keys_dev;
  const float* rows_dev;
  float alpha;
  float beta;
} b2o_char_lm;
int b2o_ctc_beam_lm_decode(b2o_ctx* ctx, const float* logits_dev, int b, int k, int beam_width, int top_paths,
                           const b2o_char_lm* lm, int32_t* labels_dev, float* logp_dev, float* fused_dev, void* stream);
int b2o_crnn_forward_beam_lm(b2o_ctx* ctx, const void* crnn_in_dev, int b, int beam_width, int top_paths,
                             const b2o_char_lm* lm, int32_t* labels_dev, float* logp_dev, float* fused_dev, void* ws_dev,
                             size_t ws_bytes, void* stream);

/* CTC prefix beam search with a bonus for a caller's word list, with or without a language model (DESIGN.md section 1,
 * "Hotwords").  The trie of the list, built on the host (recognition.Hotwords.device_arrays): n_nodes nodes numbered
 * breadth-first by (depth, parent, label), the root 0 the empty prefix; n_edges = n_nodes - 1 edges as ascending uint64
 * keys keys_dev, key = (parent << 8) | label, with child_dev (n_edges) int32 the child of each edge, so the children of
 * a node are contiguous; final_dev (n_nodes) uint8, 1 where the node's prefix is a listed word.  A prefix is live when
 * it is a node (a prefix of a listed word).  Bonus H(a) = weight * |a| for a live a, else 0; H_end(a) = weight * |a|
 * for a listed word, else 0.  Candidates rank by F = (A + G) + H and the top_paths readings by
 * F_end = ((A + G) + alpha * l(</s> | hist)) + H_end, in float32 in that order, each addition of H or H_end skipped
 * when it is 0; A and G are those of b2o_ctc_beam_lm_decode, and lm = NULL is a model of zeros (G = 0, alpha = 0).
 * Each step a beam extends by its own shortlist, the min(beam_width + 1, k - 1) labels with the largest
 * (lp[t,c] + alpha * l(c | hist)) + H(a + c) (ties: smaller label).  labels_dev, logp_dev (the acoustic A) and
 * fused_dev (F_end) as b2o_ctc_beam_lm_decode writes them.  weight = 0, or a trie of the root alone, gives
 * b2o_ctc_beam_lm_decode's labels, logp and fused bit for bit, and without a model b2o_ctc_beam_decode's labels and
 * logp.  A crop's result is a function of its logits, the model and the list alone.
 * 1 <= n_nodes <= B2O_MAX_HOTWORD_NODES, n_edges = n_nodes - 1, keys and child not NULL when n_edges > 0, final not
 * NULL, weight finite and >= 0, a valid lm (as b2o_ctc_beam_lm_decode takes it) or NULL, 2 <= k <=
 * B2O_MAX_LM_CLASSES and the beam_width / top_paths rules of beam search, otherwise B2O_ERR_ARG.
 * b2o_ctc_beam_hotword_decode: the search alone on caller-supplied (b, 48, k) float32 logits.
 * b2o_crnn_forward_beam_hotword: the CRNN of b2o_crnn_forward, its fc_12 logits into the workspace (so b2o_crnn_align
 * and b2o_crnn_char_scores work after it), then the search.                                                         */
#define B2O_MAX_HOTWORD_NODES ((1 << 24) + 1)
typedef struct {
  int n_nodes;
  int n_edges;
  const uint64_t* keys_dev;
  const int32_t* child_dev;
  const uint8_t* final_dev;
  float weight;
} b2o_hotwords;
int b2o_ctc_beam_hotword_decode(b2o_ctx* ctx, const float* logits_dev, int b, int k, int beam_width, int top_paths,
                                const b2o_char_lm* lm, const b2o_hotwords* hw, int32_t* labels_dev, float* logp_dev,
                                float* fused_dev, void* stream);
int b2o_crnn_forward_beam_hotword(b2o_ctx* ctx, const void* crnn_in_dev, int b, int beam_width, int top_paths,
                                  const b2o_char_lm* lm, const b2o_hotwords* hw, int32_t* labels_dev, float* logp_dev,
                                  float* fused_dev, void* ws_dev, size_t ws_bytes, void* stream);

/* CTC prefix beam search constrained to a pattern: a deterministic automaton over the labels (DESIGN.md section 1,
 * "Patterns"), built on the host (recognition.Pattern.device_arrays).  n_states states, trans_dev (n_states, k-1) int16:
 * trans[q][c] the state after label c in state q, -1 for none; dist_dev (n_states) uint8: the fewest labels from q to an
 * accepting state, 0 when q accepts (saturated at 255); start the state of the empty reading.  The tables are sized
 * for the k of the call.  A beam also carries its state; after step t (0 .. 47) a beam kept via blank or its last label
 * and an extension alike survive only in a state q with dist[q] <= 47 - t, so every returned reading is accepted.  Each
 * step a beam extends by its own shortlist, the min(beam_width + 1, its count) allowed labels (successor defined and
 * feasible) with the largest lp[t,c] (ties: smaller label).  Scores, merging and ranking are b2o_ctc_beam_decode's;
 * labels_dev (b, top_paths, 48) and logp_dev (b, top_paths) (NULL: not written) as it writes them, and a crop with
 * fewer than top_paths surviving readings (none: the pattern cannot be met in 48 steps) has the remaining slots -1 with
 * logp -inf; a reading of probability 0 (score -inf) is never returned.  A one-state automaton that accepts
 * everything gives b2o_ctc_beam_decode's labels and logp bit for bit, except slots that b2o_ctc_beam_decode fills
 * with -inf readings (fewer finite ones than top_paths, at tiny k), which are -1 here.
 * 1 <= n_states <= B2O_MAX_PATTERN_STATES, 0 <= start < n_states, trans and dist not NULL, 2 <= k <=
 * B2O_MAX_PATTERN_CLASSES and the beam_width / top_paths rules of beam search, otherwise B2O_ERR_ARG.
 * b2o_ctc_beam_pattern_decode: the search alone on caller-supplied (b, 48, k) float32 logits.
 * b2o_crnn_forward_beam_pattern: the CRNN of b2o_crnn_forward, its fc_12 logits into the workspace (so b2o_crnn_align
 * works after it), then the search.                                                                                  */
#define B2O_MAX_PATTERN_STATES 4096
#define B2O_MAX_PATTERN_CLASSES 127
typedef struct {
  int n_states;
  int start;
  const int16_t* trans_dev;
  const uint8_t* dist_dev;
} b2o_pattern;
int b2o_ctc_beam_pattern_decode(b2o_ctx* ctx, const float* logits_dev, int b, int k, int beam_width, int top_paths,
                                const b2o_pattern* pattern, int32_t* labels_dev, float* logp_dev, void* stream);
int b2o_crnn_forward_beam_pattern(b2o_ctx* ctx, const void* crnn_in_dev, int b, int beam_width, int top_paths,
                                  const b2o_pattern* pattern, int32_t* labels_dev, float* logp_dev, void* ws_dev,
                                  size_t ws_bytes, void* stream);

/* Lexicon-constrained CTC decoding: the top_paths most probable entries of a caller's word list, per crop.
 * Inputs: the beam decoder's lp[t,c] = log(softmax(logits_t)_c + 1e-7) over the 48 kept steps, blank = k-1.
 * Lexicon: n_words entries in CSR form, offsets_dev (n_words + 1) int32 and the concatenated labels_dev int16; entry i
 * is labels[offsets[i] .. offsets[i+1]).  An entry's score is its CTC forward log-probability: the log of the sum,
 * over every 48-step alignment that collapses (merge repeats, drop blanks) to the entry, of exp(sum_t lp[t, pi_t]).
 * A doubled letter needs a blank between its copies, so an entry of L labels with R adjacent repeats that has
 * L + R > 48 cannot be aligned and scores -inf; so does an entry that is empty, longer than 48, has a label outside
 * [0, k-2] or labels beyond index 2^24 (never read out of bounds).  Every other entry's score is finite, however
 * improbable (down to about 48 log(1e-7) ~ -774): the recursion runs in the linear domain with exact power-of-two
 * rescaling, and the score is rounded to float32 once.
 * Result: per crop the top_paths best entries, score descending, equal float32 scores by entry index ascending.
 * labels_out_dev (b, top_paths, 48) int32: entry p's labels, -1 padded; logp_dev (b, top_paths) float32 its score
 * (NULL: not written).  Slots beyond the number of finite-score entries are all -1 with logp -inf.  A (b, 1, 48)
 * result has the (b, 48) layout that b2o_pack_records(_scored) takes.
 * A crop's result is a function of its logits and the lexicon alone: bit-identical alone, in any batch and on every
 * run; an entry's score does not depend on its position in the lexicon or on the other entries.
 * 1 <= n_words <= B2O_MAX_LEXICON_WORDS, 1 <= top_paths <= B2O_MAX_LEXICON_TOP_PATHS, 2 <= k <= B2O_MAX_CLASSES,
 * otherwise B2O_ERR_ARG.  The caller owns the scratch: b2o_lexicon_workspace_bytes(b, n_words, top_paths) bytes.
 * b2o_ctc_lexicon_decode: the decoder alone on caller-supplied (b, 48, k) float32 logits; ws_dev is that scratch.
 * b2o_crnn_forward_lexicon: the CRNN of b2o_crnn_forward, its fc_12 logits into the workspace's logits slot, then the
 * decoder; ws_bytes >= b2o_crnn_workspace_bytes(b) + b2o_lexicon_workspace_bytes(b, n_words, top_paths) (the
 * decoder's scratch follows the CRNN's).                                                                        */
#define B2O_MAX_LEXICON_WORDS (1 << 20)
#define B2O_MAX_LEXICON_LABELS (1 << 24)
#define B2O_MAX_LEXICON_TOP_PATHS 128
size_t b2o_lexicon_workspace_bytes(int b, int n_words, int top_paths);
int b2o_ctc_lexicon_decode(b2o_ctx* ctx, const float* logits_dev, int b, int k, const int32_t* offsets_dev,
                           const int16_t* labels_dev, int n_words, int top_paths, int32_t* labels_out_dev,
                           float* logp_dev, void* ws_dev, size_t ws_bytes, void* stream);
int b2o_crnn_forward_lexicon(b2o_ctx* ctx, const void* crnn_in_dev, int b, const int32_t* offsets_dev,
                             const int16_t* labels_dev, int n_words, int top_paths, int32_t* labels_out_dev,
                             float* logp_dev, void* ws_dev, size_t ws_bytes, void* stream);

/* Character positions: where each character of a reading lies (DESIGN.md section 1).
 * b2o_ctc_align: the best single CTC alignment of each reading over the 48 kept steps, on lp[t,c] = log(softmax(l_t)_c +
 * 1e-7) (blank = k-1), by a Viterbi pass over the 2n + 1 states (blank, l_0, blank, ..., l_{n-1}, blank) of an n-label
 * reading: a path starts in the first blank or l_0 and ends in l_{n-1} or the trailing blank, a doubled letter needs a
 * blank between its copies.  Ties among the predecessors of a state go to staying, then to advancing by one, then to
 * skipping a blank; the trailing blank ends the path only when it scores strictly more than l_{n-1}.
 * Inputs: logits_dev (b, 48, k) float32 and labels_dev (b, top_paths, 48) int32, each reading's labels followed by -1
 * (what the decoders write).  Outputs: spans_dev (b, top_paths, 48, 2) int32, (f_j, l_j) = the first and last step (0..47)
 * at which character j's state is occupied, -1 past the last character; logp_dev (b, top_paths) float32 (NULL: not
 * written), the alignment's log-probability.  A reading with no finite alignment (too many doubled letters, a label
 * outside [0, k-2]) gets spans -1 and logp -inf; an empty reading gets its all-blank score.  A crop's result is a
 * function of its logits and labels alone: bit-identical alone, in any batch and on every run.
 * 2 <= k <= B2O_MAX_CLASSES, 1 <= top_paths <= B2O_MAX_ALIGN_PATHS, otherwise B2O_ERR_ARG.
 *
 * b2o_char_cells: the characters tile the word box along its reading direction.  The cut between characters j-1 and j
 * is grid row r = (l_{j-1} + f_j) / 2 + 2 (2 discarded steps); with the STN's theta (b, 6) it is crop column
 * x = 4u + 1.5, u = 0.5 (theta[4] gy + theta[5] + 1) 50, gy = -1 + 2r/49 (the STN's time coordinate on the grid's centre
 * column); without (theta_dev NULL, build_model(stn=False)) u = r.  Cuts are clamped to [0, sw] -- sw x sh the crop's
 * content, the float32 corners warpBox maps the box onto -- and made non-decreasing by a running max (a theta may flip
 * time).  Cell j is (a,0), (b,0), (b,sh), (a,sh) between its cuts, mapped to detector-input pixels by the inverse
 * homography of the word's warp in the turn it was read in (turns_dev (b) int32, NULL: turn 0; boxes_dev (b,4,2) the
 * boxes as they were cut, before b2o_select_rotation rolls them) in fp64 with the projective divide, rounded once to
 * float32.  The leading edge of the first cell and the trailing edge of the last are the rolled box's own corners, bit
 * for bit; corner 0 of a cell is its top-left in reading order, clockwise.  boxes_dev NULL: cells in the 200 x 31 crop
 * frame (outer edges x = 0 and 200, height 31).  cells_dev (b, top_paths, 48, 4, 2) float32, NaN past the last character,
 * for readings without spans and for boxes whose warp plan is invalid.
 *
 * The product path: b2o_crnn_forward_logits is b2o_crnn_forward_scored that also keeps the fc_12 logits in the
 * workspace's logits slot (logp_dev may be NULL), as b2o_crnn_forward_beam and _lexicon always do; b2o_crnn_align then
 * aligns labels_dev on the logits of the preceding forward in ws_dev and copies its theta (b, 6) to theta_dev (NULL, or
 * a recognizer without STN: not written).  Workspace sizes are those of the forward.  The logits must be those of the
 * context's last successful CRNN forward, with the same ws_dev and b, and that forward must have kept them (_logits,
 * _beam, _lexicon, or any greedy forward with the debug taps on; b2o_crnn_features never does): otherwise
 * B2O_ERR_STATE and nothing is written.                                                                            */
#define B2O_MAX_ALIGN_PATHS 128
int b2o_ctc_align(b2o_ctx* ctx, const float* logits_dev, int b, int k, const int32_t* labels_dev, int top_paths,
                  int32_t* spans_dev, float* logp_dev, void* stream);
int b2o_char_cells(b2o_ctx* ctx, const int32_t* spans_dev, int b, int top_paths, const float* theta_dev,
                   const float* boxes_dev, const int32_t* turns_dev, float* cells_dev, void* stream);
int b2o_crnn_forward_logits(b2o_ctx* ctx, const void* crnn_in_dev, int b, int32_t* labels_dev, float* logp_dev,
                            void* ws_dev, size_t ws_bytes, void* stream);
int b2o_crnn_align(b2o_ctx* ctx, int b, const int32_t* labels_dev, int top_paths, int32_t* spans_dev, float* logp_dev,
                   float* theta_dev, const void* ws_dev, size_t ws_bytes, void* stream);

/* Character scores: how sure the model is of each character of a reading, and what it would read there instead
 * (DESIGN.md section 1, "Character scores").  On lp[t,c] = log(softmax(l_t)_c + 1e-7) over the 48 kept steps (blank =
 * k-1), F(z) is the CTC forward log-probability of a label sequence z (b2o_ctc_lexicon_decode's entry score; -inf when
 * z cannot be aligned).  For a reading y_0..y_{n-1} and a position j the k one-character edits at j are the
 * substitutions y[j->c], c = 0..k-2 (c = y_j is y itself), and the deletion y[j->nothing], labelled k-1.  The posterior
 * of edit e is pi_j(e) = exp(F(y[j->e]) - L_j), L_j = logsumexp_e F(y[j->e]); the character's confidence is
 * pi_j(y_j); its alternatives are the A edits of largest posterior, best first, equal values by smaller label (the
 * reading's own character appears where it ranks).  Insertions are not scored.  The scores are acoustic: they do not
 * depend on the decoder that produced y.
 * Inputs: logits_dev (b, 48, k) float32 and labels_dev (b, top_paths, 48) int32, each reading's labels followed by -1
 * (what the decoders write).  Outputs: conf_dev (b, top_paths, 48) float32; alt_labels_dev (b, top_paths, 48, A) int32
 * and alt_post_dev (b, top_paths, 48, A) float32, A = alternatives (both may be NULL when A = 0); logp_dev (b, top_paths)
 * float32 = F(y) (NULL: not written).  Where L_j = -inf (and at every position of a reading with a label outside
 * [0, k-2]) the confidence and the posteriors are 0 and the labels -1; with A > k the slots past the k edits are -1
 * with posterior 0; positions past the reading's end are NaN, -1 and NaN.  A reading with a label outside [0, k-2] has
 * logp -inf.  The posteriors at a position sum to 1 up to fp32 rounding.  A crop's result is a function of its logits
 * and labels alone: bit-identical alone, in any batch and on every run.  No workspace.
 * 2 <= k <= B2O_MAX_CLASSES, 1 <= top_paths <= B2O_MAX_ALIGN_PATHS, 0 <= alternatives <= B2O_MAX_CHAR_ALTERNATIVES,
 * otherwise B2O_ERR_ARG.
 * b2o_crnn_char_scores: the same on the logits of the preceding forward in ws_dev, under b2o_crnn_align's rule (the
 * context's last successful CRNN forward, same ws_dev and b, and it kept its logits: otherwise B2O_ERR_STATE and
 * nothing is written).                                                                                             */
#define B2O_MAX_CHAR_ALTERNATIVES 8
int b2o_ctc_char_scores(b2o_ctx* ctx, const float* logits_dev, int b, int k, const int32_t* labels_dev, int top_paths,
                        int alternatives, float* conf_dev, int32_t* alt_labels_dev, float* alt_post_dev,
                        float* logp_dev, void* stream);
int b2o_crnn_char_scores(b2o_ctx* ctx, int b, const int32_t* labels_dev, int top_paths, int alternatives,
                         float* conf_dev, int32_t* alt_labels_dev, float* alt_post_dev, float* logp_dev,
                         const void* ws_dev, size_t ws_bytes, void* stream);

/* Training the output layer for a custom alphabet: Recognizer.compile() + training_model with ctc_batch_cost
 * (recognition.py:321-349, 539-545; docs/examples/fine_tuning_recognizer.rst) restricted to fc_12 (Dense 256 -> k plus
 * bias), the rest of the CRNN frozen.
 * b2o_crnn_features: the forward of b2o_crnn_forward up to the BiLSTM output l2, whose 48 kept steps (2..49,
 * rnn_steps_to_discard, recognition.py:328) go to features_dev (b, 48, 256) fp16; fc_12 and the decoder do not run.
 * Workspace: b2o_crnn_workspace_bytes(b).
 * b2o_ctc_loss_grad: per crop i the Keras ctc_batch_cost loss on the softmax output over the 48 kept steps,
 *   L_i = -log sum over the alignments of the text of prod_t q[t, path_t],  q = softmax(x_t w + bias) + 1e-7, blank = k-1,
 * i.e. minus the b2o_ctc_lexicon_decode score of the text.  x_t is row index_dev[i] of features_dev (n_rows, 48, 256)
 * fp16 (16-byte aligned; index_dev NULL: row i), after Dropout(dropout) (recognition.py:321): feature c of step t of row r
 * is kept iff splitmix64(key0 ^ (r * 12288 + t * 256 + c)) >> 40 >= floor(dropout * 2^24), key0 =
 * splitmix64(splitmix64(seed) ^ step), and kept features are multiplied by the fp32 1 / (1 - dropout); dropout = 0 uses the
 * features unchanged.  The logits are fc_ctc_kernel's (the serial fmaf chain over the features in ascending order), so
 * with dropout 0 they are bit for bit those inference decodes; logits_dev (b, 48, k) float32, when not NULL, receives them.
 * w_dev (256, k) and bias_dev (k) float32 are the caller's.  Texts: CSR as for the lexicon, offsets_dev (b + 1) int32,
 * labels_dev int16.  loss_dev (b) float32: L_i, a function of the crop's features, text, the weights and (with dropout)
 * seed, step and its row only -- bit-identical in any batch and on every run.  A text that is empty, longer than 48, has
 * a label outside [0, k-2] or cannot be aligned in 48 steps (L + adjacent repeats > 48) gets +inf, a row index outside
 * [0, n_rows) NaN; such crops add nothing to the gradient, and their logits_dev rows are all NaN.
 * grad_w_dev (256, k) and grad_b_dev (k) float32: (1/b) sum over crops and steps of x_t^T dL_i/dlogits_t and of
 * dL_i/dlogits_t, summed in a fixed order (bit-identical run to run; the order of the crops in the batch matters in the
 * last bits).  Both NULL: the loss only, and ws_dev may be NULL.  Otherwise ws_bytes >= b2o_ctc_train_workspace_bytes(b, k).
 * 2 <= k <= B2O_MAX_CLASSES, 0 <= dropout < 1, otherwise B2O_ERR_ARG.
 * b2o_rmsprop_step: Keras RMSprop with momentum 0 (the default optimizer of Recognizer.compile, recognition.py:539-545)
 * on n float32 elements: acc = rho acc + (1 - rho) g^2; param -= lr g / (sqrt(acc) + eps), in fp32, in that order.  acc
 * starts at 0; Keras' defaults are lr 1e-3, rho 0.9, eps 1e-7.
 * b2o_crnn_set_top: copies (256, k) w_dev and (k) bias_dev into the context's fc_12; every forward enqueued after it uses
 * them.  k must equal the loaded class count (B2O_ERR_ARG otherwise).                                              */
int b2o_crnn_features(b2o_ctx* ctx, const void* crnn_in_dev, int b, void* features_dev, void* ws_dev, size_t ws_bytes,
                      void* stream);
size_t b2o_ctc_train_workspace_bytes(int b, int k);
int b2o_ctc_loss_grad(b2o_ctx* ctx, const void* features_dev, int n_rows, const int32_t* index_dev, int b, int k,
                      const float* w_dev, const float* bias_dev, const int32_t* offsets_dev, const int16_t* labels_dev,
                      float dropout, uint64_t seed, uint64_t step, float* loss_dev, float* grad_w_dev,
                      float* grad_b_dev, float* logits_dev, void* ws_dev, size_t ws_bytes, void* stream);
int b2o_rmsprop_step(b2o_ctx* ctx, float* param_dev, const float* grad_dev, float* acc_dev, int64_t n, float lr,
                     float rho, float eps, void* stream);
int b2o_crnn_set_top(b2o_ctx* ctx, const float* w_dev, const float* bias_dev, int k, void* stream);

/* Fine-tuning the recurrent head: Recognizer.compile() + training_model with ctc_batch_cost (recognition.py:292-349,
 * 539-545; docs/examples/fine_tuning_recognizer.rst) restricted to lstm_10, lstm_10_back, lstm_11, lstm_11_back and fc_12;
 * the convolutions, the STN and fc_9 stay frozen.
 * b2o_crnn_sequence_features: the forward of b2o_crnn_forward up to fc_9 (recognition.py:282-290), whose output goes to
 * out_dev (b, 50, 128) fp16, bit for bit the "fc_9" tap; the BiLSTM, fc_12 and the decoder do not run.  Workspace:
 * b2o_crnn_workspace_bytes(b).  Afterwards b2o_crnn_tap reads every slot up to "fc_9", not "l1" / "l2" / "logits".
 * b2o_rnn_loss_grad: per crop i the loss of b2o_ctc_loss_grad (same q, dropout mask, +inf / NaN rules) on the l2 that the
 * BiLSTM computes from row index_dev[i] of x_dev (n_rows, 50, 128) fp16 (16-byte aligned; index_dev NULL: row i), the
 * dropout mask keyed on that row, so loss_dev (b) float32 is a function of the crop's row, text, the weights, seed and
 * step only.  params_dev is one float32 vector, per LSTM in the order lstm_10, lstm_10_back, lstm_11, lstm_11_back its
 * kernel (128, 512), recurrent_kernel (128, 512) and bias (512) (131,584 floats each), then fc_12.kernel (256, k) and
 * fc_12.bias (k): 526,336 + 257 k floats.  The forward is the inference arithmetic: kernels and recurrent kernels rounded
 * to fp16 at every call as b2o_load_crnn packs them, fp32 accumulation, h rounded to fp16 between steps, go_backwards
 * outputs kept in processing order (recognition.py:298-319), l1 = fp16(hf + hb), l2 = [h11f, h11b], steps 0 and 1
 * discarded before fc_12.  grad_dev (same layout) receives the batch means of dW = x^T dz, dU = h_prev^T dz, db = sum dz
 * of the four directions by backpropagation through time (fp16 roundings taken as the identity; the gradient of l1 at
 * processing step s goes to step s of both lstm_10 and lstm_10_back, lstm_11_back's input gradient lands at time 49 - s)
 * and fc_12's gradients as b2o_ctc_loss_grad forms them.  Fixed-order sums, no atomics: bit-identical run to run.
 * grad_dev NULL: the loss only.  ws_bytes >= b2o_rnn_train_workspace_bytes(b, k) always.  The workspace holds, in this
 * order, each slot rounded up to 256 bytes: W^T (4, 512, 128) fp16, U (4, 128, 512) fp16, xw = x W + b (4, b, 50, 512)
 * f32 in input order (row b * 50 + t; after a loss-only call it holds all four directions), then dz over it in processing
 * order, acts (4, b, 50, 5, 128) f32 = i, f, g = tanh(z_c), o, c per processing step, hf / hb (2, b, 50, 128)
 * fp16, l1 (b, 50, 128) fp16, l2 (b, 50, 256) fp16, dL/dl2 (b, 50, 256) f32, dL/dl1 (b, 50, 128) f32, the split-K
 * partials ((b + 15) / 16, 526336) f32, and b2o_ctc_train_workspace_bytes(b, k) for the CTC, which starts with dL/dlogits
 * (b, 48, k) f32.  2 <= k <= B2O_MAX_CLASSES, 0 <= dropout < 1, otherwise B2O_ERR_ARG.                             */
int b2o_crnn_sequence_features(b2o_ctx* ctx, const void* crnn_in_dev, int b, void* out_dev, void* ws_dev,
                               size_t ws_bytes, void* stream);
size_t b2o_rnn_train_workspace_bytes(int b, int k);
int b2o_rnn_loss_grad(b2o_ctx* ctx, const void* x_dev, int n_rows, const int32_t* index_dev, int b, int k,
                      const float* params_dev, const int32_t* offsets_dev, const int16_t* labels_dev, float dropout,
                      uint64_t seed, uint64_t step, float* loss_dev, float* grad_dev, void* ws_dev, size_t ws_bytes,
                      void* stream);

/* Result records of Pipeline.recognize for the multi-GPU gather (pipeline.py:66-75; SURVEY.md 8(e)): one
 * fixed-size float32 row per image = [count][rec_boxes x (4,2) boxes * inv_scale[i] (tools.adjust_boxes,
 * tools.py:232-260)][rec_boxes x 48 labels as int8, -1 padded], b2o_record_floats(rec_boxes) floats long.
 * boxes/counts as written by b2o_get_boxes, labels (sum counts, 48) int32 as written by b2o_crnn_forward
 * (NULL when no image has a box).  Rows n..rows-1 (a short last shard) get count -1.  The class count
 * must fit int8 (alphabets up to 126 characters).                                               */
size_t b2o_record_floats(int rec_boxes);
int b2o_pack_records(b2o_ctx* ctx, const float* boxes_dev, const int32_t* counts_dev, const int32_t* labels_dev,
                     const float* inv_scale_dev, int n, int max_boxes, int rows, int rec_boxes,
                     float* records_dev, void* stream);
/* Scored records: the unscored record above, unchanged, followed by [rec_boxes detection scores][rec_boxes path
 * log-probabilities S], b2o_record_floats_scored(rec_boxes) = b2o_record_floats(rec_boxes) + 2 * rec_boxes floats.
 * box_scores (n, max_boxes) as written by b2o_get_boxes_scored; logp (sum counts) as written by
 * b2o_crnn_forward_scored (NULL when no image has a box).  Slots past an image's words hold 0.                */
size_t b2o_record_floats_scored(int rec_boxes);
int b2o_pack_records_scored(b2o_ctx* ctx, const float* boxes_dev, const int32_t* counts_dev, const int32_t* labels_dev,
                            const float* box_scores_dev, const float* logp_dev, const float* inv_scale_dev, int n,
                            int max_boxes, int rows, int rec_boxes, float* records_dev, void* stream);

/* Debug / test taps (not on the product path): b2o_set_debug_taps(ctx, 1) makes b2o_crnn_forward also write the
 * fp32 fc_12 outputs ("logits") to its workspace; by default (0) the fused Dense + CTC kernel keeps them in
 * registers and only the labels reach memory.  b2o_crnn_tap copies an intermediate of the last forward pass.
 * b2o_crnn_tap names: "features" (b,50,7,512 f16), "theta" (b,6 f32), "warped" (b,50,7,512 f16),
 * "fc_9" (b,50,128 f16), "l1" (b,50,128 f16), "l2" (b,50,256 f16), "logits" (b,48,K f32); the conv backbone
 * "x1" (b,200,31,64 f16, conv_1), "x2" (128, conv_2), "x3" (256, conv_3), "p3" (b,100,15,256, its pool),
 * "x4" (256, conv_4), "x5" (512, conv_5), "p5" (b,50,7,512, its pool), "x6" (512, conv_6).  "x3" and "x5" are only
 * written by engines that do not fuse the pool into the convolution (SIMT, TC_GENERIC).
 * As for b2o_craft_tap, a tap reads the context's last successful CRNN forward (any b2o_crnn_forward*, or
 * b2o_crnn_features, which stops after "l2"), given the same ws_dev and b, and only a buffer that forward wrote: "x3"
 * and "x5" per its engine, "theta" and "warped" with a spatial transformer, "logits" when it kept them (the debug taps
 * on at the forward, or _logits, _beam, _lexicon).  Otherwise B2O_ERR_STATE, also before any forward, after a forward
 * that failed once it had begun enqueueing work, and after b2o_load_crnn (a call rejected by its argument or workspace
 * checks changes nothing).  Unknown name or out_bytes too small: B2O_ERR_ARG.                                  */
int b2o_set_debug_taps(b2o_ctx* ctx, int on);
int b2o_crnn_tap(b2o_ctx* ctx, const char* name, const void* ws_dev, int b, void* out_dev,
                 size_t out_bytes, void* stream);

/* One generic convolution through the selected engine (test hook for the conv kernels).
 * x: (n,h,w,cin) fp16, wgt: (cout, k, k, cin) fp32 host, epilogue y = relu?(acc*s1+t1)*s2+t2.
 * out: (n,h,w,cout) fp16.  s2/t2 may be NULL.                                                 */
int b2o_conv2d_test(b2o_ctx* ctx, const void* x_dev, int n, int h, int w, int cin,
                    const float* wgt_host, int cout, int ksize, int dilation,
                    const float* s1_host, const float* t1_host, int relu,
                    const float* s2_host, const float* t2_host, void* out_dev, int engine,
                    void* stream);

/* One convolution with every epilogue feature the networks use (test hook, not on the product path).  Every "_dev"
 * pointer addresses channel 0 of a channel slice of a wider NHWC buffer whose channel stride is the matching "_ld".
 *   x      (n,h,w,cin) fp16, x_ld >= cin.  wgt (cout,k,k,cin) fp32 host; y = relu?(acc*s1+t1)*s2+t2 (s2/t2 may be NULL).
 *   out    (n,h,w,cout), fp32 when out_f32 else fp16, out_ld >= cout; write_full = 0 skips it where the pool is fused.
 *   pool   optional (n,h/2,w/2,cout) fp16 2x2/2 max pool of the output (floor for odd sizes), pool_ld >= cout.
 *   up     optional (n,h/2,w/2,cout) fp16 whose exact-2x bilinear upsampling is added to the accumulator before the
 *          epilogue (the commuted decoder upsampling; tensor-core engines only).
 *   tail   optional CRAFT head tail (16-channel layers): w6 (16 in,16 out), b6 (16), w8 (16 in,2 out), b8 (2) fp32 host;
 *          scores (n,h,w,2) fp32.  B2O_CONV_AUTO fuses it into the conv epilogue when the layer allows, as
 *          b2o_craft_forward does; other engines run the separate head_tail kernel on `out`.
 * Plain and pooled layers are routed as b2o_craft_forward / b2o_crnn_forward route them for the given engine.
 * Synchronises the stream before returning.                                                              */
typedef struct {
  const void* x_dev;
  int n, h, w, cin, x_ld;
  const float* wgt_host;
  int cout, ksize, dilation;
  const float *s1_host, *t1_host;
  int relu;
  const float *s2_host, *t2_host;
  void* out_dev;
  int out_ld, out_f32, write_full;
  void* pool_dev;
  int pool_ld;
  const void* up_dev;
  int up_ld;
  const float *w6_host, *b6_host, *w8_host, *b8_host;
  float* scores_dev;
  int engine;
} b2o_conv_test_desc;
int b2o_conv_test(b2o_ctx* ctx, const b2o_conv_test_desc* desc, void* stream);

/* The plan of one tensor-core convolution (test hook, not on the product path; host only, no context and no GPU): the
 * choices the library makes before it launches a layer of (cin -> cout, ksize x ksize, dilation) over an (n, h, w, cin)
 * input, writing fp32 when out_f32, with the fused 2x2 max pool, the fused CRAFT tail or the decoder's upsample-add of a
 * (n, h/2, w/2, cout) tensor when pool, tail or up_add is set, on engine B2O_CONV_AUTO or B2O_CONV_TC_GENERIC, with the
 * channels-by-pixels bodies allowed (swap = 1, the default) or not (B2O_TC_SWAP=0), on a GPU of sm_count SMs; the other
 * switches at their defaults.  B2O_ERR_ARG where the library would refuse the launch (or the tensor cores do not run the
 * layer).  Otherwise *plan: the conv_tc_kernel<block_n, kch, mode, pair, upadd> instance (mode 0 generic tiles, 1 halo
 * tiles, 2 halo tiles with the filter bank resident in shared memory); body 0 pixels by channels, 1 channels by pixels,
 * 2 channels by pixels on 16 x 16-pixel tiles; the tile_w x tile_h x tile_n pixel tile and the number of tiles (pixel
 * tiles x output-channel tiles); the ring's stages, the bytes between stages and the bytes one stage's barrier expects;
 * the resident filter bank's bytes (0: streamed with the stages); dynamic shared memory and grid of the launch; coop_n
 * 1 where the two consumer warpgroups run paired n-tiles (tiles 2u and 2u + 1 share each activation box: a (tap,
 * chunk) step then fills one stage_tx slot and one slot of the filter rows alone).                                    */
typedef struct {
  int n, h, w, cin, cout, ksize, dilation;
  int out_f32, pool, tail, up_add;
  int engine, swap, sm_count;
} b2o_conv_plan_desc;
typedef struct {
  int32_t block_n, kch, mode, pair, upadd, body;
  int32_t tile_w, tile_h, tile_n, tiles;
  int32_t stages, stage_bytes, stage_tx, resident_bytes, smem_bytes, grid;
  int32_t coop_n;
} b2o_conv_plan;
int b2o_conv_plan_test(const b2o_conv_plan_desc* desc, b2o_conv_plan* plan);

/* The plan b2o_warp_boxes derives from each box (test hook, not on the product path): get_rotated_box ordering,
 * get_rotated_width_height, the fp64 cv2.getPerspectiveTransform solve and the closed-form 3x3 inverse.  boxes: (n,4,2)
 * float32; plans: n records of 88 bytes.  m = inverse homography (destination -> source, row major), dw, dh = dsize of
 * warpPerspective; valid = 0 where warpBox raises ZeroDivisionError (m, dw and dh are then 0) or the fp64 system is
 * singular, and b2o_warp_boxes writes an all-zero crop for such a box.                                           */
typedef struct {
  double m[9];
  int32_t dw, dh, valid;
} b2o_warp_plan;
int b2o_warp_plan_test(b2o_ctx* ctx, const float* boxes_dev, int n, b2o_warp_plan* plans_dev, void* stream);

/* b2o_get_boxes_scored, and the intermediate results of getBoxes (test hook, not on the product path).
 * labels_dev (n,hs,ws) int32: each foreground pixel's connected component, named by its root = the index inside the
 * image of the component's first pixel in raster order; -1 for background.  comps_dev (n,max_boxes,7) int32: the kept
 * components in box order, (root, left, top, width, height, area, maxtext) with maxtext the order-preserving int key
 * of the largest text score (the float's bits if >= 0, else bits ^ 0x7fffffff); entries past min(count, max_boxes)
 * are left as they were.  labels_dev or comps_dev NULL: B2O_ERR_ARG before anything is enqueued.               */
int b2o_get_boxes_test(b2o_ctx* ctx, const float* scores_dev, int n, int hs, int ws,
                       float detection_threshold, float text_threshold, float link_threshold,
                       int size_threshold, float* boxes_dev, int32_t* counts_dev, float* box_scores_dev,
                       int max_boxes, void* ws_dev, size_t ws_bytes, int32_t* labels_dev, int32_t* comps_dev,
                       void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B2OCR_H */
