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

/* getBoxes (detection.py:207-287).  scores: (n,hs,ws,2) float32.  Writes, per image i,
 * counts[i] = number of boxes found (may exceed max_boxes: then only the first max_boxes are
 * stored and the caller retries with a larger buffer) and boxes[i][k][4][2] float32 in
 * detector-input pixels, in connected-component label order (= reference order).              */
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

/* The box bookkeeping of recognize_from_boxes (recognition.py:511-521: crops are appended image after
 * image, start_end = running offsets) on the device: the (n,max_boxes,4,2) table of b2o_get_boxes becomes
 * the dense list flat (sum_i min(counts[i],max_boxes), 4, 2) with image_index[k] = image of box k, both
 * sized for n*max_boxes entries by the caller.  Runs without the host knowing the counts, i.e. BEFORE
 * the one synchronisation of the path.                                                          */
int b2o_compact_boxes(b2o_ctx* ctx, const float* boxes_dev, const int32_t* counts_dev, int n, int max_boxes,
                      float* flat_dev, int32_t* image_index_dev, void* stream);

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

/* prediction_model.predict (recognition.py:535; graph 214-333): CRNN + STN + BiLSTM + greedy CTC (beam search:
 * b2o_crnn_forward_beam below).
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
 * "fc_9" (b,50,128 f16), "l1" (b,50,128 f16), "l2" (b,50,256 f16), "logits" (b,48,K f32).      */
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

#ifdef __cplusplus
}
#endif
#endif /* B2OCR_H */
