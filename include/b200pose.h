/* b200pose - C ABI of the H100-native OpenPose (rtpose VGG19) inference path.
 *
 * Plain pointers and sizes only; no torch / numpy types.  Every entry point returns 0 on success and a
 * non-zero code on failure (b200pose_last_error() gives the text) unless stated otherwise.  A failed call leaves no
 * CUDA error pending for later calls, and the objects it was given stay usable.
 *
 * Threading: b200pose_last_error() is per thread; a net / post object and the legacy process_paf surface serialise
 * nothing themselves - use one object per host thread (or your own lock).  All work of a call is enqueued on the
 * cuda_stream argument (plus the post object's private second stream for the person assembly and result copies).
 *
 * Each declaration cites the reference interface it replaces (paths relative to the reference repository).
 * The reference-side bindings (ctypes) are shown in INTEGRATION.md.
 */
#ifndef B200POSE_H
#define B200POSE_H

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------------------------
 * 0. Library
 * ---------------------------------------------------------------------------------------------------------- */
const char* b200pose_last_error(void);
int b200pose_version(void);
/* Number of CUDA kernels launched by this library since load (the bench's gpu_launches evidence). */
long b200pose_launch_count(void);

/* ------------------------------------------------------------------------------------------------------------
 * 1. Network: replaces rtpose_model.forward                       lib/network/rtpose_vgg.py:158-198
 *    (get_model / make_vgg19_block / make_stages                  lib/network/rtpose_vgg.py:13-56, 60-225)
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct b200pose_net b200pose_net;

#define B200POSE_NUM_TENSORS 184   /* state_dict entries, reference order (model0, model{1..6}_1, model{1..6}_2) */
#define B200POSE_MODE_BF16 0       /* wgmma tensor cores, bf16 operands, fp32 accumulate                         */
#define B200POSE_MODE_FP32 1       /* fp32-parity mode: fp32 FMA everywhere (1e-3 bar of BASELINE.json)          */
#define B200POSE_MODE_BF16X3 2     /* high-precision tensor-core mode: value + residual bf16 planes for activations and
                                      weights, 3 MMA terms per K block (A_hi*W_hi + A_hi*W_lo + A_lo*W_hi); measured
                                      1.4e-3 max-abs @368x368 (bf16: 7e-2, fp32 mode: 3e-5) - the tensor core's own fp32
                                      accumulation is the floor, see DESIGN.md 2.3                                   */
#define B200POSE_MODE_FP8 3        /* fp8 tensor-core mode: the wgmma convolutions run on e4m3 operands, activations
                                      scaled by 2^ea per (launch, image) from the max |bf16| their writers stored, weights
                                      by 2^ew per output channel; activations stay bf16 in memory and conv1_1 runs as in
                                      bf16 mode (DESIGN.md 2.3).  Before this mode existed, 3 ran as bf16.             */
#define B200POSE_MODE_FP16 4       /* fp16 tensor-core mode: the bf16 plan with IEEE binary16 activations and weights
                                      (10 mantissa bits against bf16's 7), fp32 full-K accumulation; fp32 stage maps.
                                      binary16 overflows above 65504: every forward flags each image whose input or a
                                      stored value is +-inf or NaN in binary16, and weights beyond it are refused (b200pose_net_overflow, b200pose_post_overflow), the maps
                                      of a flagged image are not to be trusted (DESIGN.md 2.3).  Before this mode existed,
                                      4 ran as bf16; every value outside 0 .. 4 still does.                            */

int b200pose_net_create(b200pose_net** out, int cuda_device);
/* A net of the reference's second network, OpenPose_Model(l2_stages, l1_stages, 38, 19)    lib/network/openpose.py:111-199
 * (DESIGN.md 2.11): rtpose's trunk with PReLU after conv4_2, conv4_3_CPM and conv4_4_CPM, then l2 PAF stages and l1
 * heat-map stages, one after the other, of dense 3x3 blocks with PReLU.  1 <= l2, 1 <= l1, l2 + l1 <= 12.  The net keeps
 * its architecture: b200pose_net_set_tensor / _finalize validate against its own tensor table (the reference's
 * state_dict order, b200pose_openpose_tensor_shape), outputs[12] of every forward hold its maps in saved_for_loss order
 * [paf_1 .. paf_l2, heat_1 .. heat_l1] (the other entries must be NULL), and the final maps - what b200pose_net_last_maps
 * returns and every fused entry point post-processes - are paf_l2 and heat_l1.  Modes bf16, bf16x3 and fp32; fp8 and
 * fp16, and b200pose_net_set_stages, are refused with an error naming the architecture, leaving the net usable. */
int b200pose_net_create_openpose(b200pose_net** out, int cuda_device, int l2_stages, int l1_stages);
/* OpenPose_Model(l2_stages, l1_stages)'s state_dict, without a device: the number of tensors (< 0: no such architecture)
 * and the shape of tensor `index` (weights: 4 dims OIHW; biases and PReLU slopes: 1 dim), returning its number of dims
 * (< 0: out of range).  Each conv's tensors come in the order weight, bias, PReLU slope. */
int b200pose_openpose_num_tensors(int l2_stages, int l1_stages);
int b200pose_openpose_tensor_shape(int l2_stages, int l1_stages, int index, long dims[4]);
void b200pose_net_destroy(b200pose_net* net);
/* Shape of state_dict tensor `index` (weights: 4 dims OIHW, biases: 1 dim); returns number of dims. */
int b200pose_net_tensor_shape(int index, long dims[4]);
/* Copy one fp32 tensor (host memory, OIHW / [O]) into the net.  Replaces load_state_dict(), demo/picture_demo.py:46. */
int b200pose_net_set_tensor(b200pose_net* net, int index, const float* host_data, long count);
/* Pack weights for the device (bf16 K-major slices, padded heads, concat-permuted 7x7 inputs). */
int b200pose_net_finalize(b200pose_net* net);
/* forward: input fp32 NCHW [n,3,H,W] (H, W multiples of 8); outputs[12] fp32 NCHW in saved_for_loss order
 * [paf1, heat1, ..., paf6, heat6] (paf [n,38,H/8,W/8], heat [n,19,H/8,W/8]); entries may be NULL to skip the
 * copy-out.  With k stages (b200pose_net_set_stages) only entries 0 .. 2k-1 are written; the others must be NULL (a
 * non-NULL one is an error naming it).  *_on_device: 0 = host pointers (copies are issued on `cuda_stream` and
 * synchronised before return), 1 = device pointers (asynchronous on `cuda_stream`).  cuda_stream: a cudaStream_t cast
 * to void* (NULL = default).
 * On a real stream (not the legacy default stream, not one that is being captured) the launches (52 with six stages)
 * of a SMALL-batch (launch-bound: up to 4 frames of 368x368) tensor-core forward pass are captured at the SECOND use of
 * a (shape, mode, stages, input pointer) into a CUDA graph and replayed afterwards
 * (a caller that passes a fresh pointer every time never pays a capture); the input buffer's
 * CONTENTS may change between calls, results are those of plain launches (tests/test_gpu.py:
 * test_graph_replay_equals_plain_launches).  B200POSE_GRAPH=0 disables the capture. */
int b200pose_net_forward(b200pose_net* net, const float* input, int input_on_device, int n, int H, int W, int mode,
                         float* const* outputs, int outputs_on_device, void* cuda_stream);
/* Same, but the input is uint8 HWC BGR frames [n,H,W,3] (what cv2.imread / crop_with_factor produce) and
 * rtpose_preprocess (x/256 - 0.5, HWC -> CHW; lib/datasets/preprocessing.py:16-21, evaluate/coco_eval.py:93-94) is fused
 * into the first convolution's load: 4x less H2D traffic, no fp32 staging. */
int b200pose_net_forward_u8(b200pose_net* net, const unsigned char* images, int input_on_device, int n, int H, int W,
                            int mode, float* const* outputs, int outputs_on_device, void* cuda_stream);
/* Normalisation the uint8 entry points (b200pose_net_forward_u8, b200pose_infer_u8*, b200pose_infer_raw_u8*) fuse into
 * the first convolution: get_outputs' `preprocess` argument (evaluate/coco_eval.py:92-100; functions in
 * lib/datasets/preprocessing.py:16-86).  Default B200POSE_PRE_RTPOSE.  Bit-identical to the numpy functions. */
#define B200POSE_PRE_RTPOSE 1      /* x/256 - 0.5                                   */
#define B200POSE_PRE_VGG 2         /* BGR -> RGB, /255, (x - mean) / std            */
#define B200POSE_PRE_INCEPTION 3   /* BGR -> RGB, x/128 - 1                         */
#define B200POSE_PRE_SSD 4         /* x - (123, 117, 104) on (B, G, R)              */
int b200pose_net_set_preprocess(b200pose_net* net, int preprocess);
/* Refinement stages every later forward of the net runs (every b200pose_net_forward*, b200pose_infer* and the flip,
 * raw, ragged and multi-scale variants): the trunk, stage 1 and stages 2 .. `stages`, 1 <= stages <= 6, default 6.  The
 * stage count is part of the plan and CUDA-graph keys; the fused entry points post-process (flip-merge, resize and
 * average) stage `stages`'s maps, and b200pose_net_last_maps returns them.  Each stage's maps are those a six-stage
 * forward gives for that stage, bit for bit.  Any other value is an error and leaves the setting as it was. */
int b200pose_net_set_stages(b200pose_net* net, int stages);
/* Ragged batch (DESIGN.md 1): n already cropped uint8 HWC BGR frames of different sizes, packed back to back (frame i is
 * hw[2i] x hw[2i+1] x 3 bytes, both multiples of 8; n <= 1024).  The batch runs on the canvas Hc x Wc = (max H_i, max W_i):
 * outputs[12] as b200pose_net_forward's at canvas size [n, C, Hc/8, Wc/8]; inside its own (H_i/8) x (W_i/8) each frame's
 * maps are bit for bit those of b200pose_net_forward_u8 on that frame alone, outside they are +0.  Plans (and the CUDA
 * graphs of small batches) are keyed on (n, Hc, Wc, mode): a new mix of frames on the same canvas rebuilds nothing. */
int b200pose_net_forward_ragged_u8(b200pose_net* net, const unsigned char* frames, int on_device, int n, const int* hw,
                                   int mode, float* const* outputs, int outputs_on_device, void* cuda_stream);
/* Measurement hook: re-runs the launch list of the last tensor-core forward (conv1_1 + 16 + 7 (k - 1) tensor-core
 * launches for k stages: 51 with six) with a CUDA event pair around every launch; fills per-launch milliseconds and
 * ALGORITHMIC FLOPs (2 x MACs of the unpadded convolution).  Returns the number of launches, < 0 on error. */
int b200pose_net_profile(b200pose_net* net, float* ms, double* flops, int cap, void* cuda_stream);
/* Test hooks of the last bf16 / bf16x3 / fp8 / fp16 forward's launch list (launch 0 = conv1_1, 1 .. 16 + 7 (k - 1) = the
 * tensor-core launches of its k stages, 1 .. 51 with six);
 * they let a test check one launch against a reference computed from that launch's real inputs.
 *   b200pose_net_debug_run    : re-runs the first `launches` launches on the last forward's input (plain launches with
 *                               the plan's own arguments, PDL included, no graph), then synchronises the stream.
 *   b200pose_net_debug_launch : describes launch i in fields[0 .. B200POSE_DEBUG_LAUNCH_FIELDS - 1]:
 *       0 input buffer id (-1 = the network input)  1 in_cstride  2 in_ch_base  3 in_ch_group_stride
 *       4 output buffer id  5 out_cstride  6, 7 out_ch_off[2]  8, 9 store_ch[2]  10 H  11 W  12 ksize  13 cin_blocks
 *       14 groups  15 n_tile  16 n_tiles  17 relu  18 pool  19 split  20 chunk  21 pdl  22 tps
 *       23, 24 fp32 stage map written per group (-1 = none)  25 images  26 uint8 input normalisation (launch 0; 0 = fp32)
 *     cap >= B200POSE_DEBUG_LAUNCH_FIELDS.  With cap >= 28 it also writes
 *       27 (B200POSE_DEBUG_LAUNCH_FORMAT) format of the 16-bit activation planes: 0 bfloat16, 1 IEEE binary16 (fp16 mode)
 *     Returns the number of fields written.
 *   b200pose_net_debug_read   : copies images [img0, img0 + count) of one buffer to host memory: ids 0 .. 13 are the
 *     bf16 NHWC activation buffers t1, t2, t3, t4, t5a, t5b, t6, t7, t8, t9, cat, bra, brb, br512 (lo_plane = 1: their
 *     residual planes, bf16x3 only), 14 .. 25 the fp32 NCHW stage maps in saved_for_loss order (those of the stages the
 *     forward ran).  The activation
 *     buffers hold bfloat16 bits, or binary16 bits after an fp16 forward (debug_launch field 27). */
#define B200POSE_DEBUG_LAUNCH_FIELDS 27
#define B200POSE_DEBUG_LAUNCH_FORMAT 27
int b200pose_net_debug_run(b200pose_net* net, int launches, void* cuda_stream);
int b200pose_net_debug_launch(b200pose_net* net, int i, int* fields, int cap);
int b200pose_net_debug_read(b200pose_net* net, int buf, int lo_plane, int img0, int count, void* host, long bytes);
/* fp8 test hook: for tensor-core launch `launch` (1 .. 51 with six stages) of the last fp8 forward, the activation scale exponent ea each
 * of its n_img images used, as the kernel recorded it (act_exp[n_img], n_img = the forward's batch), and the weight
 * exponent ew of each packed output row (w_exp[cap], rows = groups * n_tiles * n_tile; pad rows 0).  Returns the number
 * of rows, < 0 on error. */
int b200pose_net_debug_fp8(b200pose_net* net, int launch, int* act_exp, int n_img, int* w_exp, int cap);
/* fp16 overflow report of the last forward (any entry point): waits for cuda_stream, then flags[i] = 1 if image i
 * (n = the forward's batch; flip: frames, then mirrors) stored a value beyond binary16's range (+-inf or NaN) in any
 * layer, else 0.  Forwards of the other modes flag nothing.  Returns the number of flagged images, < 0 on error. */
int b200pose_net_overflow(b200pose_net* net, int* flags, int n, void* cuda_stream);
/* Device pointers of the last forward's final maps (NCHW fp32): those of its last stage (stage 6 by default), valid
 * until the next forward. */
int b200pose_net_last_maps(b200pose_net* net, const float** paf, const float** heat, int* n, int* h, int* w);

/* ------------------------------------------------------------------------------------------------------------
 * 2. Post-processing: replaces NMS + paf_to_pose_cpp + pafprocess  lib/utils/paf_to_pose.py:67-145, 372-406
 *                                                                  lib/pafprocess/pafprocess.cpp:22-218
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct b200pose_post b200pose_post;

#define B200POSE_HUMAN_FLOATS 73   /* score, then 18 x (x, y, peak score, peak id or -1); x, y in input pixels */
/* status bits */
#define B200POSE_ST_PEAK_OVERFLOW 1
#define B200POSE_ST_CAND_OVERFLOW 2
#define B200POSE_ST_ROW_OVERFLOW 4
#define B200POSE_ST_HUMAN_OVERFLOW 8

int b200pose_post_create(b200pose_post** out, int cuda_device, int batch_cap, int peak_cap_per_part, int human_cap);
void b200pose_post_destroy(b200pose_post* post);
/* heat [n,19,h,w], paf [n,38,h,w] (layout 0 = NCHW) or heat [n,h,w,19], paf [n,h,w,38] (layout 1 = NHWC, what
 * get_outputs returns per image, evaluate/coco_eval.py:111-112); fp32, low resolution (stride 8).
 * thresh = cfg.TEST.THRESH_HEATMAP.  Results stay on the device until fetched. */
int b200pose_post_run(b200pose_post* post, const float* heat, const float* paf, int on_device, int layout, int n, int h,
                      int w, float thresh, void* cuda_stream);
/* Post-processing settings (lib/pafprocess/pafprocess.h:7-13, compile-time constants in the reference).  They apply
 * to the runs submitted after the call: b200pose_post_run and every fused b200pose_infer* entry point of this post
 * object.  Each run keeps the settings it was submitted with, also while another run is in flight.  Comparisons keep
 * the reference's form (pafprocess.cpp:73-90, 187-191): a sample counts iff vec . paf > paf_thresh, a pair is kept iff
 * more than paf_min_above samples count, a person is dropped iff parts < min_parts or score / parts < min_person_score.
 * The defaults run exactly the kernels of the reference's constants.  A looser prune may keep more persons than
 * human_cap; that sets B200POSE_ST_HUMAN_OVERFLOW as usual.  The legacy process_paf surface (section 4) always uses
 * the reference's constants.
 *   b200pose_post_default_params : the defaults below
 *   b200pose_post_set_params     : p = NULL restores the defaults; a value outside its range is refused with an error
 *                                  naming the field, and the settings stay as they were
 *   b200pose_post_get_params     : the settings the next run will use */
typedef struct b200pose_post_params {
    float paf_thresh;        /* THRESH_VECTOR_SCORE, pafprocess.h:7  = cfg.TEST.THRESH_PAF; finite                   0.05 */
    int paf_samples;         /* STEP_PAF, pafprocess.h:13            = cfg.TEST.NUM_INTERMED_PTS_BETWEEN_KEYPOINTS;
                                1 .. 64                                                                               10 */
    int paf_min_above;       /* THRESH_VECTOR_CNT1, pafprocess.h:8; -1 .. paf_samples                                  6 */
    int min_parts;           /* THRESH_PART_CNT, pafprocess.h:9; 0 .. 18                                               4 */
    float min_person_score;  /* THRESH_HUMAN_SCORE, pafprocess.h:10; finite                                          0.3 */
} b200pose_post_params;
int b200pose_post_default_params(b200pose_post_params* out);
int b200pose_post_set_params(b200pose_post* post, const b200pose_post_params* p);
int b200pose_post_get_params(b200pose_post* post, b200pose_post_params* out);
/* Peak refinement (NMS, lib/utils/paf_to_pose.py:67-145) and the up-sampling factor f from the maps to the peaks.
 *   B200POSE_REFINE_CUBIC       : the clipped 5x5 window around each peak, cv2.resize(INTER_CUBIC) by f, first arg-max;
 *                                 position f * window origin + arg-max, score the value there (the default)
 *   B200POSE_REFINE_CUBIC_GAUSS : as CUBIC, the resized patch first smoothed by scipy.ndimage.gaussian_filter(sigma=3)
 *                                 (bool_gaussian_filt=True); the score is the smoothed value
 *   B200POSE_REFINE_NONE        : no refinement (bool_refine_center=False): position (p + 0.5) f - 0.5 truncated to an
 *                                 int as pafprocess does, score the low-resolution map value
 *   b200pose_post_set_refine : the mode of the runs submitted after the call (b200pose_post_run, _run_scaled and every
 *                              fused entry point); each run keeps its own.  An invalid mode is refused and the setting
 *                              stays as it was
 *   b200pose_post_get_refine : the mode the next run will use, < 0 on error
 *   b200pose_post_run_scaled : b200pose_post_run with the factor as an argument, 1 .. 16; b200pose_post_run is this call
 *                              with 8.  PAF scoring reads the maps at (y / f, x / f) and h * f, w * f must not exceed
 *                              16384.  Fused runs always use 8, the network's stride. */
#define B200POSE_REFINE_NONE 0
#define B200POSE_REFINE_CUBIC 1
#define B200POSE_REFINE_CUBIC_GAUSS 2
int b200pose_post_set_refine(b200pose_post* post, int mode);
int b200pose_post_get_refine(b200pose_post* post);
int b200pose_post_run_scaled(b200pose_post* post, const float* heat, const float* paf, int on_device, int layout, int n,
                             int h, int w, int upsample, float thresh, void* cuda_stream);
/* Every run copies its results (person rows, counts, status) to pinned host memory by itself, on a second stream right
 * after the person assembly, into one of two slots (run parity) - so a caller may submit run i+1 before reading run i
 * (at most two runs in flight).  The getters below read the selected slot.
 *   b200pose_post_last_ticket : ticket (0-based index) of the most recently submitted run, -1 if none
 *   b200pose_post_select      : block until run `ticket` is on the host and make the getters read it
 *   b200pose_post_sync        : select(last ticket) */
long b200pose_post_last_ticket(b200pose_post* post);
int b200pose_post_select(b200pose_post* post, long ticket);
int b200pose_post_sync(b200pose_post* post);
/* Diagnostics: out[0..2] = max SM cycles of the limbs kernel phases (scoring, exact sort, greedy) over all blocks since
 * the last reset, out[3] = max candidates of a limb, out[4] = total candidates. */
int b200pose_post_debug(b200pose_post* post, unsigned long long* out, int n, int reset);
/* Test hook: sorts n 64-bit candidate keys (high word = ~score bits, low word = pair index) on the device with the
 * product's sorting kernels - libstdc++'s std::sort order (pafprocess.cpp:97), ties included.  Host pointers. */
int b200pose_post_debug_sort(b200pose_post* post, const unsigned long long* keys, int n, unsigned long long* out);
/* Test hook: the grids of the two work-queue kernels of PAF scoring and sorting (limb_score_kernel, range_sort_kernel),
 * for every run of this post object submitted after the call (b200pose_post_run, the fused b200pose_infer* entry points)
 * and for b200pose_post_debug_sort.  Both kernels take their work from a global cursor, so their results do not depend
 * on the grid; this lets a test check that.  0 restores a default (score: SMs x 6; sort: min(n x 19, SMs x 3), and
 * SMs x 3 for debug_sort).  A value below 0 or above 65535 is refused with an error naming it, and the grids stay as
 * they were. */
int b200pose_post_set_grids(b200pose_post* post, int score_blocks, int sort_blocks);
/* Test hook: the connections the greedy matcher (pafprocess.cpp:98-124) chose for limb `limb` of image `img` of the
 * latest run, in the order it chose them: peak indices a (part limb[0]) and b (part limb[1]) within their parts, and
 * the candidate score.  Waits for the run, copies at most cap entries to the host arrays and returns the count;
 * -1 on error. */
int b200pose_post_debug_connections(b200pose_post* post, int img, int limb, int* a, int* b, float* s, int cap);
/* Test hook: waits for the device, then copies the first heat_floats / paf_floats floats of the maps the last flip or
 * multi-scale run averaged and post-processed (NCHW fp32; a ragged run's at its canvas pitch) to host memory. */
int b200pose_post_debug_maps(b200pose_post* post, float* heat, long heat_floats, float* paf, long paf_floats);
/* OR of the status words of every image of every run since the last reset (sticky accumulator kept on the device):
 * with runs in flight a caller reads only some results back; this proves that no run at all overflowed a capacity
 * (the reference's std::vectors grow without bound, pafprocess.cpp:24-44, so an overflow is a divergence).  < 0 on error. */
int b200pose_post_status_accum(b200pose_post* post, int reset);
int b200pose_post_num_humans(b200pose_post* post, int img);             /* < 0 on error */
int b200pose_post_status(b200pose_post* post, int img);                 /* status bits of the last run */
/* fp16 mode: 1 if the network overflowed binary16 for frame img of the selected fused run (in any forward of it: either
 * orientation with flip, any scale), else 0 (always 0 for other modes and for b200pose_post_run).  < 0 on error. */
int b200pose_post_overflow(b200pose_post* post, int img);
int b200pose_post_get_humans(b200pose_post* post, int img, float* out, int max_humans);   /* returns count */
/* joint list rows (x, y, score, id, part), the array paf_to_pose.py:376-378 builds; returns count */
int b200pose_post_get_peaks(b200pose_post* post, int img, float* out, int max_peaks);

/* ------------------------------------------------------------------------------------------------------------
 * 3. Fused path: net forward + post-processing without leaving the device (the batched entry point of
 *    SURVEY.md 8b).  input: fp32 NCHW [n,3,H,W].
 * ---------------------------------------------------------------------------------------------------------- */
int b200pose_infer(b200pose_net* net, b200pose_post* post, const float* input, int input_on_device, int n, int H, int W,
                   int mode, float thresh, void* cuda_stream);

int b200pose_infer_u8(b200pose_net* net, b200pose_post* post, const unsigned char* images, int input_on_device, int n,
                      int H, int W, int mode, float thresh, void* cuda_stream);

/* ------------------------------------------------------------------------------------------------------------
 * 3b. Flip test-time averaging: replaces handle_paf_and_heat        evaluate/coco_eval.py:197-242
 *     out = (normal + mirror_W(flipped)[left/right-swapped channels, PAF x components negated]) / 2, bit-identical to
 *     the reference's float32 arithmetic.  Unlike the reference it does not modify flipped_paf in place.
 *     All six pointers are host (on_device = 0; copies on `cuda_stream`, synchronised before return) or device (1,
 *     asynchronous); layout 0 = [n,C,h,w], 1 = [n,h,w,C] (what get_outputs returns per image), C = 19 / 38.
 *     `post` provides the device and the staging buffers.
 * ---------------------------------------------------------------------------------------------------------- */
int b200pose_flip_merge(b200pose_post* post, const float* normal_heat, const float* flipped_heat,
                        const float* normal_paf, const float* flipped_paf, int on_device, int layout, int n, int h, int w,
                        float* out_heat, float* out_paf, void* cuda_stream);
/* Fused flip-TTA inference: the n frames and their W-mirrored copies (made on the device) run through the network as
 * one 2n batch, the two map sets are merged as above and the fused post-processing runs on the averaged maps; nothing
 * leaves the device but the person rows.  Equivalent to get_outputs(img) + get_outputs(img[:, ::-1]) +
 * handle_paf_and_heat + paf_to_pose_cpp for frames that need no padding in W (a padded frame must be mirrored before
 * crop_with_factor pads it: use b200pose_net_forward on both orientations + b200pose_flip_merge instead).
 * Results are fetched exactly like b200pose_infer's. */
int b200pose_infer_flip(b200pose_net* net, b200pose_post* post, const float* input, int input_on_device, int n, int H,
                        int W, int mode, float thresh, void* cuda_stream);
int b200pose_infer_u8_flip(b200pose_net* net, b200pose_post* post, const unsigned char* images, int input_on_device,
                           int n, int H, int W, int mode, float thresh, void* cuda_stream);

/* ------------------------------------------------------------------------------------------------------------
 * 3c. Device-side crop_with_factor: replaces crop_with_factor / _factor_closest   lib/network/im_transform.py:113-134
 *     (called by get_outputs, evaluate/coco_eval.py:87-91, with dest_size = cfg.DATASET.IMAGE_SIZE, factor =
 *     cfg.MODEL.DOWNSAMPLE, is_ceil = True).  uint8 HWC BGR frames of ONE source size (a video stream, or one shape
 *     bucket of a data set) -> cv2.resize(fx = fy = dest_size / min(h, w)) with OpenCV's 8-bit INTER_LINEAR arithmetic,
 *     bit for bit (csrc/resize_core.h) -> zero padding bottom/right to a multiple of `factor` (a multiple of 8).
 *   b200pose_crop_geometry         : host only; the values crop_with_factor returns / implies
 *   b200pose_net_crop_with_factor  : images [n,src_h,src_w,3] -> out [n,pad_h,pad_w,3]; host or device pointers
 *   b200pose_infer_raw_u8          : raw frames -> resize/pad -> network -> fused post-processing, all on the device;
 *                                    flip != 0 adds left/right flip test-time averaging: the RAW frame is mirrored
 *                                    before it is resized and padded, exactly like get_outputs(img[:, ::-1]) would see
 *                                    it, then the maps are merged as handle_paf_and_heat does.
 *     Person coordinates are in pixels of the padded frame (pad_h x pad_w), like the reference's.
 * ---------------------------------------------------------------------------------------------------------- */
/* (Video frames in NV12 / I420 or rotated: b200pose_infer_frames, section 3d.) */
int b200pose_crop_geometry(int src_h, int src_w, int dest_size, int factor, double* im_scale, int* res_h, int* res_w,
                           int* pad_h, int* pad_w);
int b200pose_net_crop_with_factor(b200pose_net* net, const unsigned char* images, int images_on_device, int n, int src_h,
                                  int src_w, int dest_size, int factor, unsigned char* out, int out_on_device,
                                  void* cuda_stream);
int b200pose_infer_raw_u8(b200pose_net* net, b200pose_post* post, const unsigned char* images, int input_on_device, int n,
                          int src_h, int src_w, int dest_size, int factor, int mode, float thresh, int flip,
                          void* cuda_stream);
/* b200pose_infer_raw_u8 for n raw frames of DIFFERENT sizes, packed back to back (frame i: src_hw[2i] x src_hw[2i+1] x 3
 * bytes), as one ragged batch (DESIGN.md 1): every frame is cropped to its own padded size and the batch runs on the
 * canvas of the largest; with flip the network runs 2n images.  Per frame, person rows and peaks are those
 * b200pose_infer_raw_u8 gives for that frame alone, in pixels of its own padded frame.  Fetched like b200pose_infer's. */
int b200pose_infer_raw_u8_ragged(b200pose_net* net, b200pose_post* post, const unsigned char* images, int input_on_device,
                                 int n, const int* src_hw, int dest_size, int factor, int mode, float thresh, int flip,
                                 void* cuda_stream);

/* Multi-scale (+ flip) test-time averaging, BASELINE.json configs[4].  The reference at this commit has no multi-scale
 * loop (get_outputs is single-scale, evaluate/coco_eval.py:87-91); the protocol is composed from its own functions:
 * for every scale s: crop_with_factor(img, int(base_size * s), factor) -> network (-> handle_paf_and_heat with the
 * mirrored RAW frame when flip != 0) -> bicubic resize of the 57 maps to the grid of base_size (OpenCV INTER_CUBIC
 * formula, csrc/resize_core.h) -> running float32 sum; average = sum / n_scales; fused post-processing on the average.
 * oracle/glue_port.py::multi_scale_maps restates exactly this composition. */
int b200pose_infer_raw_u8_multiscale(b200pose_net* net, b200pose_post* post, const unsigned char* images,
                                     int input_on_device, int n, int src_h, int src_w, int base_size, int factor,
                                     const double* scales, int n_scales, int mode, float thresh, int flip,
                                     void* cuda_stream);
/* b200pose_infer_raw_u8_multiscale for n raw frames of DIFFERENT sizes, packed back to back as for
 * b200pose_infer_raw_u8_ragged (frame i: src_hw[2i] x src_hw[2i+1] x 3 bytes).  Every scale runs as one ragged batch
 * on the canvas of that scale's largest padded frame; each frame's maps are resized from its own extent at that scale
 * to its own base grid and averaged on the canvas of the base padded sizes (+0 outside each frame).  Per frame, person
 * rows and peaks are those b200pose_infer_raw_u8_multiscale gives for that frame alone, in pixels of its own padded
 * base frame.  1 <= n_scales <= 16, n <= the post object's batch_cap, and with flip 2n <= 1024.  Fetched like
 * b200pose_infer's. */
int b200pose_infer_raw_u8_multiscale_ragged(b200pose_net* net, b200pose_post* post, const unsigned char* images,
                                            int input_on_device, int n, const int* src_hw, int base_size, int factor,
                                            const double* scales, int n_scales, int mode, float thresh, int flip,
                                            void* cuda_stream);

/* ------------------------------------------------------------------------------------------------------------
 * 3d. Video frames: replaces the host-side cv2.cvtColor + cv2.rotate ahead of get_outputs   video_demo.py:29-46
 *     (DESIGN.md 2.10).  Frames as decoders and capture devices hand them out - NV12 (Y plane + interleaved UV plane
 *     of h/2 rows), planar I420 (Y, U, V; U and V h/2 x w/2) or pitched BGR HWC - every plane with its own pitch, in
 *     host or device memory.  They are converted on the device to uint8 HWC BGR, rotated by `rotate` degrees clockwise
 *     (0, 90 = cv2.ROTATE_90_CLOCKWISE, 180, 270 = cv2.ROTATE_90_COUNTERCLOCKWISE), bit for bit what
 *     cv2.rotate(cv2.cvtColor(frame, COLOR_YUV2BGR_NV12 / _I420), code) gives (OpenCV 4.13; csrc/frame_core.h).
 *     4:2:0 frames need even sizes; every pitch must cover a row (BGR 3w, Y w, NV12 UV w, I420 U / V w/2 bytes).
 *     on_device = 0: host planes, copied into device staging with cudaMemcpy2DAsync (NV12 / I420 cross PCIe at half
 *     the bytes of BGR); 1: device planes, read in place.  Every frame is checked before anything is enqueued; an
 *     invalid one fails naming the frame and the field.
 * ---------------------------------------------------------------------------------------------------------- */
#define B200POSE_FRAME_BGR 0
#define B200POSE_FRAME_NV12 1
#define B200POSE_FRAME_I420 2
typedef struct b200pose_frame {
    const unsigned char* plane[3];   /* BGR: [0]; NV12: Y, UV; I420: Y, U, V */
    int pitch[3];                    /* bytes per row of each plane */
    int h, w;                        /* stored size in pixels */
} b200pose_frame;
/* n <= 1024 frames -> out: their rotated BGR HWC frames packed back to back (frame i: oh_i x ow_i x 3 bytes, (oh, ow) =
 * (h, w) or (w, h) when rotated by 90 / 270).  out_on_device: 0 = host memory (the call synchronises the stream),
 * 1 = device memory (asynchronous on cuda_stream). */
int b200pose_net_convert_frames(b200pose_net* net, const b200pose_frame* frames, int n, int format, int on_device,
                                int rotate, unsigned char* out, int out_on_device, void* cuda_stream);
/* frames -> conversion -> the b200pose_infer_raw_u8* pipeline at the rotated sizes: scales NULL runs one scale
 * (dest_size), else multi-scale averaging around dest_size; frames of one rotated size run as a uniform batch, mixed
 * sizes as a ragged one.  n <= the post object's batch_cap, and with flip 2n <= 1024.  Per frame, person rows and peaks
 * are those the b200pose_infer_raw_u8* entry point gives for the converted, rotated frame, in pixels of its padded
 * frame.  Packed BGR frames (pitch 3w, each frame right behind the previous one) with rotate 0 take that entry point
 * as they are, without a conversion launch.  Host frames stay alive until the fetch; fetched like b200pose_infer's. */
int b200pose_infer_frames(b200pose_net* net, b200pose_post* post, const b200pose_frame* frames, int n, int format,
                          int on_device, int rotate, int dest_size, int factor, const double* scales, int n_scales,
                          int mode, float thresh, int flip, void* cuda_stream);

/* ------------------------------------------------------------------------------------------------------------
 * 3e. Drawing the persons: replaces draw_humans(frame, humans_from_rows(rows, net_w, net_h))   lib/utils/common.py
 *     (DESIGN.md 2.12).  Draws, in place, the persons of images 0 .. n-1 of the SELECTED run (the rows
 *     b200pose_post_get_humans returns) on uint8 HWC BGR frames packed back to back (frame i: frame_hw[2i] x
 *     frame_hw[2i+1] x 3 bytes, the layout b200pose_net_convert_frames writes; sizes may differ).  net_hw[2i],
 *     net_hw[2i+1]: the padded network input frame i's coordinates are in.  A part's centre is
 *     (int(x / net_w * w + 0.5), int(y / net_h * h + 0.5)) in double precision; persons in row order, each with
 *     cv2.circle(c, 3, CocoColors[part], thickness 3) for its parts in part order, then cv2.line(.., CocoColors[k], 3)
 *     for the limbs k of CocoPairsRender it has, bit for bit what cv2 (OpenCV 4.13) draws (csrc/draw_core.h).
 *     on_device = 1: device frames, asynchronous on cuda_stream; 0: host frames, staged, drawn and copied back (the
 *     call synchronises the stream).  What a call draws is fixed when it returns: later runs and draw calls do not
 *     change it.  n < 1 or above batch_cap or the selected run's image count, a size < 1 and no selected run are
 *     refused, naming the field, before anything is enqueued.
 * ---------------------------------------------------------------------------------------------------------- */
int b200pose_post_draw(b200pose_post* post, unsigned char* frames, int on_device, int n, const int* frame_hw,
                       const int* net_hw, void* cuda_stream);

/* ------------------------------------------------------------------------------------------------------------
 * 3f. JPEG images: replaces cv2.imread / cv2.imdecode(buf, cv2.IMREAD_COLOR) ahead of get_outputs   (DESIGN.md 2.13)
 *     Baseline and extended sequential Huffman streams (SOF0 / SOF1, 8-bit) with one component or three YCbCr
 *     components sampled luma 1x1, 2x1, 2x2, 1x2 or 4x1 with chroma 1x1, restart intervals, any APPn / COM segments
 *     and EXIF orientations 1 .. 8 are decoded on the device, bit for bit what cv2.imdecode gives (OpenCV 4.13 with
 *     libjpeg-turbo 3.1, csrc/jpeg_core.h).  Progressive, lossless, arithmetic-coded and 12-bit streams, CMYK / YCCK,
 *     Adobe RGB and R/G/B component ids, other sampling factors and multi-scan streams are "unsupported"; a stream
 *     that is not a valid JPEG or whose frame has more than 2^28 pixels is "malformed".  Both are refused before
 *     anything is enqueued, naming the image and the reason.  Damaged entropy-coded data (an invalid code, too few or
 *     too many blocks, missing or misordered restart markers) is found on the device: it sets status bits of the image
 *     (1 invalid code, 2 data ends early, 4 data left over, 8 restart markers) where libjpeg would warn and pad.
 *
 *     b200pose_jpeg_info: host only.  The oriented size h x w of the decoded frame and whether the device decodes the
 *     stream (b200pose_last_error() holds the reason when not); returns nonzero for a malformed stream.
 *     b200pose_net_decode_jpegs: n streams data[i] of sizes[i] bytes (host memory) -> their oriented BGR frames packed
 *     back to back in `out` (host, or device when out_on_device); synchronises the stream and fails, naming the first
 *     image, when an image's status is not 0.
 *     b200pose_infer_jpegs: b200pose_infer_raw_u8* on the decoded frames - uniform when every frame has one size,
 *     ragged otherwise, multi-scale when scales is not null; n <= batch_cap, 2n <= 1024 with flip.  The streams are
 *     copied when the call returns.  b200pose_post_jpeg_status: the status bits of image img of the selected run (0
 *     for runs not made from JPEG streams), -1 when img is out of range.
 *
 *     Progressive streams (SOF2, DESIGN.md 2.18), opt-in per net: b200pose_net_set_jpeg_progressive(net, 1) makes
 *     b200pose_net_decode_jpegs and b200pose_infer_jpegs on that net decode progressive Huffman streams with 8-bit
 *     samples and the sampling set above too, bit for bit cv2.imdecode, up to 256 scans per image.  Default 0: they
 *     are refused as "unsupported: progressive (SOF2)".  Still refused as unsupported with the switch on: streams in
 *     which some component has unknown bits among zig-zag coefficients 0 .. 9 after its last scan (libjpeg smooths
 *     those blocks), bogus progressions (libjpeg only warns), undefined Huffman tables.  A scan that is not a valid
 *     progression (where libjpeg stops with JERR_BAD_PROGRESSION and cv2.imdecode returns None) is malformed.  Damaged
 *     entropy data sets the status bits above.  b200pose_net_get_jpeg_progressive: the switch (0 / 1), -1 for a null
 *     net.  b200pose_jpeg_info_ex: b200pose_jpeg_info with the switch given (b200pose_jpeg_info: 0).
 * ---------------------------------------------------------------------------------------------------------- */
int b200pose_jpeg_info(const unsigned char* data, long long size, int* h, int* w, int* supported);
int b200pose_jpeg_info_ex(const unsigned char* data, long long size, int progressive, int* h, int* w, int* supported);
int b200pose_net_set_jpeg_progressive(b200pose_net* net, int on);
int b200pose_net_get_jpeg_progressive(b200pose_net* net);
int b200pose_net_decode_jpegs(b200pose_net* net, const unsigned char* const* data, const long long* sizes, int n,
                              unsigned char* out, int out_on_device, void* cuda_stream);
int b200pose_infer_jpegs(b200pose_net* net, b200pose_post* post, const unsigned char* const* data,
                         const long long* sizes, int n, int dest_size, int factor, const double* scales, int n_scales,
                         int mode, float thresh, int flip, void* cuda_stream);
int b200pose_post_jpeg_status(b200pose_post* post, int img);

/* ------------------------------------------------------------------------------------------------------------
 * 3g. JPEG encoding: replaces cv2.imencode('.jpg', frame, [IMWRITE_JPEG_QUALITY, quality,
 *     IMWRITE_JPEG_SAMPLING_FACTOR, sampling]) and cv2.imwrite of a .jpg name   (DESIGN.md 2.14)
 *     Baseline streams with the standard Huffman tables, byte for byte what cv2 (OpenCV 4.13 with libjpeg-turbo 3.1)
 *     writes: JFIF header, quality 1 .. 100 (jpeg_set_quality with baseline tables), sampling one of cv2's
 *     IMWRITE_JPEG_SAMPLING_FACTOR values 0x221111 (4:2:0), 0x211111 (4:2:2), 0x121111 (4:4:0), 0x411111 (4:1:1) and
 *     0x111111 (4:4:4) (csrc/jpeg_enc_core.h).
 *
 *     b200pose_jpeg_encode_bound: host only.  The stream bytes that always suffice for an h x w frame at this sampling
 *     (every block at its longest codes, every byte stuffed); -1 for a size outside 1 .. 65535 or an unknown sampling.
 *     b200pose_net_encode_jpegs: n (1 .. 1024) uint8 HWC BGR frames packed back to back (frame i: frame_hw[2i] x
 *     frame_hw[2i+1] x 3 bytes, the layout b200pose_post_draw draws on; host, or device when frames_on_device) -> their
 *     streams packed back to back in `out` (host, or device when out_on_device; out_cap bytes), sizes[i] (host) the
 *     length of stream i.  Synchronises the stream (twice inside the call, to size the bit buffers and a host
 *     output's staging from what the kernels computed, and at its end).  n, a size outside 1 .. 65535, a quality outside 1 .. 100, an
 *     unknown sampling and an out_cap below the sum of the images' bounds are refused, naming the field, before
 *     anything is enqueued.  One call launches 5 kernels.
 * ---------------------------------------------------------------------------------------------------------- */
long long b200pose_jpeg_encode_bound(int h, int w, int sampling);
int b200pose_net_encode_jpegs(b200pose_net* net, const unsigned char* frames, int frames_on_device, const int* frame_hw,
                              int n, int quality, int sampling, unsigned char* out, long long out_cap, int out_on_device,
                              long long* sizes, void* cuda_stream);

/* ------------------------------------------------------------------------------------------------------------
 * 3h. PNG encoding: replaces cv2.imencode('.png', frame) and cv2.imwrite of a .png name   (DESIGN.md 2.15)
 *     Byte for byte what cv2 (OpenCV 4.13 with libpng 1.6 and zlib 1.3) writes at its defaults: 8-bit RGB, no
 *     interlace, every row Sub-filtered, zlib level 1 with strategy Z_RLE, IDAT chunks of 8 192 bytes, no ancillary
 *     chunks (csrc/png_enc_core.h).  The call takes no encoder parameters.
 *
 *     b200pose_png_encode_bound: host only.  The file bytes that always suffice for an h x w frame (every deflate
 *     block stored, plus the framing); -1 for a size outside 1 .. 65535.
 *     b200pose_net_encode_pngs: n (1 .. 1024) uint8 HWC BGR frames packed back to back (frame i: frame_hw[2i] x
 *     frame_hw[2i+1] x 3 bytes, the layout b200pose_post_draw draws on; host, or device when frames_on_device) -> their
 *     PNG files packed back to back in `out` (host, or device when out_on_device; out_cap bytes), sizes[i] (host) the
 *     length of file i.  Synchronises the stream (once inside the call, to size the deflate words and the output from
 *     what the kernels computed, and at its end).  n, a size outside 1 .. 65535 and an out_cap below the sum of the
 *     images' bounds are refused, naming the field, before anything is enqueued.  One call launches 9 kernels.
 * ---------------------------------------------------------------------------------------------------------- */
long long b200pose_png_encode_bound(int h, int w);
int b200pose_net_encode_pngs(b200pose_net* net, const unsigned char* frames, int frames_on_device, const int* frame_hw,
                             int n, unsigned char* out, long long out_cap, int out_on_device, long long* sizes,
                             void* cuda_stream);

/* ------------------------------------------------------------------------------------------------------------
 * 3i. COCO keypoint evaluation: replaces pycocotools' COCOeval(cocoGt, cocoDt, 'keypoints') .evaluate() and
 *     .accumulate() with default Params   (DESIGN.md 2.16, csrc/coco_eval_core.h)
 *     The caller has done loadRes and _prepare: the gts and detections are grouped into (category, image) units that
 *     have at least one of either, units ordered by category index (0 .. n_cats - 1, the sorted category ids) and
 *     within a category by ascending image id.  Unit u: category unit_cat[u], gts unit_gt0[u] .. unit_gt0[u+1] - 1 in
 *     the gt file's order, detections unit_dt0[u] .. unit_dt0[u+1] - 1 in the result list's order.
 *     Per gt: gt_id (non-zero, all different), gt_kpt [51] (x, y, v per part), gt_box [5] (bbox x, y, w, h, then the
 *     annotation's area), gt_crowd (iscrowd) and gt_ignore (_prepare's flag: iscrowd or num_keypoints == 0).  Per
 *     detection: dt_kpt [51] and dt_score.  thr: iouThrs [10] then recThrs [101], each ascending.
 *     Out (host): precision [10][101][n_cats][3] and recall [10][n_cats][3] (pycocotools' eval['precision'] and
 *     eval['recall'] without the maxDets axis; area ranges all, medium, large).  oks (host, may be null): each unit's
 *     computeOks block [min(nd, 20)][ng] back to back in unit order, oks_cap doubles; oks_count (may be null) gets
 *     the block sizes' sum.
 *     Runs on `device` in a stream of its own and synchronises it.  Non-finite values, a keypoint count other than
 *     51, gt id 0 or a repeated gt id, units out of order, and counts above the limits (1024 gts and 1024 detections
 *     per unit, 2^24 gts or detections per call, 2^18 detections after the cut to 20 per unit, 1024 categories) are
 *     refused, naming the argument, before anything is enqueued.  One call launches 4 kernels.
 * ---------------------------------------------------------------------------------------------------------- */
int b200pose_coco_kpt_eval(int device, int n_units, int n_cats, const int* unit_cat, const int* unit_gt0,
                           const int* unit_dt0, const long long* gt_id, const double* gt_kpt, int gt_kpt_len,
                           const double* gt_box, const unsigned char* gt_crowd, const unsigned char* gt_ignore,
                           const double* dt_kpt, int dt_kpt_len, const double* dt_score, const double* thr,
                           double* precision, double* recall, double* oks, long long oks_cap, long long* oks_count);

/* ------------------------------------------------------------------------------------------------------------
 * 3j. PNG images: replaces cv2.imread / cv2.imdecode(buf, cv2.IMREAD_COLOR) of PNG streams ahead of get_outputs
 *     (DESIGN.md 2.17)
 *     Every colour type and bit depth, Adam7 interlacing, any ancillary chunks and eXIf orientations 1 .. 8 are
 *     decoded on the device, bit for bit what cv2.imdecode gives (OpenCV 4.13 with libpng 1.6 and zlib 1.3,
 *     csrc/png_core.h): 8-bit BGR, 16-bit samples stripped to their high byte, gray below 8 bits replicated, palette
 *     entries past PLTE black, alpha dropped.  APNG streams (acTL) are "unsupported".  A bad signature or IHDR, a
 *     chunk running past the end, no IDAT, non-consecutive IDATs, no IEND, a palette image without PLTE, a CRC error
 *     on a critical chunk other than IDAT, an unknown critical chunk and a frame of more than 2^28 pixels (or a side
 *     beyond libpng's 1 000 000) are "malformed".  Both are refused before anything is enqueued, naming the image and
 *     the reason.  Damage inside the image data is found on the device and sets status bits of the image: 1 invalid
 *     deflate data, 2 data ends early, 4 Adler-32 mismatch, 8 IDAT CRC error, 16 invalid filter type - exactly the
 *     streams for which cv2.imdecode returns None.
 *
 *     b200pose_png_info: host only.  The oriented size h x w of the decoded frame and whether the device decodes the
 *     stream (b200pose_last_error() holds the reason when not); returns nonzero for a malformed stream.
 *     b200pose_net_decode_pngs: n streams data[i] of sizes[i] bytes (host memory) -> their oriented BGR frames packed
 *     back to back in `out` (host, or device when out_on_device); synchronises the stream and fails, naming the first
 *     image, when an image's status is not 0.  One call launches 4 kernels.
 *     b200pose_infer_pngs: b200pose_infer_raw_u8* on the decoded frames - uniform when every frame has one size,
 *     ragged otherwise, multi-scale when scales is not null; n <= batch_cap, 2n <= 1024 with flip.  The streams are
 *     copied when the call returns.  b200pose_post_png_status: the status bits of image img of the selected run (0
 *     for runs not made from PNG streams), -1 when img is out of range.
 * ---------------------------------------------------------------------------------------------------------- */
int b200pose_png_info(const unsigned char* data, long long size, int* h, int* w, int* supported);
int b200pose_net_decode_pngs(b200pose_net* net, const unsigned char* const* data, const long long* sizes, int n,
                             unsigned char* out, int out_on_device, void* cuda_stream);
int b200pose_infer_pngs(b200pose_net* net, b200pose_post* post, const unsigned char* const* data,
                        const long long* sizes, int n, int dest_size, int factor, const double* scales, int n_scales,
                        int mode, float thresh, int flip, void* cuda_stream);
int b200pose_post_png_status(b200pose_post* post, int img);

/* ------------------------------------------------------------------------------------------------------------
 * 3k. Training targets and stage losses: replace CocoKeypoints.get_ground_truth (lib/datasets/datasets.py:259-308) +
 *     transpose((2, 0, 1)).astype(float32), and get_loss's MSEs (train/train_VGG19.py:143-174)   (DESIGN.md 2.19)
 *   b200pose_ground_truth: keypoints (host) [sum persons][17][3] float32, COCO order, the persons of image 0 first;
 *     persons[n] per image; hw[2n] = (input_y, input_x) per image.  Writes heat [n][19][canvas_h][canvas_w] and
 *     paf [n][38][canvas_h][canvas_w] float32 (device pointers), asynchronously on cuda_stream: image i fills the
 *     top-left int(input_y / 8) x int(input_x / 8) of its slot, bit for bit the reference's maps, +0 outside.  The
 *     stage maps' own layout, ragged batches included (canvas = max H_i / 8, max W_i / 8).  An image without persons
 *     gets zero PAFs and a background of 1.0 (the reference raises IndexError there).  Refused, naming the argument,
 *     before anything is enqueued: n outside 1 .. 1024, persons outside 0 .. 256 per image, a side outside 8 .. 8192,
 *     non-finite keypoints, a canvas below an image's grid or above 1024 x 1024 cells.  heat and paf both NULL: the arguments are checked and
 *     nothing else happens.  One call: one upload and 2 kernels.
 *   b200pose_net_last_forward: what the net's last forward ran (any entry point): info[4] = n images, canvas H, canvas
 *     W (input pixels) and the stage maps it wrote (2k for k rtpose stages, l2 + l1 for OpenPose_Model); hw (may be
 *     NULL; hw_cap >= 2n) gets each image's extent {H_i, W_i}, the canvas for a uniform forward.  Later set_stages calls
 *     do not change it.  No forward yet: refused.
 *   b200pose_net_stage_losses: for the net's last forward (n images, canvas Hc x Wc, k stages or an OpenPose_Model's
 *     maps), with heat / paf its targets in the layout above at the forward's canvas (device pointers), writes on
 *     cuda_stream sums[n][maps] (double, device; `maps` must be the count b200pose_net_last_forward reports, anything
 *     else is refused): per (image, stage map in saved_for_loss order) the float64 sum of the
 *     float32 (pred - target)^2 over the image's own (H_i / 8) x (W_i / 8) cells, the PAF maps against paf and the heat
 *     maps against heat; and extrema[n][4] (float, device): max and min of the final heat map's channels 0 .. 17, then
 *     max and min of the final PAF map, over the image's own cells.  The sums are added in a fixed order without
 *     atomics: they depend on neither the canvas nor the other images.  One kernel.  No forward yet: refused.
 * ---------------------------------------------------------------------------------------------------------- */
int b200pose_ground_truth(int device, const float* keypoints, const int* persons, const int* hw, int n, float* heat,
                          float* paf, int canvas_h, int canvas_w, void* cuda_stream);
int b200pose_net_last_forward(b200pose_net* net, int* info, int* hw, int hw_cap);
int b200pose_net_stage_losses(b200pose_net* net, const float* heat, const float* paf, double* sums, int maps,
                              float* extrema, void* cuda_stream);

/* ------------------------------------------------------------------------------------------------------------
 * 3l. Training batches: replace the reference loader's per-sample image path, preprocess = Normalize,
 *     RandomApply(HFlip, 0.5), RescaleRelative (Pillow BICUBIC), Crop(edge), CenterPad(edge) (train/train_VGG19.py:124-130,
 *     lib/datasets/transforms.py), then image_transform_train = ColorJitter(0.1, 0.1, 0.1, 0.1), a JPEG quality-50
 *     round trip, RandomGrayscale(0.01), ToTensor + Normalize (transforms.py:53-65), and mask_valid_area
 *     (lib/datasets/utils.py:36-54)   (DESIGN.md 2.20)
 *   b200pose_net_augment: frames: n uint8 BGR frames packed back to back (host, or device with frames_on_device),
 *     hw[2n] = (h, w) each; params[n][B200POSE_AUG_PARAMS] the draws of each sample, as engine.augment_params makes
 *     them: hflip, resized w, resized h, crop x, crop y, ColorJitter's order (4 fn ids), brightness, contrast,
 *     saturation and hue factors, jpeg, grayscale, and the mask bounds x0, y0, x1, y1 (columns < x0 or >= x1 and rows
 *     < y0 or >= y1 become 0).  Writes out_f32 [n][3][edge][edge] (RGB, normalised, masked) and, unless out_u8 is
 *     NULL, out_u8 [n][edge][edge][3] (the BGR image ToTensor receives), bit for bit the reference's tensors; device
 *     pointers with out_on_device (written asynchronously on cuda_stream unless a sample drew the JPEG round trip,
 *     which waits for the encoded streams), else host pointers and the call waits.  Refused, naming the argument,
 *     before anything is enqueued: n outside 1 .. 1024, a side outside 2 .. 8192, an edge not a multiple of 8 or
 *     outside 8 .. 1024, and a params record that does not fit its source (non-integers, a resized size outside
 *     side / 2 .. side, a crop outside the resized image, an order that is not a permutation, a negative factor or a
 *     hue outside -0.5 .. 0.5, flags other than 0 / 1, mask bounds outside 0 .. edge).  4 kernels, plus
 *     b200pose_net_encode_jpegs' and b200pose_net_decode_jpegs' when any sample drew the JPEG round trip.
 *   b200pose_ground_truth_f64: b200pose_ground_truth for float64 keypoints (a flipped sample's, as horizontal_swap_coco
 *     returns them): add_neck and the joint centres in float64.  The same checks, layout and launches.
 * ---------------------------------------------------------------------------------------------------------- */
#define B200POSE_AUG_PARAMS 19
int b200pose_net_augment(b200pose_net* net, const unsigned char* frames, int frames_on_device, int n, const int* hw,
                         const double* params, int edge, float* out_f32, unsigned char* out_u8, int out_on_device,
                         void* cuda_stream);
int b200pose_ground_truth_f64(int device, const double* keypoints, const int* persons, const int* hw, int n,
                              float* heat, float* paf, int canvas_h, int canvas_w, void* cuda_stream);

/* ------------------------------------------------------------------------------------------------------------
 * 4. Legacy SWIG surface of lib/pafprocess (pafprocess.h:53-59, pafprocess.i:14): same names, same argument
 *    meaning; state is kept in a process-global context exactly like the reference's file-scope globals
 *    (pafprocess.cpp:12-13).  peaks [p1,p2,5] rows (x, y, score, id, part) sorted by part as paf_to_pose_cpp
 *    builds them; heatmap is not dereferenced (only h1 is used, pafprocess.cpp:83); pafmap [f1,f2,f3] is the
 *    x8 nearest-upsampled HWC array.  process_paf returns 0 like the reference, or a non-zero code if the
 *    device path failed (the reference has no failure mode).
 * ---------------------------------------------------------------------------------------------------------- */
int process_paf(int p1, int p2, int p3, float* peaks, int h1, int h2, int h3, float* heatmap, int f1, int f2, int f3,
                float* pafmap);
int get_num_humans(void);
int get_part_cid(int human_id, int part_id);
float get_score(int human_id);
int get_part_x(int cid);
int get_part_y(int cid);
float get_part_score(int cid);

#ifdef __cplusplus
}
#endif
#endif
