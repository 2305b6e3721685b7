/* libhvn -- C ABI of the H100-native HoVer-Net tile-inference + instance post-processing engine.
 *
 * Drop-in boundary for the reference's plugin seam (reference infer/base.py:56-78): the three
 * callables the reference resolves by name map onto these entry points
 *
 *   models.hovernet.net_desc.create_model      (net_desc.py:149)   -> hvn_create + hvn_load_param*
 *   models.hovernet.run_desc.infer_step        (run_desc.py:171)   -> hvn_forward
 *   models.hovernet.post_proc.process          (post_proc.py:94)   -> hvn_postproc
 *   (both, with the map never leaving the device)                  -> hvn_forward_postproc
 *
 * Plain pointers and sizes only; no torch / Python types.  Every function returns 0 on success
 * and a negative hvn_status otherwise; hvn_last_error() gives the message of the last failure on
 * the calling thread.  One context per device; calls on one context are serialised by the caller
 * (the reference calls run_step from the main thread only, infer/tile.py:308, infer/wsi.py:289).
 * Buffers are caller-owned.  "_dev" variants take device pointers on the context's device and are
 * stream-ordered on the context stream (hvn_sync waits for it).
 */
#ifndef HVN_H_
#define HVN_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HVN_ABI_VERSION 1

typedef enum {
    HVN_OK = 0,
    HVN_ERR_INVALID = -1,     /* bad argument / unsupported shape (reference: assert / shape error) */
    HVN_ERR_CUDA = -2,        /* CUDA runtime or driver failure */
    HVN_ERR_WEIGHTS = -3,     /* missing / unexpected / mis-shaped checkpoint key (strict load) */
    HVN_ERR_CAPACITY = -4,    /* caller-provided table too small */
    HVN_ERR_STATE = -5,       /* call order (e.g. forward before weights are finalised) */
    HVN_ERR_RANGE = -6        /* an activation left the representable range of the engine's fp16 hi+lo storage
                                 (|x| > 65504 * 2^act_shift); outputs of that call are invalid.  Raise option
                                 "act_shift" (exact power-of-two rescaling of all activations) and run again.  Reported
                                 by the call that synchronises: hvn_forward / hvn_forward_postproc / hvn_infer_tile(s),
                                 or, after *_dev calls, hvn_sync / hvn_timer_stop. */
} hvn_status;

/* Instance-table row: one per instance id present in inst_map, ascending id.  int64 x 10.
 * Replaces the per-instance loop of reference post_proc.py:120-181 (bbox via
 * misc/utils.py:18-28 with exclusive max; centroid = sum/area == cv2.moments m10/m00, m01/m00;
 * type vote :161-181).  type/type_count are -1/0 when nr_types == 0. */
#define HVN_ROW_LEN 10
enum { HVN_ROW_ID = 0, HVN_ROW_RMIN, HVN_ROW_CMIN, HVN_ROW_RMAX, HVN_ROW_CMAX, HVN_ROW_AREA,
       HVN_ROW_SUMX, HVN_ROW_SUMY, HVN_ROW_TYPE, HVN_ROW_TYPECNT };

/* Per-instance measurements (hvn_inst_features*): HVN_FEAT_LEN float64 per instance-table row, in this order. */
#define HVN_FEAT_LEN 18
enum { HVN_FEAT_AREA = 0, HVN_FEAT_CONTOUR_AREA, HVN_FEAT_PERIMETER, HVN_FEAT_CONVEX_AREA, HVN_FEAT_SOLIDITY,
       HVN_FEAT_CIRCULARITY, HVN_FEAT_MAJOR_AXIS_LENGTH, HVN_FEAT_MINOR_AXIS_LENGTH, HVN_FEAT_ECCENTRICITY,
       HVN_FEAT_ORIENTATION, HVN_FEAT_FERET_MAX, HVN_FEAT_MEAN_R, HVN_FEAT_MEAN_G, HVN_FEAT_MEAN_B, HVN_FEAT_STD_R,
       HVN_FEAT_STD_G, HVN_FEAT_STD_B, HVN_FEAT_NP_PROB_MEAN };

typedef struct hvn_ctx hvn_ctx;

int hvn_abi_version(void);
const char *hvn_last_error(void);

/* ---- model lifetime: reference create_model(mode, input_ch=3, nr_types, freeze) net_desc.py:149
 * mode: "original" | "fast".  nr_types: 0 means None (seg-only, 2 decoder branches). */
int hvn_create(int device, const char *mode, int nr_types, hvn_ctx **out);
void hvn_destroy(hvn_ctx *ctx);

/* ---- strict checkpoint load: reference infer/base.py:64-68 (`load_state_dict(strict=True)`).
 * Keys are the reference state_dict names (variables_tf2pytorch.csv col 1); float tensors are
 * host fp32, contiguous, shapes as in the reference (conv OIHW).  `num_batches_tracked` and
 * `upsample2x.unpool_mat` are accepted and ignored.  hvn_finalize_weights fails with
 * HVN_ERR_WEIGHTS if any expected key was not loaded. */
int hvn_num_params(const hvn_ctx *ctx);
int hvn_param_info(const hvn_ctx *ctx, int index, const char **name, int *ndim, int64_t shape[4]);
int hvn_load_param(hvn_ctx *ctx, const char *name, const float *data, int ndim, const int64_t *shape);
int hvn_finalize_weights(hvn_ctx *ctx);

/* ---- options.  keys: "conv_path" = 0 auto (wgmma where eligible), 1 CUDA-core referee only,
 *                      2 = auto + run every wgmma layer against the referee kernel and record the
 *                      per-layer max differences (hvn_debug_log);
 *                      "chunk" = patches per internal sub-batch (0 = auto);
 *                      "act_shift" = s in 0..48: store activations as x * 2^-s (see HVN_ERR_RANGE; weights are
 *                      re-derived, results are unchanged because powers of two are exact);
 *                      "precision" = 0 "highest" (default): activations feeding a convolution and its weights are
 *                      stored as fp16 hi + lo and each MAC forms hi*hi + hi*lo + lo*hi (fp32-grade products);
 *                      1 "high": hi planes only, one fp16 product per MAC with fp32 accumulation -- the operand
 *                      precision of TF32, a third of the tensor-core work and about half the activation memory.
 *                      Residual sums, BatchNorm, the 1x1 heads and post-processing stay fp32 in both; the range rules
 *                      (HVN_ERR_RANGE, "act_shift") are the same.  A change synchronises the context, re-derives the
 *                      weights and drops the cached plans; setting 0 again reproduces "highest" bit for bit.
 *                      Any other value is HVN_ERR_INVALID;
 *                      "tta" = 0 (default) | 1: test-time augmentation.  Every input patch runs as its 8 dihedral
 *                      views V_t(x) = rot90(t >= 4 ? flip(x, 1) : x, t % 4) (numpy, axes (0, 1)); each view's map is
 *                      brought back (rot90(., -(t % 4)), then flip(., 1) if t >= 4; HV vector (h, v) <- (-v, h)
 *                      t % 4 times, then h <- -h if t >= 4), and per output value the 8 are summed in view order in
 *                      fp32 and scaled by 1/8; TP is the argmax (first maximal index) of the mean softmax
 *                      probabilities.  Output layout, post-processing and the range rules are unchanged; a chunk
 *                      holds the views of max(1, chunk / 8) inputs.  Square patches only (H != W is
 *                      HVN_ERR_INVALID).  A change synchronises the context and drops the cached plans; 0 again is
 *                      the plain forward bit for bit.  Any other value is HVN_ERR_INVALID;
 *                      "profile" = 0 | 1 | 2 (see hvn_stage_ms);
 *                      tuning knobs: "tc_seg_chunks" (64-channel slices per accumulation segment), "tc_block_n",
 *                      "tc_prefetch" (L2 prefetch distance in K-slices for flat operands, 0 = off), "tc_xf_trunc"
 *                      (XF transform: truncating hi/lo split 1, round-to-nearest 0),
 *                      "xform", "fuse_shortcut", "fuse_up2", "branch_streams", "flood_impl".
 *                      The tc_* knobs are process-wide launch-time switches; every setting gives the same results to
 *                      fp32-accumulation noise (tests/test_cnn_gpu.py::test_kernel_variants_agree). */
int hvn_set_option(hvn_ctx *ctx, const char *key, int64_t value);
const char *hvn_debug_log(const hvn_ctx *ctx);
/* counters: "kernel_launches", "tc_launches", "pp_launches" (post-processing, contour and feature kernels),
 * "tile_table_rows" (rows of padded instance tables the last hvn_infer_tiles* group of two or more images held in the
 * context's workspace: min(rows_cap, H*W/6 + 8) per image, 84 B each), "last_flops" (algorithmic 2*MACs of the
 * last forward; with "tta" = 1 the 8 views' work), "precision" (0 | 1), "tta" (0 | 1), "plan_bytes" (device bytes of
 * the activation buffers, and with "tta" = 1 the per-chunk view and probability workspace, of the plan(s) the last
 * forward ran); with option "profile" = 2 also "launches:<class>" and "flops:<class>" for
 * class in {conv_tc, conv_ref, conv0, bnrelu, head, tta} (see hvn_stage_ms). */
int64_t hvn_get_counter(const hvn_ctx *ctx, const char *key);

/* ---- geometry of reference HoVerNet.forward (net_desc.py:101-145) for an in_h x in_w patch. */
int hvn_out_shape(const hvn_ctx *ctx, int in_h, int in_w, int *out_h, int *out_w, int *out_c);

/* ---- infer_step (run_desc.py:171-197): uint8 NHWC [B,H,W,3] RGB 0..255 ->
 * float32 NHWC [B,h,w,C], C = 3 (np_prob, hv_x, hv_y) or 4 (tp_argmax, np_prob, hv_x, hv_y). */
int hvn_forward(hvn_ctx *ctx, const uint8_t *imgs_host, int B, int H, int W, float *out_host);
int hvn_forward_dev(hvn_ctx *ctx, const uint8_t *imgs_dev, int B, int H, int W, float *out_dev);

/* ---- process / __proc_np_hv (post_proc.py:26-90, 94-186) on n_maps independent maps
 * pred [n_maps,H,W,C] float32 (C = 3, or 4 with nr_types > 0).
 * inst [n_maps,H,W] int32; table [n_maps,max_rows,HVN_ROW_LEN] int64; n_rows [n_maps] int32.
 * ctx may be a model context or one made with hvn_create_postproc (no weights needed). */
int hvn_create_postproc(int device, hvn_ctx **out);
int hvn_postproc(hvn_ctx *ctx, const float *pred_host, int n_maps, int H, int W, int C, int nr_types,
                 int32_t *inst_host, int64_t *table_host, int max_rows, int32_t *n_rows_host);
int hvn_postproc_dev(hvn_ctx *ctx, const float *pred_dev, int n_maps, int H, int W, int C, int nr_types,
                     int32_t *inst_dev, int64_t *table_dev, int max_rows, int32_t *n_rows_dev);

/* ---- per-instance contours (post_proc.py:133-147): for every table row the outer border of the instance,
 * point for point cv2.findContours(inst_map[rmin:rmax, cmin:cmax] == id, RETR_TREE, CHAIN_APPROX_SIMPLE)[0][0]
 * plus the (cmin, rmin) offset, traced on the device.  offs [n_maps*max_rows + 1] int32: the points of row r
 * of map m are pts[offs[m*max_rows + r] : offs[m*max_rows + r + 1]] (rows past n_rows[m] are empty);
 * pts [pts_cap,2] int32 (x, y).  HVN_ERR_CAPACITY when offs[n_maps*max_rows] > pts_cap (offs is valid then,
 * no points are written for rows that do not fit).  The caller applies the reference's "< 3 points" drop rule
 * (:140-141).  hvn_postproc_contours = hvn_postproc + contours with one round trip of the maps. */
int hvn_contours_dev(hvn_ctx *ctx, const int32_t *inst_dev, const int64_t *table_dev, const int32_t *n_rows_dev,
                     int n_maps, int H, int W, int max_rows, int32_t *pts_dev, int64_t pts_cap, int32_t *offs_dev);
int hvn_postproc_contours(hvn_ctx *ctx, const float *pred_host, int n_maps, int H, int W, int C, int nr_types,
                          int32_t *inst_host, int64_t *table_host, int max_rows, int32_t *n_rows_host,
                          int32_t *pts_host, int64_t pts_cap, int32_t *offs_host);

/* ---- fused tile path: infer_step then process on every patch, pred map stays in HBM.
 * pred_host / pred_dev may be NULL when the caller does not want the float maps back. */
int hvn_forward_postproc(hvn_ctx *ctx, const uint8_t *imgs_host, int B, int H, int W, float *pred_host,
                         int32_t *inst_host, int64_t *table_host, int max_rows, int32_t *n_rows_host);
int hvn_forward_postproc_dev(hvn_ctx *ctx, const uint8_t *imgs_dev, int B, int H, int W, float *pred_dev,
                             int32_t *inst_dev, int64_t *table_dev, int max_rows, int32_t *n_rows_dev);

/* ---- whole-image tile path (reference infer/tile.py:46-143: `_prepare_patching`, the batch loop, the stitch +
 * crop of `_post_process_patches`, then `process`): img u8 [H,W,3] RGB; patch_in = 256 (fast) / 270 (original).
 * Reflect padding, patch extraction, stitching and cropping are index arithmetic on the device; the padded image,
 * the patch list and the stitched map never exist on the host.
 *   hvn_tile_grid        : rows x cols of the patch grid (tile.py:60-69).
 *   hvn_tile_predict_dev : grid cells [cell_lo, cell_hi) (row-major) -> their region of pred_dev [H,W,C]; other
 *                          pixels are untouched (multi-GPU: each rank runs its slice into a zeroed map, then the maps
 *                          are summed -- x + 0 is exact).  batch = patches per network call (0 = default).
 *   hvn_infer_tile       : everything for one image from host buffers: pred_host [H,W,C] (may be NULL), inst [H,W],
 *                          table [max_rows,10], n_rows [1], and -- when offs_host is not NULL -- contours as in
 *                          hvn_contours (offs [max_rows + 1], pts [pts_cap,2]). */
int hvn_tile_grid(const hvn_ctx *ctx, int H, int W, int patch_in, int *rows, int *cols);
int hvn_tile_predict_dev(hvn_ctx *ctx, const uint8_t *img_dev, int H, int W, int patch_in, int cell_lo, int cell_hi,
                         int batch, float *pred_dev);
int hvn_infer_tile(hvn_ctx *ctx, const uint8_t *img_host, int H, int W, int patch_in, int batch, float *pred_host,
                   int32_t *inst_host, int64_t *table_host, int max_rows, int32_t *n_rows_host, int32_t *pts_host,
                   int64_t pts_cap, int32_t *offs_host);

/* ---- tile path over a group of images (reference infer/tile.py:236-369, which runs the patches of every cached file
 * as one stream of batches): n_images >= 1 images of any sizes, shapes [n_images][2] = (H, W) (a host array in both
 * variants), images u8 [H_i,W_i,3] packed back to back in input order.  All patches form one list, image after image,
 * cut into batches of `batch` (0 = default) that may span two or more images; each image's result is bit-identical to
 * hvn_infer_tile on that image alone.  Outputs, all in input order:
 *   pred [H_i,W_i,C] back to back (may be NULL), inst [H_i,W_i] back to back;
 *   table [rows_cap,10]: the instance rows of image i are table[row_offs[i] : row_offs[i+1]], row_offs [n_images+1];
 *   contours when pt_offs is not NULL: pt_offs [rows_cap+1], the points of packed row r are
 *   pts[pt_offs[r] : pt_offs[r+1]] (pts [pts_cap,2] (x, y); entries past row_offs[n_images] repeat the total).
 * Images of equal size are post-processed together, one call per size.  HVN_ERR_CAPACITY when row_offs[n_images] >
 * rows_cap (row_offs is valid then) or, the table fitting, when the points exceed pts_cap (pt_offs is valid then): size
 * the buffers from the offsets and call again.  HVN_ERR_INVALID on n_images < 1, a bad shape or rows_cap < 1.
 *   hvn_infer_tiles     : host buffers; synchronises, reports HVN_ERR_RANGE.
 *   hvn_infer_tiles_dev : device buffers (shapes stays on the host), stream-ordered on the context stream with no host
 *                         synchronisation, so the caller can overlap host work; the offsets are read (and range and
 *                         capacity checked) after hvn_sync, as for hvn_contours_dev.  Device workspace (context-owned,
 *                         grow-only): the padded instance tables of the group (min(rows_cap, H_i*W_i/6 + 8) rows of
 *                         84 B per image, counter "tile_table_rows"), and the maps in size order when that differs
 *                         from the input order. */
int hvn_infer_tiles(hvn_ctx *ctx, int n_images, const uint8_t *imgs_host, const int32_t *shapes, int patch_in,
                    int batch, float *pred_host, int32_t *inst_host, int64_t *table_host, int64_t rows_cap,
                    int32_t *row_offs_host, int32_t *pts_host, int64_t pts_cap, int32_t *pt_offs_host);
int hvn_infer_tiles_dev(hvn_ctx *ctx, int n_images, const uint8_t *imgs_dev, const int32_t *shapes, int patch_in,
                        int batch, float *pred_dev, int32_t *inst_dev, int64_t *table_dev, int64_t rows_cap,
                        int32_t *row_offs_dev, int32_t *pts_dev, int64_t pts_cap, int32_t *pt_offs_dev);

/* ---- end-of-batch gather support (SURVEY.md 8e; replaces the reference's DataParallel gather, infer/base.py:69):
 * hvn_pack_tables_dev compacts the padded tables of a batch, table_dev [n_maps,max_rows,10] + n_rows_dev [n_maps],
 * into packed_dev [<= cap_rows,10] (map order, no padding) and offs_dev [n_maps + 1] int32 (row range of map m =
 * [offs[m], offs[m+1]); offs[n_maps] = total; rows past cap_rows are not written) -- the buffer a rank hands to
 * ncclAllGather.  hvn_get_stream returns the context's cudaStream_t so that a collective can be ordered after the
 * library's kernels without a host synchronisation. */
int hvn_pack_tables_dev(hvn_ctx *ctx, const int64_t *table_dev, const int32_t *n_rows_dev, int n_maps, int max_rows,
                        int64_t *packed_dev, int64_t cap_rows, int32_t *offs_dev);
int hvn_get_stream(hvn_ctx *ctx, void **cuda_stream);

/* ---- instance statistics (reference metrics/stats_utils.py, compute_stats.py): contingency table of two
 * instance maps.  true/pred int32 [n_maps,H,W], ids >= 0, 0 = background; pred may be NULL (all zero, which gives
 * the ids and areas of `true`).  pairs [cap,3] int64 (t, p, count) for every (t, p) with t > 0 or p > 0 that occurs,
 * count > 0 (the (t, 0) and (0, p) rows are the parts that overlap background, so areas are row / column sums);
 * rows of map m are [offs[m], offs[m+1]), order within a map unspecified.  offs [n_maps+1] int64.
 * HVN_ERR_CAPACITY when offs[n_maps] > cap (offs valid, no rows written); HVN_ERR_INVALID on a negative id.
 * n_maps <= 65535, H*W < 2^31.  Device workspace (context-owned, grow-only): 12 B per pixel of 8x128 tiles plus
 * 12 * next_pow2(2*H*W) B per map.  Both variants synchronise the context stream to report the status. */
int hvn_inst_pairs(hvn_ctx *ctx, const int32_t *true_host, const int32_t *pred_host, int n_maps, int H, int W,
                   int64_t *pairs_host, int64_t cap, int64_t *offs_host);
int hvn_inst_pairs_dev(hvn_ctx *ctx, const int32_t *true_dev, const int32_t *pred_dev, int n_maps, int H, int W,
                       int64_t *pairs_dev, int64_t cap, int64_t *offs_dev);

/* ---- training targets (reference models/hovernet/targets.py gen_instance_hv_map, including
 * dataloader/augs.py fix_mirror_padding): inst int32 [n_maps,H,W] (ids >= 0, 0 = background) -> hv float32
 * [n_maps,H,W,2] (x, y), the full-size map before gen_targets crops it to crop_h x crop_w (the crop decides which
 * instances get offsets: those with >= 30 pixels inside it), bit for bit.  flags int32 [n_maps], HVN_TG_* bits: the
 * cases in which the reference raises ValueError (hv is undefined for such a map).  HVN_ERR_INVALID on a negative
 * id, on crop_h/crop_w outside 1..H/1..W, and when a map's largest id + its number of 4-connected components exceeds
 * 2^31 - 1 (the reference's int32 renumbering of split instances would wrap).  n_maps <= 65535, H*W < 2^31.  Device
 * workspace (context-owned, grow-only): 60 B per pixel.  Both variants synchronise the context stream. */
#define HVN_TG_NO_BACKGROUND 1       /* no 0 pixel in the map */
#define HVN_TG_NO_BACKGROUND_CROP 2  /* no 0 pixel left in the crop after removing instances < 30 px there */
#define HVN_TG_EMPTY_BOX 4           /* an instance's wrapped box holds none of its pixels (NaN centre of mass) */
int hvn_targets(hvn_ctx *ctx, const int32_t *inst_host, int n_maps, int H, int W, int crop_h, int crop_w,
                float *hv_host, int32_t *flags_host);
int hvn_targets_dev(hvn_ctx *ctx, const int32_t *inst_dev, int n_maps, int H, int W, int crop_h, int crop_w,
                    float *hv_dev, int32_t *flags_dev);

/* ---- validation step (reference run_desc.py valid_step + proc_valid_step_output) on one batch of patches already
 * cropped to the network input: imgs u8 [B,H,W,3], inst int32 [B,H,W], type int32 [B,H,W] (required when the model
 * has nr_types > 0, ignored otherwise).  Runs the forward (honouring "precision", "act_shift" and HVN_ERR_RANGE like
 * every forward), the targets on the same stream, and one reduction over the hvn_out_shape centre crop:
 * counts int64 [3 + 2*nr_types] = correct, inter, total of (np_prob > 0.5) against (inst > 0), then inter_k,
 * total_k of (tp == k) against (type == k) for k = 0..nr_types-1; hv_sse = sum of (pred_hv - true_hv)^2 (fp32
 * differences, fp64 sum); flags [B] as for hvn_targets.  Outputs are overwritten, not accumulated.  The maps never
 * leave the device.  Both variants synchronise the context stream. */
int hvn_valid(hvn_ctx *ctx, const uint8_t *imgs_host, const int32_t *inst_host, const int32_t *type_host, int B, int H,
              int W, int64_t *counts_host, double *hv_sse_host, int32_t *flags_host);
int hvn_valid_dev(hvn_ctx *ctx, const uint8_t *imgs_dev, const int32_t *inst_dev, const int32_t *type_dev, int B,
                  int H, int W, int64_t *counts_dev, double *hv_sse_dev, int32_t *flags_dev);

/* ---- validation loss: the reference's training objective (run_desc.py train_step; models/hovernet/utils.py
 * xentropy_loss, dice_loss, mse_loss, msge_loss) evaluated on the engine's eval-mode forward, on the same batch and
 * arguments as hvn_valid.  counts, hv_sse and flags are hvn_valid's (counts exactly; hv_sse to fp64 reordering).
 * sums double [10 + (nr_types ? 1 + 3*nr_types : 0)], over the B x h x w output crop, fp32 per-pixel terms added in
 * fp64 (p the softmax, t the one-hot target, q = p / sum_c p clamped to [1e-7, 1 - 1e-7] in fp32):
 *   0 np_ce = sum -log q_true;  1, 2 I_c = sum p_c t_c;  3, 4 L_c = sum p_c;  5, 6 R_c = sum t_c  (NP, t = inst > 0)
 *   7 hv_sq = sum (pred_hv - true_hv)^2 over both channels
 *   8 msge_num = sum f ((G_h(p) - G_h(t))^2 + (G_v(p) - G_v(t))^2), G_h / G_v the 5x5 kernels of get_sobel_kernel(5)
 *     on HV channels 0 / 1 as a cross-correlation, zero padding at the crop border;  9 focus = sum f, f = inst > 0
 *   with nr_types > 0: 10 tp_ce, then I_k (11 + k), L_k (11 + nt + k), R_k (11 + 2 nt + k) against type.
 * The reduction is deterministic (per-block partials in fixed slots, one fixed-order pass; no floating-point atomics):
 * equal inputs give bit-identical sums whatever "chunk" is.  probs (may be NULL) receives float32 [B,h,w,4+nr_types]
 * = [np p0, np p1, hv x, hv y, tp p0..] (with "tta" = 1 the view mean of every channel); np p1 and hv equal the plain
 * forward's bit for bit.  HVN_ERR_INVALID on a type id outside 0..nr_types-1 inside the crop (the reference's
 * F.one_hot raises; hvn_valid ignores such ids).  Device workspace (context-owned, grow-only): (4 + nr_types) * 4 B
 * per output pixel for the probabilities, 8 B per input pixel for the HV targets, 8 * sums B per 32 x 32 tile of the
 * crop for the partials, and hvn_targets' 60 B per input pixel.  Both variants synchronise the context stream. */
int hvn_valid_loss(hvn_ctx *ctx, const uint8_t *imgs_host, const int32_t *inst_host, const int32_t *type_host, int B,
                   int H, int W, int64_t *counts_host, double *hv_sse_host, int32_t *flags_host, double *sums_host,
                   float *probs_host);
int hvn_valid_loss_dev(hvn_ctx *ctx, const uint8_t *imgs_dev, const int32_t *inst_dev, const int32_t *type_dev, int B,
                       int H, int W, int64_t *counts_dev, double *hv_sse_dev, int32_t *flags_dev, double *sums_dev,
                       float *probs_dev);

/* ---- per-instance measurements (an extension; the reference has no such output): for every instance-table row, the
 * HVN_FEAT_LEN columns below, in float64.  Layout of hvn_infer_tiles: n_maps >= 1 maps of any sizes back to back,
 * shapes [n_maps][2] = (H, W) a host array in both variants; inst int32 [H_i,W_i]; img u8 [H_i,W_i,3] RGB or NULL;
 * pred float32 [H_i,W_i,C] or NULL, its NP probability at channel C - 3 (C >= 3); table [n_rows,10] with the rows of
 * map m at [row_offs[m], row_offs[m+1]); the contour of row r at pts[pt_offs[r] : pt_offs[r+1]] ((x, y) int32 in map
 * coordinates, as hvn_contours / hvn_infer_tiles write it; pts holds pt_offs[n_rows] points, the host variant stages
 * that many); feats [n_rows,HVN_FEAT_LEN].  n_rows is a host argument
 * equal to row_offs[n_maps] (0 is allowed: nothing is written).  A one-map hvn_postproc_contours result is this layout
 * with row_offs = {0, n}, pt_offs = offs.  With A the pixels of inst == id in the row's bbox, x, y relative to
 * (cmin, rmin), P the row's points:
 *   AREA A;  CONTOUR_AREA cv2.contourArea(P);  PERIMETER cv2.arcLength(P, closed) (fp32 segment lengths, fp64 sum in
 *   point order from the closing segment);  CONVEX_AREA cv2.contourArea(cv2.convexHull(P));  SOLIDITY contour_area /
 *   convex_area;  CIRCULARITY 4 pi contour_area / perimeter^2;  MAJOR/MINOR_AXIS_LENGTH 4 sqrt(l1), 4 sqrt(l2),
 *   ECCENTRICITY sqrt(1 - l2 / l1), ORIENTATION 0.5 atan2(2b, a - c) (radians from the x axis, y down), with a, b, c
 *   = mu20, mu11, mu02 of cv2.moments(crop == id, binaryImage) over A, r = sqrt(((a - c) / 2)^2 + b^2), l1 =
 *   (a + c) / 2 + r, l2 = max((a + c) / 2 - r, 0);  FERET_MAX the largest distance between two points of P;
 *   MEAN_R/G/B S_c / A and STD_R/G/B sqrt((A Q_c - S_c^2) / A^2) (population std; S_c, Q_c the exact sums of the
 *   channel and of its squares, the numerator exact and rounded once);  NP_PROB_MEAN the fp64 mean of the NP values.
 * A zero denominator gives 0.0; columns 11-16 are NaN without img, column 17 NaN without pred.  Columns 0-16 are
 * bit-exact (ORIENTATION within 4 ulp); NP_PROB_MEAN's sum has a fixed order, so repeated calls are bit-identical.
 * HVN_ERR_INVALID on a bad shape, C < 3 with pred, row_offs not rising from 0 to n_rows, falling pt_offs, a bbox
 * outside its map or empty, or a point outside its row's bbox.  Device workspace (context-owned, grow-only): 16 B per
 * map, and 24 B per contour point of the call when a row has more than 512 points (rows up to 512 points are hulled in
 * shared memory).  Both variants synchronise the context stream once, after the argument check, to report the status;
 * the _dev variant's measurements are then stream-ordered on the context stream (hvn_sync waits for them).  Option
 * "profile" = 1 reports the call's device time as stage "features"; the kernels count towards "pp_launches". */
int hvn_inst_features(hvn_ctx *ctx, int n_maps, const int32_t *shapes, const int32_t *inst_host, const uint8_t *img_host,
                      const float *pred_host, int C, const int64_t *table_host, const int32_t *row_offs_host,
                      int64_t n_rows, const int32_t *pts_host, const int32_t *pt_offs_host, double *feats_host);
int hvn_inst_features_dev(hvn_ctx *ctx, int n_maps, const int32_t *shapes, const int32_t *inst_dev, const uint8_t *img_dev,
                          const float *pred_dev, int C, const int64_t *table_dev, const int32_t *row_offs_dev,
                          int64_t n_rows, const int32_t *pts_dev, const int32_t *pt_offs_dev, double *feats_dev);

/* ---- device memory / stream helpers for callers without a CUDA binding of their own. */
int hvn_malloc(hvn_ctx *ctx, size_t bytes, void **dev_ptr);
int hvn_free(hvn_ctx *ctx, void *dev_ptr);
int hvn_malloc_host(hvn_ctx *ctx, size_t bytes, void **host_ptr); /* pinned */
int hvn_free_host(hvn_ctx *ctx, void *host_ptr);
int hvn_memcpy_h2d(hvn_ctx *ctx, void *dst_dev, const void *src_host, size_t bytes);
int hvn_memcpy_d2h(hvn_ctx *ctx, void *dst_host, const void *src_dev, size_t bytes);
int hvn_sync(hvn_ctx *ctx);
/* cudaMemGetInfo on the context's device: free and total bytes (e.g. to size a tile group). */
int hvn_mem_info(hvn_ctx *ctx, size_t *free_bytes, size_t *total_bytes);
/* CUDA-event timing on the context stream (the stream every kernel of this library is launched
 * on): hvn_timer_start .. hvn_timer_stop returns elapsed milliseconds. */
int hvn_timer_start(hvn_ctx *ctx);
int hvn_timer_stop(hvn_ctx *ctx, float *ms);
/* device time (ms) of the last forward / postproc call.  option "profile" = 1: name in
 * {"cnn","postproc","loss","features"} (whole stage, CUDA events on the context stream; "loss": the reduction of the
 * last hvn_valid_loss* call; "features": the last hvn_inst_features* call).  "profile" = 2 additionally
 * brackets every CNN launch with its own event pair and sums per kernel class:
 * {"conv_tc","conv_ref","conv0","bnrelu","head","tta"} ("tta": the view and merge kernels of option "tta"). */
int hvn_stage_ms(const hvn_ctx *ctx, const char *name, float *ms);

#ifdef __cplusplus
}
#endif
#endif /* HVN_H_ */
