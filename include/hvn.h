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
                                 by the call that synchronises: hvn_forward / hvn_forward_postproc / hvn_infer_tile,
                                 or, after *_dev calls, hvn_sync / hvn_timer_stop. */
} hvn_status;

/* Instance-table row: one per instance id present in inst_map, ascending id.  int64 x 10.
 * Replaces the per-instance loop of reference post_proc.py:120-181 (bbox via
 * misc/utils.py:18-28 with exclusive max; centroid = sum/area == cv2.moments m10/m00, m01/m00;
 * type vote :161-181).  type/type_count are -1/0 when nr_types == 0. */
#define HVN_ROW_LEN 10
enum { HVN_ROW_ID = 0, HVN_ROW_RMIN, HVN_ROW_CMIN, HVN_ROW_RMAX, HVN_ROW_CMAX, HVN_ROW_AREA,
       HVN_ROW_SUMX, HVN_ROW_SUMY, HVN_ROW_TYPE, HVN_ROW_TYPECNT };

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
 *                      "profile" = 0 | 1 | 2 (see hvn_stage_ms);
 *                      tuning knobs: "tc_seg_chunks" (64-channel slices per accumulation segment), "tc_block_n",
 *                      "tc_prefetch" (L2 prefetch distance in K-slices for flat operands, 0 = off), "tc_xf_trunc"
 *                      (XF transform: truncating hi/lo split 1, round-to-nearest 0),
 *                      "xform", "fuse_shortcut", "fuse_up2", "branch_streams", "flood_impl".
 *                      The tc_* knobs are process-wide launch-time switches; every setting gives the same results to
 *                      fp32-accumulation noise (tests/test_cnn_gpu.py::test_kernel_variants_agree). */
int hvn_set_option(hvn_ctx *ctx, const char *key, int64_t value);
const char *hvn_debug_log(const hvn_ctx *ctx);
/* counters: "kernel_launches", "tc_launches", "pp_launches" (post-processing and contour kernels), "last_flops" (algorithmic 2*MACs of the
 * last forward); with option "profile" = 2 also "launches:<class>" and "flops:<class>" for
 * class in {conv_tc, conv_ref, conv0, bnrelu, head} (see hvn_stage_ms). */
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

/* ---- device memory / stream helpers for callers without a CUDA binding of their own. */
int hvn_malloc(hvn_ctx *ctx, size_t bytes, void **dev_ptr);
int hvn_free(hvn_ctx *ctx, void *dev_ptr);
int hvn_malloc_host(hvn_ctx *ctx, size_t bytes, void **host_ptr); /* pinned */
int hvn_free_host(hvn_ctx *ctx, void *host_ptr);
int hvn_memcpy_h2d(hvn_ctx *ctx, void *dst_dev, const void *src_host, size_t bytes);
int hvn_memcpy_d2h(hvn_ctx *ctx, void *dst_host, const void *src_dev, size_t bytes);
int hvn_sync(hvn_ctx *ctx);
/* CUDA-event timing on the context stream (the stream every kernel of this library is launched
 * on): hvn_timer_start .. hvn_timer_stop returns elapsed milliseconds. */
int hvn_timer_start(hvn_ctx *ctx);
int hvn_timer_stop(hvn_ctx *ctx, float *ms);
/* device time (ms) of the last forward / postproc call.  option "profile" = 1: name in
 * {"cnn","postproc"} (whole stage, CUDA events on the context stream).  "profile" = 2 additionally
 * brackets every CNN launch with its own event pair and sums per kernel class:
 * {"conv_tc","conv_ref","conv0","bnrelu","head"}. */
int hvn_stage_ms(const hvn_ctx *ctx, const char *name, float *ms);

#ifdef __cplusplus
}
#endif
#endif /* HVN_H_ */
