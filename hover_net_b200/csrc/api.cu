// C ABI of libhvn (include/hvn.h).  Thin: argument checks, host<->device staging, error mapping.
#include <cstring>
#include <memory>
#include <string>

#include "../../include/hvn.h"
#include "cnn.h"
#include "postproc.h"
#include "stats.h"
#include "tile.h"

using namespace hvn;

static thread_local std::string g_err;

struct hvn_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    std::unique_ptr<Model> model;  // null for post-processing-only contexts
    Arena pp_arena;                // post-processing workspace
    Arena io_arena;                // staging for the host-pointer entry points
    Arena tile_arena;              // patch / output batches of the tile path
    Arena stats_arena;             // pair-table workspace of hvn_inst_pairs*
    int chunk = 0;
    int profile = 0;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t tev[2] = {nullptr, nullptr};
    float ms_cnn = 0.f, ms_pp = 0.f;
    long long pp_launches = 0;
    std::string pp_log;  // per-kernel post-processing times of the last call ("profile" >= 3)
    std::string log_out;
};

#define API_BEGIN try {
#define API_END                                                     \
    }                                                               \
    catch (const hvn::Error &e) { g_err = e.what(); return e.code; } \
    catch (const std::exception &e) { g_err = e.what(); return HVN_ERR_INVALID; } \
    return HVN_OK;

// After the context stream has been synchronised: a raised range flag becomes HVN_ERR_RANGE (once), never a silently
// clamped result.
static void check_range(hvn_ctx *c) {
    if (c->model && c->model->range_overflow()) {
        c->model->reset_range_flag(c->stream);
        throw Error(HVN_ERR_RANGE, "an activation exceeded the fp16-split range (|x| > 65504 * 2^act_shift, act_shift = " +
                                       std::to_string(c->model->act_shift) + "); set option \"act_shift\" higher and run again");
    }
}

static void use(hvn_ctx *c) {
    HVN_CHECK(c != nullptr, HVN_ERR_INVALID, "null context");
    HVN_CUDA(cudaSetDevice(c->device));
}

extern "C" {

int hvn_abi_version(void) { return HVN_ABI_VERSION; }
const char *hvn_last_error(void) { return g_err.c_str(); }

static int create_common(int device, hvn_ctx **out, const char *mode, int nr_types, bool with_model) {
    API_BEGIN
    HVN_CHECK(out != nullptr, HVN_ERR_INVALID, "null out pointer");
    int ndev = 0;
    HVN_CUDA(cudaGetDeviceCount(&ndev));
    HVN_CHECK(device >= 0 && device < ndev, HVN_ERR_INVALID, "no such CUDA device " + std::to_string(device));
    std::unique_ptr<hvn_ctx> c(new hvn_ctx());
    c->device = device;
    HVN_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    HVN_CUDA(cudaGetDeviceProperties(&prop, device));
    HVN_CHECK(prop.major == 9 && prop.minor == 0, HVN_ERR_CUDA,
              std::string("libhvn is built for sm_90a only; device is ") + prop.name);
    if (with_model) c->model.reset(new Model(mode ? mode : "", nr_types));
    HVN_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    for (auto &e : c->ev) HVN_CUDA(cudaEventCreate(&e));
    for (auto &e : c->tev) HVN_CUDA(cudaEventCreate(&e));
    *out = c.release();
    API_END
}
int hvn_create(int device, const char *mode, int nr_types, hvn_ctx **out) {
    return create_common(device, out, mode, nr_types, true);
}
int hvn_create_postproc(int device, hvn_ctx **out) { return create_common(device, out, nullptr, 0, false); }

void hvn_destroy(hvn_ctx *c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    c->model.reset();
    c->pp_arena.release();
    c->io_arena.release();
    c->tile_arena.release();
    c->stats_arena.release();
    for (auto &e : c->ev) cudaEventDestroy(e);
    for (auto &e : c->tev) cudaEventDestroy(e);
    cudaStreamDestroy(c->stream);
    delete c;
}

int hvn_num_params(const hvn_ctx *c) { return (c && c->model) ? (int)c->model->spec.size() : 0; }

int hvn_param_info(const hvn_ctx *c, int index, const char **name, int *ndim, int64_t shape[4]) {
    API_BEGIN
    HVN_CHECK(c && c->model, HVN_ERR_STATE, "context has no model");
    HVN_CHECK(index >= 0 && index < (int)c->model->spec.size(), HVN_ERR_INVALID, "param index out of range");
    const ParamSpec &s = c->model->spec[index];
    if (name) *name = s.name.c_str();
    if (ndim) *ndim = s.ndim;
    if (shape) for (int i = 0; i < 4; ++i) shape[i] = s.shape[i];
    API_END
}

int hvn_load_param(hvn_ctx *c, const char *name, const float *data, int ndim, const int64_t *shape) {
    API_BEGIN
    use(c);
    HVN_CHECK(c->model, HVN_ERR_STATE, "context has no model");
    HVN_CHECK(name != nullptr, HVN_ERR_INVALID, "null name");
    c->model->load(name, data, ndim, shape);
    API_END
}

int hvn_finalize_weights(hvn_ctx *c) {
    API_BEGIN
    use(c);
    HVN_CHECK(c->model, HVN_ERR_STATE, "context has no model");
    c->model->finalize();
    API_END
}

int hvn_set_option(hvn_ctx *c, const char *key, int64_t value) {
    API_BEGIN
    use(c);
    std::string k = key ? key : "";
    if (k == "conv_path") { HVN_CHECK(c->model, HVN_ERR_STATE, "context has no model"); c->model->conv_path = (int)value; }
    else if (k == "chunk") c->chunk = (int)value;
    else if (k == "flood_impl") postproc_set_flood_impl((int)value);
    else if (k == "fuse_up2") { HVN_CHECK(c->model, HVN_ERR_STATE, "context has no model"); c->model->fuse_up2 = (int)value; }
    else if (k == "fuse_shortcut") { HVN_CHECK(c->model, HVN_ERR_STATE, "context has no model"); c->model->fuse_shortcut = (int)value; }
    else if (k == "stem_tc") { HVN_CHECK(c->model, HVN_ERR_STATE, "context has no model"); c->model->stem_tc = (int)value; }
    else if (k == "xform") { HVN_CHECK(c->model, HVN_ERR_STATE, "context has no model"); c->model->xform = (int)value; }
    else if (k == "branch_streams") { HVN_CHECK(c->model, HVN_ERR_STATE, "context has no model"); c->model->branch_streams = (int)value; }
    else if (k == "tc_seg_chunks") tc_set_seg_chunks((int)value);
    else if (k == "tc_block_n") tc_set_block_n((int)value);
    else if (k == "tc_xf_trunc") tc_set_xf_trunc((int)value);
    else if (k == "tc_prefetch") tc_set_prefetch((int)value);
    else if (k == "act_shift") {
        HVN_CHECK(c->model, HVN_ERR_STATE, "context has no model");
        HVN_CHECK(value >= 0 && value <= 48, HVN_ERR_INVALID, "act_shift out of range (0..48)");
        if (c->model->act_shift != (int)value) {
            HVN_CUDA(cudaStreamSynchronize(c->stream));
            c->model->act_shift = (int)value;
            if (c->model->finalized) c->model->finalize();  // re-derives the BN shifts / head weights; plans are rebuilt
        }
    }
    else if (k == "profile") { c->profile = (int)value; if (c->model) c->model->profile_ops = value >= 3 ? 2 : (value >= 2 ? 1 : 0); }
    else throw Error(HVN_ERR_INVALID, "unknown option " + k);
    API_END
}

int64_t hvn_get_counter(const hvn_ctx *c, const char *key) {
    if (!c || !key) return -1;
    std::string k = key;
    if (k == "act_shift") return c->model ? c->model->act_shift : 0;
    if (k == "kernel_launches") return (c->model ? c->model->kernel_launches : 0) + c->pp_launches;
    if (k == "tc_launches") return c->model ? c->model->tc_launches : 0;
    if (k == "pp_launches") return c->pp_launches;
    if (c->model) {
        if (k == "last_flops") return (int64_t)c->model->last_flops;
        if (k.rfind("launches:", 0) == 0) { auto it = c->model->class_launches.find(k.substr(9)); return it == c->model->class_launches.end() ? 0 : it->second; }
        if (k.rfind("flops:", 0) == 0) { auto it = c->model->class_flops.find(k.substr(6)); return it == c->model->class_flops.end() ? 0 : (int64_t)it->second; }
    }
    return -1;
}

const char *hvn_debug_log(const hvn_ctx *c) {
    if (!c) return "";
    hvn_ctx *m = const_cast<hvn_ctx *>(c);
    m->log_out = (c->model ? c->model->debug_log : std::string()) + c->pp_log;
    return m->log_out.c_str();
}

int hvn_out_shape(const hvn_ctx *c, int in_h, int in_w, int *out_h, int *out_w, int *out_c) {
    API_BEGIN
    HVN_CHECK(c && c->model, HVN_ERR_STATE, "context has no model");
    int oh, ow, oc;
    c->model->out_shape(in_h, in_w, oh, ow, oc);
    if (out_h) *out_h = oh;
    if (out_w) *out_w = ow;
    if (out_c) *out_c = oc;
    API_END
}

// ---------------------------------------------------------------------------------------------------
static void run_forward(hvn_ctx *c, const uint8_t *imgs, int B, int H, int W, float *out) {
    HVN_CHECK(c->model, HVN_ERR_STATE, "context has no model");
    if (c->profile) HVN_CUDA(cudaEventRecord(c->ev[0], c->stream));
    c->model->forward(imgs, B, H, W, out, c->chunk, c->stream);
    if (c->profile) HVN_CUDA(cudaEventRecord(c->ev[1], c->stream));
}
static void run_postproc(hvn_ctx *c, const float *pred, int n, int H, int W, int C, int nr_types, int32_t *inst,
                         int64_t *table, int max_rows, int32_t *n_rows) {
    HVN_CHECK(max_rows >= 1, HVN_ERR_INVALID, "max_rows must be >= 1");
    HVN_CHECK(nr_types >= 0 && nr_types <= HVN_MAX_TYPES, HVN_ERR_INVALID, "nr_types out of range");
    if (c->profile) HVN_CUDA(cudaEventRecord(c->ev[2], c->stream));
    c->pp_launches += postproc_run(c->pp_arena, c->stream, pred, n, H, W, C, nr_types, inst, (long long *)table,
                                   max_rows, n_rows, c->profile >= 3 ? &c->pp_log : nullptr);
    if (c->profile) HVN_CUDA(cudaEventRecord(c->ev[3], c->stream));
}
static void finish_profile(hvn_ctx *c, bool cnn, bool pp) {
    if (!c->profile) return;
    HVN_CUDA(cudaStreamSynchronize(c->stream));
    if (cnn) HVN_CUDA(cudaEventElapsedTime(&c->ms_cnn, c->ev[0], c->ev[1]));
    if (pp) HVN_CUDA(cudaEventElapsedTime(&c->ms_pp, c->ev[2], c->ev[3]));
}
static void check_rows(const int32_t *n_rows, int n, int max_rows) {
    for (int i = 0; i < n; ++i)
        HVN_CHECK(n_rows[i] <= max_rows, HVN_ERR_CAPACITY,
                  "instance table too small: map " + std::to_string(i) + " has " + std::to_string(n_rows[i]) +
                      " instances, max_rows=" + std::to_string(max_rows));
}

int hvn_forward_dev(hvn_ctx *c, const uint8_t *imgs, int B, int H, int W, float *out) {
    API_BEGIN
    use(c);
    HVN_CHECK(imgs && out, HVN_ERR_INVALID, "null buffer");
    run_forward(c, imgs, B, H, W, out);
    finish_profile(c, true, false);
    API_END
}

int hvn_forward(hvn_ctx *c, const uint8_t *imgs, int B, int H, int W, float *out) {
    API_BEGIN
    use(c);
    HVN_CHECK(imgs && out, HVN_ERR_INVALID, "null buffer");
    HVN_CHECK(c->model, HVN_ERR_STATE, "context has no model");
    int oh, ow, oc;
    c->model->out_shape(H, W, oh, ow, oc);
    size_t in_b = (size_t)B * H * W * 3, out_b = (size_t)B * oh * ow * oc * sizeof(float);
    c->io_arena.reset();
    c->io_arena.reserve(in_b + out_b + 1024);
    uint8_t *d_in = c->io_arena.take<uint8_t>(in_b);
    float *d_out = c->io_arena.take<float>(out_b / sizeof(float));
    HVN_CUDA(cudaMemcpyAsync(d_in, imgs, in_b, cudaMemcpyHostToDevice, c->stream));
    run_forward(c, d_in, B, H, W, d_out);
    HVN_CUDA(cudaMemcpyAsync(out, d_out, out_b, cudaMemcpyDeviceToHost, c->stream));
    HVN_CUDA(cudaStreamSynchronize(c->stream));
    finish_profile(c, true, false);
    check_range(c);
    API_END
}

int hvn_postproc_dev(hvn_ctx *c, const float *pred, int n, int H, int W, int C, int nr_types, int32_t *inst,
                     int64_t *table, int max_rows, int32_t *n_rows) {
    API_BEGIN
    use(c);
    HVN_CHECK(pred && inst && table && n_rows, HVN_ERR_INVALID, "null buffer");
    run_postproc(c, pred, n, H, W, C, nr_types, inst, table, max_rows, n_rows);
    finish_profile(c, false, true);
    API_END
}

int hvn_postproc(hvn_ctx *c, const float *pred, int n, int H, int W, int C, int nr_types, int32_t *inst,
                 int64_t *table, int max_rows, int32_t *n_rows) {
    API_BEGIN
    use(c);
    HVN_CHECK(pred && inst && table && n_rows, HVN_ERR_INVALID, "null buffer");
    HVN_CHECK(n >= 1 && H >= 1 && W >= 1, HVN_ERR_INVALID, "empty input");
    size_t px = (size_t)n * H * W;
    size_t tb = (size_t)n * max_rows * HVN_ROW_LEN;
    c->io_arena.reset();
    c->io_arena.reserve(px * C * 4 + px * 4 + tb * 8 + (size_t)n * 4 + 4096);
    float *d_pred = c->io_arena.take<float>(px * C);
    int32_t *d_inst = c->io_arena.take<int32_t>(px);
    int64_t *d_tab = c->io_arena.take<int64_t>(tb);
    HVN_CUDA(cudaMemsetAsync(d_tab, 0, tb * 8, c->stream));  // rows past n_rows go back to the caller as zeros
    int32_t *d_nr = c->io_arena.take<int32_t>(n);
    HVN_CUDA(cudaMemcpyAsync(d_pred, pred, px * C * 4, cudaMemcpyHostToDevice, c->stream));
    run_postproc(c, d_pred, n, H, W, C, nr_types, d_inst, d_tab, max_rows, d_nr);
    HVN_CUDA(cudaMemcpyAsync(inst, d_inst, px * 4, cudaMemcpyDeviceToHost, c->stream));
    HVN_CUDA(cudaMemcpyAsync(n_rows, d_nr, (size_t)n * 4, cudaMemcpyDeviceToHost, c->stream));
    HVN_CUDA(cudaMemcpyAsync(table, d_tab, tb * 8, cudaMemcpyDeviceToHost, c->stream));
    HVN_CUDA(cudaStreamSynchronize(c->stream));
    finish_profile(c, false, true);
    check_rows(n_rows, n, max_rows);
    API_END
}

int hvn_contours_dev(hvn_ctx *c, const int32_t *inst, const int64_t *table, const int32_t *n_rows, int n, int H, int W,
                     int max_rows, int32_t *pts, int64_t cap, int32_t *offs) {
    API_BEGIN
    use(c);
    HVN_CHECK(inst && table && n_rows && offs && (pts || cap == 0), HVN_ERR_INVALID, "null buffer");
    HVN_CHECK(n >= 1 && H >= 1 && W >= 1 && max_rows >= 1 && cap >= 0, HVN_ERR_INVALID, "bad shape");
    HVN_CHECK((long long)n * max_rows < (1ll << 31), HVN_ERR_INVALID, "too many table rows");
    c->pp_launches += contours_run(c->stream, inst, (const long long *)table, n_rows, n, H, W, max_rows, pts, cap, offs);
    API_END
}

int hvn_postproc_contours(hvn_ctx *c, const float *pred, int n, int H, int W, int C, int nr_types, int32_t *inst,
                          int64_t *table, int max_rows, int32_t *n_rows, int32_t *pts, int64_t cap, int32_t *offs) {
    API_BEGIN
    use(c);
    HVN_CHECK(pred && inst && table && n_rows && offs && (pts || cap == 0), HVN_ERR_INVALID, "null buffer");
    HVN_CHECK(n >= 1 && H >= 1 && W >= 1 && cap >= 0, HVN_ERR_INVALID, "empty input");
    HVN_CHECK((long long)n * max_rows < (1ll << 31), HVN_ERR_INVALID, "too many table rows");
    size_t px = (size_t)n * H * W;
    size_t tb = (size_t)n * max_rows * HVN_ROW_LEN;
    size_t no = (size_t)n * max_rows + 1;
    c->io_arena.reset();
    c->io_arena.reserve(px * C * 4 + px * 4 + tb * 8 + (size_t)n * 4 + no * 4 + (size_t)cap * 8 + 8192);
    float *d_pred = c->io_arena.take<float>(px * C);
    int32_t *d_inst = c->io_arena.take<int32_t>(px);
    int64_t *d_tab = c->io_arena.take<int64_t>(tb);
    HVN_CUDA(cudaMemsetAsync(d_tab, 0, tb * 8, c->stream));  // rows past n_rows go back to the caller as zeros
    int32_t *d_nr = c->io_arena.take<int32_t>(n);
    int32_t *d_offs = c->io_arena.take<int32_t>(no);
    int32_t *d_pts = c->io_arena.take<int32_t>((size_t)cap * 2 + 2);
    HVN_CUDA(cudaMemcpyAsync(d_pred, pred, px * C * 4, cudaMemcpyHostToDevice, c->stream));
    run_postproc(c, d_pred, n, H, W, C, nr_types, d_inst, d_tab, max_rows, d_nr);
    c->pp_launches += contours_run(c->stream, d_inst, (const long long *)d_tab, d_nr, n, H, W, max_rows, d_pts, cap, d_offs);
    HVN_CUDA(cudaMemcpyAsync(inst, d_inst, px * 4, cudaMemcpyDeviceToHost, c->stream));
    HVN_CUDA(cudaMemcpyAsync(n_rows, d_nr, (size_t)n * 4, cudaMemcpyDeviceToHost, c->stream));
    HVN_CUDA(cudaMemcpyAsync(table, d_tab, tb * 8, cudaMemcpyDeviceToHost, c->stream));
    HVN_CUDA(cudaMemcpyAsync(offs, d_offs, no * 4, cudaMemcpyDeviceToHost, c->stream));
    HVN_CUDA(cudaStreamSynchronize(c->stream));
    finish_profile(c, false, true);
    check_rows(n_rows, n, max_rows);
    const long long total = offs[no - 1];
    HVN_CHECK(total <= cap, HVN_ERR_CAPACITY, "contour buffer too small: " + std::to_string(total) + " points, pts_cap=" + std::to_string(cap));
    if (total > 0) {
        HVN_CUDA(cudaMemcpyAsync(pts, d_pts, (size_t)total * 8, cudaMemcpyDeviceToHost, c->stream));
        HVN_CUDA(cudaStreamSynchronize(c->stream));
    }
    API_END
}

int hvn_forward_postproc_dev(hvn_ctx *c, const uint8_t *imgs, int B, int H, int W, float *pred, int32_t *inst,
                             int64_t *table, int max_rows, int32_t *n_rows) {
    API_BEGIN
    use(c);
    HVN_CHECK(imgs && inst && table && n_rows, HVN_ERR_INVALID, "null buffer");
    HVN_CHECK(c->model, HVN_ERR_STATE, "context has no model");
    int oh, ow, oc;
    c->model->out_shape(H, W, oh, ow, oc);
    float *d_pred = pred;
    if (!d_pred) {
        c->io_arena.reset();
        c->io_arena.reserve((size_t)B * oh * ow * oc * 4 + 1024);
        d_pred = c->io_arena.take<float>((size_t)B * oh * ow * oc);
    }
    run_forward(c, imgs, B, H, W, d_pred);
    run_postproc(c, d_pred, B, oh, ow, oc, c->model->nr_types, inst, table, max_rows, n_rows);
    finish_profile(c, true, true);
    API_END
}

int hvn_forward_postproc(hvn_ctx *c, const uint8_t *imgs, int B, int H, int W, float *pred, int32_t *inst,
                         int64_t *table, int max_rows, int32_t *n_rows) {
    API_BEGIN
    use(c);
    HVN_CHECK(imgs && inst && table && n_rows, HVN_ERR_INVALID, "null buffer");
    HVN_CHECK(c->model, HVN_ERR_STATE, "context has no model");
    int oh, ow, oc;
    c->model->out_shape(H, W, oh, ow, oc);
    size_t in_b = (size_t)B * H * W * 3, px = (size_t)B * oh * ow, tb = (size_t)B * max_rows * HVN_ROW_LEN;
    c->io_arena.reset();
    c->io_arena.reserve(in_b + px * oc * 4 + px * 4 + tb * 8 + (size_t)B * 4 + 8192);
    uint8_t *d_in = c->io_arena.take<uint8_t>(in_b);
    float *d_pred = c->io_arena.take<float>(px * oc);
    int32_t *d_inst = c->io_arena.take<int32_t>(px);
    int64_t *d_tab = c->io_arena.take<int64_t>(tb);
    HVN_CUDA(cudaMemsetAsync(d_tab, 0, tb * 8, c->stream));  // rows past n_rows go back to the caller as zeros
    int32_t *d_nr = c->io_arena.take<int32_t>(B);
    HVN_CUDA(cudaMemcpyAsync(d_in, imgs, in_b, cudaMemcpyHostToDevice, c->stream));
    run_forward(c, d_in, B, H, W, d_pred);
    run_postproc(c, d_pred, B, oh, ow, oc, c->model->nr_types, d_inst, d_tab, max_rows, d_nr);
    if (pred) HVN_CUDA(cudaMemcpyAsync(pred, d_pred, px * oc * 4, cudaMemcpyDeviceToHost, c->stream));
    HVN_CUDA(cudaMemcpyAsync(inst, d_inst, px * 4, cudaMemcpyDeviceToHost, c->stream));
    HVN_CUDA(cudaMemcpyAsync(n_rows, d_nr, (size_t)B * 4, cudaMemcpyDeviceToHost, c->stream));
    HVN_CUDA(cudaMemcpyAsync(table, d_tab, tb * 8, cudaMemcpyDeviceToHost, c->stream));
    HVN_CUDA(cudaStreamSynchronize(c->stream));
    finish_profile(c, true, true);
    check_range(c);
    check_rows(n_rows, B, max_rows);
    API_END
}

// ---------------------------------------------------------------------------------------------------
int hvn_tile_grid(const hvn_ctx *c, int H, int W, int patch_in, int *rows, int *cols) {
    API_BEGIN
    HVN_CHECK(c && c->model, HVN_ERR_STATE, "context has no model");
    HVN_CHECK(H >= 1 && W >= 1 && rows && cols, HVN_ERR_INVALID, "bad argument");
    int oh, ow, oc;
    c->model->out_shape(patch_in, patch_in, oh, ow, oc);
    tile_grid(H, W, oh, rows, cols);
    API_END
}

static int run_tile_predict(hvn_ctx *c, const uint8_t *img, int H, int W, int patch_in, int lo, int hi, int batch, float *pred) {
    int oh, ow, oc;
    c->model->out_shape(patch_in, patch_in, oh, ow, oc);
    if (batch < 1) batch = 64;
    c->tile_arena.reset();
    c->tile_arena.reserve(tile_workspace_bytes(patch_in, oh, oc, batch) + 1024);
    return tile_predict(*c->model, c->tile_arena, c->stream, img, H, W, patch_in, lo, hi, batch, c->chunk, pred);
}

int hvn_tile_predict_dev(hvn_ctx *c, const uint8_t *img, int H, int W, int patch_in, int cell_lo, int cell_hi, int batch,
                         float *pred) {
    API_BEGIN
    use(c);
    HVN_CHECK(c->model, HVN_ERR_STATE, "context has no model");
    HVN_CHECK(img && pred && H >= 1 && W >= 1, HVN_ERR_INVALID, "bad argument");
    if (c->profile) HVN_CUDA(cudaEventRecord(c->ev[0], c->stream));
    c->model->kernel_launches += run_tile_predict(c, img, H, W, patch_in, cell_lo, cell_hi, batch, pred);
    if (c->profile) HVN_CUDA(cudaEventRecord(c->ev[1], c->stream));
    finish_profile(c, true, false);
    API_END
}

int hvn_infer_tile(hvn_ctx *c, const uint8_t *img, int H, int W, int patch_in, int batch, float *pred, int32_t *inst,
                   int64_t *table, int max_rows, int32_t *n_rows, int32_t *pts, int64_t cap, int32_t *offs) {
    API_BEGIN
    use(c);
    HVN_CHECK(c->model, HVN_ERR_STATE, "context has no model");
    HVN_CHECK(img && inst && table && n_rows && H >= 1 && W >= 1 && max_rows >= 1, HVN_ERR_INVALID, "bad argument");
    HVN_CHECK(!offs || pts || cap == 0, HVN_ERR_INVALID, "contours requested without a point buffer");
    int oh, ow, oc, rows, cols;
    c->model->out_shape(patch_in, patch_in, oh, ow, oc);
    tile_grid(H, W, oh, &rows, &cols);
    const size_t px = (size_t)H * W, tb = (size_t)max_rows * HVN_ROW_LEN, no = (size_t)max_rows + 1;
    if (!offs) cap = 0;
    c->io_arena.reset();
    c->io_arena.reserve(px * 3 + px * oc * 4 + px * 4 + tb * 8 + no * 4 + (size_t)cap * 8 + 16384);
    uint8_t *d_img = c->io_arena.take<uint8_t>(px * 3);
    float *d_pred = c->io_arena.take<float>(px * oc);
    int32_t *d_inst = c->io_arena.take<int32_t>(px);
    int64_t *d_tab = c->io_arena.take<int64_t>(tb);
    HVN_CUDA(cudaMemsetAsync(d_tab, 0, tb * 8, c->stream));  // rows past n_rows go back to the caller as zeros
    int32_t *d_nr = c->io_arena.take<int32_t>(1);
    int32_t *d_offs = c->io_arena.take<int32_t>(no);
    int32_t *d_pts = c->io_arena.take<int32_t>((size_t)cap * 2 + 2);
    HVN_CUDA(cudaMemcpyAsync(d_img, img, px * 3, cudaMemcpyHostToDevice, c->stream));
    if (c->profile) HVN_CUDA(cudaEventRecord(c->ev[0], c->stream));
    c->model->kernel_launches += run_tile_predict(c, d_img, H, W, patch_in, 0, rows * cols, batch, d_pred);
    if (c->profile) HVN_CUDA(cudaEventRecord(c->ev[1], c->stream));
    run_postproc(c, d_pred, 1, H, W, oc, c->model->nr_types, d_inst, d_tab, max_rows, d_nr);
    if (offs) c->pp_launches += contours_run(c->stream, d_inst, (const long long *)d_tab, d_nr, 1, H, W, max_rows, d_pts, cap, d_offs);
    if (pred) HVN_CUDA(cudaMemcpyAsync(pred, d_pred, px * oc * 4, cudaMemcpyDeviceToHost, c->stream));
    HVN_CUDA(cudaMemcpyAsync(inst, d_inst, px * 4, cudaMemcpyDeviceToHost, c->stream));
    HVN_CUDA(cudaMemcpyAsync(n_rows, d_nr, 4, cudaMemcpyDeviceToHost, c->stream));
    HVN_CUDA(cudaMemcpyAsync(table, d_tab, tb * 8, cudaMemcpyDeviceToHost, c->stream));
    if (offs) HVN_CUDA(cudaMemcpyAsync(offs, d_offs, no * 4, cudaMemcpyDeviceToHost, c->stream));
    HVN_CUDA(cudaStreamSynchronize(c->stream));
    finish_profile(c, true, true);
    check_range(c);
    check_rows(n_rows, 1, max_rows);
    if (offs) {
        const long long total = offs[no - 1];
        HVN_CHECK(total <= cap, HVN_ERR_CAPACITY, "contour buffer too small: " + std::to_string(total) + " points, pts_cap=" + std::to_string(cap));
        if (total > 0) {
            HVN_CUDA(cudaMemcpyAsync(pts, d_pts, (size_t)total * 8, cudaMemcpyDeviceToHost, c->stream));
            HVN_CUDA(cudaStreamSynchronize(c->stream));
        }
    }
    API_END
}

// ---------------------------------------------------------------------------------------------------
static void check_pairs_args(const int32_t *tru, const int64_t *pairs, int64_t cap, const int64_t *offs, int n, int H,
                             int W) {
    HVN_CHECK(tru && offs && (pairs || cap == 0), HVN_ERR_INVALID, "null buffer");
    HVN_CHECK(n >= 1 && n <= 65535 && H >= 1 && W >= 1 && cap >= 0, HVN_ERR_INVALID, "bad shape");
    HVN_CHECK((long long)H * W <= 0x7fffffffll, HVN_ERR_INVALID, "map larger than 2^31 - 1 pixels");
}
static void check_pairs_result(int err, long long total, int64_t cap) {
    HVN_CHECK(!err, HVN_ERR_INVALID, "negative instance id");
    HVN_CHECK(total <= cap, HVN_ERR_CAPACITY,
              "pair table too small: " + std::to_string(total) + " pairs, cap=" + std::to_string(cap));
}

int hvn_inst_pairs_dev(hvn_ctx *c, const int32_t *tru, const int32_t *pred, int n, int H, int W, int64_t *pairs,
                       int64_t cap, int64_t *offs) {
    API_BEGIN
    use(c);
    check_pairs_args(tru, pairs, cap, offs, n, H, W);
    PairWork w;
    inst_pairs_count(c->stats_arena, c->stream, tru, pred, n, H, W, (long long *)offs, w);
    inst_pairs_emit(c->stream, w, (long long *)pairs, cap);
    int err = 0;
    long long total = 0;
    HVN_CUDA(cudaMemcpyAsync(&err, w.err, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    HVN_CUDA(cudaMemcpyAsync(&total, offs + n, sizeof(long long), cudaMemcpyDeviceToHost, c->stream));
    HVN_CUDA(cudaStreamSynchronize(c->stream));
    check_pairs_result(err, total, cap);
    API_END
}

int hvn_inst_pairs(hvn_ctx *c, const int32_t *tru, const int32_t *pred, int n, int H, int W, int64_t *pairs,
                   int64_t cap, int64_t *offs) {
    API_BEGIN
    use(c);
    check_pairs_args(tru, pairs, cap, offs, n, H, W);
    const size_t px = (size_t)n * H * W;
    c->io_arena.reset();
    c->io_arena.reserve(px * 4 * (pred ? 2 : 1) + (size_t)(n + 1) * 8 + 4096);
    int32_t *d_t = c->io_arena.take<int32_t>(px);
    int32_t *d_p = pred ? c->io_arena.take<int32_t>(px) : nullptr;
    long long *d_offs = c->io_arena.take<long long>((size_t)n + 1);
    HVN_CUDA(cudaMemcpyAsync(d_t, tru, px * 4, cudaMemcpyHostToDevice, c->stream));
    if (pred) HVN_CUDA(cudaMemcpyAsync(d_p, pred, px * 4, cudaMemcpyHostToDevice, c->stream));
    PairWork w;
    inst_pairs_count(c->stats_arena, c->stream, d_t, d_p, n, H, W, d_offs, w);
    int err = 0;
    HVN_CUDA(cudaMemcpyAsync(&err, w.err, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    HVN_CUDA(cudaMemcpyAsync(offs, d_offs, (size_t)(n + 1) * 8, cudaMemcpyDeviceToHost, c->stream));
    HVN_CUDA(cudaStreamSynchronize(c->stream));
    const long long total = offs[n];
    check_pairs_result(err, total, cap);
    if (total == 0) return HVN_OK;
    // the maps are no longer needed: the staging arena now holds the rows
    c->io_arena.reset();
    c->io_arena.reserve((size_t)total * 24 + (size_t)(n + 1) * 8 + 1024);
    long long *d_pairs = c->io_arena.take<long long>((size_t)total * 3);
    w.offs = c->io_arena.take<long long>((size_t)n + 1);
    HVN_CUDA(cudaMemcpyAsync(w.offs, offs, (size_t)(n + 1) * 8, cudaMemcpyHostToDevice, c->stream));
    inst_pairs_emit(c->stream, w, d_pairs, total);
    HVN_CUDA(cudaMemcpyAsync(pairs, d_pairs, (size_t)total * 24, cudaMemcpyDeviceToHost, c->stream));
    HVN_CUDA(cudaStreamSynchronize(c->stream));
    API_END
}

// ---------------------------------------------------------------------------------------------------
int hvn_malloc(hvn_ctx *c, size_t bytes, void **p) {
    API_BEGIN
    use(c);
    HVN_CHECK(p, HVN_ERR_INVALID, "null out pointer");
    HVN_CUDA(cudaMalloc(p, bytes ? bytes : 1));
    API_END
}
int hvn_free(hvn_ctx *c, void *p) {
    API_BEGIN
    use(c);
    HVN_CUDA(cudaFree(p));
    API_END
}
int hvn_malloc_host(hvn_ctx *c, size_t bytes, void **p) {
    API_BEGIN
    use(c);
    HVN_CHECK(p, HVN_ERR_INVALID, "null out pointer");
    HVN_CUDA(cudaMallocHost(p, bytes ? bytes : 1));
    API_END
}
int hvn_free_host(hvn_ctx *c, void *p) {
    API_BEGIN
    use(c);
    HVN_CUDA(cudaFreeHost(p));
    API_END
}
int hvn_memcpy_h2d(hvn_ctx *c, void *dst, const void *src, size_t bytes) {
    API_BEGIN
    use(c);
    HVN_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, c->stream));
    API_END
}
int hvn_memcpy_d2h(hvn_ctx *c, void *dst, const void *src, size_t bytes) {
    API_BEGIN
    use(c);
    HVN_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, c->stream));
    API_END
}
int hvn_pack_tables_dev(hvn_ctx *c, const int64_t *table, const int32_t *n_rows, int n, int max_rows, int64_t *packed,
                        int64_t cap, int32_t *offs) {
    API_BEGIN
    use(c);
    HVN_CHECK(table && n_rows && packed && offs && n >= 1 && max_rows >= 1 && cap >= 0, HVN_ERR_INVALID, "bad argument");
    c->pp_launches += pack_tables(c->stream, (const long long *)table, n_rows, n, max_rows, (long long *)packed, cap, offs);
    API_END
}
int hvn_get_stream(hvn_ctx *c, void **stream) {
    API_BEGIN
    HVN_CHECK(c && stream, HVN_ERR_INVALID, "null argument");
    *stream = (void *)c->stream;
    API_END
}
int hvn_sync(hvn_ctx *c) {
    API_BEGIN
    use(c);
    HVN_CUDA(cudaStreamSynchronize(c->stream));
    check_range(c);
    API_END
}
int hvn_timer_start(hvn_ctx *c) {
    API_BEGIN
    use(c);
    HVN_CUDA(cudaEventRecord(c->tev[0], c->stream));
    API_END
}
int hvn_timer_stop(hvn_ctx *c, float *ms) {
    API_BEGIN
    use(c);
    HVN_CHECK(ms, HVN_ERR_INVALID, "null out pointer");
    HVN_CUDA(cudaEventRecord(c->tev[1], c->stream));
    HVN_CUDA(cudaEventSynchronize(c->tev[1]));
    HVN_CUDA(cudaEventElapsedTime(ms, c->tev[0], c->tev[1]));
    check_range(c);
    API_END
}
int hvn_stage_ms(const hvn_ctx *c, const char *name, float *ms) {
    API_BEGIN
    HVN_CHECK(c && name && ms, HVN_ERR_INVALID, "null argument");
    std::string k = name;
    if (k == "cnn") *ms = c->ms_cnn;
    else if (k == "postproc") *ms = c->ms_pp;
    else if (c->model && c->model->class_ms.count(k)) *ms = (float)c->model->class_ms.at(k);
    else if (k == "conv_tc" || k == "conv_ref" || k == "conv0" || k == "bnrelu" || k == "head") *ms = 0.f;
    else throw Error(HVN_ERR_INVALID, "unknown stage " + k);
    API_END
}

}  // extern "C"
