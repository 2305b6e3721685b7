// C ABI of libhvn (include/hvn.h).  Thin: argument checks, host<->device staging, error mapping.
#include <algorithm>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "../../include/hvn.h"
#include "cnn.h"
#include "features.h"
#include "loss.h"
#include "postproc.h"
#include "stats.h"
#include "targets.h"
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
    Arena targets_arena;           // workspace of hvn_targets* and hvn_valid*
    Arena valid_arena;             // maps and counts of hvn_valid*
    Arena loss_arena;              // per-block partials of hvn_valid_loss*
    Arena group_arena;             // slot table, padded instance tables and slot-order maps of the tile-group path
    Arena feat_arena;              // map table, status and long-contour scratch of hvn_inst_features*
    void *pin = nullptr;           // pinned staging of the tile-group slot table (uploaded stream-ordered)
    size_t pin_bytes = 0;
    cudaEvent_t pin_ev = nullptr;  // recorded after the last upload from `pin`
    long long group_table_rows = 0;  // padded instance-table rows the last tile group took from group_arena
    int chunk = 0;
    int profile = 0;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t tev[2] = {nullptr, nullptr};
    float ms_cnn = 0.f, ms_pp = 0.f, ms_loss = 0.f, ms_feat = 0.f;
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

// The device buffers of one call, taken from one of the context's arenas.  The call's layout declares each buffer once:
// in() is copied from the host as it is declared, out() is copied back to the host by copy_back() (which then
// synchronises the stream), scratch() stays on the device.  The constructor runs the layout over an ArenaSizer first,
// so the arena is reserved for exactly the takes that follow.
class Buffers {
  public:
    template <typename F> Buffers(hvn_ctx *c, Arena &a, F &&layout) : c_(c), a_(a) {
        layout(*this);
        a.reset();
        a.reserve(sizer_.top);
        sizing_ = false;
        layout(*this);
    }
    template <typename T> T *scratch(size_t n) { return sizing_ ? sizer_.take<T>(n) : a_.take<T>(n); }
    template <typename T> T *in(const T *host, size_t n) {
        T *d = scratch<T>(n);
        if (!sizing_) HVN_CUDA(cudaMemcpyAsync(d, host, n * sizeof(T), cudaMemcpyHostToDevice, c_->stream));
        return d;
    }
    // zero: the device buffer is cleared first, so whatever the work leaves unwritten goes back as zeros
    template <typename T> T *out(T *host, size_t n, bool zero = false) {
        T *d = scratch<T>(n);
        if (sizing_) return d;
        if (zero) HVN_CUDA(cudaMemsetAsync(d, 0, n * sizeof(T), c_->stream));
        HVN_CHECK(n_back_ < kMaxOut, HVN_ERR_INVALID, "too many staged outputs");
        back_[n_back_++] = {host, d, n * sizeof(T)};
        return d;
    }
    void copy_back() {
        for (int i = 0; i < n_back_; ++i)
            HVN_CUDA(cudaMemcpyAsync(back_[i].host, back_[i].dev, back_[i].bytes, cudaMemcpyDeviceToHost, c_->stream));
        HVN_CUDA(cudaStreamSynchronize(c_->stream));
    }

  private:
    static constexpr int kMaxOut = 8;
    struct Out { void *host; const void *dev; size_t bytes; };
    hvn_ctx *c_;
    Arena &a_;
    ArenaSizer sizer_;
    bool sizing_ = true;
    Out back_[kMaxOut];
    int n_back_ = 0;
};

// Second phase of a two-phase host call, after the stream has been synchronised: `count` items of `item` bytes are
// ready in dev.  More than `cap` is HVN_ERR_CAPACITY with the exact count; otherwise they are copied to host.  Returns
// whether a copy was enqueued (the caller synchronises).
static bool copy_fitting(hvn_ctx *c, void *host, const void *dev, long long count, long long cap, size_t item,
                         const char *buffer, const char *items, const char *cap_name) {
    HVN_CHECK(count <= cap, HVN_ERR_CAPACITY, std::string(buffer) + " too small: " + std::to_string(count) + " " + items +
                                                  ", " + cap_name + "=" + std::to_string(cap));
    if (count > 0) HVN_CUDA(cudaMemcpyAsync(host, dev, (size_t)count * item, cudaMemcpyDeviceToHost, c->stream));
    return count > 0;
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
    HVN_CUDA(cudaEventCreateWithFlags(&c->pin_ev, cudaEventDisableTiming));
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
    c->targets_arena.release();
    c->valid_arena.release();
    c->loss_arena.release();
    c->group_arena.release();
    c->feat_arena.release();
    if (c->pin) cudaFreeHost(c->pin);
    if (c->pin_ev) cudaEventDestroy(c->pin_ev);
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
    else if (k == "precision") {
        HVN_CHECK(c->model, HVN_ERR_STATE, "context has no model");
        HVN_CHECK(value == 0 || value == 1, HVN_ERR_INVALID, "precision must be 0 (highest) or 1 (high)");
        if (c->model->precision != (int)value) {
            HVN_CUDA(cudaStreamSynchronize(c->stream));
            c->model->precision = (int)value;
            if (c->model->finalized) c->model->finalize();  // weight planes re-derived (lo dropped / restored); plans rebuilt
        }
    }
    else if (k == "tta") {
        HVN_CHECK(c->model, HVN_ERR_STATE, "context has no model");
        HVN_CHECK(value == 0 || value == 1, HVN_ERR_INVALID, "tta must be 0 (off) or 1 (eight dihedral views, merged)");
        if (c->model->tta != (int)value) {
            HVN_CUDA(cudaStreamSynchronize(c->stream));
            c->model->tta = (int)value;
            c->model->drop_plans();  // a context keeps the buffers of one mode only
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
    if (k == "precision") return c->model ? c->model->precision : 0;
    if (k == "tta") return c->model ? c->model->tta : 0;
    if (k == "plan_bytes") return c->model ? (int64_t)c->model->last_plan_bytes : 0;
    if (k == "kernel_launches") return (c->model ? c->model->kernel_launches : 0) + c->pp_launches;
    if (k == "tc_launches") return c->model ? c->model->tc_launches : 0;
    if (k == "pp_launches") return c->pp_launches;
    if (k == "tile_table_rows") return c->group_table_rows;
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
static void run_forward(hvn_ctx *c, const uint8_t *imgs, int B, int H, int W, float *out, int layout = OUT_PLAIN) {
    HVN_CHECK(c->model, HVN_ERR_STATE, "context has no model");
    if (c->profile) HVN_CUDA(cudaEventRecord(c->ev[0], c->stream));
    c->model->forward(imgs, B, H, W, out, c->chunk, c->stream, layout);
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
static void run_forward_postproc(hvn_ctx *c, const uint8_t *imgs, int B, int H, int W, float *pred, int32_t *inst,
                                 int64_t *table, int max_rows, int32_t *n_rows) {
    int oh, ow, oc;
    c->model->out_shape(H, W, oh, ow, oc);
    run_forward(c, imgs, B, H, W, pred);
    run_postproc(c, pred, B, oh, ow, oc, c->model->nr_types, inst, table, max_rows, n_rows);
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
    uint8_t *d_in;
    float *d_out;
    Buffers io(c, c->io_arena, [&](Buffers &s) {
        d_in = s.in(imgs, (size_t)B * H * W * 3);
        d_out = s.out(out, (size_t)B * oh * ow * oc);
    });
    run_forward(c, d_in, B, H, W, d_out);
    io.copy_back();
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

// hvn_postproc, and with `contours` hvn_postproc_contours.
static int postproc_host(hvn_ctx *c, const float *pred, int n, int H, int W, int C, int nr_types, int32_t *inst,
                         int64_t *table, int max_rows, int32_t *n_rows, bool contours, int32_t *pts, int64_t cap,
                         int32_t *offs) {
    API_BEGIN
    use(c);
    HVN_CHECK(pred && inst && table && n_rows && (!contours || (offs && (pts || cap == 0))), HVN_ERR_INVALID, "null buffer");
    HVN_CHECK(n >= 1 && H >= 1 && W >= 1 && cap >= 0, HVN_ERR_INVALID, "empty input");
    HVN_CHECK(!contours || (long long)n * max_rows < (1ll << 31), HVN_ERR_INVALID, "too many table rows");
    const size_t px = (size_t)n * H * W, no = (size_t)n * max_rows + 1;
    float *d_pred;
    int32_t *d_inst, *d_nr, *d_offs, *d_pts;
    int64_t *d_tab;
    Buffers io(c, c->io_arena, [&](Buffers &s) {
        d_pred = s.in(pred, px * C);
        d_inst = s.out(inst, px);
        d_tab = s.out(table, (size_t)n * max_rows * HVN_ROW_LEN, true);
        d_nr = s.out(n_rows, (size_t)n);
        d_offs = contours ? s.out(offs, no) : nullptr;
        d_pts = contours ? s.scratch<int32_t>((size_t)cap * 2 + 2) : nullptr;
    });
    run_postproc(c, d_pred, n, H, W, C, nr_types, d_inst, d_tab, max_rows, d_nr);
    if (contours)
        c->pp_launches += contours_run(c->stream, d_inst, (const long long *)d_tab, d_nr, n, H, W, max_rows, d_pts, cap,
                                       d_offs);
    io.copy_back();
    finish_profile(c, false, true);
    check_rows(n_rows, n, max_rows);
    if (contours && copy_fitting(c, pts, d_pts, offs[no - 1], cap, 8, "contour buffer", "points", "pts_cap"))
        HVN_CUDA(cudaStreamSynchronize(c->stream));
    API_END
}

int hvn_postproc(hvn_ctx *c, const float *pred, int n, int H, int W, int C, int nr_types, int32_t *inst,
                 int64_t *table, int max_rows, int32_t *n_rows) {
    return postproc_host(c, pred, n, H, W, C, nr_types, inst, table, max_rows, n_rows, false, nullptr, 0, nullptr);
}

int hvn_postproc_contours(hvn_ctx *c, const float *pred, int n, int H, int W, int C, int nr_types, int32_t *inst,
                          int64_t *table, int max_rows, int32_t *n_rows, int32_t *pts, int64_t cap, int32_t *offs) {
    return postproc_host(c, pred, n, H, W, C, nr_types, inst, table, max_rows, n_rows, true, pts, cap, offs);
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
    if (!pred) Buffers io(c, c->io_arena, [&](Buffers &s) { d_pred = s.scratch<float>((size_t)B * oh * ow * oc); });
    run_forward_postproc(c, imgs, B, H, W, d_pred, inst, table, max_rows, n_rows);
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
    const size_t px = (size_t)B * oh * ow;
    uint8_t *d_in;
    float *d_pred;
    int32_t *d_inst, *d_nr;
    int64_t *d_tab;
    Buffers io(c, c->io_arena, [&](Buffers &s) {
        d_in = s.in(imgs, (size_t)B * H * W * 3);
        d_pred = pred ? s.out(pred, px * oc) : s.scratch<float>(px * oc);
        d_inst = s.out(inst, px);
        d_tab = s.out(table, (size_t)B * max_rows * HVN_ROW_LEN, true);
        d_nr = s.out(n_rows, (size_t)B);
    });
    run_forward_postproc(c, d_in, B, H, W, d_pred, d_inst, d_tab, max_rows, d_nr);
    io.copy_back();
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

// A group of images laid out for the tile path (tile_plan): slot order groups equal sizes, `identity` when that is the
// input order already.
struct TileGroup {
    std::vector<TileImage> slots;
    std::vector<int> slot_of;
    int n = 0, oc = 0;
    long long table_rows = 0;  // rows of the group's padded instance tables (sum of the slots' max_rows)
    size_t px = 0;         // pixels of the whole group
    long long cells = 0;   // patches of the whole group
    bool identity = true;
};

static void plan_tiles(hvn_ctx *c, int n, const int32_t *shapes, int patch_in, long long rows_cap, TileGroup &g) {
    HVN_CHECK(c->model, HVN_ERR_STATE, "context has no model");
    HVN_CHECK(n >= 1 && shapes, HVN_ERR_INVALID, "a tile group needs n_images >= 1 and their shapes");
    HVN_CHECK(rows_cap >= 1 && rows_cap < (1ll << 31) - 1, HVN_ERR_INVALID, "rows_cap must be in 1 .. 2^31 - 2");
    int oh, ow;
    c->model->out_shape(patch_in, patch_in, oh, ow, g.oc);
    HVN_CHECK(oh == ow && oh >= 1, HVN_ERR_INVALID, "unsupported patch size for this model mode");
    tile_plan(shapes, n, oh, g.oc, g.slots, g.slot_of);
    g.n = n;
    for (int i = 0; i < n; ++i) {
        g.px += (size_t)g.slots[i].H * g.slots[i].W;
        g.cells += (long long)g.slots[i].rows * g.slots[i].cols;
        g.identity = g.identity && g.slot_of[i] == i;
    }
    // each slot's padded table holds min(rows_cap, its own id bound) rows -- no map has more rows than its id bound,
    // and a map with more than rows_cap rows makes the packed table overflow anyway -- so the tables take about 14 B
    // per pixel of the group whatever its mix of sizes; equal sizes share a stride, as one postproc_run needs
    for (auto &t : g.slots) {
        t.max_rows = (int)std::min<long long>(rows_cap, postproc_max_ids(t.H, t.W));
        t.row0 = g.table_rows;
        g.table_rows += t.max_rows;
    }
}

// Uploads the slot table through the context's pinned buffer, stream-ordered: no host synchronisation beyond waiting
// for the previous upload to have left the buffer.
static void upload_slots(hvn_ctx *c, const TileGroup &g, TileImage *d_slots, int *d_slot_of) {
    const size_t tb = g.slots.size() * sizeof(TileImage), bytes = tb + (size_t)g.n * sizeof(int);
    HVN_CUDA(cudaEventSynchronize(c->pin_ev));
    if (bytes > c->pin_bytes) {
        if (c->pin) HVN_CUDA(cudaFreeHost(c->pin));
        c->pin = nullptr;
        c->pin_bytes = 0;
        HVN_CUDA(cudaMallocHost(&c->pin, bytes));
        c->pin_bytes = bytes;
    }
    std::memcpy(c->pin, g.slots.data(), tb);
    HVN_CUDA(cudaMemcpyAsync(d_slots, c->pin, tb, cudaMemcpyHostToDevice, c->stream));
    if (d_slot_of) {
        std::memcpy((char *)c->pin + tb, g.slot_of.data(), (size_t)g.n * sizeof(int));
        HVN_CUDA(cudaMemcpyAsync(d_slot_of, (char *)c->pin + tb, (size_t)g.n * sizeof(int), cudaMemcpyHostToDevice, c->stream));
    }
    HVN_CUDA(cudaEventRecord(c->pin_ev, c->stream));
}

static int run_tile_predict(hvn_ctx *c, const uint8_t *imgs, const TileImage *d_slots, int n, long long lo, long long hi,
                            int patch_in, int batch, float *pred) {
    int oh, ow, oc;
    c->model->out_shape(patch_in, patch_in, oh, ow, oc);
    if (batch < 1) batch = 64;
    batch = std::min(batch, 65535);
    c->tile_arena.reset();
    c->tile_arena.reserve(tile_workspace_bytes(patch_in, oh, oc, batch));
    return tile_predict(*c->model, c->tile_arena, c->stream, imgs, d_slots, n, lo, hi, patch_in, batch, c->chunk, pred);
}

// The device work of a tile group, enqueued on the context stream: patches of every image in one stream of batches,
// then per size class one post-processing call over its maps and one contour count, then the packed tables
// (input order) and -- when pt_offs is not null -- the packed contour points.  pred / inst are slot-ordered maps; null
// takes them from the context's workspace.  *pred_out / *inst_out receive the maps that were written.
static void run_tiles(hvn_ctx *c, const TileGroup &g, const uint8_t *imgs, int patch_in, int batch, float *pred,
                      int32_t *inst, int64_t *table, long long rows_cap, int32_t *row_offs, int32_t *pts, long long pts_cap,
                      int32_t *pt_offs, float **pred_out, int32_t **inst_out) {
    const int n = g.n, nt = c->model->nr_types;
    const size_t R = (size_t)g.table_rows;
    const bool contours = pt_offs != nullptr, one = n == 1;
    c->group_table_rows = one ? 0 : (long long)R;
    TileImage *d_slots;
    int *d_slot_of, *d_nrows, *cnt;
    long long *pad;
    // a group of one writes its table and its point counts in place (the packing is the identity)
    Buffers ws(c, c->group_arena, [&](Buffers &b) {
        d_slots = b.scratch<TileImage>(n);
        d_slot_of = b.scratch<int>(n);
        d_nrows = b.scratch<int>(n);
        pad = one ? (long long *)table : b.scratch<long long>(R * 10);
        cnt = !contours ? nullptr : (one ? pt_offs : b.scratch<int>(R));
        *pred_out = pred ? pred : b.scratch<float>(g.px * g.oc);
        *inst_out = inst ? inst : b.scratch<int32_t>(g.px);
    });
    pred = *pred_out;
    inst = *inst_out;
    upload_slots(c, g, d_slots, d_slot_of);

    if (c->profile) HVN_CUDA(cudaEventRecord(c->ev[0], c->stream));
    c->model->kernel_launches += run_tile_predict(c, imgs, d_slots, n, 0, g.cells, patch_in, batch, pred);
    if (c->profile) HVN_CUDA(cudaEventRecord(c->ev[1], c->stream));
    if (c->profile) HVN_CUDA(cudaEventRecord(c->ev[2], c->stream));
    if (contours) HVN_CUDA(cudaMemsetAsync(pt_offs, 0, (size_t)(rows_cap + 1) * 4, c->stream));
    std::vector<std::pair<int, int>> classes;  // (first slot, maps) of each size class
    for (int s = 0; s < n; ++s) {
        if (s && g.slots[s].H == g.slots[s - 1].H && g.slots[s].W == g.slots[s - 1].W) ++classes.back().second;
        else classes.push_back({s, 1});
    }
    for (auto &k : classes) {
        const TileImage &t = g.slots[k.first];
        const size_t p0 = (size_t)(t.pred_off / g.oc);
        c->pp_launches += postproc_run(c->pp_arena, c->stream, pred + t.pred_off, k.second, t.H, t.W, g.oc, nt, inst + p0,
                                       pad + (size_t)t.row0 * 10, t.max_rows, d_nrows + k.first,
                                       c->profile >= 3 ? &c->pp_log : nullptr);
        if (contours)
            c->pp_launches += contours_count(c->stream, inst + p0, pad + (size_t)t.row0 * 10, d_nrows + k.first, k.second,
                                             t.H, t.W, t.max_rows, cnt + t.row0);
    }
    c->pp_launches += pack_tables(c->stream, pad, d_nrows, n, 0, (long long *)table, rows_cap, row_offs, d_slot_of,
                                  d_slots, cnt, pt_offs);
    if (contours) {
        c->pp_launches += contours_scan(c->stream, pt_offs, (int)rows_cap);
        for (auto &k : classes) {
            const TileImage &t = g.slots[k.first];
            c->pp_launches += contours_write_packed(c->stream, inst + t.pred_off / g.oc, pad + (size_t)t.row0 * 10,
                                                    d_nrows + k.first, k.second, t.H, t.W, t.max_rows, d_slots + k.first, row_offs,
                                                    n, rows_cap, pt_offs, pts, pts_cap);
        }
    }
    if (c->profile) HVN_CUDA(cudaEventRecord(c->ev[3], c->stream));
}

// Copies slot-ordered maps (elem_px bytes per pixel) to dst in input order.
static void copy_maps(hvn_ctx *c, const TileGroup &g, void *dst, const void *src, size_t elem_px, cudaMemcpyKind kind) {
    if (g.identity) {
        HVN_CUDA(cudaMemcpyAsync(dst, src, g.px * elem_px, kind, c->stream));
        return;
    }
    size_t o = 0;
    for (int i = 0; i < g.n; ++i) {
        const TileImage &t = g.slots[g.slot_of[i]];
        const size_t b = (size_t)t.H * t.W * elem_px;
        HVN_CUDA(cudaMemcpyAsync((char *)dst + o, (const char *)src + (size_t)(t.pred_off / g.oc) * elem_px, b, kind, c->stream));
        o += b;
    }
}

static void check_tiles_args(hvn_ctx *c, const void *imgs, const void *inst, const void *table, const void *row_offs,
                             const void *pts, long long pts_cap, const void *pt_offs) {
    HVN_CHECK(c->model, HVN_ERR_STATE, "context has no model");
    HVN_CHECK(imgs && inst && table && row_offs, HVN_ERR_INVALID, "null buffer");
    HVN_CHECK(pts_cap >= 0 && (!pt_offs || pts || pts_cap == 0), HVN_ERR_INVALID, "contours requested without a point buffer");
}

int hvn_tile_predict_dev(hvn_ctx *c, const uint8_t *img, int H, int W, int patch_in, int cell_lo, int cell_hi, int batch,
                         float *pred) {
    API_BEGIN
    use(c);
    HVN_CHECK(c->model, HVN_ERR_STATE, "context has no model");
    HVN_CHECK(img && pred && H >= 1 && W >= 1, HVN_ERR_INVALID, "bad argument");
    const int32_t shape[2] = {H, W};
    TileGroup g;
    plan_tiles(c, 1, shape, patch_in, 1, g);
    HVN_CHECK(cell_lo >= 0 && cell_hi <= g.cells && cell_lo <= cell_hi, -1, "patch range outside the grid");
    TileImage *d_slots;
    Buffers ws(c, c->group_arena, [&](Buffers &b) { d_slots = b.scratch<TileImage>(1); });
    upload_slots(c, g, d_slots, nullptr);
    if (c->profile) HVN_CUDA(cudaEventRecord(c->ev[0], c->stream));
    c->model->kernel_launches += run_tile_predict(c, img, d_slots, 1, cell_lo, cell_hi, patch_in, batch, pred);
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
    const int32_t shape[2] = {H, W};
    TileGroup g;
    plan_tiles(c, 1, shape, patch_in, max_rows, g);
    const size_t px = (size_t)H * W;
    if (!offs) cap = 0;
    int32_t ro[2] = {0, 0};
    uint8_t *d_img;
    float *d_pred, *wp;
    int32_t *d_inst, *d_ro, *d_offs, *d_pts, *wi;
    int64_t *d_tab;
    Buffers io(c, c->io_arena, [&](Buffers &s) {
        d_img = s.in(img, px * 3);
        d_pred = pred ? s.out(pred, px * g.oc) : s.scratch<float>(px * g.oc);
        d_inst = s.out(inst, px);
        d_tab = s.out(table, (size_t)max_rows * HVN_ROW_LEN, true);
        d_ro = s.out(ro, 2);
        d_offs = offs ? s.out(offs, (size_t)max_rows + 1) : nullptr;
        d_pts = s.scratch<int32_t>((size_t)cap * 2 + 2);
    });
    run_tiles(c, g, d_img, patch_in, batch, d_pred, d_inst, d_tab, max_rows, d_ro, d_pts, cap, d_offs, &wp, &wi);
    io.copy_back();
    finish_profile(c, true, true);
    check_range(c);
    n_rows[0] = ro[1];
    check_rows(n_rows, 1, max_rows);
    if (offs && copy_fitting(c, pts, d_pts, offs[max_rows], cap, 8, "contour buffer", "points", "pts_cap"))
        HVN_CUDA(cudaStreamSynchronize(c->stream));
    API_END
}

int hvn_infer_tiles(hvn_ctx *c, int n, const uint8_t *imgs, const int32_t *shapes, int patch_in, int batch, float *pred,
                    int32_t *inst, int64_t *table, int64_t rows_cap, int32_t *row_offs, int32_t *pts, int64_t pts_cap,
                    int32_t *pt_offs) {
    API_BEGIN
    use(c);
    check_tiles_args(c, imgs, inst, table, row_offs, pts, pts_cap, pt_offs);
    TileGroup g;
    plan_tiles(c, n, shapes, patch_in, rows_cap, g);
    if (!pt_offs) pts_cap = 0;
    const size_t px = g.px;
    uint8_t *d_imgs;
    float *d_pred, *wp;
    int32_t *d_inst, *d_ro, *d_po, *d_pts, *wi;
    int64_t *d_tab;
    Buffers io(c, c->io_arena, [&](Buffers &s) {
        d_imgs = s.in(imgs, px * 3);
        d_pred = s.scratch<float>(px * g.oc);
        d_inst = s.scratch<int32_t>(px);
        d_tab = s.scratch<int64_t>((size_t)rows_cap * HVN_ROW_LEN);
        d_ro = s.out(row_offs, (size_t)n + 1);
        d_po = pt_offs ? s.out(pt_offs, (size_t)rows_cap + 1) : nullptr;
        d_pts = s.scratch<int32_t>((size_t)pts_cap * 2 + 2);
    });
    run_tiles(c, g, d_imgs, patch_in, batch, d_pred, d_inst, d_tab, rows_cap, d_ro, d_pts, pts_cap, d_po, &wp, &wi);
    if (pred) copy_maps(c, g, pred, d_pred, (size_t)g.oc * 4, cudaMemcpyDeviceToHost);
    copy_maps(c, g, inst, d_inst, 4, cudaMemcpyDeviceToHost);
    io.copy_back();
    finish_profile(c, true, true);
    check_range(c);
    const long long rows = row_offs[n];
    copy_fitting(c, table, d_tab, rows, rows_cap, HVN_ROW_LEN * 8, "instance table", "rows", "rows_cap");
    if (pt_offs) copy_fitting(c, pts, d_pts, pt_offs[rows], pts_cap, 8, "contour buffer", "points", "pts_cap");
    HVN_CUDA(cudaStreamSynchronize(c->stream));
    API_END
}

int hvn_infer_tiles_dev(hvn_ctx *c, int n, const uint8_t *imgs, const int32_t *shapes, int patch_in, int batch,
                        float *pred, int32_t *inst, int64_t *table, int64_t rows_cap, int32_t *row_offs, int32_t *pts,
                        int64_t pts_cap, int32_t *pt_offs) {
    API_BEGIN
    use(c);
    check_tiles_args(c, imgs, inst, table, row_offs, pts, pts_cap, pt_offs);
    TileGroup g;
    plan_tiles(c, n, shapes, patch_in, rows_cap, g);
    if (!pt_offs) pts_cap = 0;
    // the caller's maps are in input order: written in place when that is the slot order, else copied from the
    // context's slot-order maps afterwards
    float *wp;
    int32_t *wi;
    run_tiles(c, g, imgs, patch_in, batch, g.identity ? pred : nullptr, g.identity ? inst : nullptr, table, rows_cap,
              row_offs, pts, pts_cap, pt_offs, &wp, &wi);
    if (pred && wp != pred) copy_maps(c, g, pred, wp, (size_t)g.oc * 4, cudaMemcpyDeviceToDevice);
    if (wi != inst) copy_maps(c, g, inst, wi, 4, cudaMemcpyDeviceToDevice);
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
    long long *h_offs = (long long *)offs, *d_offs, *d_pairs;
    int32_t *d_t, *d_p;
    Buffers maps(c, c->io_arena, [&](Buffers &s) {
        d_t = s.in(tru, px);
        d_p = pred ? s.in(pred, px) : nullptr;
        d_offs = s.out(h_offs, (size_t)n + 1);
    });
    PairWork w;
    inst_pairs_count(c->stats_arena, c->stream, d_t, d_p, n, H, W, d_offs, w);
    int err = 0;
    HVN_CUDA(cudaMemcpyAsync(&err, w.err, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    maps.copy_back();
    const long long total = offs[n];
    check_pairs_result(err, total, cap);
    if (total == 0) return HVN_OK;
    // the maps are no longer needed: the staging arena now holds the rows
    Buffers rows(c, c->io_arena, [&](Buffers &s) {
        d_pairs = s.out((long long *)pairs, (size_t)total * 3);
        w.offs = s.in(h_offs, (size_t)n + 1);
    });
    inst_pairs_emit(c->stream, w, d_pairs, total);
    rows.copy_back();
    API_END
}

// ---------------------------------------------------------------------------------------------------
static void check_targets_args(int n, int H, int W, int crop_h, int crop_w) {
    HVN_CHECK(n >= 1 && n <= 65535 && H >= 1 && W >= 1, HVN_ERR_INVALID, "bad shape");
    HVN_CHECK((long long)H * W <= 0x7fffffffll, HVN_ERR_INVALID, "map larger than 2^31 - 1 pixels");
    HVN_CHECK(crop_h >= 1 && crop_h <= H && crop_w >= 1 && crop_w <= W, HVN_ERR_INVALID,
              "crop shape must lie within the map");
}
// After the context stream has been synchronised.
static void check_targets_result(const TargetWork &w) {
    std::vector<int> per((size_t)5 * w.n + 1);
    HVN_CUDA(cudaMemcpy(per.data(), w.maxid, per.size() * sizeof(int), cudaMemcpyDeviceToHost));
    HVN_CHECK(!per[(size_t)5 * w.n], HVN_ERR_INVALID, "negative instance id");
    for (int m = 0; m < w.n; ++m)
        HVN_CHECK((long long)per[m] + per[(size_t)w.n + m] <= 0x7fffffffll, HVN_ERR_INVALID,
                  "map " + std::to_string(m) + ": largest id " + std::to_string(per[m]) + " + " +
                      std::to_string(per[(size_t)w.n + m]) +
                      " components exceeds 2^31 - 1 (the fresh ids of split instances would not fit in int32)");
}

int hvn_targets_dev(hvn_ctx *c, const int32_t *inst, int n, int H, int W, int crop_h, int crop_w, float *hv,
                    int32_t *flags) {
    API_BEGIN
    use(c);
    HVN_CHECK(inst && hv && flags, HVN_ERR_INVALID, "null buffer");
    check_targets_args(n, H, W, crop_h, crop_w);
    TargetWork w;
    targets_run(c->targets_arena, c->stream, inst, n, H, W, crop_h, crop_w, hv, flags, w);
    HVN_CUDA(cudaStreamSynchronize(c->stream));
    check_targets_result(w);
    API_END
}

int hvn_targets(hvn_ctx *c, const int32_t *inst, int n, int H, int W, int crop_h, int crop_w, float *hv,
                int32_t *flags) {
    API_BEGIN
    use(c);
    HVN_CHECK(inst && hv && flags, HVN_ERR_INVALID, "null buffer");
    check_targets_args(n, H, W, crop_h, crop_w);
    const size_t px = (size_t)n * H * W;
    int32_t *d_inst, *d_flags;
    float *d_hv;
    Buffers io(c, c->io_arena, [&](Buffers &s) {
        d_inst = s.in(inst, px);
        d_hv = s.out(hv, px * 2);
        d_flags = s.out(flags, (size_t)n);
    });
    TargetWork w;
    targets_run(c->targets_arena, c->stream, d_inst, n, H, W, crop_h, crop_w, d_hv, d_flags, w);
    io.copy_back();
    check_targets_result(w);
    API_END
}

// Forward, targets and the reduction of one validation batch, enqueued on the context stream.  Without `loss`
// (hvn_valid): the plain head and the counts.  With it (hvn_valid_loss): the full head, the loss sums and the counts;
// probs (may be null) receives the [B,h,w,4+nt] probabilities by a copy of kind pk.  The caller synchronises and calls
// finish_valid.
static void run_valid(hvn_ctx *c, const uint8_t *imgs, const int32_t *inst, const int32_t *type, int B, int H, int W,
                      int64_t *counts, double *sse, int32_t *flags, bool loss, double *sums, float *probs,
                      cudaMemcpyKind pk, TargetWork &w, LossWork &lw) {
    HVN_CHECK(c->model, HVN_ERR_STATE, "context has no model");
    const int nt = c->model->nr_types;
    HVN_CHECK(imgs && inst && counts && sse && flags && (sums || !loss), HVN_ERR_INVALID, "null buffer");
    HVN_CHECK(nt == 0 || type, HVN_ERR_INVALID, "a model with nr_types > 0 needs a type map");
    int oh, ow, oc;
    c->model->out_shape(H, W, oh, ow, oc);
    check_targets_args(B, H, W, oh, ow);
    if (loss) oc = nt + 4;
    const size_t opx = (size_t)B * oh * ow, px = (size_t)B * H * W;
    float *d_pred, *d_hv;
    Buffers ws(c, c->valid_arena, [&](Buffers &b) {
        d_pred = b.scratch<float>(opx * oc);
        d_hv = b.scratch<float>(px * 2);
    });
    HVN_CUDA(cudaMemsetAsync(counts, 0, (size_t)(3 + 2 * nt) * 8, c->stream));
    if (!loss) {
        HVN_CUDA(cudaMemsetAsync(sse, 0, sizeof(double), c->stream));
        run_forward(c, imgs, B, H, W, d_pred);
        targets_run(c->targets_arena, c->stream, inst, B, H, W, oh, ow, d_hv, flags, w);
        valid_reduce(c->stream, d_pred, inst, nt ? type : nullptr, d_hv, B, H, W, oh, ow, oc, nt, (long long *)counts, sse);
        return;
    }
    run_forward(c, imgs, B, H, W, d_pred, OUT_FULL);
    targets_run(c->targets_arena, c->stream, inst, B, H, W, oh, ow, d_hv, flags, w);
    if (c->profile) HVN_CUDA(cudaEventRecord(c->ev[2], c->stream));
    loss_reduce(c->loss_arena, c->stream, d_pred, inst, nt ? type : nullptr, d_hv, B, H, W, oh, ow, nt, sums,
                (long long *)counts, lw);
    if (c->profile) HVN_CUDA(cudaEventRecord(c->ev[3], c->stream));
    HVN_CUDA(cudaMemcpyAsync(sse, sums + LS_HV_SQ, sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
    if (probs) HVN_CUDA(cudaMemcpyAsync(probs, d_pred, opx * oc * 4, pk, c->stream));
}
// After the context stream has been synchronised.
static void finish_valid(hvn_ctx *c, bool loss, const TargetWork &w, const LossWork &lw) {
    finish_profile(c, true, false);
    if (loss && c->profile) HVN_CUDA(cudaEventElapsedTime(&c->ms_loss, c->ev[2], c->ev[3]));
    check_range(c);
    check_targets_result(w);
    if (!loss) return;
    int err = 0;
    HVN_CUDA(cudaMemcpy(&err, lw.err, sizeof(int), cudaMemcpyDeviceToHost));
    HVN_CHECK(!err, HVN_ERR_INVALID,
              "type id outside 0.." + std::to_string(c->model->nr_types - 1) + " inside the output crop");
}

static int valid_dev(hvn_ctx *c, const uint8_t *imgs, const int32_t *inst, const int32_t *type, int B, int H, int W,
                     int64_t *counts, double *sse, int32_t *flags, bool loss, double *sums, float *probs) {
    API_BEGIN
    use(c);
    TargetWork w;
    LossWork lw;
    run_valid(c, imgs, inst, type, B, H, W, counts, sse, flags, loss, sums, probs, cudaMemcpyDeviceToDevice, w, lw);
    HVN_CUDA(cudaStreamSynchronize(c->stream));
    finish_valid(c, loss, w, lw);
    API_END
}

static int valid_host(hvn_ctx *c, const uint8_t *imgs, const int32_t *inst, const int32_t *type, int B, int H, int W,
                      int64_t *counts, double *sse, int32_t *flags, bool loss, double *sums, float *probs) {
    API_BEGIN
    use(c);
    HVN_CHECK(c->model, HVN_ERR_STATE, "context has no model");
    HVN_CHECK(imgs && inst && counts && sse && flags && (sums || !loss), HVN_ERR_INVALID, "null buffer");
    check_targets_args(B, H, W, 1, 1);
    const int nt = c->model->nr_types;
    const size_t px = (size_t)B * H * W;
    uint8_t *d_imgs;
    int32_t *d_inst, *d_type, *d_flags;
    int64_t *d_counts;
    double *d_sse, *d_sums;
    Buffers io(c, c->io_arena, [&](Buffers &s) {
        d_imgs = s.in(imgs, px * 3);
        d_inst = s.in(inst, px);
        d_type = nt && type ? s.in(type, px) : nullptr;
        d_counts = s.out(counts, 3 + 2 * (size_t)nt);
        d_sse = s.out(sse, 1);
        d_sums = loss ? s.out(sums, (size_t)loss_nsums(nt)) : nullptr;
        d_flags = s.out(flags, (size_t)B);
    });
    TargetWork w;
    LossWork lw;
    run_valid(c, d_imgs, d_inst, d_type, B, H, W, d_counts, d_sse, d_flags, loss, d_sums, probs, cudaMemcpyDeviceToHost,
              w, lw);
    io.copy_back();
    finish_valid(c, loss, w, lw);
    API_END
}

int hvn_valid_dev(hvn_ctx *c, const uint8_t *imgs, const int32_t *inst, const int32_t *type, int B, int H, int W,
                  int64_t *counts, double *sse, int32_t *flags) {
    return valid_dev(c, imgs, inst, type, B, H, W, counts, sse, flags, false, nullptr, nullptr);
}

int hvn_valid(hvn_ctx *c, const uint8_t *imgs, const int32_t *inst, const int32_t *type, int B, int H, int W,
              int64_t *counts, double *sse, int32_t *flags) {
    return valid_host(c, imgs, inst, type, B, H, W, counts, sse, flags, false, nullptr, nullptr);
}

int hvn_valid_loss_dev(hvn_ctx *c, const uint8_t *imgs, const int32_t *inst, const int32_t *type, int B, int H, int W,
                       int64_t *counts, double *sse, int32_t *flags, double *sums, float *probs) {
    return valid_dev(c, imgs, inst, type, B, H, W, counts, sse, flags, true, sums, probs);
}

int hvn_valid_loss(hvn_ctx *c, const uint8_t *imgs, const int32_t *inst, const int32_t *type, int B, int H, int W,
                   int64_t *counts, double *sse, int32_t *flags, double *sums, float *probs) {
    return valid_host(c, imgs, inst, type, B, H, W, counts, sse, flags, true, sums, probs);
}

// ---------------------------------------------------------------------------------------------------
// The map table of a packed feature call; checks the host-side arguments.
static std::vector<FeatMap> feature_maps(int n, const int32_t *shapes, const float *pred, int C, long long n_rows) {
    HVN_CHECK(n >= 1 && shapes, HVN_ERR_INVALID, "a feature call needs n_maps >= 1 and their shapes");
    HVN_CHECK(!pred || C >= 3, HVN_ERR_INVALID, "a prediction map needs C >= 3 channels (NP at C - 3)");
    HVN_CHECK(n_rows >= 0 && n_rows < (1ll << 31) - 1, HVN_ERR_INVALID, "n_rows must be in 0 .. 2^31 - 2");
    std::vector<FeatMap> maps(n);
    long long off = 0;
    for (int m = 0; m < n; ++m) {
        const int H = shapes[2 * m], W = shapes[2 * m + 1];
        HVN_CHECK(H >= 1 && W >= 1 && (long long)H * W < (1ll << 31), HVN_ERR_INVALID,
                  "map " + std::to_string(m) + ": bad shape " + std::to_string(H) + "x" + std::to_string(W));
        maps[m] = {off, H, W};
        off += (long long)H * W;
    }
    return maps;
}

// hvn_inst_features_dev on device buffers: the check, one synchronisation to read its status, then the measurements.
static void run_features(hvn_ctx *c, const std::vector<FeatMap> &maps, const int32_t *inst, const uint8_t *img,
                         const float *pred, int C, const int64_t *table, const int32_t *row_offs, long long n_rows,
                         const int32_t *pts, const int32_t *pt_offs, double *feats) {
    HVN_CHECK(inst && table && row_offs && pt_offs && (feats || n_rows == 0), HVN_ERR_INVALID, "null buffer");
    const int n = (int)maps.size();
    FeatMap *d_maps;
    FeatStatus *d_st, st;
    void *scratch = nullptr;
    size_t scratch_bytes = 0;
    auto layout = [&](Buffers &b) {
        d_maps = b.in(maps.data(), maps.size());
        d_st = b.scratch<FeatStatus>(1);
        scratch = scratch_bytes ? b.scratch<char>(scratch_bytes) : nullptr;
    };
    Buffers ws(c, c->feat_arena, layout);
    if (c->profile) HVN_CUDA(cudaEventRecord(c->ev[2], c->stream));
    c->pp_launches += features_check(c->stream, d_maps, n, row_offs, n_rows, (const long long *)table, pts, pt_offs, d_st);
    HVN_CUDA(cudaMemcpyAsync(&st, d_st, sizeof(st), cudaMemcpyDeviceToHost, c->stream));
    HVN_CUDA(cudaStreamSynchronize(c->stream));
    HVN_CHECK(!(st.err & 1), HVN_ERR_INVALID, "row_offs must rise from 0 to n_rows = " + std::to_string(n_rows));
    HVN_CHECK(!(st.err & 2), HVN_ERR_INVALID, "a table row's bbox is empty or outside its map");
    HVN_CHECK(!(st.err & 4), HVN_ERR_INVALID, "pt_offs must not fall (and pt_offs[0] >= 0)");
    HVN_CHECK(!(st.err & 8), HVN_ERR_INVALID, "a contour point lies outside its row's bbox");
    if (st.max_pts > FEAT_SMEM_POINTS) {  // long contours: the arena again, now with their scratch (the stream is idle)
        scratch_bytes = FEAT_SCRATCH_BYTES_PER_POINT * (size_t)st.total_pts;
        Buffers again(c, c->feat_arena, layout);
    }
    c->pp_launches += features_rows(c->stream, d_maps, n, inst, img, pred, C, (const long long *)table, row_offs, n_rows,
                                    pts, pt_offs, scratch, feats, st.total_pts);
    if (c->profile) {
        HVN_CUDA(cudaEventRecord(c->ev[3], c->stream));
        HVN_CUDA(cudaStreamSynchronize(c->stream));
        HVN_CUDA(cudaEventElapsedTime(&c->ms_feat, c->ev[2], c->ev[3]));
    }
}

int hvn_inst_features_dev(hvn_ctx *c, int n, const int32_t *shapes, const int32_t *inst, const uint8_t *img,
                          const float *pred, int C, const int64_t *table, const int32_t *row_offs, int64_t n_rows,
                          const int32_t *pts, const int32_t *pt_offs, double *feats) {
    API_BEGIN
    use(c);
    run_features(c, feature_maps(n, shapes, pred, C, n_rows), inst, img, pred, C, table, row_offs, n_rows, pts, pt_offs,
                 feats);
    API_END
}

int hvn_inst_features(hvn_ctx *c, int n, const int32_t *shapes, const int32_t *inst, const uint8_t *img,
                      const float *pred, int C, const int64_t *table, const int32_t *row_offs, int64_t n_rows,
                      const int32_t *pts, const int32_t *pt_offs, double *feats) {
    API_BEGIN
    use(c);
    const std::vector<FeatMap> maps = feature_maps(n, shapes, pred, C, n_rows);
    HVN_CHECK(inst && table && row_offs && pt_offs && (feats || n_rows == 0), HVN_ERR_INVALID, "null buffer");
    // the points the offsets reach are staged; the device check sees the offsets themselves
    HVN_CHECK(pt_offs[0] >= 0 && pt_offs[n_rows] >= pt_offs[0] && (pts || pt_offs[n_rows] == 0), HVN_ERR_INVALID,
              "pt_offs must not fall (and pt_offs[0] >= 0)");
    const size_t px = (size_t)(maps.back().px_off + (long long)maps.back().H * maps.back().W);
    const uint8_t *d_img;
    const float *d_pred;
    const int32_t *d_inst, *d_ro, *d_pts, *d_po;
    const int64_t *d_tab;
    double *d_feats;
    Buffers io(c, c->io_arena, [&](Buffers &s) {
        d_inst = s.in(inst, px);
        d_img = img ? s.in(img, px * 3) : nullptr;
        d_pred = pred ? s.in(pred, px * C) : nullptr;
        d_tab = s.in(table, (size_t)n_rows * HVN_ROW_LEN);
        d_ro = s.in(row_offs, (size_t)n + 1);
        d_pts = s.in(pts, (size_t)pt_offs[n_rows] * 2);
        d_po = s.in(pt_offs, (size_t)n_rows + 1);
        d_feats = s.out(feats, (size_t)n_rows * HVN_FEAT_LEN);
    });
    run_features(c, maps, d_inst, d_img, d_pred, C, d_tab, d_ro, n_rows, d_pts, d_po, d_feats);
    io.copy_back();
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
int hvn_mem_info(hvn_ctx *c, size_t *free_bytes, size_t *total_bytes) {
    API_BEGIN
    use(c);
    HVN_CHECK(free_bytes && total_bytes, HVN_ERR_INVALID, "null out pointer");
    HVN_CUDA(cudaMemGetInfo(free_bytes, total_bytes));
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
    else if (k == "loss") *ms = c->ms_loss;
    else if (k == "features") *ms = c->ms_feat;
    else if (c->model && c->model->class_ms.count(k)) *ms = (float)c->model->class_ms.at(k);
    else if (k == "conv_tc" || k == "conv_ref" || k == "conv0" || k == "bnrelu" || k == "head" || k == "tta") *ms = 0.f;
    else throw Error(HVN_ERR_INVALID, "unknown stage " + k);
    API_END
}

}  // extern "C"
