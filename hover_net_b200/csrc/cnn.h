// HoVer-Net model state + layer plan + executor (host side of the CNN path).
#pragma once
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "cnn_kernels.h"
#include "common.cuh"

namespace hvn {

struct ParamSpec {
    std::string name;
    int ndim = 0;
    int64_t shape[4] = {0, 0, 0, 0};
    bool ignored = false;  // num_batches_tracked / upsample2x.unpool_mat: accepted, unused
    bool loaded = false;
    size_t numel() const {
        size_t n = 1;
        for (int i = 0; i < ndim; ++i) n *= (size_t)shape[i];
        return n;
    }
};

struct BNParams { float *scale = nullptr, *shift = nullptr; int c = 0; };

struct Op {
    enum Kind { CONV0, CONV, BNRELU, HEAD, UP2ADD } kind = CONV;
    std::string name;
    ConvParams cp;          // CONV
    TcPlan tc;              // CONV: tensor-core plan (ok=false -> referee kernel)
    // CONV0
    SplitRef c0_out; int c0_pad = 0;
    // BNRELU
    RawRef bn_in; SplitRef bn_out; BNParams bn;
    // HEAD
    HeadParams head;
    // UP2ADD
    RawRef up_in; SplitRef up_skip, up_out;
    double flops = 0;       // 2*MACs of the reference layer (algorithmic)
    int stream = 0;         // 0 = context stream; 1,2 = side streams (decoder branches run concurrently)
    bool fork_point = false; // side streams may start once everything before this op has been issued
};

struct Plan {
    int B = 0, H = 0, W = 0, oh = 0, ow = 0, oc = 0;
    // tta: B network patches are the eight views of B / 8 inputs; the stem reads tta_views, the head stores
    // probabilities (k_head_probs) into tta_probs [B,oh,ow,nr_types+3], which k_tta_merge reduces into the output
    int tta = 0;
    uint8_t *tta_views = nullptr;
    float *tta_probs = nullptr;
    // the views' k_head_full maps [B,oh,ow,nr_types+4] for a forward with layout OUT_FULL, allocated by the first one
    float *tta_full = nullptr;
    std::vector<Op> ops;
    std::vector<void *> allocs;
    size_t bytes = 0;
    double flops = 0;       // algorithmic 2*MACs for B patches
    ~Plan();
};

class Model {
  public:
    Model(const std::string &mode, int nr_types);
    ~Model();
    std::string mode;
    int nr_types;  // 0 == None
    int k;         // decoder kernel size
    std::vector<ParamSpec> spec;
    std::map<std::string, int> index;
    std::map<std::string, std::vector<float>> host;
    bool finalized = false;
    int fuse_up2 = 0;        // 1: 2x upsample + skip add inside the conv epilogue; 0: separate streaming pass (faster)
    int fuse_shortcut = 1;   // fold each residual group's 1x1 shortcut into unit 0's conv3 (one GEMM over [a2 | x])
    int stem_tc = 1;         // stem (conv0) on the tensor core (k_conv0_tc); 0: CUDA-core k_conv0
    int xform = 1;           // fuse pre-activation BN+ReLU into the consuming 1x1 conv's A-operand load
    int branch_streams = 1;  // run the decoder branches on separate streams
    int conv_path = 0;  // 0 auto (wgmma where eligible), 1 referee only, 2 auto + per-layer self test
    // Activations travel as fp16 hi + lo, finite up to 65504.  act_shift = s stores every activation as x * 2^-s:
    // the stem's BN scale, every BN shift and (inversely) the head weights absorb the factor, so the network function
    // is unchanged (powers of two are exact) while the representable range grows to 65504 * 2^s.  0 by default; raise
    // it when a forward reports HVN_ERR_RANGE (the Python binding retries with +6 automatically).
    int act_shift = 0;
    // Convolution operand precision.  0 "highest": activations that feed a convolution and its weights are stored as
    // fp16 hi + lo and every MAC forms hi*hi + hi*lo + lo*hi.  1 "high": hi planes only (no lo is allocated), one fp16
    // product per MAC -- the operand precision of TF32.  Accumulation, residual sums, BN and heads stay fp32 in both.
    // Weights are re-finalised on a change.
    int precision = 0;
    // Test-time augmentation.  1: every input patch runs as its eight dihedral views (tta.h), whose maps are brought
    // back to the input's frame and averaged on the device; each chunk holds the views of chunk / 8 inputs (at least
    // one).  0 (default): the plain forward.  Square patches only.
    int tta = 0;
    // true if the last forward() stored a value outside the fp16 range (valid after the stream was synchronised)
    bool range_overflow() const { return h_flag_ && *h_flag_ != 0; }
    void reset_range_flag(cudaStream_t s);  // after the host has seen (and reported) an overflow
    void drop_plans() { plans_.clear(); }   // frees the cached plans' buffers (the caller has synchronised)

    void load(const std::string &name, const float *data, int ndim, const int64_t *shape);
    void finalize();
    void out_shape(int H, int W, int &oh, int &ow, int &oc) const;
    // builds (and caches) the plan for a sub-batch geometry
    Plan &plan(int B, int H, int W);
    // runs B patches: imgs u8 [B,H,W,3] (device) -> out f32 [B,oh,ow,oc] (device).  layout OUT_FULL (the validation
    // loss) stores every probability instead, out f32 [B,oh,ow,nr_types+4] = [np p0, np p1, hv x, hv y, tp p0..];
    // np p1 and hv equal the OUT_PLAIN forward's bit for bit, with and without tta.
    void forward(const uint8_t *imgs, int B, int H, int W, float *out, int chunk, cudaStream_t s,
                 int layout = OUT_PLAIN);

    long long kernel_launches = 0, tc_launches = 0;
    // per-kernel-class device time of the last forward() when profile_ops != 0 (CUDA events per launch)
    int profile_ops = 0;
    std::map<std::string, double> class_ms, class_flops;
    std::map<std::string, long long> class_launches;
    double last_flops = 0;  // algorithmic 2*MACs of the last forward()
    size_t last_plan_bytes = 0;  // device bytes of the plan(s) the last forward() ran
    std::string debug_log;  // conv_path == 2: per-layer wgmma-vs-referee report of the last forward()
    void selftest_conv(const Op &op, cudaStream_t s);

  private:
    std::map<std::string, ConvWeights> conv_;
    std::map<std::string, BNParams> bn_;
    float *conv0_w_ = nullptr;
    ConvWeights conv0_tc_w_;  // the stem's weights as a [1][64][192] GEMM operand (k = ky * 24 + kx * 3 + ch)
    std::map<std::string, float *> head_w_, head_b_;
    std::vector<void *> wallocs_;
    std::map<std::string, std::unique_ptr<Plan>> plans_;
    std::vector<std::string> branches_;
    unsigned int *d_flag_ = nullptr;          // device range flag (raised by split stores)
    unsigned int *h_flag_ = nullptr;          // pinned host copy, refreshed at the end of every forward()
    cudaStream_t side_[2] = {nullptr, nullptr};
    cudaEvent_t ev_fork_ = nullptr, ev_join_[2] = {nullptr, nullptr};
    void add_spec(const std::string &name, std::initializer_list<int64_t> shape, bool ignored = false);
    void add_bn(const std::string &prefix, int c);
    const std::vector<float> &hostp(const std::string &name) const;
    void make_conv(const std::string &name, int groups);
    void make_conv_concat(const std::string &key, const std::string &name1, const std::string &name2);
    void make_bn(const std::string &prefix);
    void upload_planes(ConvWeights &cw, const std::vector<__half> &hi, const std::vector<__half> &lo);
    template <typename T> T *dalloc(size_t n, std::vector<void *> &owner, bool zero);
};

}  // namespace hvn
