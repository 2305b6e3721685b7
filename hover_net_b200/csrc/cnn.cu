// HoVer-Net model state, layer plan and executor.
//
// The plan is the reference graph (reference models/hovernet/net_desc.py:17-145,
// net_utils.py:71-294) re-expressed as a flat list of fused device ops over NHWC buffers:
//   * post-conv BatchNorm+ReLU (conv1/bn, conv2/bn, conv0/bn, u0/bn) folds into the producing conv's epilogue;
//   * the pre-activation BN+ReLU of the *next* residual unit (and the group's blk_bna) is a second
//     output of conv3's epilogue, next to the raw running sum that feeds the residual add;
//   * dense-block concatenation is a channel-offset write into one buffer, the centre crops are
//     window offsets (no copies); each dense unit's preact BN is an elementwise pass over that window;
//   * 2x nearest upsample + skip add is the epilogue of conv_bot / convf;
//   * TF-"same" padding and valid crops are operand addressing (zero fill outside the view).
#include "cnn.h"
#include "tta.h"

#include <algorithm>
#include <cmath>
#include <cstring>

namespace hvn {

static const struct { const char *name; int cin, c1, c3, units, stride; } kGroups[4] = {
    {"d0", 64, 64, 256, 3, 1}, {"d1", 256, 128, 512, 4, 2}, {"d2", 512, 256, 1024, 6, 2}, {"d3", 1024, 512, 2048, 3, 2}};

Plan::~Plan() {
    for (void *p : allocs) cudaFree(p);
}

template <typename T> T *Model::dalloc(size_t n, std::vector<void *> &owner, bool zero) {
    T *p = nullptr;
    HVN_CUDA(cudaMalloc((void **)&p, std::max<size_t>(n, 1) * sizeof(T)));
    owner.push_back(p);
    if (zero) HVN_CUDA(cudaMemset(p, 0, std::max<size_t>(n, 1) * sizeof(T)));
    return p;
}

void Model::add_spec(const std::string &name, std::initializer_list<int64_t> shape, bool ignored) {
    ParamSpec s;
    s.name = name;
    s.ndim = (int)shape.size();
    int i = 0;
    for (auto v : shape) s.shape[i++] = v;
    s.ignored = ignored;
    index[name] = (int)spec.size();
    spec.push_back(s);
}
void Model::add_bn(const std::string &p, int c) {
    add_spec(p + ".weight", {c});
    add_spec(p + ".bias", {c});
    add_spec(p + ".running_mean", {c});
    add_spec(p + ".running_var", {c});
    add_spec(p + ".num_batches_tracked", {}, true);
}

// Checkpoint key inventory == reference state_dict (module registration order).
Model::Model(const std::string &mode_, int nr_types_) : mode(mode_), nr_types(nr_types_) {
    HVN_CHECK(mode == "original" || mode == "fast", -1,
              "Unknown mode `" + mode + "` for HoVerNet. Only support `original` or `fast`.");
    HVN_CHECK(nr_types >= 0 && nr_types <= HVN_MAX_TYPES, -1, "nr_types out of range");
    k = mode == "original" ? 5 : 3;
    add_spec("conv0./.weight", {64, 3, 7, 7});
    add_bn("conv0.bn", 64);
    for (auto &g : kGroups) {
        int unit_in = g.cin;
        for (int u = 0; u < g.units; ++u) {
            std::string p = std::string(g.name) + ".units." + std::to_string(u) + ".";
            if (u != 0) add_bn(p + "preact/bn", unit_in);
            add_spec(p + "conv1.weight", {g.c1, unit_in, 1, 1});
            add_bn(p + "conv1/bn", g.c1);
            add_spec(p + "conv2.weight", {g.c1, g.c1, 3, 3});
            add_bn(p + "conv2/bn", g.c1);
            add_spec(p + "conv3.weight", {g.c3, g.c1, 1, 1});
            unit_in = g.c3;
        }
        add_spec(std::string(g.name) + ".shortcut.weight", {g.c3, g.cin, 1, 1});
        add_bn(std::string(g.name) + ".blk_bna.bn", g.c3);
    }
    add_spec("conv_bot.weight", {1024, 2048, 1, 1});
    if (nr_types > 0) branches_ = {"tp", "np", "hv"};
    else branches_ = {"np", "hv"};
    for (auto &b : branches_) {
        int out_ch = b == "tp" ? nr_types : 2;
        const struct { const char *u; int cin, ca, units; } us[2] = {{"u3", 1024, 256, 8}, {"u2", 512, 128, 4}};
        for (auto &u : us) {
            std::string p = "decoder." + b + "." + u.u + ".";
            add_spec(p + "conva.weight", {u.ca, u.cin, k, k});
            int c = u.ca;
            for (int i = 0; i < u.units; ++i) {
                std::string q = p + "dense.units." + std::to_string(i) + ".";
                add_bn(q + "preact_bna/bn", c);
                add_spec(q + "conv1.weight", {128, c, 1, 1});
                add_bn(q + "conv1/bn", 128);
                add_spec(q + "conv2.weight", {32, 32, k, k});
                c += 32;
            }
            add_bn(p + "dense.blk_bna.bn", c);
            add_spec(p + "convf.weight", {c, c, 1, 1});
        }
        add_spec("decoder." + b + ".u1.conva.weight", {64, 256, k, k});
        add_bn("decoder." + b + ".u0.bn", 64);
        add_spec("decoder." + b + ".u0.conv.weight", {out_ch, 64, 1, 1});
        add_spec("decoder." + b + ".u0.conv.bias", {out_ch});
    }
    add_spec("upsample2x.unpool_mat", {2, 2}, true);
}

Model::~Model() {
    for (auto &st : side_) if (st) cudaStreamDestroy(st);
    if (ev_fork_) cudaEventDestroy(ev_fork_);
    for (auto &e : ev_join_) if (e) cudaEventDestroy(e);
    plans_.clear();
    for (void *p : wallocs_) cudaFree(p);
    if (d_flag_) cudaFree(d_flag_);
    if (h_flag_) cudaFreeHost(h_flag_);
}

void Model::load(const std::string &name_in, const float *data, int ndim, const int64_t *shape) {
    std::string name = name_in;
    if (name.rfind("module.", 0) == 0) name = name.substr(7);  // run_utils/utils.py:15-29
    auto it = index.find(name);
    HVN_CHECK(it != index.end(), -3, "Unexpected key(s) in state_dict: \"" + name + "\"");
    ParamSpec &s = spec[it->second];
    if (!s.ignored) {
        bool same = ndim == s.ndim;
        for (int i = 0; same && i < ndim; ++i) same = shape[i] == s.shape[i];
        HVN_CHECK(same, -3, "size mismatch for " + name);
        HVN_CHECK(data != nullptr, -1, "null data for " + name);
        host[name].assign(data, data + s.numel());
    }
    s.loaded = true;
    finalized = false;
}

const std::vector<float> &Model::hostp(const std::string &name) const {
    auto it = host.find(name);
    HVN_CHECK(it != host.end(), -3, "Missing key(s) in state_dict: \"" + name + "\"");
    return it->second;
}

// Exponent e with max|w| * 2^e in [2^13, 2^14): see ConvWeights::oscale.  Inf / NaN weights are a checkpoint error.
static int weight_exponent(float mx) {
    HVN_CHECK(std::isfinite(mx), -3, "non-finite convolution weight in the checkpoint");
    if (mx == 0.f) return 0;
    int ex = 0;
    std::frexp(mx, &ex);  // mx = m * 2^ex, m in [0.5, 1)  ->  mx in [2^(ex-1), 2^ex)
    return 14 - ex;
}

// hi (and, in precision "highest", lo) weight planes -> device
void Model::upload_planes(ConvWeights &cw, const std::vector<__half> &hi, const std::vector<__half> &lo) {
    cw.hi = dalloc<__half>(hi.size(), wallocs_, false);
    HVN_CUDA(cudaMemcpy(cw.hi, hi.data(), hi.size() * sizeof(__half), cudaMemcpyHostToDevice));
    cw.lo = nullptr;
    if (precision == 0) {
        cw.lo = dalloc<__half>(lo.size(), wallocs_, false);
        HVN_CUDA(cudaMemcpy(cw.lo, lo.data(), lo.size() * sizeof(__half), cudaMemcpyHostToDevice));
    }
}

// OIHW fp32 -> [tap][cout][cin_pad] split fp16 (grouped convs become block-diagonal dense)
void Model::make_conv(const std::string &name, int groups) {
    const ParamSpec &s = spec[index.at(name)];
    const std::vector<float> &w = hostp(name);
    int O = (int)s.shape[0], I = (int)s.shape[1], KH = (int)s.shape[2], KW = (int)s.shape[3];
    int cin = I * groups, og = O / groups;
    ConvWeights cw;
    cw.taps = KH * KW; cw.kh = KH; cw.kw = KW; cw.cout = O; cw.cin = cin;
    cw.cin_pad = (cin + 63) / 64 * 64;
    size_t n = (size_t)cw.taps * O * cw.cin_pad;
    std::vector<__half> hi(n, __float2half_rn(0.f)), lo(n, __float2half_rn(0.f));
    std::vector<float> osc(O, 1.f);
    for (int o = 0; o < O; ++o) {
        int g = o / og;
        float mx = 0.f;
        for (size_t j = 0; j < (size_t)I * cw.taps; ++j) mx = std::max(mx, std::fabs(w[(size_t)o * I * cw.taps + j]));
        const int e = weight_exponent(mx);
        osc[o] = std::ldexp(1.f, -e);
        for (int i = 0; i < I; ++i)
            for (int t = 0; t < cw.taps; ++t) {
                float v = std::ldexp(w[((size_t)o * I + i) * cw.taps + t], e);
                __half h = __float2half_rn(v);
                __half l = __float2half_rn(v - __half2float(h));
                size_t d = ((size_t)t * O + o) * cw.cin_pad + (size_t)g * I + i;
                hi[d] = h;
                lo[d] = l;
            }
    }
    upload_planes(cw, hi, lo);
    float *d_osc = dalloc<float>(O, wallocs_, false);
    HVN_CUDA(cudaMemcpy(d_osc, osc.data(), O * sizeof(float), cudaMemcpyHostToDevice));
    cw.oscale = d_osc;
    conv_[name] = cw;
}

// two 1x1 convolutions with the same cout, concatenated along K: [cout][cin1 + cin2]
void Model::make_conv_concat(const std::string &key, const std::string &name1, const std::string &name2) {
    const ParamSpec &s1 = spec[index.at(name1)], &s2 = spec[index.at(name2)];
    const std::vector<float> &w1 = hostp(name1), &w2 = hostp(name2);
    const int O = (int)s1.shape[0], I1 = (int)s1.shape[1], I2 = (int)s2.shape[1];
    HVN_CHECK(s2.shape[0] == O && s1.shape[2] == 1 && s2.shape[2] == 1 && I1 % 64 == 0 && I2 % 64 == 0, -1,
              "internal: cannot concatenate " + name1 + " and " + name2);
    ConvWeights cw;
    cw.taps = 1; cw.kh = cw.kw = 1; cw.cout = O; cw.cin = I1 + I2; cw.cin_pad = I1 + I2;
    size_t n = (size_t)O * cw.cin_pad;
    std::vector<__half> hi(n), lo(n);
    std::vector<float> osc(O, 1.f);
    for (int o = 0; o < O; ++o) {
        float mx = 0.f;
        for (int i = 0; i < I1; ++i) mx = std::max(mx, std::fabs(w1[(size_t)o * I1 + i]));
        for (int i = 0; i < I2; ++i) mx = std::max(mx, std::fabs(w2[(size_t)o * I2 + i]));
        const int e = weight_exponent(mx);  // one exponent per output channel: both sources accumulate into it
        osc[o] = std::ldexp(1.f, -e);
        for (int i = 0; i < I1 + I2; ++i) {
            float v = std::ldexp(i < I1 ? w1[(size_t)o * I1 + i] : w2[(size_t)o * I2 + (i - I1)], e);
            __half h = __float2half_rn(v);
            hi[(size_t)o * cw.cin_pad + i] = h;
            lo[(size_t)o * cw.cin_pad + i] = __float2half_rn(v - __half2float(h));
        }
    }
    upload_planes(cw, hi, lo);
    float *d_osc = dalloc<float>(O, wallocs_, false);
    HVN_CUDA(cudaMemcpy(d_osc, osc.data(), O * sizeof(float), cudaMemcpyHostToDevice));
    cw.oscale = d_osc;
    conv_[key] = cw;
}

// BatchNorm and head parameters must be finite: the reference would return NaN maps for them, which the engine's ReLU
// and range clamp would otherwise turn into finite, plausible-looking ones
static void check_finite(const std::vector<float> &v, const std::string &name) {
    for (float x : v) HVN_CHECK(std::isfinite(x), -3, "non-finite value in checkpoint parameter " + name);
}

// eval-mode BatchNorm2d(eps=1e-5) as y = x*scale + shift
void Model::make_bn(const std::string &p) {
    const auto &g = hostp(p + ".weight"), &b = hostp(p + ".bias"), &m = hostp(p + ".running_mean"),
               &v = hostp(p + ".running_var");
    for (const char *f : {".weight", ".bias", ".running_mean", ".running_var"}) check_finite(hostp(p + f), p + f);
    int c = (int)g.size();
    for (int i = 0; i < c; ++i)
        HVN_CHECK((double)v[i] + 1e-5 > 0.0, -3, "running_var + eps <= 0 in checkpoint parameter " + p + ".running_var");
    std::vector<float> sc(c), sh(c);
    for (int i = 0; i < c; ++i) {
        double s = (double)g[i] / std::sqrt((double)v[i] + 1e-5);
        sc[i] = (float)s;
        sh[i] = (float)((double)b[i] - (double)m[i] * s);
        // act_shift: activations are stored as x * 2^-s.  A BN whose input is already scaled keeps its scale and
        // shrinks its shift; the stem's BN sees the unscaled image and shrinks both.  (ldexp: exact.)
        sh[i] = std::ldexp(sh[i], -act_shift);
        if (p == "conv0.bn") sc[i] = std::ldexp(sc[i], -act_shift);
    }
    BNParams bp;
    bp.c = c;
    bp.scale = dalloc<float>(c, wallocs_, false);
    bp.shift = dalloc<float>(c, wallocs_, false);
    HVN_CUDA(cudaMemcpy(bp.scale, sc.data(), c * 4, cudaMemcpyHostToDevice));
    HVN_CUDA(cudaMemcpy(bp.shift, sh.data(), c * 4, cudaMemcpyHostToDevice));
    bn_[p] = bp;
}

void Model::reset_range_flag(cudaStream_t s) {
    if (d_flag_) HVN_CUDA(cudaMemsetAsync(d_flag_, 0, sizeof(unsigned int), s));
    if (h_flag_) *h_flag_ = 0;
}

void Model::finalize() {
    std::string missing;
    for (auto &s : spec)
        if (!s.loaded && !s.ignored) missing += (missing.empty() ? "\"" : ", \"") + s.name + "\"";
    HVN_CHECK(missing.empty(), -3, "Missing key(s) in state_dict: " + missing);
    plans_.clear();
    for (void *p : wallocs_) cudaFree(p);
    wallocs_.clear();
    conv_.clear(); bn_.clear(); head_w_.clear(); head_b_.clear();
    HVN_CHECK(act_shift >= 0 && act_shift <= 48, -1, "act_shift out of range (0..48)");
    HVN_CHECK(precision == 0 || precision == 1, -1, "precision must be 0 (highest) or 1 (high)");
    if (!d_flag_) {
        HVN_CUDA(cudaMalloc((void **)&d_flag_, sizeof(unsigned int)));
        HVN_CUDA(cudaMemset(d_flag_, 0, sizeof(unsigned int)));
        HVN_CUDA(cudaMallocHost((void **)&h_flag_, sizeof(unsigned int)));
        *h_flag_ = 0;
    }
    for (auto &s : spec) {
        if (s.ignored) continue;
        const std::string &n = s.name;
        if (n == "conv0./.weight") {
            const auto &w = hostp(n);  // OIHW [64][3][7][7] -> [ky][kx][ch][64]
            std::vector<float> t(7 * 7 * 3 * 64);
            for (int o = 0; o < 64; ++o) {
                // precision "high": the CUDA-core stem multiplies by the same fp16 weights as the tensor-core one,
                // fp16(w * 2^e) * 2^-e with the channel's exponent (exact)
                float mx = 0.f;
                for (int j = 0; j < 147; ++j) mx = std::max(mx, std::fabs(w[(size_t)o * 147 + j]));
                const int e = weight_exponent(mx);
                for (int ch = 0; ch < 3; ++ch)
                    for (int ky = 0; ky < 7; ++ky)
                        for (int kx = 0; kx < 7; ++kx) {
                            float v = w[((o * 3 + ch) * 7 + ky) * 7 + kx];
                            if (precision == 1) v = std::ldexp(__half2float(__float2half_rn(std::ldexp(v, e))), -e);
                            t[((ky * 7 + kx) * 3 + ch) * 64 + o] = v;
                        }
            }
            conv0_w_ = dalloc<float>(t.size(), wallocs_, false);
            HVN_CUDA(cudaMemcpy(conv0_w_, t.data(), t.size() * 4, cudaMemcpyHostToDevice));
            {   // tensor-core stem operand: [64 cout][192 k] split fp16, k = ky * 24 + kx * 3 + ch, zeros elsewhere
                ConvWeights cw;
                cw.taps = 1; cw.kh = cw.kw = 1; cw.cout = 64; cw.cin = 168; cw.cin_pad = 192;
                std::vector<__half> hi((size_t)64 * 192, __float2half_rn(0.f)), lo(hi);
                std::vector<float> osc(64, 1.f);
                for (int o = 0; o < 64; ++o) {
                    float mx = 0.f;
                    for (int j = 0; j < 147; ++j) mx = std::max(mx, std::fabs(w[(size_t)o * 147 + j]));
                    const int e = weight_exponent(mx);
                    osc[o] = std::ldexp(1.f, -e);
                    for (int ch = 0; ch < 3; ++ch)
                        for (int ky = 0; ky < 7; ++ky)
                            for (int kx = 0; kx < 7; ++kx) {
                                const float v = std::ldexp(w[((o * 3 + ch) * 7 + ky) * 7 + kx], e);
                                const __half h = __float2half_rn(v);
                                const size_t d = (size_t)o * 192 + ky * 24 + kx * 3 + ch;
                                hi[d] = h;
                                lo[d] = __float2half_rn(v - __half2float(h));
                            }
                }
                upload_planes(cw, hi, lo);
                float *d_osc = dalloc<float>(64, wallocs_, false);
                HVN_CUDA(cudaMemcpy(d_osc, osc.data(), 64 * sizeof(float), cudaMemcpyHostToDevice));
                cw.oscale = d_osc;
                conv0_tc_w_ = cw;
            }
        } else if (n.size() > 15 && n.compare(n.size() - 15, 15, ".u0.conv.weight") == 0) {
            std::vector<float> w = hostp(n);
            check_finite(w, n);
            for (auto &x : w) x = std::ldexp(x, act_shift);  // the heads see features scaled by 2^-act_shift
            float *d = dalloc<float>(w.size(), wallocs_, false);
            HVN_CUDA(cudaMemcpy(d, w.data(), w.size() * 4, cudaMemcpyHostToDevice));
            head_w_[n.substr(0, n.size() - 7)] = d;
        } else if (n.size() > 13 && n.compare(n.size() - 13, 13, ".u0.conv.bias") == 0) {
            const auto &w = hostp(n);
            check_finite(w, n);
            float *d = dalloc<float>(w.size(), wallocs_, false);
            HVN_CUDA(cudaMemcpy(d, w.data(), w.size() * 4, cudaMemcpyHostToDevice));
            head_b_[n.substr(0, n.size() - 5)] = d;
        } else if (s.ndim == 4) {
            bool grouped = n.find(".dense.units.") != std::string::npos && n.find("conv2.weight") != std::string::npos;
            make_conv(n, grouped ? 4 : 1);
        } else if (n.size() > 13 && n.compare(n.size() - 13, 13, ".running_mean") == 0) {
            make_bn(n.substr(0, n.size() - 13));
        }
    }
    for (auto &g : kGroups) {
        const std::string gn = g.name;
        make_conv_concat(gn + ".fused3", gn + ".units.0.conv3.weight", gn + ".shortcut.weight");
    }
    finalized = true;
}

void Model::out_shape(int H, int W, int &oh, int &ow, int &oc) const {
    auto f = [&](int in) {
        int s = mode == "fast" ? in : in - 6;
        HVN_CHECK(s >= 8 && s % 8 == 0, -1,
                  "unsupported patch size " + std::to_string(in) + " for mode `" + mode +
                      "` (skip connections only line up when the stem output is a multiple of 8)");
        int d3 = s / 8;
        int u3 = 2 * d3 - (k - 1) * 9;
        int u2 = 2 * u3 - (k - 1) * 5;
        HVN_CHECK(u3 > 0 && u2 > 0, -1, "patch too small for the decoder's valid convolutions");
        return 2 * u2;
    };
    oh = f(H);
    ow = f(W);
    oc = nr_types > 0 ? 4 : 3;
}

// ------------------------------------------------------------------------------------------------
// conv_path = 2: per-layer self test of the wgmma kernel against the CUDA-core referee
__global__ void k_cmp_raw(const float *a, const float *b, int B, int h, int w, int c, long long sN, int sH, int sW,
                          unsigned int *out) {
    long long total = (long long)B * h * w * c;
    float md = 0.f, mr = 0.f;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        int ch = (int)(i % c); long long t = i / c;
        int x = (int)(t % w); t /= w;
        int y = (int)(t % h); int n = (int)(t / h);
        long long o = n * sN + (long long)y * sH + (long long)x * sW + ch;
        float va = a[o], vb = b[o];
        float d = fabsf(va - vb);
        if (!(d == d)) d = 3.0e38f;  // NaN -> huge
        md = fmaxf(md, d); mr = fmaxf(mr, fabsf(vb));
    }
    atomicMax(out + 0, __float_as_uint(md));
    atomicMax(out + 1, __float_as_uint(mr));
}
__global__ void k_cmp_split(const __half *ah, const __half *al, const __half *bh, const __half *bl, int B, int h, int w,
                            int c, long long sN, int sH, int sW, unsigned int *out) {
    long long total = (long long)B * h * w * c;
    float md = 0.f, mr = 0.f;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        int ch = (int)(i % c); long long t = i / c;
        int x = (int)(t % w); t /= w;
        int y = (int)(t % h); int n = (int)(t / h);
        long long o = n * sN + (long long)y * sH + (long long)x * sW + ch;
        float va = __half2float(ah[o]), vb = __half2float(bh[o]);
        if (al) { va += __half2float(al[o]); vb += __half2float(bl[o]); }  // single-plane tensors: hi only
        float d = fabsf(va - vb);
        if (!(d == d)) d = 3.0e38f;
        md = fmaxf(md, d); mr = fmaxf(mr, fabsf(vb));
    }
    atomicMax(out + 2, __float_as_uint(md));
    atomicMax(out + 3, __float_as_uint(mr));
}

void Model::selftest_conv(const Op &op, cudaStream_t s) {
    ConvParams a = op.cp, b = op.cp;
    std::vector<void *> tmp;
    auto dz = [&](size_t bytes) { void *p = nullptr; HVN_CUDA(cudaMalloc(&p, bytes)); HVN_CUDA(cudaMemsetAsync(p, 0, bytes, s)); tmp.push_back(p); return p; };
    const int B = op.cp.B;
    if (op.cp.out_raw.p) {
        size_t n = (size_t)B * op.cp.out_raw.sN;
        a.out_raw.p = (float *)dz(n * 4); b.out_raw.p = (float *)dz(n * 4);
    }
    if (op.cp.out_split.hi) {
        size_t n = (size_t)B * op.cp.out_split.sN;
        const bool lo = op.cp.out_split.lo != nullptr;
        a.out_split.hi = (__half *)dz(n * 2); a.out_split.lo = lo ? (__half *)dz(n * 2) : nullptr;
        b.out_split.hi = (__half *)dz(n * 2); b.out_split.lo = lo ? (__half *)dz(n * 2) : nullptr;
    }
    unsigned int *d_out = (unsigned int *)dz(16);
    const bool trace = getenv("HVN_TRACE") != nullptr;
    if (trace) { fprintf(stderr, "[selftest] %s ...\n", op.name.c_str()); fflush(stderr); }
    TcPlan pa;   // the plan's tensor maps address the epilogue tensors: planned again for the scratch outputs
    HVN_CHECK(tc_plan(a, pa), -1, "selftest: tc_plan declined the scratch outputs of a planned layer");
    tc_launch(a, pa, s);
    if (b.in_scale) {  // referee path of a transformed-input layer: BN+ReLU pass into the scratch view, then the conv
        launch_bnrelu(b.a_raw, B, b.in_scale, b.in_shift, b.a, s);
        b.in_scale = b.in_shift = nullptr;
    }
    launch_conv_ref(b, s);
    if (op.cp.out_raw.p) {
        const RawRef &r = op.cp.out_raw;
        k_cmp_raw<<<296, 256, 0, s>>>(a.out_raw.p, b.out_raw.p, B, r.h, r.w, op.cp.w.cout, r.sN, r.sH, r.sW, d_out);
    }
    if (op.cp.out_split.hi) {
        const SplitRef &r = op.cp.out_split;
        int hh = op.cp.up2 ? 2 * op.cp.ho : op.cp.ho, ww = op.cp.up2 ? 2 * op.cp.wo : op.cp.wo;
        k_cmp_split<<<296, 256, 0, s>>>(a.out_split.hi, a.out_split.lo, b.out_split.hi, b.out_split.lo, B, hh, ww,
                                        op.cp.w.cout, r.sN, r.sH, r.sW, d_out);
    }
    unsigned int h_out[4] = {0, 0, 0, 0};
    HVN_CUDA(cudaMemcpyAsync(h_out, d_out, 16, cudaMemcpyDeviceToHost, s));
    cudaError_t e = cudaStreamSynchronize(s);
    float f[4];
    memcpy(f, h_out, 16);
    char line[512];
    snprintf(line, sizeof(line), "%-44s k%dx%d s%d cin%-4d cout%-4d %dx%d flat=%d box=%dx%d bn=%d | raw diff %.3e (ref %.3e) | split diff %.3e (ref %.3e)%s\n",
             op.name.c_str(), op.cp.w.kh, op.cp.w.kw, op.cp.stride, op.cp.w.cin, op.cp.w.cout, op.cp.ho, op.cp.wo,
             op.tc.flat, op.tc.bw, op.tc.bh, op.tc.block_n, f[0], f[1], f[2], f[3],
             e == cudaSuccess ? "" : (std::string("  CUDA ERROR: ") + cudaGetErrorString(e)).c_str());
    debug_log += line;
    if (trace) { fputs(line, stderr); fflush(stderr); }
    for (void *p : tmp) cudaFree(p);
    HVN_CHECK(e == cudaSuccess, -2, std::string("selftest: ") + cudaGetErrorString(e) + " at " + op.name);
}

// ------------------------------------------------------------------------------------------------
namespace {
SplitRef sview(const SplitRef &b, int y0, int x0, int h, int w, int c0, int c) {
    SplitRef v = b;
    long long off = (long long)y0 * b.sH + (long long)x0 * b.sW + c0;
    v.hi += off;
    if (v.lo) v.lo += off;
    v.h = h; v.w = w; v.c = c;
    return v;
}
RawRef rview(const RawRef &b, int y0, int x0, int h, int w, int c0, int c) {
    RawRef v = b;
    v.p += (long long)y0 * b.sH + (long long)x0 * b.sW + c0;
    v.h = h; v.w = w; v.c = c;
    return v;
}
}  // namespace

Plan &Model::plan(int B, int H, int W) {
    HVN_CHECK(finalized, -5, "weights not finalised (call hvn_finalize_weights)");
    HVN_CHECK(H == W, -1, "only square patches are supported (reference patch geometry is square)");
    std::string key = std::to_string(B) + "x" + std::to_string(H) + "x" + std::to_string(W) + "p" + std::to_string(conv_path) +
                      "b" + std::to_string(branch_streams) + "x" + std::to_string(xform) + "f" + std::to_string(fuse_shortcut) + "u" + std::to_string(fuse_up2) + "t" + std::to_string(tta);
    auto it = plans_.find(key);
    if (it != plans_.end()) return *it->second;
    std::unique_ptr<Plan> pl(new Plan());
    Plan &P = *pl;
    P.B = B; P.H = H; P.W = W;
    out_shape(H, W, P.oh, P.ow, P.oc);
    P.tta = tta;
    if (tta) {
        const size_t nv = (size_t)B * H * W * 3, np = (size_t)B * P.oh * P.ow * (nr_types + 3);
        P.tta_views = dalloc<uint8_t>(nv, P.allocs, false);
        P.tta_probs = dalloc<float>(np, P.allocs, false);
        P.bytes += nv + np * sizeof(float);
    }

    auto new_split = [&](int h, int w, int c) {
        SplitRef r;
        size_t n = (size_t)B * h * w * c;
        r.hi = dalloc<__half>(n, P.allocs, true);
        r.lo = precision == 0 ? dalloc<__half>(n, P.allocs, true) : nullptr;  // "high": one plane
        P.bytes += (precision == 0 ? 2 : 1) * n * sizeof(__half);
        r.sN = (long long)h * w * c; r.sH = w * c; r.sW = c; r.h = h; r.w = w; r.c = c;
        r.flag = d_flag_;
        return r;
    };
    auto new_raw = [&](int h, int w, int c) {
        RawRef r;
        size_t n = (size_t)B * h * w * c;
        r.p = dalloc<float>(n, P.allocs, true);
        P.bytes += n * sizeof(float);
        r.sN = (long long)h * w * c; r.sH = w * c; r.sW = c; r.h = h; r.w = w; r.c = c;
        return r;
    };
    int cur_stream = 0;
    auto add_conv = [&](const std::string &wname, const SplitRef &a, int stride, int pad, int ho, int wo) -> Op & {
        Op op;
        op.stream = cur_stream;
        op.kind = Op::CONV;
        op.name = wname;
        op.cp.a = a;
        op.cp.w = conv_.at(wname);
        op.cp.stride = stride; op.cp.pad_t = pad; op.cp.pad_l = pad;
        op.cp.B = B; op.cp.ho = ho; op.cp.wo = wo;
        const ParamSpec &ps = spec[index.at(wname)];
        op.flops = 2.0 * B * ho * wo * (double)ps.numel();  // grouped conv counted at its true (sparse) size
        P.ops.push_back(op);
        return P.ops.back();
    };
    auto set_bn = [&](Op &op, const std::string &bnp, const SplitRef &out) {
        const BNParams &b = bn_.at(bnp);
        op.cp.out_split = out; op.cp.scale = b.scale; op.cp.shift = b.shift; op.cp.relu = 1;
    };
    auto add_bnrelu = [&](const std::string &bnp, const RawRef &in, const SplitRef &out) {
        Op op;
        op.stream = cur_stream;
        op.kind = Op::BNRELU;
        op.name = bnp;
        op.bn_in = in; op.bn_out = out; op.bn = bn_.at(bnp);
        P.ops.push_back(op);
    };
    auto add_up2 = [&](const std::string &name, const RawRef &in, const SplitRef &skip, const SplitRef &out) {
        Op op;
        op.stream = cur_stream;
        op.kind = Op::UP2ADD;
        op.name = name + "+up2add";
        op.up_in = in; op.up_skip = skip; op.up_out = out;
        P.ops.push_back(op);
    };
    auto tf_same_lo = [](int size, int ksize, int stride) {  // net_utils.py:51-63
        int pad = (size % stride == 0) ? std::max(ksize - stride, 0) : std::max(ksize - (size % stride), 0);
        return pad / 2;
    };

    const bool use_xf = xform && conv_path != 1;
    // ---- stem
    const int s0 = mode == "fast" ? H : H - 6;
    SplitRef X0 = new_split(s0, s0, 64);
    {
        Op op;
        op.kind = Op::CONV0; op.name = "conv0";
        op.c0_out = X0; op.c0_pad = mode == "fast" ? 3 : 0;
        op.bn = bn_.at("conv0.bn");
        op.flops = 2.0 * B * s0 * s0 * 64 * 147;
        P.ops.push_back(op);
    }
    // ---- encoder
    SplitRef x = X0, D[4];
    int si = s0, ds[4];
    for (int gi = 0; gi < 4; ++gi) {
        const auto &g = kGroups[gi];
        const std::string gn = g.name;
        int so = (si + g.stride - 1) / g.stride;
        RawRef S = new_raw(so, so, g.c3);
        SplitRef A1 = new_split(si, si, g.c1), A2 = new_split(so, so, g.c1), Pp = new_split(so, so, g.c3);
        const bool fuse = fuse_shortcut != 0;
        if (!fuse) { Op &op = add_conv(gn + ".shortcut.weight", x, g.stride, 0, so, so); op.cp.out_raw = S; }
        for (int u = 0; u < g.units; ++u) {
            std::string p = gn + ".units." + std::to_string(u) + ".";
            const SplitRef &in = u == 0 ? x : Pp;
            int ri = u == 0 ? si : so, st = u == 0 ? g.stride : 1;
            SplitRef a1 = A1;  // unit 0 runs conv1 at the group's input resolution; later units reuse the
                               // same allocation as a compact [ri,ri,c1] tensor
            if (ri != A1.h) { a1.h = ri; a1.w = ri; a1.sH = ri * g.c1; a1.sN = (long long)ri * ri * g.c1; }
            {
                Op &op = add_conv(p + "conv1.weight", in, 1, 0, ri, ri);
                set_bn(op, p + "conv1/bn", a1);
                if (u != 0 && use_xf) {  // A = relu(bn_preact(S)) formed in the kernel from the raw running sum
                    const BNParams &pb = bn_.at(p + "preact/bn");
                    op.cp.a_raw = S; op.cp.in_scale = pb.scale; op.cp.in_shift = pb.shift;
                }
            }
            int lo = tf_same_lo(ri, 3, st);
            { Op &op = add_conv(p + "conv2.weight", a1, st, lo, so, so); set_bn(op, p + "conv2/bn", A2); }
            {
                Op &op = add_conv(p + "conv3.weight", A2, 1, 0, so, so);
                if (u == 0 && fuse) {  // conv3(a2) + shortcut(x) as one GEMM over K = [c1 | cin]
                    op.cp.w = conv_.at(gn + ".fused3");
                    op.cp.a2 = x; op.cp.a2_stride = g.stride; op.cp.cin1 = g.c1;
                    op.flops += 2.0 * B * so * so * (double)g.cin * g.c3;
                    op.name = gn + ".units.0.conv3+shortcut";
                } else op.cp.res = S;
                if (u + 1 < g.units) {
                    op.cp.out_raw = S;
                    if (!use_xf) set_bn(op, gn + ".units." + std::to_string(u + 1) + ".preact/bn", Pp);
                } else set_bn(op, gn + ".blk_bna.bn", Pp);
            }
        }
        x = Pp; D[gi] = Pp; ds[gi] = so; si = so;
    }
    HVN_CHECK(2 * ds[3] == ds[2] && 2 * ds[2] == ds[1] && 2 * ds[1] == ds[0], -1, "patch size breaks the skip geometry");
    auto crop_to = [&](const SplitRef &d, int t) {
        int c = d.h - t;
        HVN_CHECK(c >= 0, -1, "skip connection smaller than decoder tensor");
        return sview(d, c / 2, c / 2, t, t, 0, d.c);  // utils.py:11-28 : crop_t = c // 2
    };
    // ---- bottleneck: conv_bot, upsample x2, + d2
    SplitRef U3in = new_split(2 * ds[3], 2 * ds[3], 1024);
    if (fuse_up2) {
        Op &op = add_conv("conv_bot.weight", D[3], 1, 0, ds[3], ds[3]);
        op.cp.up2 = 1; op.cp.skip = crop_to(D[2], 2 * ds[3]); op.cp.out_split = U3in;
    } else {
        RawRef Rb = new_raw(ds[3], ds[3], 1024);
        { Op &op = add_conv("conv_bot.weight", D[3], 1, 0, ds[3], ds[3]); op.cp.out_raw = Rb; }
        add_up2("conv_bot", Rb, crop_to(D[2], 2 * ds[3]), U3in);
    }
    // ---- decoder
    const int km1 = k - 1;
    const int h3 = 2 * ds[3] - km1, w8 = h3 - 8 * km1;
    const int h2 = 2 * w8 - km1, w4 = h2 - 4 * km1;
    const int ho = 2 * w4;
    HVN_CHECK(ho == P.oh, -1, "internal: output size mismatch");
    const int nsets = branch_streams ? (int)branches_.size() : 1;  // private scratch per concurrent branch
    RawRef C3[3], C2[3], RS[3];
    SplitRef T3[3], T2[3], B3[3], B2[3], U2in[3], U1in[3];
    for (int i = 0; i < nsets; ++i) {
        C3[i] = new_raw(h3, h3, 512); C2[i] = new_raw(h2, h2, 256);
        T3[i] = new_split(h3, h3, 512); T2[i] = new_split(h2, h2, 256);
        B3[i] = new_split(h3, h3, 128); B2[i] = new_split(h2, h2, 128);
        U2in[i] = new_split(2 * w8, 2 * w8, 512); U1in[i] = new_split(ho, ho, 256);
        if (!fuse_up2) RS[i] = new_raw(1, 1, std::max(w8 * w8 * 512, w4 * w4 * 256));  // convf output before up2+add
    }
    SplitRef Hf[3];
    for (size_t b = 0; b < branches_.size(); ++b) Hf[b] = new_split(ho, ho, 64);

    auto dense = [&](const std::string &pfx, const SplitRef &uin, const RawRef &Cb, const SplitRef &Tb,
                     const SplitRef &Bb, int hin, int c0, int units, const SplitRef &skip, const SplitRef &out,
                     const RawRef &Rscratch) {
        int hh = hin - km1;  // after conva (valid)
        { Op &op = add_conv(pfx + "conva.weight", uin, 1, 0, hh, hh); op.cp.out_raw = rview(Cb, 0, 0, hh, hh, 0, c0); }
        int c = c0;
        for (int i = 0; i < units; ++i) {
            int wi = hh - i * km1, oi = i * km1 / 2, wn = wi - km1, on = oi + km1 / 2;
            std::string q = pfx + "dense.units." + std::to_string(i) + ".";
            if (!use_xf) add_bnrelu(q + "preact_bna/bn", rview(Cb, oi, oi, wi, wi, 0, c), sview(Tb, oi, oi, wi, wi, 0, c));
            { Op &op = add_conv(q + "conv1.weight", sview(Tb, oi, oi, wi, wi, 0, c), 1, 0, wi, wi);
              set_bn(op, q + "conv1/bn", sview(Bb, oi, oi, wi, wi, 0, 128));
              if (use_xf) {
                  const BNParams &pb = bn_.at(q + "preact_bna/bn");
                  op.cp.a_raw = rview(Cb, oi, oi, wi, wi, 0, c); op.cp.in_scale = pb.scale; op.cp.in_shift = pb.shift;
              } }
            { Op &op = add_conv(q + "conv2.weight", sview(Bb, oi, oi, wi, wi, 0, 128), 1, 0, wn, wn);
              op.cp.out_raw = rview(Cb, on, on, wn, wn, c, 32); }
            c += 32;
        }
        int wl = hh - units * km1, ol = units * km1 / 2;
        if (!use_xf) add_bnrelu(pfx + "dense.blk_bna.bn", rview(Cb, ol, ol, wl, wl, 0, c), sview(Tb, ol, ol, wl, wl, 0, c));
        Op &op = add_conv(pfx + "convf.weight", sview(Tb, ol, ol, wl, wl, 0, c), 1, 0, wl, wl);
        RawRef Rf;
        if (fuse_up2) { op.cp.up2 = 1; op.cp.skip = skip; op.cp.out_split = out; }
        else { Rf = rview(Rscratch, 0, 0, wl, wl, 0, c); Rf.sH = wl * c; Rf.sW = c; Rf.sN = (long long)wl * wl * c; op.cp.out_raw = Rf; }
        if (use_xf) {
            const BNParams &pb = bn_.at(pfx + "dense.blk_bna.bn");
            op.cp.a_raw = rview(Cb, ol, ol, wl, wl, 0, c); op.cp.in_scale = pb.scale; op.cp.in_shift = pb.shift;
        }
        if (!fuse_up2) add_up2(pfx + "convf", Rf, skip, out);
    };

    Op head;
    head.kind = Op::HEAD; head.name = "head";
    head.head.nbranch = (int)branches_.size();
    head.head.B = B; head.head.h = ho; head.head.w_ = ho; head.head.C = tta ? nr_types + 3 : P.oc;
    for (size_t b = 0; b < branches_.size(); ++b) {
        const std::string bp = "decoder." + branches_[b] + ".";
        const int si_ = branch_streams ? (int)b : 0;
        cur_stream = si_;
        const size_t first_op = P.ops.size();
        dense(bp + "u3.", U3in, C3[si_], T3[si_], B3[si_], 2 * ds[3], 256, 8, crop_to(D[1], 2 * w8), U2in[si_], RS[si_]);
        dense(bp + "u2.", U2in[si_], C2[si_], T2[si_], B2[si_], 2 * w8, 128, 4, crop_to(D[0], ho), U1in[si_], RS[si_]);
        { Op &op = add_conv(bp + "u1.conva.weight", U1in[si_], 1, km1 / 2, ho, ho); set_bn(op, bp + "u0.bn", Hf[b]); }
        if (b == 0) P.ops[first_op].fork_point = true;
        head.head.feat[b] = Hf[b];
        head.head.w[b] = head_w_.at(bp + "u0.conv");
        head.head.bias[b] = head_b_.at(bp + "u0.conv");
        head.head.out_ch[b] = branches_[b] == "tp" ? nr_types : 2;
        head.head.kind[b] = branches_[b] == "tp" ? HEAD_TP : (branches_[b] == "np" ? HEAD_NP : HEAD_HV);
        head.flops += 2.0 * B * ho * ho * 64 * head.head.out_ch[b];
    }
    cur_stream = 0;
    P.ops.push_back(head);

    for (auto &op : P.ops) {
        P.flops += op.flops;
        if (op.kind == Op::CONV && conv_path != 1) tc_plan(op.cp, op.tc);
    }
    plans_[key] = std::move(pl);
    return *plans_[key];
}

void Model::forward(const uint8_t *imgs, int B, int H, int W, float *out, int chunk, cudaStream_t s, int layout) {
    HVN_CHECK(finalized, -5, "weights not finalised (call hvn_finalize_weights)");
    HVN_CHECK(B >= 1, -1, "empty batch");
    HVN_CHECK(!tta || H == W, -1,
              "test-time augmentation needs square patches (the rotated views of a " + std::to_string(H) + "x" +
                  std::to_string(W) + " patch are " + std::to_string(W) + "x" + std::to_string(H) + ")");
    HVN_CHECK(layout == OUT_PLAIN || layout == OUT_FULL, -1, "bad forward output layout");
    const bool full = layout == OUT_FULL;
    int oh, ow, oc;
    out_shape(H, W, oh, ow, oc);
    if (full) oc = nr_types + 4;
    if (chunk <= 0) chunk = 32;  // sub-batch size: large enough to fill 132 persistent CTAs on the thin decoder layers
    // inputs per chunk: with TTA a chunk of network patches holds the eight views of chunk / 8 whole inputs
    const int per = tta ? std::max(1, chunk / 8) : chunk;
    if (!side_[0]) {
        for (auto &st : side_) HVN_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
        HVN_CUDA(cudaEventCreateWithFlags(&ev_fork_, cudaEventDisableTiming));
        for (auto &e : ev_join_) HVN_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    }
    cudaStream_t main_stream = s;
    struct Rec { const char *cls; double flops; cudaEvent_t a, b; const Op *op; const char *name; };
    std::vector<Rec> recs;
    // the TTA kernels run on the context stream, outside the op list; profiled as class "tta"
    auto tta_launch = [&](const char *name, auto &&launch) {
        Rec r{"tta", 0.0, nullptr, nullptr, nullptr, name};
        if (profile_ops) {
            HVN_CUDA(cudaEventCreate(&r.a));
            HVN_CUDA(cudaEventCreate(&r.b));
            HVN_CUDA(cudaEventRecord(r.a, main_stream));
        }
        launch();
        ++kernel_launches;
        if (profile_ops) { HVN_CUDA(cudaEventRecord(r.b, main_stream)); recs.push_back(r); }
    };
    if (profile_ops) { class_ms.clear(); class_flops.clear(); class_launches.clear(); }
    last_flops = 0;
    last_plan_bytes = 0;
    const Plan *last_plan = nullptr;
    if (conv_path == 2 || profile_ops >= 2) debug_log.clear();

    for (int b0 = 0; b0 < B; b0 += per) {
        const int nb = std::min(per, B - b0);   // inputs of this chunk
        const int bc = tta ? 8 * nb : nb;       // network patches of this chunk
        Plan &P = plan(bc, H, W);
        if (tta && full && !P.tta_full) {
            const size_t n = (size_t)bc * oh * ow * oc;
            P.tta_full = dalloc<float>(n, P.allocs, false);
            P.bytes += n * sizeof(float);
        }
        last_flops += P.flops;
        if (&P != last_plan) last_plan_bytes += P.bytes;  // a tail chunk runs a second, smaller plan
        last_plan = &P;
        const uint8_t *in_c = imgs + (size_t)b0 * H * W * 3;
        if (tta) {
            tta_launch("tta_views", [&] { launch_tta_views(in_c, nb, H, P.tta_views, main_stream); });
            in_c = P.tta_views;
        }
        int prev_stream = 0;
        bool forked[3] = {true, false, false};
        for (auto &op : P.ops) {
            // fork: a side stream starts after everything issued so far on the context stream;
            // join: the context stream waits for the side streams before the op that follows them
            if (op.fork_point && branch_streams) {
                HVN_CUDA(cudaEventRecord(ev_fork_, main_stream));
                for (int i = 1; i < 3; ++i) { HVN_CUDA(cudaStreamWaitEvent(side_[i - 1], ev_fork_, 0)); forked[i] = true; }
            }
            if (op.stream == 0 && prev_stream != 0) {
                for (int i = 1; i < 3; ++i)
                    if (forked[i]) {
                        HVN_CUDA(cudaEventRecord(ev_join_[i - 1], side_[i - 1]));
                        HVN_CUDA(cudaStreamWaitEvent(main_stream, ev_join_[i - 1], 0));
                    }
            }
            prev_stream = op.stream;
            s = op.stream == 0 ? main_stream : side_[op.stream - 1];
            Rec r{nullptr, op.flops, nullptr, nullptr, &op};
            if (profile_ops) {
                HVN_CUDA(cudaEventCreate(&r.a));
                HVN_CUDA(cudaEventCreate(&r.b));
                HVN_CUDA(cudaEventRecord(r.a, s));
            }
            switch (op.kind) {
            case Op::CONV0:
                if (stem_tc && conv_path != 1 && conv0_tc_supported(H, W, op.c0_pad, op.c0_out)) {
                    launch_conv0_tc(in_c, bc, H, W, op.c0_pad, conv0_tc_w_, op.bn.scale, op.bn.shift, op.c0_out, s);
                    ++tc_launches;
                } else
                    launch_conv0(in_c, bc, H, W, op.c0_pad, conv0_w_, op.bn.scale, op.bn.shift, op.c0_out, s);
                r.cls = "conv0";
                break;
            case Op::CONV:
                if (op.tc.ok && conv_path == 2) selftest_conv(op, s);
                if (op.tc.ok) { tc_launch(op.cp, op.tc, s); ++tc_launches; r.cls = "conv_tc"; }
                else {
                    ConvParams q = op.cp;
                    if (q.in_scale) {  // materialise the pre-activated operand for the referee kernel
                        launch_bnrelu(q.a_raw, bc, q.in_scale, q.in_shift, q.a, s);
                        q.in_scale = q.in_shift = nullptr;
                    }
                    launch_conv_ref(q, s);
                    r.cls = "conv_ref";
                }
                break;
            case Op::BNRELU:
                launch_bnrelu(op.bn_in, bc, op.bn.scale, op.bn.shift, op.bn_out, s);
                r.cls = "bnrelu";
                break;
            case Op::UP2ADD:
                launch_up2_add(op.up_in, bc, op.up_skip, op.up_out, s);
                r.cls = "bnrelu";  // elementwise class
                break;
            case Op::HEAD: {
                HeadParams hp = op.head;
                if (full) {
                    hp.C = oc;
                    hp.out = P.tta ? P.tta_full : out + (size_t)b0 * oh * ow * oc;
                    launch_head_full(hp, s);
                } else if (P.tta) {
                    hp.out = P.tta_probs;
                    launch_head_probs(hp, s);
                } else {
                    hp.out = out + (size_t)b0 * oh * ow * oc;
                    launch_head(hp, s);
                }
                r.cls = "head";
                break;
            }
            }
            ++kernel_launches;
            if (profile_ops) { HVN_CUDA(cudaEventRecord(r.b, s)); recs.push_back(r); }
        }
        if (tta)  // the head ran on the context stream, after the branches joined
            tta_launch("tta_merge", [&] {
                float *o = out + (size_t)b0 * oh * ow * oc;
                if (full) launch_tta_merge_full(P.tta_full, nb, oh, nr_types, o, main_stream);
                else launch_tta_merge(P.tta_probs, nb, oh, nr_types, o, main_stream);
            });
    }
    s = main_stream;
    HVN_CUDA(cudaMemcpyAsync(h_flag_, d_flag_, sizeof(unsigned int), cudaMemcpyDeviceToHost, s));
    HVN_CUDA(cudaGetLastError());
    if (profile_ops) {
        HVN_CUDA(cudaStreamSynchronize(s));
        for (auto &r : recs) {
            float ms = 0.f;
            HVN_CUDA(cudaEventElapsedTime(&ms, r.a, r.b));
            class_ms[r.cls] += ms; class_flops[r.cls] += r.flops; class_launches[r.cls] += 1;
            if (profile_ops >= 2) {
                char line[384];
                const Op *o = r.op;
                if (o && o->kind == Op::CONV) {
                    // algorithmic HBM bytes: every input read once, every output written once, weights ignored
                    const ConvParams &c = o->cp;
                    const double px = (double)c.B * c.ho * c.wo, up = c.up2 ? 4.0 : 1.0;
                    auto split_b = [](const SplitRef &v) { return v.lo ? 4.0 : 2.0; };
                    double by = c.in_scale ? (double)c.B * c.a_raw.h * c.a_raw.w * c.a_raw.c * 4.0
                                           : (double)c.B * c.a.h * c.a.w * c.a.c * split_b(c.a);
                    if (c.a2.hi) by += (double)c.B * c.a2.h * c.a2.w * c.a2.c * split_b(c.a2);
                    if (c.res.p) by += px * c.w.cout * 4.0;
                    if (c.out_raw.p) by += px * c.w.cout * 4.0;
                    if (c.out_split.hi) by += up * px * c.w.cout * split_b(c.out_split);
                    if (c.up2) by += up * px * c.w.cout * split_b(c.skip);
                    snprintf(line, sizeof(line), "%-44s %-8s k%dx%d s%d cin%-4d cout%-4d out%dx%d box=%dx%d bn=%d %8.4f ms %8.2f GFLOP %7.1f TFLOP/s %8.4f GB\n",
                             o->name.c_str(), r.cls, o->cp.w.kh, o->cp.w.kw, o->cp.stride, o->cp.w.cin, o->cp.w.cout, o->cp.ho, o->cp.wo,
                             o->tc.bw, o->tc.bh, o->tc.block_n, ms, r.flops / 1e9, r.flops / 1e9 / std::max(ms, 1e-6f), by / 1e9);
                } else
                    snprintf(line, sizeof(line), "%-44s %-8s %8.4f ms\n", o ? o->name.c_str() : r.name, r.cls, ms);
                debug_log += line;
            }
            cudaEventDestroy(r.a); cudaEventDestroy(r.b);
        }
    }
}

}  // namespace hvn
