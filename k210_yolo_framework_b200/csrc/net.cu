// Native graph builder, weight folding/packing, activation arena and executor behind the
// k2y_net_* C-ABI.  One k2y_net == one Keras model pair (yolo_model / yolo_model_warpper) of
// /root/reference/models/yolonet.py; the four builders below restate :12-46 (yolo_mobilev1 over
// keras_mobilenet.py:215-229,291-436), :49-104 (yolo_mobilev2 over keras_mobilenet_v2.py:311-382,
// 426-485), :107-158 (tiny_yolo) and :161-229 (yolo / Darknet-53) as a static layer schedule.
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>
#include <stdarg.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <map>
#include <memory>
#include <string>
#include <tuple>
#include <vector>

#include "common.h"
#include "gemm_tc.h"

namespace k2y {

static thread_local char g_err[512] = "";
void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

namespace {

constexpr float BN_EPS = 1e-3f;  // Keras BatchNormalization epsilon used by every reference model

enum LayerKind { L_CONV = 0, L_DW = 1, L_POOL = 2 };

struct Tensor {
    int h = 0, w = 0, c = 0;
    int def = -1, last_use = -1;  // layer indices
    int out_index = -1;           // >= 0: network output l (bound head buffer)
    bool is_input = false;
    size_t off = 0;               // float offset inside the arena
};

struct Layer {
    int kind = L_CONV;
    std::string name, bn_name;
    int src0 = -1, src1 = -1, res = -1, dst = -1;
    bool up0 = false;
    int kh = 1, kw = 1, stride = 1, pad_t = 0, pad_l = 0;
    int cin = 0, cout = 0;
    int act = ACT_NONE;
    float alpha = 0.f;
    bool has_bias = false;
    // raw Keras variables (host)
    std::vector<float> kernel, bias, gamma, beta, mean, var;
    // device
    float *d_w = nullptr, *d_scale = nullptr, *d_shift = nullptr;
    std::vector<float> h_scale, h_shift;  // folded BN (host copy; the first conv takes its constants by value)
    // "pixel pair" form of a narrow 1x1 conv (Cin <= 32): [M][K] x [K][N] run as [M/2][2K] x blockdiag(W, W)[2K][2N] — the same
    // memory on both sides, half as many 128-row tiles, full-width TMA boxes (gemm_tc.cu per-tile costs dominate these layers)
    TcWeights tc2;
    float *d_scale2 = nullptr, *d_shift2 = nullptr;
    TcWeights tc;  // tensor-core packing (gemm_tc.cu)
};

}  // namespace
}  // namespace k2y

using namespace k2y;

struct k2y_net {
    std::string model_def;
    int in_h = 0, in_w = 0, A = 0, C = 0, max_batch = 0, device = 0;
    float alpha = 1.f;
    std::vector<Tensor> tensors;
    std::vector<Layer> layers;
    std::vector<int> outputs;  // tensor ids
    std::map<std::string, int> auto_count;
    bool finalized = false, bound = false, keep_all = false, use_graph = true;
    int math = K2Y_MATH_TC_BF16X3;  // default: bf16 tensor cores on (hi, mid) split operands
    size_t arena_floats = 0;
    float *arena = nullptr;
    const float *x_dev = nullptr;
    const unsigned char *x_u8 = nullptr;  // optional uint8 input (k2y_net_bind_u8)
    int *img_max = nullptr;
    std::vector<float *> heads_dev;
    // one captured graph per (batch, input binding): re-binding the input to an alternate buffer (double-buffered H2D) reuses
    // the graph captured for that buffer instead of re-capturing
    std::map<std::tuple<int, const void *, const void *, const void *, const void *>, cudaGraphExec_t> graphs;  // (batch, x, x_u8, img_max, head 0)
    int last_batch = 0;
    int launches = 0;  // kernels issued by the last issue_layers() pass
    int sm_limit = 0;              // SM budget of the persistent tensor-core kernels (0 = whole device), k2y_net_set_sm_limit
    float *tc_scratch = nullptr;   // this net's split-K partials (never shared with another net / stream)
    size_t tc_scratch_bytes = 0;

    std::string auto_name(const std::string &base) {
        int n = auto_count[base]++;
        return n == 0 ? base : base + "_" + std::to_string(n);
    }
    int add_tensor(int h, int w, int c) {
        Tensor t;
        t.h = h;
        t.w = w;
        t.c = c;
        tensors.push_back(t);
        return (int)tensors.size() - 1;
    }
    // Dense conv. pad_mode: 0 = SAME (stride 1), 1 = ZeroPadding2D((1,1),(1,1)) + VALID, 2 = ZeroPadding2D((1,0),(1,0)) + VALID
    int conv(int src, const std::string &name, int cout, int k, int stride, int pad_mode, const std::string &bn, int act,
             float alpha_, bool bias, int src1 = -1, bool up0 = false, int res = -1) {
        Layer L;
        L.kind = L_CONV;
        L.name = name;
        L.bn_name = bn;
        L.src0 = src;
        L.src1 = src1;
        L.up0 = up0;
        L.res = res;
        const Tensor &s = tensors[src];
        const int H = up0 ? s.h * 2 : s.h, W = up0 ? s.w * 2 : s.w;
        L.cin = s.c + (src1 >= 0 ? tensors[src1].c : 0);
        L.cout = cout;
        L.kh = L.kw = k;
        L.stride = stride;
        int oh, ow;
        if (pad_mode == 0) {
            L.pad_t = L.pad_l = k / 2;
            oh = H;
            ow = W;
        } else if (pad_mode == 1) {
            L.pad_t = L.pad_l = 1;
            oh = (H + 2 - k) / stride + 1;
            ow = (W + 2 - k) / stride + 1;
        } else {
            L.pad_t = L.pad_l = 1;
            oh = (H + 1 - k) / stride + 1;
            ow = (W + 1 - k) / stride + 1;
        }
        L.act = act;
        L.alpha = alpha_;
        L.has_bias = bias;
        L.dst = add_tensor(oh, ow, cout);
        layers.push_back(L);
        return L.dst;
    }
    int dwconv(int src, const std::string &name, int stride, const std::string &bn, int act) {
        Layer L;
        L.kind = L_DW;
        L.name = name;
        L.bn_name = bn;
        L.src0 = src;
        const Tensor &s = tensors[src];
        L.cin = L.cout = s.c;
        L.kh = L.kw = 3;
        L.stride = stride;
        L.pad_t = L.pad_l = 1;  // SAME for stride 1; ZeroPadding2D((1,1),(1,1)) + VALID for stride 2
        const int oh = stride == 1 ? s.h : (s.h + 2 - 3) / 2 + 1;
        const int ow = stride == 1 ? s.w : (s.w + 2 - 3) / 2 + 1;
        L.act = act;
        L.dst = add_tensor(oh, ow, s.c);
        layers.push_back(L);
        return L.dst;
    }
    int maxpool(int src, int stride) {
        Layer L;
        L.kind = L_POOL;
        L.name = auto_name("max_pooling2d");
        L.src0 = src;
        const Tensor &s = tensors[src];
        L.cin = L.cout = s.c;
        L.stride = stride;
        L.dst = add_tensor((s.h + stride - 1) / stride, (s.w + stride - 1) / stride, s.c);
        layers.push_back(L);
        return L.dst;
    }
    // DarknetConv2D_BN_Leaky (yolonet.py:253-260): conv (no bias) -> BN -> LeakyReLU(0.1)
    int dbl(int src, int cout, int k, int stride = 1, int src1 = -1, bool up0 = false, int res = -1) {
        const std::string cn = auto_name("conv2d");
        const std::string bn = auto_name("batch_normalization");
        auto_name("leaky_re_lu");
        return conv(src, cn, cout, k, stride, stride == 2 ? 2 : 0, bn, ACT_LEAKY, 0.1f, false, src1, up0, res);
    }
    // DarknetConv2D (yolonet.py:244-250): plain conv with bias, linear
    int dconv_out(int src, int cout) {
        return conv(src, auto_name("conv2d"), cout, 1, 1, 0, "", ACT_NONE, 0.f, true);
    }
};

namespace {

// Keras stores LeakyReLU() default alpha as float32(0.3) = 0.30000001192...
constexpr float LEAKY_DEFAULT = 0.3f;

int make_divisible(float v, int divisor) {
    int new_v = std::max(divisor, (int)(v + divisor / 2.0f) / divisor * divisor);
    if (new_v < 0.9f * v) new_v += divisor;
    return new_v;
}

void two_scale_heads(k2y_net *n, int x1, int x2, int f1, int f2, int out_ch) {
    // y1 = compose(DBL(f1,3x3), DarknetConv2D(out))(x2)
    int y1 = n->dbl(x2, f1, 3);
    y1 = n->dconv_out(y1, out_ch);
    // x2 = compose(DBL(128,1x1), UpSampling2D(2))(x2);  y2 = compose(Concatenate, DBL(f2,3x3), DarknetConv2D(out))([x2, x1])
    int lat = n->dbl(x2, 128, 1);
    int y2 = n->dbl(lat, f2, 3, 1, x1, /*up0=*/true);
    y2 = n->dconv_out(y2, out_ch);
    n->outputs = {y1, y2};
}

void build_mobilev1(k2y_net *n, int out_ch) {
    const float a = n->alpha;
    int x = 0;
    x = n->conv(x, "conv1", (int)(32 * a), 3, 2, 1, "conv1_bn", ACT_LEAKY, LEAKY_DEFAULT, false);
    const int f[13] = {a == 1.0f ? 40 : 64, 128, 128, 256, 256, 512, 512, 512, 512, 512, 512, 1024, 1024};
    const int s[13] = {1, 2, 1, 2, 1, 2, 1, 1, 1, 1, 1, 2, 1};
    int x1 = -1;
    for (int i = 0; i < 13; ++i) {
        const std::string id = std::to_string(i + 1);
        x = n->dwconv(x, "conv_dw_" + id, s[i], "conv_dw_" + id + "_bn", ACT_RELU);
        x = n->conv(x, "conv_pw_" + id, (int)(f[i] * a), 1, 1, 0, "conv_pw_" + id + "_bn", ACT_LEAKY, LEAKY_DEFAULT, false);
        if (i + 1 == 11) x1 = x;
    }
    two_scale_heads(n, x1, x, a > 0.8f ? 128 : 192, 128, out_ch);
}

void build_mobilev2(k2y_net *n, int out_ch) {
    const float a = n->alpha;
    int x = 0;
    x = n->conv(x, "Conv1", 32, 3, 2, 1, "bn_Conv1", ACT_RELU6, 0.f, false);
    struct B {
        int filters, stride, expansion, id, expand_channel;
    };
    const B blocks[17] = {{16, 1, 1, 0, 0},
                          {24, 2, 6, 1, a > 0.6f ? 48 : 0}, {24, 1, 6, 2, a > 0.6f ? 124 : 0},
                          {32, 2, 6, 3, 0}, {32, 1, 6, 4, 0}, {32, 1, 6, 5, 0},
                          {64, 2, 6, 6, 0}, {64, 1, 6, 7, 0}, {64, 1, 6, 8, 0}, {64, 1, 6, 9, 0},
                          {96, 1, 6, 10, 0}, {96, 1, 6, 11, 0}, {96, 1, 6, 12, 0},
                          {160, 2, 6, 13, 0}, {160, 1, 6, 14, 0}, {160, 1, 6, 15, 0},
                          {320, 1, 6, 16, 0}};
    int x1 = -1;
    for (const B &b : blocks) {
        const int inputs = x;
        const int in_ch = n->tensors[x].c;
        const int pw = make_divisible((float)(int)(b.filters * a), 8);
        std::string prefix = "block_" + std::to_string(b.id) + "_";
        if (b.id) {
            const int ec = b.expand_channel ? b.expand_channel : b.expansion * in_ch;
            x = n->conv(x, prefix + "expand", ec, 1, 1, 0, prefix + "expand_BN", ACT_RELU6, 0.f, false);
            if (b.id == 13) x1 = x;
        } else {
            prefix = "expanded_conv_";
        }
        x = n->dwconv(x, prefix + "depthwise", b.stride, prefix + "depthwise_BN", ACT_RELU6);
        const bool add = (in_ch == pw && b.stride == 1);
        x = n->conv(x, prefix + "project", pw, 1, 1, 0, prefix + "project_BN", ACT_NONE, 0.f, false, -1, false, add ? inputs : -1);
    }
    const int last = a > 1.0f ? make_divisible(1280 * a, 8) : 1280;
    x = n->conv(x, "Conv_1", last, 1, 1, 0, "Conv_1_bn", ACT_RELU6, 0.f, false);
    const int f = a > 0.7f ? 128 : 192;
    two_scale_heads(n, x1, x, f, f, out_ch);
}

void build_tiny(k2y_net *n, int out_ch) {
    int x = 0;
    const int f[4] = {16, 32, 64, 128};
    for (int i = 0; i < 4; ++i) {
        x = n->dbl(x, f[i], 3);
        x = n->maxpool(x, 2);
    }
    const int x1 = n->dbl(x, 256, 3);
    x = n->maxpool(x1, 2);
    x = n->dbl(x, 512, 3);
    x = n->maxpool(x, 1);
    x = n->dbl(x, 1024, 3);
    const int x2 = n->dbl(x, 256, 1);
    two_scale_heads(n, x1, x2, 512, 256, out_ch);
}

// make_last_layers (yolonet.py:218-229); `src1`/`up0` describe the (upsampled lateral ‖ skip) input of the first 1x1
int last_layers(k2y_net *n, int x, int nf, int out_ch, int *y, int src1 = -1, bool up0 = false) {
    x = n->dbl(x, nf, 1, 1, src1, up0);
    x = n->dbl(x, nf * 2, 3);
    x = n->dbl(x, nf, 1);
    x = n->dbl(x, nf * 2, 3);
    x = n->dbl(x, nf, 1);
    int t = n->dbl(x, nf * 2, 3);
    *y = n->dconv_out(t, out_ch);
    return x;
}

void build_darknet(k2y_net *n, int out_ch) {
    int x = n->dbl(0, 32, 3);
    const int nf[5] = {64, 128, 256, 512, 1024}, nb[5] = {1, 2, 8, 8, 4};
    int stage_out[5];
    for (int s = 0; s < 5; ++s) {
        x = n->dbl(x, nf[s], 3, 2);
        for (int i = 0; i < nb[s]; ++i) {
            int y = n->dbl(x, nf[s] / 2, 1);
            x = n->dbl(y, nf[s], 3, 1, -1, false, /*res=*/x);
        }
        stage_out[s] = x;
    }
    int y1, y2, y3;
    x = last_layers(n, stage_out[4], 512, out_ch, &y1);
    int lat = n->dbl(x, 256, 1);
    x = last_layers(n, lat, 256, out_ch, &y2, stage_out[3], true);
    lat = n->dbl(x, 128, 1);
    x = last_layers(n, lat, 128, out_ch, &y3, stage_out[2], true);
    n->outputs = {y1, y2, y3};
}

size_t round_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// Makes the net's device current for the duration of a call (function attributes, allocations and launches are per device).
struct DeviceGuard {
    int prev = -1;
    bool switched = false;
    explicit DeviceGuard(int dev) {
        if (cudaGetDevice(&prev) == cudaSuccess && prev != dev) switched = cudaSetDevice(dev) == cudaSuccess;
    }
    ~DeviceGuard() {
        if (switched) cudaSetDevice(prev);
    }
};

void plan_arena(k2y_net *n) {
    auto &T = n->tensors;
    for (auto &t : T) {
        t.def = -1;
        t.last_use = -1;
        t.out_index = -1;
    }
    T[0].is_input = true;
    for (size_t i = 0; i < n->layers.size(); ++i) {
        const Layer &L = n->layers[i];
        T[L.dst].def = (int)i;
        for (int s : {L.src0, L.src1, L.res})
            if (s >= 0) T[s].last_use = (int)i;
    }
    for (size_t o = 0; o < n->outputs.size(); ++o) T[n->outputs[o]].out_index = (int)o;
    // greedy first-fit over a free list, in layer order
    struct Block {
        size_t off, size;
    };
    std::vector<Block> free_list;
    size_t top = 0;
    const size_t B = (size_t)n->max_batch;
    for (size_t i = 0; i < n->layers.size(); ++i) {
        const Layer &L = n->layers[i];
        Tensor &d = T[L.dst];
        if (d.out_index < 0) {
            const size_t need = round_up(B * d.h * d.w * d.c, 64);  // 256-byte granules
            size_t best = (size_t)-1;
            for (size_t k = 0; k < free_list.size(); ++k)
                if (free_list[k].size >= need && (best == (size_t)-1 || free_list[k].size < free_list[best].size)) best = k;
            if (!n->keep_all && best != (size_t)-1) {
                d.off = free_list[best].off;
                if (free_list[best].size > need) {
                    free_list[best].off += need;
                    free_list[best].size -= need;
                } else {
                    free_list.erase(free_list.begin() + best);
                }
            } else {
                d.off = top;
                top += need;
            }
        }
        // release inputs whose last use is this layer (each layer is its own kernel, and every kernel waits for its
        // predecessor to complete before it touches activations)
        for (int s : {L.src0, L.src1, L.res}) {
            if (s < 0) continue;
            Tensor &t = T[s];
            if (t.last_use == (int)i && !t.is_input && t.out_index < 0 && !n->keep_all) {
                bool dup = false;
                for (auto &fb : free_list) dup |= (fb.off == t.off);
                if (dup) continue;
                free_list.push_back({t.off, round_up(B * t.h * t.w * t.c, 64)});
                // coalesce neighbours
                std::sort(free_list.begin(), free_list.end(), [](const Block &a, const Block &b) { return a.off < b.off; });
                for (size_t k = 0; k + 1 < free_list.size();) {
                    if (free_list[k].off + free_list[k].size == free_list[k + 1].off) {
                        free_list[k].size += free_list[k + 1].size;
                        free_list.erase(free_list.begin() + k + 1);
                    } else {
                        ++k;
                    }
                }
            }
        }
    }
    n->arena_floats = top;
}

const float *tensor_ptr(const k2y_net *n, int id) {
    const Tensor &t = n->tensors[id];
    if (t.is_input) return n->x_dev;
    if (t.out_index >= 0) return n->heads_dev[t.out_index];
    return n->arena + t.off;
}

int check_net(const k2y_net *n, const char *fn) {
    if (!n) {
        set_error("%s: net is NULL", fn);
        return K2Y_ERR_INVALID;
    }
    return K2Y_OK;
}

int issue_layers(k2y_net *n, int batch, cudaStream_t st, cudaEvent_t *ev = nullptr) {
    n->launches = 0;
    if (ev) cudaEventRecord(ev[0], st);
    if (n->x_u8) {  // np.max(img) per image, consumed by the first conv's u8 -> f32 look-up table
        cudaError_t e0 = launch_image_max_u8(n->x_u8, batch, (size_t)n->in_h * n->in_w * 3, n->img_max, st);
        if (e0 != cudaSuccess) {
            set_error("image max: launch failed: %s", cudaGetErrorString(e0));
            return K2Y_ERR_CUDA;
        }
        n->launches += 1;
    }
    auto conv_args = [&](const Layer &L) {
        const Tensor &s0 = n->tensors[L.src0];
        const Tensor &d = n->tensors[L.dst];
        ConvArgs a;
        a.src0 = tensor_ptr(n, L.src0);
        a.src1 = L.src1 >= 0 ? tensor_ptr(n, L.src1) : nullptr;
        a.residual = L.res >= 0 ? tensor_ptr(n, L.res) : nullptr;
        a.dst = const_cast<float *>(tensor_ptr(n, L.dst));
        a.w = L.d_w;
        a.scale = L.d_scale;
        a.shift = L.d_shift;
        a.w_host = L.kernel.data();
        a.scale_host = L.h_scale.data();
        a.shift_host = L.h_shift.data();
        a.B = batch;
        a.H = L.up0 ? s0.h * 2 : s0.h;
        a.W = L.up0 ? s0.w * 2 : s0.w;
        a.C0 = s0.c;
        a.C1 = L.src1 >= 0 ? n->tensors[L.src1].c : 0;
        a.up0 = L.up0 ? 1 : 0;
        a.OH = d.h;
        a.OW = d.w;
        a.N = L.cout;
        a.kh = L.kh;
        a.kw = L.kw;
        a.stride = L.stride;
        a.pad_t = L.pad_t;
        a.pad_l = L.pad_l;
        a.act = L.act;
        a.alpha = L.alpha;
        a.tc_scratch = n->tc_scratch;
        a.tc_scratch_bytes = n->tc_scratch_bytes;
        a.sm_limit = n->sm_limit;
        return a;
    };
    // one NVTX range per layer (header-only NVTX 3: a no-op unless a tool is attached); under graph capture the ranges
    // bracket the capture-time issue of each node, in eager mode (k2y_net_set_use_graph(0), k2y_net_profile) the launches
    struct NvtxRange {
        explicit NvtxRange(const char *name) { nvtxRangePushA(name); }
        ~NvtxRange() { nvtxRangePop(); }
    };
    for (size_t idx = 0; idx < n->layers.size(); ++idx) {
        const Layer &L = n->layers[idx];
        NvtxRange range(L.name.c_str());
        const Tensor &s0 = n->tensors[L.src0];
        const Tensor &d = n->tensors[L.dst];
        cudaError_t e = cudaSuccess;
        if (L.kind == L_CONV) {
            ConvArgs a = conv_args(L);
            if (n->x_u8 && n->tensors[L.src0].is_input) {
                if (!(L.kh == 3 && s0.c == 3 && L.src1 < 0 && (L.cout == 16 || L.cout == 24 || L.cout == 32))) {
                    set_error("uint8 input is only supported in front of a 3x3, Cin=3 first convolution");
                    return K2Y_ERR_STATE;
                }
                a.src_u8 = n->x_u8;
                a.img_max = n->img_max;
            }
            const long long Mrows = (long long)batch * d.h * d.w;
            ConvArgs pa = a;  // pixel-pair form (see Layer::tc2)
            const bool pair = n->math != K2Y_MATH_FP32_SIMT && L.tc2.d_hi && L.d_scale2 && (Mrows % 2) == 0;
            if (pair) {
                pa.B = 1;
                pa.H = pa.OH = 1;
                pa.W = pa.OW = (int)(Mrows / 2);
                pa.C0 = 2 * L.cin;
                pa.N = 2 * L.cout;
                pa.scale = L.d_scale2;
                pa.shift = L.d_shift2;
            }
            if (pair && tc_supported(pa, L.tc2)) {
                e = launch_conv_tc(pa, L.tc2, n->math, st);
                n->launches += tc_launch_count(pa, L.tc2, n->math);
            } else if (n->math != K2Y_MATH_FP32_SIMT && tc_supported(a, L.tc)) {
                e = launch_conv_tc(a, L.tc, n->math, st);
                n->launches += tc_launch_count(a, L.tc, n->math);
            } else {
                e = launch_conv_simt(a, st);
                n->launches += 1;
            }
        } else if (L.kind == L_DW) {
            DwArgs a;
            a.src = tensor_ptr(n, L.src0);
            a.dst = const_cast<float *>(tensor_ptr(n, L.dst));
            a.w = L.d_w;
            a.scale = L.d_scale;
            a.shift = L.d_shift;
            a.B = batch;
            a.H = s0.h;
            a.W = s0.w;
            a.C = s0.c;
            a.OH = d.h;
            a.OW = d.w;
            a.stride = L.stride;
            a.pad_t = L.pad_t;
            a.pad_l = L.pad_l;
            a.act = L.act;
            a.alpha = L.alpha;
            e = launch_dwconv(a, st);
            n->launches += 1;
        } else {
            PoolArgs a;
            a.src = tensor_ptr(n, L.src0);
            a.dst = const_cast<float *>(tensor_ptr(n, L.dst));
            a.B = batch;
            a.H = s0.h;
            a.W = s0.w;
            a.C = s0.c;
            a.OH = d.h;
            a.OW = d.w;
            a.stride = L.stride;
            e = launch_maxpool(a, st);
            n->launches += 1;
        }
        if (e != cudaSuccess) {
            set_error("layer %s: launch failed: %s", L.name.c_str(), cudaGetErrorString(e));
            return K2Y_ERR_CUDA;
        }
        if (ev) cudaEventRecord(ev[idx + 1], st);
    }
    return K2Y_OK;
}

void drop_graphs(k2y_net *n) {
    for (auto &kv : n->graphs) cudaGraphExecDestroy(kv.second);
    n->graphs.clear();
}

}  // namespace

extern "C" const char *k2y_last_error(void) { return g_err; }
extern "C" int k2y_version(void) { return 100; }
extern "C" int k2y_cuda_available(void) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n > 0 ? 1 : 0;
}

extern "C" int k2y_net_create(const char *model_def, int in_h, int in_w, float alpha, int anchor_num, int class_num,
                              int max_batch, int device, k2y_net **out) {
    if (!model_def || !out || in_h <= 0 || in_w <= 0 || anchor_num <= 0 || class_num <= 0 || max_batch <= 0) {
        set_error("k2y_net_create: bad arguments");
        return K2Y_ERR_INVALID;
    }
    if (in_h % 32 || in_w % 32) {
        set_error("k2y_net_create: input size %dx%d must be a multiple of 32", in_h, in_w);
        return K2Y_ERR_INVALID;
    }
    std::unique_ptr<k2y_net> n(new k2y_net());
    n->model_def = model_def;
    n->in_h = in_h;
    n->in_w = in_w;
    n->alpha = alpha;
    n->A = anchor_num;
    n->C = class_num;
    n->max_batch = max_batch;
    n->device = device;
    n->add_tensor(in_h, in_w, 3);
    const int out_ch = anchor_num * (class_num + 5);
    if (n->model_def == "yolo_mobilev1")
        build_mobilev1(n.get(), out_ch);
    else if (n->model_def == "yolo_mobilev2")
        build_mobilev2(n.get(), out_ch);
    else if (n->model_def == "tiny_yolo")
        build_tiny(n.get(), out_ch);
    else if (n->model_def == "yolo")
        build_darknet(n.get(), out_ch);
    else {
        set_error("k2y_net_create: unknown model_def '%s' (yolo_mobilev1|yolo_mobilev2|tiny_yolo|yolo)", model_def);
        return K2Y_ERR_INVALID;
    }
    // the depthwise and max-pool kernels move 4 channels per float4 load and store; there is no scalar form of either
    // (yolo_mobilev1 reaches such widths at alphas like 0.35 or 0.6: conv_dw_1 gets int(32 * alpha) channels)
    for (const Layer &L : n->layers)
        if ((L.kind == L_DW || L.kind == L_POOL) && L.cin % 4 != 0) {
            set_error("k2y_net_create: %s at alpha %g has %d channels; depthwise and max-pool layers need a multiple of 4",
                      L.name.c_str(), alpha, L.cin);
            return K2Y_ERR_INVALID;
        }
    plan_arena(n.get());
    *out = n.release();
    return K2Y_OK;
}

extern "C" int k2y_net_destroy(k2y_net *net) {
    if (!net) return K2Y_OK;
    drop_graphs(net);
    cudaFree(net->tc_scratch);
    net->tc_scratch = nullptr;
    for (Layer &L : net->layers) {
        cudaFree(L.d_w);
        cudaFree(L.d_scale);
        cudaFree(L.d_shift);
        tc_free(L.tc);
        tc_free(L.tc2);
        cudaFree(L.d_scale2);
        cudaFree(L.d_shift2);
        L.d_scale2 = L.d_shift2 = nullptr;
    }
    delete net;
    return K2Y_OK;
}

extern "C" int k2y_net_num_layers(const k2y_net *net, int *n) {
    if (check_net(net, "k2y_net_num_layers") || !n) return K2Y_ERR_INVALID;
    int c = 0;
    for (const Layer &L : net->layers) c += (L.kind != L_POOL);
    *n = c;
    return K2Y_OK;
}

extern "C" int k2y_net_layer_info(const k2y_net *net, int i, k2y_layer_info *info) {
    if (check_net(net, "k2y_net_layer_info") || !info) return K2Y_ERR_INVALID;
    int c = 0;
    for (const Layer &L : net->layers) {
        if (L.kind == L_POOL) continue;
        if (c++ == i) {
            memset(info, 0, sizeof(*info));
            snprintf(info->name, sizeof(info->name), "%s", L.name.c_str());
            snprintf(info->bn_name, sizeof(info->bn_name), "%s", L.bn_name.c_str());
            info->kind = L.kind == L_DW ? 1 : 0;
            info->kh = L.kh;
            info->kw = L.kw;
            info->cin = L.cin;
            info->cout = L.cout;
            info->stride = L.stride;
            info->has_bias = L.has_bias;
            return K2Y_OK;
        }
    }
    set_error("k2y_net_layer_info: index %d out of range", i);
    return K2Y_ERR_INVALID;
}

extern "C" int k2y_net_set_weight(k2y_net *net, const char *layer, const char *var, const float *data,
                                  const int64_t *dims, int ndim) {
    if (check_net(net, "k2y_net_set_weight") || !layer || !var || !data || !dims) {
        set_error("k2y_net_set_weight: bad arguments");
        return K2Y_ERR_INVALID;
    }
    const std::string ln(layer), vn(var);
    size_t count = 1;
    for (int i = 0; i < ndim; ++i) count *= (size_t)dims[i];
    for (Layer &L : net->layers) {
        if (L.kind == L_POOL) continue;
        std::vector<float> *dst = nullptr;
        size_t expect = 0;
        bool shape_ok = true;
        if (L.name == ln) {
            if (L.kind == L_CONV && vn == "kernel") {
                dst = &L.kernel;
                expect = (size_t)L.kh * L.kw * L.cin * L.cout;
                shape_ok = ndim == 4 && dims[0] == L.kh && dims[1] == L.kw && dims[2] == L.cin && dims[3] == L.cout;
            } else if (L.kind == L_DW && vn == "depthwise_kernel") {
                dst = &L.kernel;
                expect = (size_t)9 * L.cin;
                shape_ok = ndim == 4 && dims[0] == 3 && dims[1] == 3 && dims[2] == L.cin && dims[3] == 1;
            } else if (vn == "bias" && L.has_bias) {
                dst = &L.bias;
                expect = L.cout;
                shape_ok = ndim == 1;
            }
        } else if (!L.bn_name.empty() && L.bn_name == ln) {
            expect = L.cout;
            shape_ok = ndim == 1;
            if (vn == "gamma") dst = &L.gamma;
            else if (vn == "beta") dst = &L.beta;
            else if (vn == "moving_mean") dst = &L.mean;
            else if (vn == "moving_variance") dst = &L.var;
        } else {
            continue;
        }
        if (!dst) {
            set_error("k2y_net_set_weight: layer '%s' has no variable '%s'", layer, var);
            return K2Y_ERR_INVALID;
        }
        if (!shape_ok || count != expect) {
            set_error("k2y_net_set_weight: %s/%s has %zu elements (ndim %d), graph expects %zu", layer, var, count, ndim,
                      expect);
            return K2Y_ERR_INVALID;
        }
        dst->assign(data, data + count);
        net->finalized = false;
        return K2Y_OK;
    }
    set_error("k2y_net_set_weight: no layer named '%s' in %s", layer, net->model_def.c_str());
    return K2Y_ERR_INVALID;
}

extern "C" int k2y_net_finalize(k2y_net *net) {
    if (check_net(net, "k2y_net_finalize")) return K2Y_ERR_INVALID;
    DeviceGuard guard(net->device);
    drop_graphs(net);
    for (Layer &L : net->layers) {
        if (L.kind == L_POOL) continue;
        std::string missing;
        if (L.kernel.empty()) missing = L.name + (L.kind == L_DW ? "/depthwise_kernel" : "/kernel");
        else if (L.has_bias && L.bias.empty()) missing = L.name + "/bias";
        else if (!L.bn_name.empty()) {
            if (L.gamma.empty()) missing = L.bn_name + "/gamma";
            else if (L.beta.empty()) missing = L.bn_name + "/beta";
            else if (L.mean.empty()) missing = L.bn_name + "/moving_mean";
            else if (L.var.empty()) missing = L.bn_name + "/moving_variance";
        }
        if (!missing.empty()) {
            set_error("k2y_net_finalize: weights not set: %s", missing.c_str());
            return K2Y_ERR_STATE;
        }
        // Fold BN:  y = (x - mean) * gamma * rsqrt(var + eps) + beta  ->  x * scale + shift
        std::vector<float> scale(L.cout, 1.f), shift(L.cout, 0.f);
        for (int c = 0; c < L.cout; ++c) {
            if (!L.bn_name.empty()) {
                const float inv = L.gamma[c] / std::sqrt(L.var[c] + BN_EPS);
                scale[c] = inv;
                shift[c] = L.beta[c] - L.mean[c] * inv;
            }
            if (L.has_bias) shift[c] += L.bias[c] * scale[c];
        }
        cudaFree(L.d_w);
        cudaFree(L.d_scale);
        cudaFree(L.d_shift);
        L.d_w = L.d_scale = L.d_shift = nullptr;
        K2Y_CUDA_CHECK(cudaMalloc(&L.d_w, L.kernel.size() * sizeof(float)));
        K2Y_CUDA_CHECK(cudaMalloc(&L.d_scale, L.cout * sizeof(float)));
        K2Y_CUDA_CHECK(cudaMalloc(&L.d_shift, L.cout * sizeof(float)));
        // Keras HWIO flattened == [K][N]; depthwise (3,3,C,1) flattened == [9][C]
        K2Y_CUDA_CHECK(cudaMemcpy(L.d_w, L.kernel.data(), L.kernel.size() * sizeof(float), cudaMemcpyHostToDevice));
        K2Y_CUDA_CHECK(cudaMemcpy(L.d_scale, scale.data(), L.cout * sizeof(float), cudaMemcpyHostToDevice));
        K2Y_CUDA_CHECK(cudaMemcpy(L.d_shift, shift.data(), L.cout * sizeof(float), cudaMemcpyHostToDevice));
        L.h_scale = scale;
        L.h_shift = shift;
        if (L.kind == L_CONV) {
            int rc = tc_pack(L.tc, L.kernel.data(), L.kh * L.kw * L.cin, L.cout);
            if (rc != K2Y_OK) return rc;
            tc_free(L.tc2);
            cudaFree(L.d_scale2);
            cudaFree(L.d_shift2);
            L.d_scale2 = L.d_shift2 = nullptr;
            if (L.kh == 1 && L.stride == 1 && L.src1 < 0 && !L.up0 && L.cin <= 32 && (L.cin % 2) == 0 && L.cout <= 128 && (L.cout % 4) == 0) {
                const int K = L.cin, N = L.cout;
                std::vector<float> wd((size_t)4 * K * N, 0.f), sc2(2 * N), sh2(2 * N);
                for (int k = 0; k < K; ++k)
                    for (int nn = 0; nn < N; ++nn) {
                        wd[(size_t)k * 2 * N + nn] = L.kernel[(size_t)k * N + nn];
                        wd[(size_t)(K + k) * 2 * N + N + nn] = L.kernel[(size_t)k * N + nn];
                    }
                for (int nn = 0; nn < N; ++nn) {
                    sc2[nn] = sc2[N + nn] = scale[nn];
                    sh2[nn] = sh2[N + nn] = shift[nn];
                }
                rc = tc_pack(L.tc2, wd.data(), 2 * K, 2 * N);
                if (rc != K2Y_OK) return rc;
                K2Y_CUDA_CHECK(cudaMalloc(&L.d_scale2, 2 * N * sizeof(float)));
                K2Y_CUDA_CHECK(cudaMalloc(&L.d_shift2, 2 * N * sizeof(float)));
                K2Y_CUDA_CHECK(cudaMemcpy(L.d_scale2, sc2.data(), 2 * N * sizeof(float), cudaMemcpyHostToDevice));
                K2Y_CUDA_CHECK(cudaMemcpy(L.d_shift2, sh2.data(), 2 * N * sizeof(float), cudaMemcpyHostToDevice));
            }
        }
    }
    // split-K scratch of this net: the largest bound over its dense convs at max_batch
    size_t scratch = 0;
    for (const Layer &L : net->layers) {
        if (L.kind != L_CONV) continue;
        const Tensor &d = net->tensors[L.dst];
        ConvArgs a;
        memset(&a, 0, sizeof(a));
        a.B = net->max_batch;
        a.OH = d.h;
        a.OW = d.w;
        a.N = L.cout;
        scratch = std::max(scratch, tc_scratch_bound(a, L.tc));
    }
    if (scratch != net->tc_scratch_bytes) {
        cudaFree(net->tc_scratch);
        net->tc_scratch = nullptr;
        net->tc_scratch_bytes = 0;
        if (scratch) {
            K2Y_CUDA_CHECK(cudaMalloc(&net->tc_scratch, scratch));
            net->tc_scratch_bytes = scratch;
        }
    }
    net->finalized = true;
    return K2Y_OK;
}

extern "C" int k2y_net_set_math(k2y_net *net, int math_mode) {
    if (check_net(net, "k2y_net_set_math")) return K2Y_ERR_INVALID;
    if (math_mode != K2Y_MATH_FP32_SIMT && math_mode != K2Y_MATH_TC_3XTF32 && math_mode != K2Y_MATH_TC_TF32 &&
        math_mode != K2Y_MATH_TC_BF16X3) {
        set_error("k2y_net_set_math: unknown mode %d", math_mode);
        return K2Y_ERR_INVALID;
    }
    if (math_mode != net->math) drop_graphs(net);
    net->math = math_mode;
    return K2Y_OK;
}
extern "C" int k2y_net_get_math(const k2y_net *net, int *math_mode) {
    if (check_net(net, "k2y_net_get_math") || !math_mode) return K2Y_ERR_INVALID;
    *math_mode = net->math;
    return K2Y_OK;
}
extern "C" int k2y_net_set_use_graph(k2y_net *net, int use_graph) {
    if (check_net(net, "k2y_net_set_use_graph")) return K2Y_ERR_INVALID;
    net->use_graph = use_graph != 0;
    return K2Y_OK;
}
extern "C" int k2y_net_set_keep_all(k2y_net *net, int keep_all) {
    if (check_net(net, "k2y_net_set_keep_all")) return K2Y_ERR_INVALID;
    net->keep_all = keep_all != 0;
    net->bound = false;
    drop_graphs(net);
    plan_arena(net);
    return K2Y_OK;
}

extern "C" int k2y_net_num_outputs(const k2y_net *net, int *n) {
    if (check_net(net, "k2y_net_num_outputs") || !n) return K2Y_ERR_INVALID;
    *n = (int)net->outputs.size();
    return K2Y_OK;
}
extern "C" int k2y_net_output_shape(const k2y_net *net, int l, int *h, int *w, int *c) {
    if (check_net(net, "k2y_net_output_shape") || l < 0 || l >= (int)net->outputs.size()) {
        set_error("k2y_net_output_shape: bad output index");
        return K2Y_ERR_INVALID;
    }
    const Tensor &t = net->tensors[net->outputs[l]];
    if (h) *h = t.h;
    if (w) *w = t.w;
    if (c) *c = t.c;
    return K2Y_OK;
}
extern "C" int k2y_net_workspace_bytes(const k2y_net *net, size_t *bytes) {
    if (check_net(net, "k2y_net_workspace_bytes") || !bytes) return K2Y_ERR_INVALID;
    *bytes = net->arena_floats * sizeof(float) + 256;
    return K2Y_OK;
}

extern "C" int k2y_net_bind(k2y_net *net, void *workspace, size_t workspace_bytes, const float *x_dev,
                            float *const *heads_dev, int n_heads) {
    if (check_net(net, "k2y_net_bind")) return K2Y_ERR_INVALID;
    if (!workspace || !x_dev || !heads_dev || n_heads != (int)net->outputs.size()) {
        set_error("k2y_net_bind: null pointer or wrong number of heads (%d, expected %zu)", n_heads, net->outputs.size());
        return K2Y_ERR_INVALID;
    }
    const uintptr_t base = ((uintptr_t)workspace + 255) & ~(uintptr_t)255;
    if (base + net->arena_floats * sizeof(float) > (uintptr_t)workspace + workspace_bytes) {
        set_error("k2y_net_bind: workspace too small (%zu bytes, need %zu)", workspace_bytes,
                  net->arena_floats * sizeof(float) + 256);
        return K2Y_ERR_INVALID;
    }
    if (((uintptr_t)x_dev & 15) != 0) {
        set_error("k2y_net_bind: x_dev must be 16-byte aligned");
        return K2Y_ERR_INVALID;
    }
    net->arena = (float *)base;
    net->x_dev = x_dev;
    net->heads_dev.assign(heads_dev, heads_dev + n_heads);
    for (float *h : net->heads_dev)
        if (!h || ((uintptr_t)h & 15) != 0) {
            set_error("k2y_net_bind: head buffers must be non-null and 16-byte aligned");
            return K2Y_ERR_INVALID;
        }
    net->bound = true;
    drop_graphs(net);
    return K2Y_OK;
}

extern "C" int k2y_net_bind_u8(k2y_net *net, const unsigned char *x_u8_dev, int32_t *img_max_dev) {
    if (check_net(net, "k2y_net_bind_u8")) return K2Y_ERR_INVALID;
    if ((x_u8_dev == nullptr) != (img_max_dev == nullptr) || (((uintptr_t)x_u8_dev) & 15) != 0) {
        set_error("k2y_net_bind_u8: pass both pointers (16-byte aligned input) or both NULL");
        return K2Y_ERR_INVALID;
    }
    net->x_u8 = x_u8_dev;
    net->img_max = img_max_dev;
    return K2Y_OK;
}

extern "C" int k2y_net_bind_input(k2y_net *net, const float *x_dev) {
    if (check_net(net, "k2y_net_bind_input")) return K2Y_ERR_INVALID;
    if (!net->bound) {
        set_error("k2y_net_bind_input: call k2y_net_bind first");
        return K2Y_ERR_STATE;
    }
    if (!x_dev || ((uintptr_t)x_dev & 15) != 0) {
        set_error("k2y_net_bind_input: x_dev must be non-null and 16-byte aligned");
        return K2Y_ERR_INVALID;
    }
    net->x_dev = x_dev;
    return K2Y_OK;
}

extern "C" int k2y_net_set_sm_limit(k2y_net *net, int sms) {
    if (check_net(net, "k2y_net_set_sm_limit")) return K2Y_ERR_INVALID;
    if (sms < 0) {
        set_error("k2y_net_set_sm_limit: sms must be >= 0 (0 = whole device)");
        return K2Y_ERR_INVALID;
    }
    if (sms != net->sm_limit) drop_graphs(net);
    net->sm_limit = sms;
    return K2Y_OK;
}

extern "C" int k2y_net_bind_heads(k2y_net *net, float *const *heads_dev, int n_heads) {
    if (check_net(net, "k2y_net_bind_heads")) return K2Y_ERR_INVALID;
    if (!net->bound) {
        set_error("k2y_net_bind_heads: call k2y_net_bind first");
        return K2Y_ERR_STATE;
    }
    if (!heads_dev || n_heads != (int)net->outputs.size()) {
        set_error("k2y_net_bind_heads: null pointer or wrong number of heads (%d, expected %zu)", n_heads, net->outputs.size());
        return K2Y_ERR_INVALID;
    }
    for (int l = 0; l < n_heads; ++l)
        if (!heads_dev[l] || ((uintptr_t)heads_dev[l] & 15) != 0) {
            set_error("k2y_net_bind_heads: head buffers must be non-null and 16-byte aligned");
            return K2Y_ERR_INVALID;
        }
    net->heads_dev.assign(heads_dev, heads_dev + n_heads);
    return K2Y_OK;
}

extern "C" int k2y_net_run(k2y_net *net, int batch, void *stream) {
    if (check_net(net, "k2y_net_run")) return K2Y_ERR_INVALID;
    if (!net->finalized || !net->bound) {
        set_error("k2y_net_run: net must be finalized (weights) and bound (buffers) first");
        return K2Y_ERR_STATE;
    }
    if (batch <= 0 || batch > net->max_batch) {
        set_error("k2y_net_run: batch %d outside 1..%d", batch, net->max_batch);
        return K2Y_ERR_INVALID;
    }
    cudaStream_t st = (cudaStream_t)stream;
    DeviceGuard guard(net->device);
    net->last_batch = batch;
    if (!net->use_graph) return issue_layers(net, batch, st);
    const auto key = std::make_tuple(batch, (const void *)net->x_dev, (const void *)net->x_u8, (const void *)net->img_max,
                                     (const void *)net->heads_dev[0]);
    auto it = net->graphs.find(key);
    if (it == net->graphs.end()) {
        cudaGraph_t g = nullptr;
        cudaStream_t cap = st;
        bool own = false;
        if (cap == nullptr || cap == cudaStreamLegacy) {  // the legacy default stream cannot be captured
            K2Y_CUDA_CHECK(cudaStreamCreateWithFlags(&cap, cudaStreamNonBlocking));
            own = true;
        }
        K2Y_CUDA_CHECK(cudaStreamBeginCapture(cap, cudaStreamCaptureModeThreadLocal));
        int rc = issue_layers(net, batch, cap);
        cudaError_t e = cudaStreamEndCapture(cap, &g);
        if (own) cudaStreamDestroy(cap);
        if (rc != K2Y_OK) {
            if (g) cudaGraphDestroy(g);
            return rc;
        }
        K2Y_CUDA_CHECK(e);
        cudaGraphExec_t ge = nullptr;
        K2Y_CUDA_CHECK(cudaGraphInstantiate(&ge, g, 0));
        cudaGraphDestroy(g);
        it = net->graphs.emplace(key, ge).first;
    }
    K2Y_CUDA_CHECK(cudaGraphLaunch(it->second, st));
    return K2Y_OK;
}

extern "C" int k2y_net_predict_host(k2y_net *net, const float *x_host, int batch, float *const *heads_host, void *stream) {
    if (check_net(net, "k2y_net_predict_host")) return K2Y_ERR_INVALID;
    if (!x_host || !heads_host) {
        set_error("k2y_net_predict_host: null pointer");
        return K2Y_ERR_INVALID;
    }
    if (!net->bound) {
        set_error("k2y_net_predict_host: net must be bound first");
        return K2Y_ERR_STATE;
    }
    if (batch <= 0 || batch > net->max_batch) {
        set_error("k2y_net_predict_host: batch %d outside 1..%d", batch, net->max_batch);
        return K2Y_ERR_INVALID;
    }
    cudaStream_t st = (cudaStream_t)stream;
    DeviceGuard guard(net->device);
    if (net->x_u8) {  // predict() takes float32 pixels: leave the uint8 front end, or the first conv would read the stale u8 buffer
        net->x_u8 = nullptr;
        net->img_max = nullptr;
    }
    const size_t in_bytes = (size_t)batch * net->in_h * net->in_w * 3 * sizeof(float);
    K2Y_CUDA_CHECK(cudaMemcpyAsync(const_cast<float *>(net->x_dev), x_host, in_bytes, cudaMemcpyHostToDevice, st));
    int rc = k2y_net_run(net, batch, stream);
    if (rc != K2Y_OK) return rc;
    for (size_t l = 0; l < net->outputs.size(); ++l) {
        const Tensor &t = net->tensors[net->outputs[l]];
        K2Y_CUDA_CHECK(cudaMemcpyAsync(heads_host[l], net->heads_dev[l], (size_t)batch * t.h * t.w * t.c * sizeof(float),
                                       cudaMemcpyDeviceToHost, st));
    }
    K2Y_CUDA_CHECK(cudaStreamSynchronize(st));
    return K2Y_OK;
}

extern "C" int k2y_net_launches_per_run(const k2y_net *net, int *n) {
    if (check_net(net, "k2y_net_launches_per_run") || !n) return K2Y_ERR_INVALID;
    *n = net->launches > 0 ? net->launches : (int)net->layers.size();  // exact after the first run (split-K adds reducers)
    return K2Y_OK;
}

extern "C" int k2y_net_read_layer(k2y_net *net, const char *name, int batch, float *host, size_t host_floats, int *h,
                                  int *w, int *c) {
    if (check_net(net, "k2y_net_read_layer") || !name || !host) return K2Y_ERR_INVALID;
    if (!net->keep_all || !net->bound) {
        set_error("k2y_net_read_layer: requires set_keep_all(1) before bind");
        return K2Y_ERR_STATE;
    }
    for (const Layer &L : net->layers) {
        if (L.name != name) continue;
        const Tensor &t = net->tensors[L.dst];
        const size_t cnt = (size_t)batch * t.h * t.w * t.c;
        if (cnt > host_floats) {
            set_error("k2y_net_read_layer: host buffer too small (%zu < %zu)", host_floats, cnt);
            return K2Y_ERR_INVALID;
        }
        K2Y_CUDA_CHECK(cudaDeviceSynchronize());
        K2Y_CUDA_CHECK(cudaMemcpy(host, tensor_ptr(net, L.dst), cnt * sizeof(float), cudaMemcpyDeviceToHost));
        if (h) *h = t.h;
        if (w) *w = t.w;
        if (c) *c = t.c;
        return K2Y_OK;
    }
    set_error("k2y_net_read_layer: no layer named '%s'", name);
    return K2Y_ERR_INVALID;
}

extern "C" int k2y_net_schedule_len(const k2y_net *net, int *n) {
    if (check_net(net, "k2y_net_schedule_len") || !n) return K2Y_ERR_INVALID;
    *n = (int)net->layers.size();
    return K2Y_OK;
}

extern "C" int k2y_net_profile(k2y_net *net, int batch, void *stream, float *ms_per_launch, int n) {
    if (check_net(net, "k2y_net_profile") || !ms_per_launch) return K2Y_ERR_INVALID;
    if (!net->finalized || !net->bound) {
        set_error("k2y_net_profile: net must be finalized and bound first");
        return K2Y_ERR_STATE;
    }
    const int L = (int)net->layers.size();
    if (n < L || batch <= 0 || batch > net->max_batch) {
        set_error("k2y_net_profile: need room for %d launches, batch 1..%d", L, net->max_batch);
        return K2Y_ERR_INVALID;
    }
    DeviceGuard guard(net->device);
    std::vector<cudaEvent_t> ev(L + 1);
    for (auto &e : ev) K2Y_CUDA_CHECK(cudaEventCreate(&e));
    cudaStream_t st = (cudaStream_t)stream;
    int rc = issue_layers(net, batch, st, ev.data());
    if (rc == K2Y_OK) {
        cudaError_t e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) {
            set_error("k2y_net_profile: %s", cudaGetErrorString(e));
            rc = K2Y_ERR_CUDA;
        }
    }
    if (rc == K2Y_OK)
        for (int i = 0; i < L; ++i) cudaEventElapsedTime(&ms_per_launch[i], ev[i], ev[i + 1]);
    for (auto &e : ev) cudaEventDestroy(e);
    return rc;
}

extern "C" int k2y_net_launch_info(const k2y_net *net, int i, char *name, int name_len, double *flops_per_image,
                                   double *bytes_per_image) {
    if (check_net(net, "k2y_net_launch_info") || i < 0 || i >= (int)net->layers.size()) {
        set_error("k2y_net_launch_info: index out of range");
        return K2Y_ERR_INVALID;
    }
    const Layer &L = net->layers[i];
    const Tensor &d = net->tensors[L.dst];
    if (name && name_len > 0) snprintf(name, name_len, "%s", L.name.c_str());
    double in_elems = 0;
    for (int s : {L.src0, L.src1, L.res})
        if (s >= 0) in_elems += (double)net->tensors[s].h * net->tensors[s].w * net->tensors[s].c;
    const double out_elems = (double)d.h * d.w * d.c;
    double macs = 0;
    if (L.kind == L_CONV) macs = out_elems * L.kh * L.kw * L.cin;
    else if (L.kind == L_DW) macs = out_elems * 9;
    const double bytes = 4.0 * (in_elems + out_elems);  // algorithmic: activations read once + written once
    if (flops_per_image) *flops_per_image = 2.0 * macs;
    if (bytes_per_image) *bytes_per_image = bytes;
    return K2Y_OK;
}

// Single-layer hook for kernel parity tests: one dense conv on device tensors, weights given in the Keras layout.
extern "C" int k2y_conv2d(const float *src0_dev, const float *src1_dev, const float *residual_dev, float *dst_dev,
                          const float *kernel_host, const float *scale_host, const float *shift_host, int batch, int h, int w,
                          int c0, int c1, int up0, int cout, int ksize, int stride, int pad_mode, int act, float alpha,
                          int math_mode, void *stream) {
    if (!src0_dev || !dst_dev || !kernel_host || !scale_host || !shift_host || batch <= 0) {
        set_error("k2y_conv2d: bad arguments");
        return K2Y_ERR_INVALID;
    }
    ConvArgs a;
    a.src0 = src0_dev;
    a.src1 = c1 > 0 ? src1_dev : nullptr;
    a.residual = residual_dev;
    a.dst = dst_dev;
    a.B = batch;
    a.H = h;
    a.W = w;
    a.C0 = c0;
    a.C1 = c1;
    a.up0 = up0;
    a.N = cout;
    a.kh = a.kw = ksize;
    a.stride = stride;
    if (pad_mode == 0) {
        a.pad_t = a.pad_l = ksize / 2;
        a.OH = h;
        a.OW = w;
    } else if (pad_mode == 1) {
        a.pad_t = a.pad_l = 1;
        a.OH = (h + 2 - ksize) / stride + 1;
        a.OW = (w + 2 - ksize) / stride + 1;
    } else {
        a.pad_t = a.pad_l = 1;
        a.OH = (h + 1 - ksize) / stride + 1;
        a.OW = (w + 1 - ksize) / stride + 1;
    }
    a.act = act;
    a.alpha = alpha;
    const int K = ksize * ksize * (c0 + c1);
    float *d_w = nullptr, *d_sc = nullptr, *d_sh = nullptr;
    K2Y_CUDA_CHECK(cudaMalloc(&d_w, (size_t)K * cout * sizeof(float)));
    K2Y_CUDA_CHECK(cudaMalloc(&d_sc, cout * sizeof(float)));
    K2Y_CUDA_CHECK(cudaMalloc(&d_sh, cout * sizeof(float)));
    K2Y_CUDA_CHECK(cudaMemcpy(d_w, kernel_host, (size_t)K * cout * sizeof(float), cudaMemcpyHostToDevice));
    K2Y_CUDA_CHECK(cudaMemcpy(d_sc, scale_host, cout * sizeof(float), cudaMemcpyHostToDevice));
    K2Y_CUDA_CHECK(cudaMemcpy(d_sh, shift_host, cout * sizeof(float), cudaMemcpyHostToDevice));
    a.w = d_w;
    a.scale = d_sc;
    a.shift = d_sh;
    a.w_host = kernel_host;
    a.scale_host = scale_host;
    a.shift_host = shift_host;
    TcWeights tw;
    int rc = K2Y_OK;
    cudaError_t e = cudaSuccess;
    if (math_mode == K2Y_MATH_FP32_SIMT) {
        e = launch_conv_simt(a, (cudaStream_t)stream);
    } else {
        rc = tc_pack(tw, kernel_host, K, cout);
        if (rc == K2Y_OK) {
            if (!tc_supported(a, tw)) {
                set_error("k2y_conv2d: shape not supported by the tensor-core path");
                rc = K2Y_ERR_INVALID;
            } else {
                e = launch_conv_tc(a, tw, math_mode, (cudaStream_t)stream);
            }
        }
    }
    if (rc == K2Y_OK && e == cudaSuccess) e = cudaStreamSynchronize((cudaStream_t)stream);
    if (rc == K2Y_OK && e != cudaSuccess) {
        set_error("k2y_conv2d: %s", cudaGetErrorString(e));
        rc = K2Y_ERR_CUDA;
    }
    tc_free(tw);
    cudaFree(d_w);
    cudaFree(d_sc);
    cudaFree(d_sh);
    return rc;
}
