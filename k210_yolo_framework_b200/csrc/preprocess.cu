// Image pre-processing on the GPU: the reference's aspect-preserving "letterbox" resize (tools/utils.py:372-400) for
// uint8 HWC images of any size -> uint8 [in_h, in_w, 3], the tensor the uint8 front end of the network consumes
// (k2y_net_bind_u8: per-image max + `img / np.max(img)` fused into the first convolution).
//
// The resampling restates skimage 0.15 `warp(img, aff.inverse, output_shape, order=1, mode='constant', cval=0, clip=True,
// preserve_range=True).astype('uint8')` (third-party, unpinned — see oracle/preprocess_ref.py): float64 bilinear
// interpolation between floor/ceil neighbours with zero outside the image, no half-pixel shift, clip to the input's
// [min, max] (exact-zero fill pixels stay zero when 0 is outside that range), truncation to uint8.  Every double
// operation is an explicit round-to-nearest intrinsic so that nvcc cannot contract a*b+c into an FMA: results are
// bit-identical to the numpy oracle.
#include <vector>

#include "common.h"

// A batch is n images of different sizes packed back to back in one device buffer.  What is letterboxed is a VIEW: a window
// (y0, x0, th, tw) of one of those images, treated as an image of its own (the whole image is the window (0, 0, h, w)); several
// views may share an image.  A mirrored view is the window flipped left to right: the warp samples the same positions and
// fetches column tw - 1 - c where it would fetch c, so it equals the letterbox of np.fliplr(window) bit for bit (folding the
// flip into the inverse matrix instead would round tw - 1 - x differently).  The descriptors travel by value in the kernel parameters (__grid_constant__: indexed in place,
// never copied to local memory), LB_MAX_IMAGES views per launch.  Pass 1 reduces each window's min and max into the scratch as
// (255 - min, max), both with atomicMax, so that one memset to zero initialises it; pass 2 is the bilinear warp, one thread
// per output pixel, grid (pixel tile, view).
namespace k2y {
namespace {

constexpr int LB_MAX_IMAGES = 48;
constexpr int LB_THREADS = 256;
constexpr int LB_CHUNK = LB_THREADS * 64;   // source bytes per block of pass 1

struct LbImage {
    long long offset;   // byte offset of the window's first pixel in the packed source buffer
    int pitch;          // pixels per row of the image the window lies in
    int h, w;           // the window's size
    int y0, x0;         // its origin in the image (only reported, view_yx)
    int mirror;         // nonzero: the window flipped left to right
    double m[6];        // the first two rows of the inverse affine matrix, in window coordinates
};

struct LbBatch {
    const unsigned char *src;
    unsigned char *dst;     // [n][dh][dw][3]
    int *minmax;            // [n][2]: 255 - min, max
    float *image_hw;        // [n][2] (h, w) of the window, or null
    float *view_yx;         // [n][2] (y0, x0) of the window, or null
    int dh, dw;
    LbImage img[LB_MAX_IMAGES];
};
static_assert(sizeof(LbBatch) <= 4096, "letterbox descriptors must fit the kernel parameter space");

__device__ __forceinline__ unsigned fold_min4(unsigned v) { return min(min(v & 255u, (v >> 8) & 255u), min((v >> 16) & 255u, v >> 24)); }
__device__ __forceinline__ unsigned fold_max4(unsigned v) { return max(max(v & 255u, (v >> 8) & 255u), max((v >> 16) & 255u, v >> 24)); }

// min / max of the bytes [s, s + len) into four byte lanes each: single bytes up to the first 16-byte boundary, then 16 bytes
// per load, then the rest
__device__ __forceinline__ void minmax_run(const unsigned char *s, size_t len, unsigned &lo4, unsigned &hi4) {
    const size_t head = min(len, (size_t)((16 - ((uintptr_t)s & 15)) & 15));
    const uint4 *v = reinterpret_cast<const uint4 *>(s + head);
    const int nv = (int)((len - head) / 16);
    for (int i = threadIdx.x; i < nv; i += LB_THREADS) {
        const uint4 q = __ldg(v + i);
        lo4 = __vminu4(lo4, __vminu4(__vminu4(q.x, q.y), __vminu4(q.z, q.w)));
        hi4 = __vmaxu4(hi4, __vmaxu4(__vmaxu4(q.x, q.y), __vmaxu4(q.z, q.w)));
    }
    const size_t body = head + (size_t)nv * 16;
    for (size_t i = threadIdx.x; i < head + (len - body); i += LB_THREADS) {
        const unsigned b = __ldg(s + (i < head ? i : body + (i - head))) * 0x01010101u;
        lo4 = __vminu4(lo4, b);
        hi4 = __vmaxu4(hi4, b);
    }
}

// A window is `rows` runs of `run` bytes, `pitch` bytes apart (one run when its rows are whole image rows).  A block takes one
// LB_CHUNK piece of a run longer than LB_CHUNK, else as many whole runs as fit LB_CHUNK.
struct LbRuns {
    size_t run, pitch;
    int rows, pieces, per_block;
    __host__ __device__ LbRuns(const LbImage &im) {
        const bool whole_rows = im.w == im.pitch;
        run = (size_t)im.w * 3 * (whole_rows ? (size_t)im.h : 1);
        pitch = (size_t)im.pitch * 3;
        rows = whole_rows ? 1 : im.h;
        pieces = (int)((run + LB_CHUNK - 1) / LB_CHUNK);
        per_block = pieces > 1 ? 1 : (int)(LB_CHUNK / run);
    }
    __host__ __device__ size_t blocks() const { return pieces > 1 ? (size_t)rows * pieces : ((size_t)rows + per_block - 1) / per_block; }
};

__global__ void __launch_bounds__(LB_THREADS) letterbox_minmax_kernel(const __grid_constant__ LbBatch p) {
    const LbImage &im = p.img[blockIdx.y];
    const LbRuns r(im);
    if (blockIdx.x >= r.blocks()) return;
    const unsigned char *s = p.src + im.offset;
    unsigned lo4 = 0xffffffffu, hi4 = 0u;   // four byte lanes each
    if (r.pieces > 1) {
        const size_t row = blockIdx.x / r.pieces, begin = (size_t)(blockIdx.x % r.pieces) * LB_CHUNK;
        minmax_run(s + row * r.pitch + begin, min(r.run - begin, (size_t)LB_CHUNK), lo4, hi4);
    } else {
        const int row0 = blockIdx.x * r.per_block, row1 = min(r.rows, row0 + r.per_block);
        for (int row = row0; row < row1; ++row) minmax_run(s + row * r.pitch, r.run, lo4, hi4);
    }
    int lo = (int)fold_min4(lo4), hi = (int)fold_max4(hi4);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
        hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    }
    __shared__ int s_lo[LB_THREADS / 32], s_hi[LB_THREADS / 32];
    if ((threadIdx.x & 31) == 0) {
        s_lo[threadIdx.x >> 5] = lo;
        s_hi[threadIdx.x >> 5] = hi;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int k = 1; k < LB_THREADS / 32; ++k) {
            lo = min(lo, s_lo[k]);
            hi = max(hi, s_hi[k]);
        }
        atomicMax(&p.minmax[2 * blockIdx.y], 255 - lo);
        atomicMax(&p.minmax[2 * blockIdx.y + 1], hi);
    }
}

// the bounds test is on the sampled column c; a mirrored view fetches the window's column sw - 1 - c
__device__ __forceinline__ double pix_or_zero(const unsigned char *src, int sh, int sw, int pitch, bool mirror, double r, double c,
                                              int ch) {
    if (!(r >= 0.0 && r < (double)sh && c >= 0.0 && c < (double)sw)) return 0.0;
    const int col = mirror ? sw - 1 - (int)c : (int)c;
    return (double)src[((size_t)(int)r * pitch + col) * 3 + ch];
}

__global__ void __launch_bounds__(LB_THREADS) letterbox_warp_kernel(const __grid_constant__ LbBatch p) {
    const int b = blockIdx.y;
    const LbImage &im = p.img[b];
    if (p.image_hw && blockIdx.x == 0 && threadIdx.x == 0) {
        p.image_hw[2 * b] = (float)im.h;
        p.image_hw[2 * b + 1] = (float)im.w;
    }
    if (p.view_yx && blockIdx.x == 0 && threadIdx.x == 0) {
        p.view_yx[2 * b] = (float)im.y0;
        p.view_yx[2 * b + 1] = (float)im.x0;
    }
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= p.dh * p.dw) return;
    const unsigned char *src = p.src + im.offset;
    const int sh = im.h, sw = im.w, pitch = im.pitch;
    const bool mir = im.mirror != 0;
    const double r = (double)(idx / p.dw), c = (double)(idx % p.dw);
    const double x = __dadd_rn(__dadd_rn(__dmul_rn(im.m[0], c), __dmul_rn(im.m[1], r)), im.m[2]);
    const double y = __dadd_rn(__dadd_rn(__dmul_rn(im.m[3], c), __dmul_rn(im.m[4], r)), im.m[5]);
    const double minr = floor(y), minc = floor(x), maxr = ceil(y), maxc = ceil(x);
    const double dr = __dsub_rn(y, minr), dc = __dsub_rn(x, minc);
    const double wr = __dsub_rn(1.0, dr), wc = __dsub_rn(1.0, dc);
    const double lo = (double)(255 - p.minmax[2 * b]), hi = (double)p.minmax[2 * b + 1];
    const bool keep_fill = lo > 0.0;  // 0 (cval) lies outside [min, max]: exact-zero pixels are preserved by the clip
    unsigned char *dst = p.dst + ((size_t)b * p.dh * p.dw + idx) * 3;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        const double p00 = pix_or_zero(src, sh, sw, pitch, mir, minr, minc, ch), p01 = pix_or_zero(src, sh, sw, pitch, mir, minr, maxc, ch);
        const double p10 = pix_or_zero(src, sh, sw, pitch, mir, maxr, minc, ch), p11 = pix_or_zero(src, sh, sw, pitch, mir, maxr, maxc, ch);
        const double top = __dadd_rn(__dmul_rn(wc, p00), __dmul_rn(dc, p01));
        const double bot = __dadd_rn(__dmul_rn(wc, p10), __dmul_rn(dc, p11));
        double o = __dadd_rn(__dmul_rn(wr, top), __dmul_rn(dr, bot));
        if (!(keep_fill && o == 0.0)) o = fmin(fmax(o, lo), hi);
        dst[ch] = (unsigned char)(int)o;
    }
}

}  // namespace
}  // namespace k2y

extern "C" int k2y_letterbox_u8_views_mirror(const unsigned char *src_dev, int n_views, const long long *offsets_host,
                                             const int *hw_host, const int *windows_host, const int *mirror_host,
                                             const double *inv_matrices_host, unsigned char *dst_dev, int dst_h, int dst_w,
                                             float *image_hw_dev, float *view_yx_dev, int *minmax_dev, void *stream) {
    using namespace k2y;
    if (!src_dev || n_views <= 0 || !offsets_host || !hw_host || !windows_host || !inv_matrices_host || !dst_dev || !minmax_dev ||
        dst_h <= 0 || dst_w <= 0 || (long long)dst_h * dst_w > (1LL << 30)) {
        set_error("k2y_letterbox_u8_views: bad arguments");
        return K2Y_ERR_INVALID;
    }
    for (int i = 0; i < n_views; ++i) {
        const int h = hw_host[2 * i], w = hw_host[2 * i + 1], *win = windows_host + 4 * i;
        if (offsets_host[i] < 0 || h <= 0 || w <= 0) {
            set_error("k2y_letterbox_u8_views: the image of view %d has offset %lld and size %dx%d", i, offsets_host[i], h, w);
            return K2Y_ERR_INVALID;
        }
        if (win[0] < 0 || win[1] < 0 || win[2] <= 0 || win[3] <= 0 || win[2] > h - win[0] || win[3] > w - win[1]) {
            set_error("k2y_letterbox_u8_views: window (%d, %d, %d, %d) of view %d is not inside its %dx%d image", win[0], win[1], win[2],
                      win[3], i, h, w);
            return K2Y_ERR_INVALID;
        }
    }
    cudaStream_t st = (cudaStream_t)stream;
    K2Y_CUDA_CHECK(cudaMemsetAsync(minmax_dev, 0, sizeof(int) * 2 * (size_t)n_views, st));
    const size_t plane = (size_t)dst_h * dst_w * 3;
    for (int g0 = 0; g0 < n_views; g0 += LB_MAX_IMAGES) {
        const int g = n_views - g0 < LB_MAX_IMAGES ? n_views - g0 : LB_MAX_IMAGES;
        LbBatch p;
        memset(&p, 0, sizeof(p));
        p.src = src_dev;
        p.dst = dst_dev + plane * g0;
        p.minmax = minmax_dev + 2 * g0;
        p.image_hw = image_hw_dev ? image_hw_dev + 2 * g0 : nullptr;
        p.view_yx = view_yx_dev ? view_yx_dev + 2 * g0 : nullptr;
        p.dh = dst_h;
        p.dw = dst_w;
        size_t max_blocks = 0;
        for (int i = 0; i < g; ++i) {
            LbImage &im = p.img[i];
            const int *win = windows_host + 4 * (g0 + i);
            im.pitch = hw_host[2 * (g0 + i) + 1];
            im.y0 = win[0];
            im.x0 = win[1];
            im.h = win[2];
            im.w = win[3];
            im.mirror = mirror_host ? (mirror_host[g0 + i] != 0) : 0;
            im.offset = offsets_host[g0 + i] + ((long long)im.y0 * im.pitch + im.x0) * 3;
            for (int k = 0; k < 6; ++k) im.m[k] = inv_matrices_host[6 * (g0 + i) + k];
            const size_t blocks = LbRuns(im).blocks();
            if (blocks > max_blocks) max_blocks = blocks;
        }
        letterbox_minmax_kernel<<<dim3((unsigned)max_blocks, g), LB_THREADS, 0, st>>>(p);
        letterbox_warp_kernel<<<dim3((unsigned)((dst_h * dst_w + LB_THREADS - 1) / LB_THREADS), g), LB_THREADS, 0, st>>>(p);
        K2Y_CUDA_CHECK(cudaGetLastError());
    }
    return K2Y_OK;
}

extern "C" int k2y_letterbox_u8_views(const unsigned char *src_dev, int n_views, const long long *offsets_host, const int *hw_host,
                                      const int *windows_host, const double *inv_matrices_host, unsigned char *dst_dev, int dst_h,
                                      int dst_w, float *image_hw_dev, float *view_yx_dev, int *minmax_dev, void *stream) {
    return k2y_letterbox_u8_views_mirror(src_dev, n_views, offsets_host, hw_host, windows_host, nullptr, inv_matrices_host, dst_dev,
                                         dst_h, dst_w, image_hw_dev, view_yx_dev, minmax_dev, stream);
}

extern "C" int k2y_letterbox_u8_batch(const unsigned char *src_dev, int n, const long long *offsets_host, const int *hw_host,
                                      const double *inv_matrices_host, unsigned char *dst_dev, int dst_h, int dst_w,
                                      float *image_hw_dev, int *minmax_dev, void *stream) {
    using namespace k2y;
    if (n <= 0 || !hw_host) {
        set_error("k2y_letterbox_u8_batch: bad arguments");
        return K2Y_ERR_INVALID;
    }
    std::vector<int> windows(4 * (size_t)n, 0);   // every image whole
    for (int i = 0; i < n; ++i) {
        windows[4 * i + 2] = hw_host[2 * i];
        windows[4 * i + 3] = hw_host[2 * i + 1];
    }
    return k2y_letterbox_u8_views(src_dev, n, offsets_host, hw_host, windows.data(), inv_matrices_host, dst_dev, dst_h, dst_w,
                                  image_hw_dev, nullptr, minmax_dev, stream);
}

extern "C" int k2y_letterbox_u8(const unsigned char *src_dev, int src_h, int src_w, const double *inv_matrix_host,
                                unsigned char *dst_dev, int dst_h, int dst_w, int *minmax_dev, void *stream) {
    if (!src_dev || !dst_dev || !inv_matrix_host || !minmax_dev || src_h <= 0 || src_w <= 0 || dst_h <= 0 || dst_w <= 0) {
        k2y::set_error("k2y_letterbox_u8: bad arguments");
        return K2Y_ERR_INVALID;
    }
    const long long offset = 0;
    const int hw[2] = {src_h, src_w};
    return k2y_letterbox_u8_batch(src_dev, 1, &offset, hw, inv_matrix_host, dst_dev, dst_h, dst_w, nullptr, minmax_dev, stream);
}

// ---------------------------------------------------------------------------------------------------------------------
// Precision / recall counters of the reference's training-time metrics (tools/custom.py:13-75 Yolo_Precision / Yolo_Recall),
// evaluated on device head tensors: per box, true_conf = y_true[..., 4], pred_conf = y_pred[..., 4];
//   tp += (true > thr) & (pred > thr);  fp += !(true > thr) & (pred > thr);  fn += (true > thr) & !(pred > thr).
// The reference compares the RAW predicted logit with the threshold (it computes the sigmoid and never uses it, :33-35);
// apply_sigmoid = 1 evaluates the evidently intended sigmoid(pred) > thr instead.
// ---------------------------------------------------------------------------------------------------------------------
namespace {
__global__ void __launch_bounds__(256) pr_counts_kernel(const float *__restrict__ y_true, const float *__restrict__ y_pred, long long n_boxes,
                                                        int entry, float thr, int apply_sigmoid, unsigned long long *__restrict__ counts) {
    unsigned tp = 0, fp = 0, fn = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_boxes; i += (long long)gridDim.x * blockDim.x) {
        const float t = __ldg(y_true + i * entry + 4);
        float p = __ldg(y_pred + i * entry + 4);
        if (apply_sigmoid) p = __fdiv_rn(1.0f, __fadd_rn(1.0f, __double2float_rn(exp(-(double)p))));
        const bool tt = t > thr, pp = p > thr;
        tp += tt && pp;
        fp += !tt && pp;
        fn += tt && !pp;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        tp += __shfl_xor_sync(0xffffffffu, tp, o);
        fp += __shfl_xor_sync(0xffffffffu, fp, o);
        fn += __shfl_xor_sync(0xffffffffu, fn, o);
    }
    if ((threadIdx.x & 31) == 0) {
        if (tp) atomicAdd(counts + 0, (unsigned long long)tp);
        if (fp) atomicAdd(counts + 1, (unsigned long long)fp);
        if (fn) atomicAdd(counts + 2, (unsigned long long)fn);
    }
}
}  // namespace

extern "C" int k2y_pr_counts(const float *y_true_dev, const float *y_pred_dev, long long n_boxes, int entry_floats, float threshold,
                             int apply_sigmoid, unsigned long long *counts_dev, void *stream) {
    if (!y_true_dev || !y_pred_dev || !counts_dev || n_boxes < 0 || entry_floats < 5) {
        k2y::set_error("k2y_pr_counts: bad arguments (entry_floats = 5 + classes >= 5)");
        return K2Y_ERR_INVALID;
    }
    if (n_boxes == 0) return K2Y_OK;
    long long blocks = (n_boxes + 255) / 256;
    if (blocks > 132 * 8) blocks = 132 * 8;
    pr_counts_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(y_true_dev, y_pred_dev, n_boxes, entry_floats, threshold,
                                                                       apply_sigmoid, counts_dev);
    K2Y_CUDA_CHECK(cudaGetLastError());
    return K2Y_OK;
}
