// Detection mAP on the device: VOC matching per update, then at result() the per-class ranking and the AP reductions.
// The protocol (ground-truth conversion, IoU, matching rule, ranking, AP formulas) is written down in oracle/ap_ref.py.
//
//   ap_match_kernel    one warp per (image, class) of an update.  It reads the image's records and count with per-image
//                      strides (the layout k2y_detect_keras_strided writes, so gather blocks go in as they are), compacts the
//                      image's ground truth of its class into shared memory with a taken word (one bit per threshold) per
//                      box, walks the records in order and writes each record's score bits and TP bits to its slot of the
//                      store.  The store has one slot per (image, class, k < max_per_class) in stream order; slots past the
//                      count hold EMPTY_KEY.  So stream order is slot order and the store grows with the image count only.
//   sort               rank_slots: five stable counting passes (hist -> per-digit scan over tiles -> digit bases ->
//                      scatter) of 64-bit elements (VocElem: ~score bits | class << 32 | tp bits << 48): four over the 8-bit
//                      digits of the score key, then one over the class, the most significant digit, which buckets the
//                      classes.  The first pass reads the slot store and drops empty slots.  Every pass keeps the input
//                      order of equal digits (warp-ordered ranks with __match_any_sync), so the result is (class, score
//                      descending, stream order).  The launch count does not depend on the number of images or classes.
//                      The COCO evaluator below sorts CocoElem (~score bits | slot << 32) with the same passes.
//   ap_curve_kernel    one CTA per (class, threshold): the TP total, then one sweep from the lowest-ranked detection up
//                      with block scans for the cumulative TP count and the precision envelope (suffix max), all in
//                      float64, reducing the all-point AP and (first threshold) the 11 VOC 2007 recall points.
#include <algorithm>
#include <cmath>
#include <vector>

#include "common.h"

struct k2y_ap {
    int device, C, K, T;
    float thr[16];
    long long n_images, cap_images;     // images matched so far / images the slot store holds
    uint32_t *key;                      // [cap_images * C * K] score bits, EMPTY_KEY for a slot without a record
    uint16_t *tp;                       // [cap_images * C * K] bit t: TP at threshold t
    unsigned long long *npos;           // [C]
    unsigned *status;                   // [1] K2Y_AP_* bits
    cudaEvent_t done;                   // the handle's last operation, so successive calls on different streams stay ordered
};

namespace k2y {

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr uint32_t EMPTY_KEY = 0xffffffffu;        // a NaN pattern: never a valid score
constexpr uint32_t MAX_SCORE_BITS = 0x7f800000u;   // +inf; every larger pattern is NaN or has the sign bit set
constexpr int MAX_T = 16;
constexpr int MAX_CLASSES = 1024;                  // the class pass keeps SORT_WARPS * class_num counters in shared memory
constexpr int MATCH_WARPS = 4;
constexpr int SORT_WARPS = 8, SORT_ITEMS = 8, SORT_TILE = SORT_WARPS * SORT_ITEMS * 32;
constexpr int SCORE_PASSES = 4;
constexpr unsigned NO_DIGIT = 0xffffffffu;
constexpr int CURVE_THREADS = 512;
constexpr int SCAN_THREADS = 256;

struct Thresholds {
    float t[MAX_T];
};

__device__ __forceinline__ float4 norm_box(float y0, float x0, float y1, float x1) {
    return make_float4(fminf(y0, y1), fminf(x0, x1), fmaxf(y0, y1), fmaxf(x0, x1));
}
__device__ __forceinline__ float box_area(float4 b) { return __fmul_rn(__fsub_rn(b.z, b.x), __fsub_rn(b.w, b.y)); }

// oracle/ap_ref.iou: no "+1 pixel" term, 0 when the union is not positive
__device__ __forceinline__ float box_iou(float4 a, float area_a, float4 b, float area_b) {
    const float ih = fmaxf(__fsub_rn(fminf(a.z, b.z), fmaxf(a.x, b.x)), 0.f);
    const float iw = fmaxf(__fsub_rn(fminf(a.w, b.w), fmaxf(a.y, b.y)), 0.f);
    const float inter = __fmul_rn(ih, iw);
    const float uni = __fsub_rn(__fadd_rn(area_a, area_b), inter);
    return uni > 0.f ? __fdiv_rn(inter, uni) : 0.f;
}

struct MatchArgs {
    const int32_t *dets, *counts;
    long long det_stride, count_stride;
    int n, C, K, T, max_gt;
    const float *gt;                 // [total][5] (class, ymin, xmin, ymax, xmax)
    const long long *gt_off;         // [n + 1]
    Thresholds thr;
    uint32_t *key;
    uint16_t *tp;
    long long slot0;                 // first slot of this update's image 0
    unsigned long long *npos;
    unsigned *status;
};

__global__ void __launch_bounds__(MATCH_WARPS * 32) ap_match_kernel(MatchArgs a) {
    extern __shared__ float4 sm_gt[];                       // [MATCH_WARPS][max_gt] normalised boxes, then taken words
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long item = (long long)blockIdx.x * MATCH_WARPS + warp;
    if (item >= (long long)a.n * a.C) return;               // warp-uniform; the kernel has no block barrier
    const int b = (int)(item / a.C), c = (int)(item % a.C);
    float4 *box = sm_gt + (size_t)warp * a.max_gt;
    uint16_t *taken = reinterpret_cast<uint16_t *>(sm_gt + (size_t)MATCH_WARPS * a.max_gt) + (size_t)warp * a.max_gt;

    long long g0 = a.gt_off[b], g1 = a.gt_off[b + 1];
    if (g1 - g0 > a.max_gt) {
        if (lane == 0) atomicOr(a.status, (unsigned)K2Y_AP_GT_OVERFLOW);
        g1 = g0 + a.max_gt;
    }
    // this class's ground truth, in index order (so the lowest compact index is the lowest ground-truth index)
    int ng = 0;
    for (long long j0 = g0; j0 < g1; j0 += 32) {
        const long long j = j0 + lane;
        const bool mine = j < g1 && a.gt[j * 5] == (float)c;
        const unsigned m = __ballot_sync(FULL, mine);
        if (mine) {
            const int pos = ng + __popc(m & ((1u << lane) - 1));
            const float *g = a.gt + j * 5;
            box[pos] = norm_box(g[1], g[2], g[3], g[4]);
            taken[pos] = 0;
        }
        ng += __popc(m);
    }
    __syncwarp();
    if (lane == 0 && ng) atomicAdd(a.npos + c, (unsigned long long)ng);

    int cnt = a.counts[(long long)b * a.count_stride + c];
    if (cnt < 0 || cnt > a.K) {
        if (lane == 0) atomicOr(a.status, (unsigned)K2Y_AP_BAD_COUNT);
        cnt = max(0, min(cnt, a.K));
    }
    const long long slot = (a.slot0 + b) * a.C * a.K + (long long)c * a.K;
    for (int k = cnt + lane; k < a.K; k += 32) {
        a.key[slot + k] = EMPTY_KEY;
        a.tp[slot + k] = 0;
    }
    const int32_t *rec = a.dets + (long long)b * a.det_stride + (long long)c * a.K * 6;
    for (int k = 0; k < cnt; ++k) {
        const int32_t *r = rec + k * 6;
        const float4 d = norm_box(__int_as_float(r[0]), __int_as_float(r[1]), __int_as_float(r[2]), __int_as_float(r[3]));
        const float area_d = box_area(d);
        float best = -1.f;       // a NaN IoU never compares greater, so it never becomes the best box
        int bj = -1;
        for (int j = lane; j < ng; j += 32) {
            const float v = box_iou(d, area_d, box[j], box_area(box[j]));
            if (v > best) best = v, bj = j;
        }
        for (int o = 16; o; o >>= 1) {          // arg-max over the warp, ties to the lowest index
            const float ob = __shfl_xor_sync(FULL, best, o);
            const int oj = __shfl_xor_sync(FULL, bj, o);
            if (ob > best || (ob == best && (unsigned)oj < (unsigned)bj)) best = ob, bj = oj;
        }
        if (lane == 0) {
            const uint32_t bits = (uint32_t)r[4];
            unsigned hit = 0;
            if (bj >= 0) {
                unsigned ge = 0;
                for (int t = 0; t < a.T; ++t) ge |= (unsigned)(best >= a.thr.t[t]) << t;
                hit = ge & ~(unsigned)taken[bj];
                taken[bj] = (uint16_t)(taken[bj] | hit);
            }
            if (bits > MAX_SCORE_BITS) atomicOr(a.status, (unsigned)K2Y_AP_BAD_SCORE);
            a.key[slot + k] = bits > MAX_SCORE_BITS ? EMPTY_KEY : bits;
            a.tp[slot + k] = (uint16_t)hit;
        }
        __syncwarp();
    }
}

// inclusive scan over the block (blockDim.x a multiple of 32); ws: 32 entries of shared scratch; total: the block's result
template <typename T, typename Op>
__device__ __forceinline__ T block_incl_scan(T v, Op op, T identity, T *ws, T &total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    for (int o = 1; o < 32; o <<= 1) {
        const T y = __shfl_up_sync(FULL, v, o);
        if (lane >= o) v = op(y, v);
    }
    if (lane == 31) ws[warp] = v;
    __syncthreads();
    if (warp == 0) {
        T s = lane < nw ? ws[lane] : identity;
        for (int o = 1; o < 32; o <<= 1) {
            const T y = __shfl_up_sync(FULL, s, o);
            if (lane >= o) s = op(y, s);
        }
        ws[lane] = s;
    }
    __syncthreads();
    if (warp > 0) v = op(ws[warp - 1], v);
    total = ws[nw - 1];
    __syncthreads();
    return v;
}
struct AddOp {
    template <typename T> __device__ T operator()(T x, T y) const { return x + y; }
};
struct MaxOp {
    __device__ double operator()(double x, double y) const { return fmax(x, y); }
};

struct SortPass {
    const uint32_t *slot_key;        // pass 0 reads the slot store
    const uint16_t *slot_tp;
    const uint64_t *src;             // later passes
    uint64_t *dst;
    long long n;                     // source elements
    int C, K, pass, bins, nblocks;
    uint32_t *block_hist;            // [bins][nblocks]
    const uint32_t *digit_base;      // [bins]
};

// The element each evaluator sorts, made from slot i of its store in the first pass.  Both keep ~score bits in the low 32
// bits; the class of slot i is (i / K) % C.
struct VocElem {            // ~score | class << 32 | tp bits << 48
    static __device__ __forceinline__ uint64_t make(const SortPass &p, uint32_t key, long long i) {
        const uint64_t cls = (uint64_t)((i / p.K) % p.C);
        return (uint64_t)(~key) | (cls << 32) | ((uint64_t)p.slot_tp[i] << 48);
    }
    static __device__ __forceinline__ unsigned cls(const SortPass &, uint64_t e) { return (unsigned)(e >> 32) & 0xffffu; }
};
struct CocoElem {           // ~score | slot << 32 (the slot's match bits are read through it)
    static __device__ __forceinline__ uint64_t make(const SortPass &, uint32_t key, long long i) {
        return (uint64_t)(~key) | ((uint64_t)i << 32);
    }
    static __device__ __forceinline__ unsigned cls(const SortPass &p, uint64_t e) {
        return ((unsigned)(e >> 32) / (unsigned)p.K) % (unsigned)p.C;
    }
};

template <typename Elem>
__device__ __forceinline__ uint64_t sort_load(const SortPass &p, long long i, bool &valid) {
    valid = i < p.n;
    if (!valid) return 0;
    if (p.pass > 0) return p.src[i];
    const uint32_t key = p.slot_key[i];
    valid = key != EMPTY_KEY;
    return Elem::make(p, key, i);
}

// Loads this thread's items of the tile and ranks them among the equal digits of its warp's span, in span order; cnt (this
// warp's row of bins counters, zeroed) ends as the span's histogram.
template <typename Elem>
__device__ __forceinline__ void rank_tile(const SortPass &p, uint32_t *cnt, uint64_t (&e)[SORT_ITEMS], unsigned (&d)[SORT_ITEMS],
                                          unsigned (&r)[SORT_ITEMS]) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long base = (long long)blockIdx.x * SORT_TILE + warp * SORT_ITEMS * 32 + lane;
#pragma unroll
    for (int it = 0; it < SORT_ITEMS; ++it) {
        bool v;
        e[it] = sort_load<Elem>(p, base + it * 32, v);
        d[it] = !v ? NO_DIGIT : p.pass < SCORE_PASSES ? (unsigned)(e[it] >> (8 * p.pass)) & 255u : Elem::cls(p, e[it]);
    }
#pragma unroll
    for (int it = 0; it < SORT_ITEMS; ++it) {
        const unsigned peers = __match_any_sync(FULL, d[it]);
        const unsigned lower = peers & ((1u << lane) - 1);
        const unsigned c0 = d[it] != NO_DIGIT ? cnt[d[it]] : 0;
        __syncwarp();
        if (d[it] != NO_DIGIT && lower == 0) cnt[d[it]] = c0 + __popc(peers);
        r[it] = c0 + __popc(lower);
        __syncwarp();
    }
}

template <typename Elem>
__global__ void __launch_bounds__(SORT_WARPS * 32) ap_hist_kernel(SortPass p) {
    extern __shared__ uint32_t cnt[];                       // [SORT_WARPS][bins]
    for (int i = threadIdx.x; i < SORT_WARPS * p.bins; i += blockDim.x) cnt[i] = 0;
    __syncthreads();
    uint64_t e[SORT_ITEMS];
    unsigned d[SORT_ITEMS], r[SORT_ITEMS];
    rank_tile<Elem>(p, cnt + (threadIdx.x >> 5) * p.bins, e, d, r);
    __syncthreads();
    for (int g = threadIdx.x; g < p.bins; g += blockDim.x) {
        uint32_t s = 0;
        for (int w = 0; w < SORT_WARPS; ++w) s += cnt[w * p.bins + g];
        p.block_hist[(long long)g * p.nblocks + blockIdx.x] = s;
    }
}

// one CTA per digit: exclusive scan of the digit's tile counts in place, and the digit's total
__global__ void __launch_bounds__(SCAN_THREADS) ap_colscan_kernel(uint32_t *block_hist, int nblocks, uint32_t *totals) {
    __shared__ uint32_t ws[32];
    uint32_t *row = block_hist + (long long)blockIdx.x * nblocks;
    uint32_t carry = 0;
    for (int i0 = 0; i0 < nblocks; i0 += blockDim.x) {
        const int i = i0 + threadIdx.x;
        const uint32_t v = i < nblocks ? row[i] : 0u;
        uint32_t tot;
        const uint32_t inc = block_incl_scan(v, AddOp{}, 0u, ws, tot);
        if (i < nblocks) row[i] = carry + inc - v;
        carry += tot;
    }
    if (threadIdx.x == 0) totals[blockIdx.x] = carry;
}

// one CTA of MAX_CLASSES threads: exclusive scan of the digit totals, and the grand total
__global__ void __launch_bounds__(MAX_CLASSES) ap_basescan_kernel(const uint32_t *totals, int bins, uint32_t *bases, uint32_t *grand) {
    __shared__ uint32_t ws[32];
    const uint32_t v = (int)threadIdx.x < bins ? totals[threadIdx.x] : 0u;
    uint32_t tot;
    const uint32_t inc = block_incl_scan(v, AddOp{}, 0u, ws, tot);
    if ((int)threadIdx.x < bins) bases[threadIdx.x] = inc - v;
    if (threadIdx.x == 0) *grand = tot;
}

template <typename Elem>
__global__ void __launch_bounds__(SORT_WARPS * 32) ap_scatter_kernel(SortPass p) {
    extern __shared__ uint32_t cnt[];
    for (int i = threadIdx.x; i < SORT_WARPS * p.bins; i += blockDim.x) cnt[i] = 0;
    __syncthreads();
    uint64_t e[SORT_ITEMS];
    unsigned d[SORT_ITEMS], r[SORT_ITEMS];
    const int warp = threadIdx.x >> 5;
    rank_tile<Elem>(p, cnt + warp * p.bins, e, d, r);
    __syncthreads();
    for (int g = threadIdx.x; g < p.bins; g += blockDim.x) {    // per-warp histograms -> per-warp output offsets
        uint32_t run = p.digit_base[g] + p.block_hist[(long long)g * p.nblocks + blockIdx.x];
        for (int w = 0; w < SORT_WARPS; ++w) {
            const uint32_t t = cnt[w * p.bins + g];
            cnt[w * p.bins + g] = run;
            run += t;
        }
    }
    __syncthreads();
#pragma unroll
    for (int it = 0; it < SORT_ITEMS; ++it)
        if (d[it] != NO_DIGIT) p.dst[cnt[warp * p.bins + d[it]] + r[it]] = e[it];
}

struct CurveArgs {
    const uint64_t *e;               // sorted (class, score descending, stream order)
    const uint32_t *class_start, *class_count;
    const unsigned long long *npos;
    int C;
    double *ap;                      // [T][C]
    double *ap07;                    // [C]
};

__global__ void __launch_bounds__(CURVE_THREADS) ap_curve_kernel(CurveArgs a) {
    __shared__ uint32_t wsu[32];
    __shared__ double wsd[32];
    __shared__ double p07[11];
    const int c = blockIdx.x, t = blockIdx.y, tid = threadIdx.x;
    const unsigned long long np = a.npos[c];
    if (np == 0) {
        if (tid == 0) {
            a.ap[t * a.C + c] = nan("");
            if (t == 0) a.ap07[c] = nan("");
        }
        return;
    }
    const uint64_t *e = a.e + a.class_start[c];
    const long long m = a.class_count[c];
    const int sh = 48 + t;
    uint32_t s = 0;
    for (long long i = tid; i < m; i += blockDim.x) s += (uint32_t)(e[i] >> sh) & 1u;
    uint32_t tp_total;
    block_incl_scan(s, AddOp{}, 0u, wsu, tp_total);
    if (tid < 11) p07[tid] = 0.0;
    const double npd = (double)np;
    uint32_t after = 0;              // TPs ranked below the current chunk
    double carry_max = -1.0;         // precision envelope of the ranks below the current chunk
    double acc = 0.0;
    for (long long hi = m; hi > 0; hi -= blockDim.x) {
        const long long r = hi - 1 - tid;            // thread order runs from the lowest rank up: scans are suffix scans
        const bool v = r >= 0;
        const uint32_t x = v ? (uint32_t)(e[r] >> sh) & 1u : 0u;
        uint32_t chunk_tp;
        const uint32_t suffix = block_incl_scan(x, AddOp{}, 0u, wsu, chunk_tp);
        const uint32_t cum = tp_total - after - suffix + x;           // cumTP_r
        const double prec = v ? (double)cum / (double)(r + 1) : -1.0;
        double chunk_max;
        const double env = fmax(block_incl_scan(prec, MaxOp{}, -1.0, wsd, chunk_max), carry_max);
        if (v && x) acc += env;
        if (t == 0 && v) {
            const double rec = (double)cum / npd, rec_prev = (double)(cum - x) / npd;
            for (int k = 0; k < 11; ++k) {           // the first rank whose recall reaches t_k = np.arange(0, 1.1, 0.1)[k]
                const double tk = __dmul_rn((double)k, 0.1);
                if (rec >= tk && (r == 0 || rec_prev < tk)) p07[k] = env;
            }
        }
        after += chunk_tp;
        carry_max = fmax(carry_max, chunk_max);
    }
    double sum;
    block_incl_scan(acc, AddOp{}, 0.0, wsd, sum);
    if (tid == 0) {
        a.ap[t * a.C + c] = sum / npd;
        if (t == 0) {
            double s07 = 0.0;
            for (int k = 0; k < 11; ++k) s07 += p07[k];
            a.ap07[c] = s07 / 11.0;
        }
    }
}

struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) {
        if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
        if (prev != dev) cudaSetDevice(dev);
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

// one stable counting pass: hist -> per-digit tile scan -> digit bases (+ grand total) -> scatter
template <typename Elem>
cudaError_t sort_pass(SortPass p, uint32_t *totals, uint32_t *bases, uint32_t *grand, bool scatter, cudaStream_t st) {
    const size_t smem = (size_t)SORT_WARPS * p.bins * sizeof(uint32_t);
    p.digit_base = bases;
    ap_hist_kernel<Elem><<<p.nblocks, SORT_WARPS * 32, smem, st>>>(p);
    ap_colscan_kernel<<<p.bins, SCAN_THREADS, 0, st>>>(p.block_hist, p.nblocks, totals);
    ap_basescan_kernel<<<1, MAX_CLASSES, 0, st>>>(totals, p.bins, bases, grand);
    if (scatter) ap_scatter_kernel<Elem><<<p.nblocks, SORT_WARPS * 32, smem, st>>>(p);
    return cudaGetLastError();
}

// Scratch words rank_slots needs for n_slots slots of C classes: totals, bases, the grand total, the tile histograms.
size_t rank_scratch_words(long long n_slots, int C) {
    const int nb0 = (int)((n_slots + SORT_TILE - 1) / SORT_TILE);
    return 2 * MAX_CLASSES + 2 + (size_t)std::max(256, C) * std::max(nb0, 1);
}

// Ranks the slot store p.slot_key[0, p.n) (p.C, p.K set): the non-empty slots as Elem, ordered by (class, score
// descending, slot order).  Synchronises st once (to size the buffers).  On return class c's elements lie at
// [bases[c], bases[c] + totals[c]) of *sorted (nullptr when there are none); the caller frees buf[0] and buf[1] on st.
template <typename Elem>
int rank_slots(SortPass p, uint32_t *words, uint64_t *(&buf)[2], const uint64_t *&sorted, cudaStream_t st) {
    uint32_t *totals = words, *bases = totals + MAX_CLASSES, *grand = bases + MAX_CLASSES, *hist = grand + 2;
    uint32_t m = 0;
    if (p.n > 0) {
        p.bins = 256;
        p.nblocks = (int)((p.n + SORT_TILE - 1) / SORT_TILE);
        p.block_hist = hist;
        K2Y_CUDA_CHECK(sort_pass<Elem>(p, totals, bases, grand, false, st));
        K2Y_CUDA_CHECK(cudaMemcpyAsync(&m, grand, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        K2Y_CUDA_CHECK(cudaStreamSynchronize(st));
        if (m > 0) {
            K2Y_CUDA_CHECK(cudaMallocAsync(&buf[0], (size_t)m * sizeof(uint64_t), st));
            K2Y_CUDA_CHECK(cudaMallocAsync(&buf[1], (size_t)m * sizeof(uint64_t), st));
            p.digit_base = bases;
            p.dst = buf[0];
            ap_scatter_kernel<Elem><<<p.nblocks, SORT_WARPS * 32, (size_t)SORT_WARPS * p.bins * sizeof(uint32_t), st>>>(p);
            K2Y_CUDA_CHECK(cudaGetLastError());
            p.n = m;
            p.nblocks = (int)((m + SORT_TILE - 1) / SORT_TILE);
            for (int pass = 1; pass <= SCORE_PASSES; ++pass) {     // pass SCORE_PASSES: the class digit
                p.pass = pass;
                p.bins = pass < SCORE_PASSES ? 256 : p.C;
                p.src = buf[(pass - 1) & 1];
                p.dst = buf[pass & 1];
                K2Y_CUDA_CHECK(sort_pass<Elem>(p, totals, bases, grand, true, st));
            }
        }
    }
    if (m == 0) K2Y_CUDA_CHECK(cudaMemsetAsync(totals, 0, 2 * MAX_CLASSES * sizeof(uint32_t), st));
    sorted = buf[SCORE_PASSES & 1];
    return K2Y_OK;
}

template <typename Handle>
int begin(Handle *ap, cudaStream_t st) {
    K2Y_CUDA_CHECK(cudaStreamWaitEvent(st, ap->done, 0));
    return K2Y_OK;
}
template <typename Handle>
int finish(Handle *ap, cudaStream_t st) {
    K2Y_CUDA_CHECK(cudaEventRecord(ap->done, st));
    return K2Y_OK;
}

}  // namespace
}  // namespace k2y

using namespace k2y;

extern "C" int k2y_ap_create(int class_num, int max_per_class, const float *iou_thresholds, int n_thresholds, int device,
                             k2y_ap **out) {
    if (!out || !iou_thresholds || class_num < 1 || class_num > MAX_CLASSES || max_per_class < 1 || n_thresholds < 1 ||
        n_thresholds > MAX_T) {
        set_error("k2y_ap_create: class_num must be 1..%d, max_per_class >= 1 and 1..%d IoU thresholds", MAX_CLASSES, MAX_T);
        return K2Y_ERR_INVALID;
    }
    for (int t = 0; t < n_thresholds; ++t)
        if (!(iou_thresholds[t] > 0.f && iou_thresholds[t] <= 1.f)) {
            set_error("k2y_ap_create: IoU threshold %d is %g, not in (0, 1]", t, (double)iou_thresholds[t]);
            return K2Y_ERR_INVALID;
        }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) {
        cudaGetLastError();
        set_error("k2y_ap_create: no CUDA device %d", device);
        return K2Y_ERR_CUDA;
    }
    DeviceGuard g(device);
    k2y_ap *ap = new k2y_ap();
    ap->device = device;
    ap->C = class_num;
    ap->K = max_per_class;
    ap->T = n_thresholds;
    for (int t = 0; t < n_thresholds; ++t) ap->thr[t] = iou_thresholds[t];
    if (cudaMalloc(&ap->npos, class_num * sizeof(unsigned long long)) != cudaSuccess ||
        cudaMalloc(&ap->status, sizeof(unsigned)) != cudaSuccess ||
        cudaMemset(ap->npos, 0, class_num * sizeof(unsigned long long)) != cudaSuccess ||
        cudaMemset(ap->status, 0, sizeof(unsigned)) != cudaSuccess ||
        cudaEventCreateWithFlags(&ap->done, cudaEventDisableTiming) != cudaSuccess) {
        set_error("k2y_ap_create: %s", cudaGetErrorString(cudaGetLastError()));
        k2y_ap_destroy(ap);
        return K2Y_ERR_CUDA;
    }
    *out = ap;
    return K2Y_OK;
}

extern "C" int k2y_ap_destroy(k2y_ap *ap) {
    if (!ap) return K2Y_OK;
    DeviceGuard g(ap->device);
    if (ap->done) cudaEventSynchronize(ap->done);
    if (ap->key) cudaFreeAsync(ap->key, 0);     // stream-ordered allocations (k2y_ap_match grows the store with cudaMallocAsync)
    if (ap->tp) cudaFreeAsync(ap->tp, 0);
    cudaStreamSynchronize(0);
    cudaFree(ap->npos);
    cudaFree(ap->status);
    if (ap->done) cudaEventDestroy(ap->done);
    delete ap;
    return K2Y_OK;
}

extern "C" int k2y_ap_match(k2y_ap *ap, const int32_t *dets_dev, const int32_t *counts_dev, long long det_image_stride_words,
                            long long count_image_stride_words, int n_images, const float *gt_dev,
                            const long long *gt_offsets_dev, int max_gt_per_image, void *stream) {
    if (!ap || n_images < 0 || max_gt_per_image < 0 || (n_images > 0 && (!dets_dev || !counts_dev || !gt_offsets_dev)) ||
        (max_gt_per_image > 0 && !gt_dev)) {
        set_error("k2y_ap_match: bad arguments");
        return K2Y_ERR_INVALID;
    }
    if (det_image_stride_words < (long long)ap->C * ap->K * 6 || count_image_stride_words < ap->C) {
        set_error("k2y_ap_match: image strides smaller than one image's records / counts");
        return K2Y_ERR_INVALID;
    }
    if (n_images == 0) return K2Y_OK;
    const size_t smem = (size_t)MATCH_WARPS * max_gt_per_image * (sizeof(float4) + sizeof(uint16_t));
    DeviceGuard g(ap->device);
    int dev_smem = 0;
    K2Y_CUDA_CHECK(cudaDeviceGetAttribute(&dev_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, ap->device));
    if (smem > (size_t)dev_smem) {
        set_error("k2y_ap_match: an image has %d ground-truth boxes, more than the %d the match kernel holds", max_gt_per_image,
                  (int)(dev_smem / (MATCH_WARPS * (sizeof(float4) + sizeof(uint16_t)))));
        return K2Y_ERR_INVALID;
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (int rc = begin(ap, st)) return rc;
    const long long per_image = (long long)ap->C * ap->K;
    const long long need = ap->n_images + n_images;
    if (need > ap->cap_images) {        // grow the slot store by doubling, stream-ordered
        const long long cap = std::max(need, 2 * ap->cap_images);
        uint32_t *key = nullptr;
        uint16_t *tp = nullptr;
        K2Y_CUDA_CHECK(cudaMallocAsync(&key, cap * per_image * sizeof(uint32_t), st));
        K2Y_CUDA_CHECK(cudaMallocAsync(&tp, cap * per_image * sizeof(uint16_t), st));
        if (ap->n_images) {
            K2Y_CUDA_CHECK(cudaMemcpyAsync(key, ap->key, ap->n_images * per_image * sizeof(uint32_t), cudaMemcpyDeviceToDevice, st));
            K2Y_CUDA_CHECK(cudaMemcpyAsync(tp, ap->tp, ap->n_images * per_image * sizeof(uint16_t), cudaMemcpyDeviceToDevice, st));
        }
        if (ap->key) K2Y_CUDA_CHECK(cudaFreeAsync(ap->key, st));
        if (ap->tp) K2Y_CUDA_CHECK(cudaFreeAsync(ap->tp, st));
        ap->key = key;
        ap->tp = tp;
        ap->cap_images = cap;
    }
    MatchArgs a;
    a.dets = dets_dev;
    a.counts = counts_dev;
    a.det_stride = det_image_stride_words;
    a.count_stride = count_image_stride_words;
    a.n = n_images;
    a.C = ap->C;
    a.K = ap->K;
    a.T = ap->T;
    a.max_gt = max_gt_per_image;
    a.gt = gt_dev;
    a.gt_off = gt_offsets_dev;
    for (int t = 0; t < MAX_T; ++t) a.thr.t[t] = t < ap->T ? ap->thr[t] : 2.f;
    a.key = ap->key;
    a.tp = ap->tp;
    a.slot0 = ap->n_images;
    a.npos = ap->npos;
    a.status = ap->status;
    if (smem > 48 * 1024) K2Y_CUDA_CHECK(cudaFuncSetAttribute(ap_match_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const long long warps = (long long)n_images * ap->C;
    ap_match_kernel<<<(unsigned)((warps + MATCH_WARPS - 1) / MATCH_WARPS), MATCH_WARPS * 32, smem, st>>>(a);
    K2Y_CUDA_CHECK(cudaGetLastError());
    ap->n_images = need;
    return finish(ap, st);
}

extern "C" int k2y_ap_result(k2y_ap *ap, double *ap_host, double *ap07_host, long long *npos_host, unsigned *status_host,
                             void *stream) {
    if (!ap || !ap_host || !ap07_host || !npos_host || !status_host) {
        set_error("k2y_ap_result: null pointer");
        return K2Y_ERR_INVALID;
    }
    const long long n_slots = ap->n_images * ap->C * ap->K;
    if (n_slots >= (1ll << 32) - SORT_TILE) {
        set_error("k2y_ap_result: %lld record slots (images x classes x max_per_class); the ranking counts with 32 bits", n_slots);
        return K2Y_ERR_INVALID;
    }
    DeviceGuard g(ap->device);
    cudaStream_t st = (cudaStream_t)stream;
    if (int rc = begin(ap, st)) return rc;
    const int C = ap->C, T = ap->T;
    // scratch: the AP outputs, then rank_slots' words
    const size_t words = rank_scratch_words(n_slots, C);
    const size_t out_doubles = (size_t)T * C + C;
    char *scratch = nullptr;
    K2Y_CUDA_CHECK(cudaMallocAsync(&scratch, out_doubles * sizeof(double) + words * sizeof(uint32_t), st));
    double *ap_dev = reinterpret_cast<double *>(scratch), *ap07_dev = ap_dev + (size_t)T * C;
    uint32_t *totals = reinterpret_cast<uint32_t *>(ap_dev + out_doubles), *bases = totals + MAX_CLASSES;
    uint64_t *buf[2] = {nullptr, nullptr};
    const uint64_t *sorted = nullptr;
    SortPass p = {};
    p.slot_key = ap->key;
    p.slot_tp = ap->tp;
    p.n = n_slots;
    p.C = C;
    p.K = ap->K;
    if (int rc = rank_slots<VocElem>(p, totals, buf, sorted, st)) return rc;
    CurveArgs ca;
    ca.e = sorted;
    ca.class_start = bases;
    ca.class_count = totals;
    ca.npos = ap->npos;
    ca.C = C;
    ca.ap = ap_dev;
    ca.ap07 = ap07_dev;
    ap_curve_kernel<<<dim3(C, T), CURVE_THREADS, 0, st>>>(ca);
    K2Y_CUDA_CHECK(cudaGetLastError());
    K2Y_CUDA_CHECK(cudaMemcpyAsync(ap_host, ap_dev, (size_t)T * C * sizeof(double), cudaMemcpyDeviceToHost, st));
    K2Y_CUDA_CHECK(cudaMemcpyAsync(ap07_host, ap07_dev, (size_t)C * sizeof(double), cudaMemcpyDeviceToHost, st));
    static_assert(sizeof(long long) == sizeof(unsigned long long), "npos is copied as is");
    K2Y_CUDA_CHECK(cudaMemcpyAsync(npos_host, ap->npos, (size_t)C * sizeof(long long), cudaMemcpyDeviceToHost, st));
    K2Y_CUDA_CHECK(cudaMemcpyAsync(status_host, ap->status, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    for (uint64_t *b : buf)
        if (b) K2Y_CUDA_CHECK(cudaFreeAsync(b, st));
    K2Y_CUDA_CHECK(cudaFreeAsync(scratch, st));
    if (int rc = finish(ap, st)) return rc;
    K2Y_CUDA_CHECK(cudaStreamSynchronize(st));
    return K2Y_OK;
}

extern "C" int k2y_ap_reset(k2y_ap *ap, void *stream) {
    if (!ap) {
        set_error("k2y_ap_reset: null handle");
        return K2Y_ERR_INVALID;
    }
    DeviceGuard g(ap->device);
    cudaStream_t st = (cudaStream_t)stream;
    if (int rc = begin(ap, st)) return rc;
    K2Y_CUDA_CHECK(cudaMemsetAsync(ap->npos, 0, ap->C * sizeof(unsigned long long), st));
    K2Y_CUDA_CHECK(cudaMemsetAsync(ap->status, 0, sizeof(unsigned), st));
    ap->n_images = 0;
    return finish(ap, st);
}

extern "C" int k2y_ap_tp_flags(k2y_ap *ap, uint16_t *tp_host, long long capacity, long long *n_images, void *stream) {
    if (!ap || !n_images) {
        set_error("k2y_ap_tp_flags: null pointer");
        return K2Y_ERR_INVALID;
    }
    *n_images = ap->n_images;
    const long long n = ap->n_images * ap->C * ap->K;
    if (!tp_host) return K2Y_OK;
    if (capacity < n) {
        set_error("k2y_ap_tp_flags: capacity %lld < %lld flags", capacity, n);
        return K2Y_ERR_INVALID;
    }
    DeviceGuard g(ap->device);
    cudaStream_t st = (cudaStream_t)stream;
    if (int rc = begin(ap, st)) return rc;
    if (n) K2Y_CUDA_CHECK(cudaMemcpyAsync(tp_host, ap->tp, n * sizeof(uint16_t), cudaMemcpyDeviceToHost, st));
    if (int rc = finish(ap, st)) return rc;
    K2Y_CUDA_CHECK(cudaStreamSynchronize(st));
    return K2Y_OK;
}

// ------------------------------------------------------------------------------------------------------------------------
// COCO protocol (COCOeval, iouType "bbox", default parameters), written down in oracle/coco_ref.py.
//
//   coco_match_kernel  one warp per (image, class) of an update.  It copies the image's ground truth of the class (grouped
//                      per (image position, class) at create, JSON order) and the first min(count, 100) records into shared
//                      memory, computes their IoU matrix once in float64 (maskApi bbIou), then runs COCOeval's greedy
//                      matching for the 40 (area range, threshold) pairs, lane l taking pairs l and l + 32.  Each record's
//                      TP and not-ignored bits (bit a * 10 + t) go to its slot, addressed by the image's position in the
//                      sorted image-id list, so updates may arrive in any order.
//   sort               rank_slots<CocoElem>: (class, score descending, slot order), slot order being COCOeval's tie order
//                      (sorted image ids, then record order).
//   coco_curve_kernel  one CTA per (threshold, area, maxDet, class): cumulative TP / FP counts, the precision envelope
//                      (suffix max) and the 101 searchsorted lookups in float64, each TP record writing the recall points
//                      its recall reaches first.
struct k2y_coco {
    int device, C, K, KD;               // KD = min(K, 100): COCOeval keeps the 100 best detections per (image, class)
    long long n_images;
    int max_g, warps;                   // most ground-truth boxes of one (image, class); warps per match CTA
    size_t warp_smem;                   // match kernel shared memory per warp
    double *gt;                         // [n_gt][6] (x, y, w, h, area, iscrowd), grouped per (image position, class)
    long long *gt_off;                  // [n_images * C + 1]
    long long *npig;                    // [C][4] non-ignored ground truth per (class, area range)
    double *params;                     // [10] IoU thresholds, then [101] recall points
    uint32_t *key;                      // [n_images * C * KD] score bits, EMPTY_KEY for a slot without a record
    uint64_t *tp, *nig;                 // [n_images * C * KD] bit a * 10 + t: TP / not ignored, area range a, threshold t
    unsigned *seen;                     // [n_images] matched since the last reset
    unsigned *status;                   // [1] K2Y_COCO_* bits
    cudaEvent_t done;
};

namespace k2y {
namespace {

constexpr int COCO_T = 10, COCO_R = 101, COCO_A = 4, COCO_M = 3, COCO_MAX_DETS = 100;
constexpr int COCO_PAIRS = COCO_A * COCO_T;        // (area range, threshold) pairs of one record's bits
constexpr int COCO_GT_FIELDS = 6;
constexpr int COCO_MATCH_MAX_WARPS = 4;
__constant__ double COCO_AREA_RNG[COCO_A][2] = {{0.0, 1e10}, {0.0, 1024.0}, {1024.0, 9216.0}, {9216.0, 1e10}};
__constant__ int COCO_MAX_DET[COCO_M] = {1, 10, 100};

size_t coco_warp_smem(int KD, int max_g) {
    const size_t doubles = (size_t)KD * max_g + (size_t)COCO_GT_FIELDS * max_g + 4 * (size_t)KD;
    return (doubles * sizeof(double) + (size_t)max_g * COCO_PAIRS + 15) & ~(size_t)15;
}

// maskApi.c bbIou of a detection D and a ground-truth box G, both (x, y, w, h), G[5] its crowd flag; no contraction
__device__ __forceinline__ double bb_iou(const double *D, const double *G) {
    const double w = __dsub_rn(fmin(__dadd_rn(D[2], D[0]), __dadd_rn(G[2], G[0])), fmax(D[0], G[0]));
    if (w <= 0.0) return 0.0;
    const double h = __dsub_rn(fmin(__dadd_rn(D[3], D[1]), __dadd_rn(G[3], G[1])), fmax(D[1], G[1]));
    if (h <= 0.0) return 0.0;
    const double i = __dmul_rn(w, h), da = __dmul_rn(D[2], D[3]);
    const double u = G[5] != 0.0 ? da : __dsub_rn(__dadd_rn(da, __dmul_rn(G[2], G[3])), i);
    return __ddiv_rn(i, u);
}

struct CocoMatchArgs {
    const int32_t *dets, *counts;
    long long det_stride, count_stride;
    const long long *pos;            // [n] positions in the sorted image-id list
    int n, C, K, KD, max_g;
    long long n_images;
    size_t warp_doubles;             // per-warp shared memory, in doubles
    const double *gt;
    const long long *gt_off;
    const double *thr;               // [10]
    uint32_t *key;
    uint64_t *tp, *nig;
    unsigned *seen, *status;
};

// COCOeval.evaluateImg for record k at one (area range, threshold) pair: the ground truth walked non-ignored first, then
// (only when nothing matched) ignored, each in JSON order; a taken box is skipped unless crowd, and the last box with the
// highest IoU >= min(t, 1 - 1e-10) wins.  Returns the TP and not-ignored bits.
__device__ __forceinline__ void coco_match_pair(const CocoMatchArgs &a, int pair, int k, int ng, const double *iou,
                                                const double *g, uint8_t *taken, double area_d, bool &tp, bool &nig) {
    const int ar = pair / COCO_T, t = pair % COCO_T;
    const double lo = COCO_AREA_RNG[ar][0], hi = COCO_AREA_RNG[ar][1];
    double best = fmin(a.thr[t], 1.0 - 1e-10);
    int m = -1;
    bool m_ig = false;
    for (int pass = 0; pass < 2 && m < 0; ++pass)
        for (int j = 0; j < ng; ++j) {
            const double *G = g + j * COCO_GT_FIELDS;
            const bool crowd = G[5] != 0.0;
            const bool ig = crowd || G[4] < lo || G[4] > hi;
            if (ig != (pass == 1)) continue;
            if (taken[j * COCO_PAIRS + pair] && !crowd) continue;
            const double v = iou[k * ng + j];
            if (v < best) continue;
            best = v;
            m = j;
            m_ig = ig;
        }
    if (m >= 0) {
        taken[m * COCO_PAIRS + pair] = 1;
        tp = nig = !m_ig;
    } else {
        tp = false;
        nig = !(area_d < lo || area_d > hi);
    }
}

__global__ void __launch_bounds__(COCO_MATCH_MAX_WARPS * 32) coco_match_kernel(CocoMatchArgs a) {
    extern __shared__ double sm_coco[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long item = (long long)blockIdx.x * (blockDim.x >> 5) + warp;
    if (item >= (long long)a.n * a.C) return;               // warp-uniform; the kernel has no block barrier
    const int b = (int)(item / a.C), c = (int)(item % a.C);
    double *iou = sm_coco + (size_t)warp * a.warp_doubles;   // [KD][max_g]
    double *g = iou + (size_t)a.KD * a.max_g;                 // [max_g][6]
    double *d = g + (size_t)COCO_GT_FIELDS * a.max_g;        // [KD][4] (x, y, w, h)
    uint8_t *taken = reinterpret_cast<uint8_t *>(d + 4 * (size_t)a.KD);    // [max_g][40]

    const long long pos = a.pos[b];
    if (pos < 0 || pos >= a.n_images) {
        if (lane == 0) atomicOr(a.status, (unsigned)K2Y_COCO_BAD_POSITION);
        return;
    }
    if (c == 0 && lane == 0 && atomicExch(a.seen + pos, 1u)) atomicOr(a.status, (unsigned)K2Y_COCO_REPEATED_IMAGE);
    int cnt = a.counts[(long long)b * a.count_stride + c];
    if (cnt < 0 || cnt > a.K) {
        if (lane == 0) atomicOr(a.status, (unsigned)K2Y_COCO_BAD_COUNT);
        cnt = max(0, min(cnt, a.K));
    }
    const int32_t *rec = a.dets + (long long)b * a.det_stride + (long long)c * a.K * 6;
    for (int k = lane; k < cnt; k += 32)
        if ((uint32_t)rec[k * 6 + 4] > MAX_SCORE_BITS) atomicOr(a.status, (unsigned)K2Y_COCO_BAD_SCORE);
    const int nd = min(cnt, a.KD);
    const long long g0 = a.gt_off[pos * a.C + c];
    const int ng = (int)(a.gt_off[pos * a.C + c + 1] - g0);
    for (int i = lane; i < ng * COCO_GT_FIELDS; i += 32) g[i] = a.gt[g0 * COCO_GT_FIELDS + i];
    for (int i = lane; i < ng * COCO_PAIRS; i += 32) taken[i] = 0;
    for (int k = lane; k < nd; k += 32) {       // (ymin, xmin, ymax, xmax) float32 -> (x, y, w, h) float64
        const int32_t *r = rec + k * 6;
        const double y0 = __int_as_float(r[0]), x0 = __int_as_float(r[1]), y1 = __int_as_float(r[2]), x1 = __int_as_float(r[3]);
        d[k * 4 + 0] = x0;
        d[k * 4 + 1] = y0;
        d[k * 4 + 2] = __dsub_rn(x1, x0);
        d[k * 4 + 3] = __dsub_rn(y1, y0);
    }
    __syncwarp();
    for (int i = lane; i < nd * ng; i += 32) iou[i] = bb_iou(d + (i / ng) * 4, g + (i % ng) * COCO_GT_FIELDS);
    __syncwarp();
    const long long slot = (pos * a.C + c) * a.KD;
    for (int k = 0; k < nd; ++k) {
        const double area_d = __dmul_rn(d[k * 4 + 2], d[k * 4 + 3]);
        bool tp0, nig0, tp1 = false, nig1 = false;
        coco_match_pair(a, lane, k, ng, iou, g, taken, area_d, tp0, nig0);
        if (lane + 32 < COCO_PAIRS) coco_match_pair(a, lane + 32, k, ng, iou, g, taken, area_d, tp1, nig1);
        const unsigned t0 = __ballot_sync(FULL, tp0), n0 = __ballot_sync(FULL, nig0);
        const unsigned t1 = __ballot_sync(FULL, tp1), n1 = __ballot_sync(FULL, nig1);
        if (lane == 0) {
            const uint32_t bits = (uint32_t)rec[k * 6 + 4];
            a.key[slot + k] = bits > MAX_SCORE_BITS ? EMPTY_KEY : bits;
            a.tp[slot + k] = (uint64_t)t0 | (uint64_t)t1 << 32;
            a.nig[slot + k] = (uint64_t)n0 | (uint64_t)n1 << 32;
        }
    }
    for (int k = nd + lane; k < a.KD; k += 32) a.key[slot + k] = EMPTY_KEY;
}

struct CocoCurveArgs {
    const uint64_t *e;               // sorted (class, score descending, slot order), CocoElem
    const uint32_t *class_start, *class_count;
    const uint64_t *tp, *nig;
    const long long *npig;           // [C][4]
    const double *rec_thr;           // [101]
    int C, KD;
    double *precision;               // [10][101][C][4][3]
    double *recall;                  // [10][C][4][3]
};

// the number of recall points <= v (rthr ascending)
__device__ __forceinline__ int recall_points_upto(const double *rthr, double v) {
    int lo = 0, hi = COCO_R;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (rthr[mid] <= v) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(CURVE_THREADS) coco_curve_kernel(CocoCurveArgs a) {
    __shared__ unsigned long long wsu[32];
    __shared__ double wsd[32];
    __shared__ double rthr[COCO_R], q[COCO_R];
    const int combo = blockIdx.x, c = blockIdx.y, tid = threadIdx.x;
    const int t = combo / (COCO_A * COCO_M), ar = (combo / COCO_M) % COCO_A, mi = combo % COCO_M;
    const int max_det = COCO_MAX_DET[mi];
    const size_t cell = (size_t)c * COCO_A * COCO_M + ar * COCO_M + mi;
    const size_t plane = (size_t)a.C * COCO_A * COCO_M;
    double *prec = a.precision + (size_t)t * COCO_R * plane + cell;
    const long long np = a.npig[c * COCO_A + ar];
    if (np == 0) {                   // COCOeval leaves -1 where the class has no non-ignored ground truth
        for (int j = tid; j < COCO_R; j += blockDim.x) prec[j * plane] = -1.0;
        if (tid == 0) a.recall[t * plane + cell] = -1.0;
        return;
    }
    for (int j = tid; j < COCO_R; j += blockDim.x) {
        rthr[j] = a.rec_thr[j];
        q[j] = 0.0;
    }
    const uint64_t *e = a.e + a.class_start[c];
    const long long n = a.class_count[c];
    const int bit = ar * COCO_T + t;
    // a record counts as fp << 32 | tp; records ranked >= max_det in their image are left out (they count 0, and their
    // precision repeats a kept record's, so the envelope is unchanged)
    auto load = [&](long long r) -> unsigned long long {
        const uint32_t slot = (uint32_t)(e[r] >> 32);
        if ((int)(slot % (uint32_t)a.KD) >= max_det) return 0ull;
        if ((a.tp[slot] >> bit) & 1u) return 1ull;
        return ((a.nig[slot] >> bit) & 1u) ? 1ull << 32 : 0ull;
    };
    unsigned long long s = 0;
    for (long long i = tid; i < n; i += blockDim.x) s += load(i);
    unsigned long long total;
    block_incl_scan(s, AddOp{}, 0ull, wsu, total);
    const double npd = (double)np, eps = 0x1p-52;     // np.spacing(1)
    unsigned long long after = 0;    // counts ranked below the current chunk
    double carry_max = -1.0;         // precision envelope of the ranks below the current chunk
    for (long long hi = n; hi > 0; hi -= blockDim.x) {
        const long long r = hi - 1 - tid;             // thread order runs from the lowest rank up: scans are suffix scans
        const bool v = r >= 0;
        const unsigned long long x = v ? load(r) : 0ull;
        unsigned long long chunk;
        const unsigned long long suffix = block_incl_scan(x, AddOp{}, 0ull, wsu, chunk);
        const unsigned long long cum = total - after - suffix + x;     // counts ranked at or above r
        const double tpc = (double)(cum & 0xffffffffull), fpc = (double)(cum >> 32);
        const double pr = v ? __ddiv_rn(tpc, __dadd_rn(__dadd_rn(fpc, tpc), eps)) : -1.0;
        double chunk_max;
        const double env = fmax(block_incl_scan(pr, MaxOp{}, -1.0, wsd, chunk_max), carry_max);
        if (v && (x & 1ull)) {       // recall rises here: the points in (rc_prev, rc] look up this rank
            const int j0 = recall_points_upto(rthr, __ddiv_rn(tpc - 1.0, npd));
            const int j1 = recall_points_upto(rthr, __ddiv_rn(tpc, npd));
            for (int j = j0; j < j1; ++j) q[j] = env;
        }
        after += chunk;
        carry_max = fmax(carry_max, chunk_max);
    }
    __syncthreads();
    if (tid == 0) {
        q[0] = fmax(carry_max, 0.0);                  // recall point 0 looks up the first rank (0 without records)
        a.recall[t * plane + cell] = __ddiv_rn((double)(total & 0xffffffffull), npd);
    }
    __syncthreads();
    for (int j = tid; j < COCO_R; j += blockDim.x) prec[j * plane] = q[j];
}

int coco_clear(k2y_coco *h, cudaStream_t st) {
    const size_t slots = (size_t)h->n_images * h->C * h->KD;
    if (slots) K2Y_CUDA_CHECK(cudaMemsetAsync(h->key, 0xff, slots * sizeof(uint32_t), st));
    if (h->n_images) K2Y_CUDA_CHECK(cudaMemsetAsync(h->seen, 0, h->n_images * sizeof(unsigned), st));
    K2Y_CUDA_CHECK(cudaMemsetAsync(h->status, 0, sizeof(unsigned), st));
    return K2Y_OK;
}

}  // namespace
}  // namespace k2y

extern "C" int k2y_coco_create(const double *gt_host, const long long *gt_offsets_host, long long n_images, int class_num,
                               int max_per_class, const double *iou_thresholds, const double *recall_thresholds, int device,
                               k2y_coco **out) {
    if (!out || !gt_offsets_host || !iou_thresholds || !recall_thresholds || n_images < 0 || class_num < 1 ||
        class_num > MAX_CLASSES || max_per_class < 1) {
        set_error("k2y_coco_create: bad arguments (class_num must be 1..%d, max_per_class >= 1)", MAX_CLASSES);
        return K2Y_ERR_INVALID;
    }
    for (int t = 0; t < COCO_T; ++t)
        if (!(iou_thresholds[t] > 0.0 && iou_thresholds[t] <= 1.0) || (t && !(iou_thresholds[t] > iou_thresholds[t - 1]))) {
            set_error("k2y_coco_create: the 10 IoU thresholds must increase within (0, 1]");
            return K2Y_ERR_INVALID;
        }
    for (int j = 0; j < COCO_R; ++j)
        if (!(recall_thresholds[j] >= 0.0 && recall_thresholds[j] <= 1.0) || (j && !(recall_thresholds[j] > recall_thresholds[j - 1]))) {
            set_error("k2y_coco_create: the 101 recall points must increase within [0, 1]");
            return K2Y_ERR_INVALID;
        }
    const int C = class_num;
    const long long n_gt = gt_offsets_host[n_images];
    if (gt_offsets_host[0] != 0 || (n_gt > 0 && !gt_host)) {
        set_error("k2y_coco_create: gt_offsets must start at 0");
        return K2Y_ERR_INVALID;
    }
    // group the rows per (image, class), keeping their order; count the non-ignored boxes per (class, area range)
    std::vector<long long> off((size_t)n_images * C + 1, 0);
    std::vector<long long> npig((size_t)C * COCO_A, 0);
    for (long long i = 0; i < n_images; ++i) {
        if (gt_offsets_host[i + 1] < gt_offsets_host[i]) {
            set_error("k2y_coco_create: gt_offsets decrease at image %lld", i);
            return K2Y_ERR_INVALID;
        }
        for (long long r = gt_offsets_host[i]; r < gt_offsets_host[i + 1]; ++r) {
            const double *row = gt_host + r * 7;
            const double cls = row[0], area = row[5], crowd = row[6];
            if (!(cls >= 0.0 && cls < C && cls == (double)(int)cls) || !(crowd == 0.0 || crowd == 1.0)) {
                set_error("k2y_coco_create: ground-truth row %lld has class %g (must be an integer in [0, %d)) and iscrowd %g "
                          "(must be 0 or 1)", r, cls, C, crowd);
                return K2Y_ERR_INVALID;
            }
            ++off[(size_t)i * C + (int)cls + 1];
            if (crowd == 0.0) {
                const double rng[COCO_A][2] = {{0.0, 1e10}, {0.0, 1024.0}, {1024.0, 9216.0}, {9216.0, 1e10}};
                for (int ar = 0; ar < COCO_A; ++ar) npig[(size_t)cls * COCO_A + ar] += !(area < rng[ar][0] || area > rng[ar][1]);
            }
        }
    }
    int max_g = 0;
    for (size_t i = 1; i < off.size(); ++i) {
        max_g = (int)std::max<long long>(max_g, off[i]);
        off[i] += off[i - 1];
    }
    std::vector<double> grouped((size_t)n_gt * COCO_GT_FIELDS);
    {
        std::vector<long long> fill(off.begin(), off.end() - 1);
        for (long long i = 0; i < n_images; ++i)
            for (long long r = gt_offsets_host[i]; r < gt_offsets_host[i + 1]; ++r) {
                const double *row = gt_host + r * 7;
                const long long dst = fill[(size_t)i * C + (int)row[0]]++;
                std::copy(row + 1, row + 7, grouped.begin() + dst * COCO_GT_FIELDS);
            }
    }
    const int KD = std::min(max_per_class, COCO_MAX_DETS);
    const size_t warp_smem = coco_warp_smem(KD, max_g);
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) {
        cudaGetLastError();
        set_error("k2y_coco_create: no CUDA device %d", device);
        return K2Y_ERR_CUDA;
    }
    DeviceGuard g(device);
    int dev_smem = 0;
    K2Y_CUDA_CHECK(cudaDeviceGetAttribute(&dev_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
    if (warp_smem > (size_t)dev_smem) {
        set_error("k2y_coco_create: an image has %d ground-truth boxes of one category, more than the match kernel holds", max_g);
        return K2Y_ERR_INVALID;
    }
    const long long slots = n_images * C * KD;
    if (slots >= (1ll << 32) - SORT_TILE) {
        set_error("k2y_coco_create: %lld record slots (images x classes x min(max_per_class, 100)); the ranking counts with 32 "
                  "bits", slots);
        return K2Y_ERR_INVALID;
    }
    k2y_coco *h = new k2y_coco();
    h->device = device;
    h->C = C;
    h->K = max_per_class;
    h->KD = KD;
    h->n_images = n_images;
    h->max_g = max_g;
    h->warp_smem = warp_smem;
    h->warps = (int)std::max<size_t>(1, std::min<size_t>(COCO_MATCH_MAX_WARPS, (size_t)dev_smem / 2 / warp_smem));
    const size_t nslot = std::max<long long>(slots, 1), nimg = std::max<long long>(n_images, 1);
    if (cudaMalloc(&h->gt, std::max<size_t>(grouped.size(), 1) * sizeof(double)) != cudaSuccess ||
        cudaMalloc(&h->gt_off, off.size() * sizeof(long long)) != cudaSuccess ||
        cudaMalloc(&h->npig, npig.size() * sizeof(long long)) != cudaSuccess ||
        cudaMalloc(&h->params, (COCO_T + COCO_R) * sizeof(double)) != cudaSuccess ||
        cudaMalloc(&h->key, nslot * sizeof(uint32_t)) != cudaSuccess ||
        cudaMalloc(&h->tp, nslot * sizeof(uint64_t)) != cudaSuccess ||
        cudaMalloc(&h->nig, nslot * sizeof(uint64_t)) != cudaSuccess ||
        cudaMalloc(&h->seen, nimg * sizeof(unsigned)) != cudaSuccess ||
        cudaMalloc(&h->status, sizeof(unsigned)) != cudaSuccess ||
        cudaMemcpy(h->gt, grouped.data(), grouped.size() * sizeof(double), cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(h->gt_off, off.data(), off.size() * sizeof(long long), cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(h->npig, npig.data(), npig.size() * sizeof(long long), cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(h->params, iou_thresholds, COCO_T * sizeof(double), cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(h->params + COCO_T, recall_thresholds, COCO_R * sizeof(double), cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaEventCreateWithFlags(&h->done, cudaEventDisableTiming) != cudaSuccess || coco_clear(h, 0) != K2Y_OK ||
        cudaStreamSynchronize(0) != cudaSuccess) {
        set_error("k2y_coco_create: %s", cudaGetErrorString(cudaGetLastError()));
        k2y_coco_destroy(h);
        return K2Y_ERR_CUDA;
    }
    *out = h;
    return K2Y_OK;
}

extern "C" int k2y_coco_destroy(k2y_coco *h) {
    if (!h) return K2Y_OK;
    DeviceGuard g(h->device);
    if (h->done) cudaEventSynchronize(h->done);
    for (void *p : {(void *)h->gt, (void *)h->gt_off, (void *)h->npig, (void *)h->params, (void *)h->key, (void *)h->tp,
                    (void *)h->nig, (void *)h->seen, (void *)h->status})
        cudaFree(p);
    if (h->done) cudaEventDestroy(h->done);
    delete h;
    return K2Y_OK;
}

extern "C" int k2y_coco_match(k2y_coco *h, const int32_t *dets_dev, const int32_t *counts_dev, long long det_image_stride_words,
                              long long count_image_stride_words, int n_images, const long long *image_positions_dev,
                              void *stream) {
    if (!h || n_images < 0 || (n_images > 0 && (!dets_dev || !counts_dev || !image_positions_dev))) {
        set_error("k2y_coco_match: bad arguments");
        return K2Y_ERR_INVALID;
    }
    if (det_image_stride_words < (long long)h->C * h->K * 6 || count_image_stride_words < h->C) {
        set_error("k2y_coco_match: image strides smaller than one image's records / counts");
        return K2Y_ERR_INVALID;
    }
    if (n_images == 0) return K2Y_OK;
    DeviceGuard g(h->device);
    cudaStream_t st = (cudaStream_t)stream;
    if (int rc = begin(h, st)) return rc;
    CocoMatchArgs a;
    a.dets = dets_dev;
    a.counts = counts_dev;
    a.det_stride = det_image_stride_words;
    a.count_stride = count_image_stride_words;
    a.pos = image_positions_dev;
    a.n = n_images;
    a.C = h->C;
    a.K = h->K;
    a.KD = h->KD;
    a.max_g = h->max_g;
    a.n_images = h->n_images;
    a.warp_doubles = h->warp_smem / sizeof(double);
    a.gt = h->gt;
    a.gt_off = h->gt_off;
    a.thr = h->params;
    a.key = h->key;
    a.tp = h->tp;
    a.nig = h->nig;
    a.seen = h->seen;
    a.status = h->status;
    const size_t smem = h->warp_smem * h->warps;
    if (smem > 48 * 1024) K2Y_CUDA_CHECK(cudaFuncSetAttribute(coco_match_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const long long warps = (long long)n_images * h->C;
    coco_match_kernel<<<(unsigned)((warps + h->warps - 1) / h->warps), h->warps * 32, smem, st>>>(a);
    K2Y_CUDA_CHECK(cudaGetLastError());
    return finish(h, st);
}

extern "C" int k2y_coco_result(k2y_coco *h, double *precision_host, double *recall_host, unsigned *status_host, void *stream) {
    if (!h || !precision_host || !recall_host || !status_host) {
        set_error("k2y_coco_result: null pointer");
        return K2Y_ERR_INVALID;
    }
    DeviceGuard g(h->device);
    cudaStream_t st = (cudaStream_t)stream;
    if (int rc = begin(h, st)) return rc;
    const int C = h->C;
    const long long n_slots = h->n_images * C * h->KD;
    const size_t n_prec = (size_t)COCO_T * COCO_R * C * COCO_A * COCO_M, n_rec = (size_t)COCO_T * C * COCO_A * COCO_M;
    // scratch: precision, recall, then rank_slots' words
    char *scratch = nullptr;
    K2Y_CUDA_CHECK(cudaMallocAsync(&scratch, (n_prec + n_rec) * sizeof(double) + rank_scratch_words(n_slots, C) * sizeof(uint32_t), st));
    double *prec_dev = reinterpret_cast<double *>(scratch), *rec_dev = prec_dev + n_prec;
    uint32_t *totals = reinterpret_cast<uint32_t *>(rec_dev + n_rec), *bases = totals + MAX_CLASSES;
    uint64_t *buf[2] = {nullptr, nullptr};
    const uint64_t *sorted = nullptr;
    SortPass p = {};
    p.slot_key = h->key;
    p.n = n_slots;
    p.C = C;
    p.K = h->KD;
    if (int rc = rank_slots<CocoElem>(p, totals, buf, sorted, st)) return rc;
    CocoCurveArgs ca;
    ca.e = sorted;
    ca.class_start = bases;
    ca.class_count = totals;
    ca.tp = h->tp;
    ca.nig = h->nig;
    ca.npig = h->npig;
    ca.rec_thr = h->params + COCO_T;
    ca.C = C;
    ca.KD = h->KD;
    ca.precision = prec_dev;
    ca.recall = rec_dev;
    coco_curve_kernel<<<dim3(COCO_T * COCO_A * COCO_M, C), CURVE_THREADS, 0, st>>>(ca);
    K2Y_CUDA_CHECK(cudaGetLastError());
    K2Y_CUDA_CHECK(cudaMemcpyAsync(precision_host, prec_dev, n_prec * sizeof(double), cudaMemcpyDeviceToHost, st));
    K2Y_CUDA_CHECK(cudaMemcpyAsync(recall_host, rec_dev, n_rec * sizeof(double), cudaMemcpyDeviceToHost, st));
    K2Y_CUDA_CHECK(cudaMemcpyAsync(status_host, h->status, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    for (uint64_t *b : buf)
        if (b) K2Y_CUDA_CHECK(cudaFreeAsync(b, st));
    K2Y_CUDA_CHECK(cudaFreeAsync(scratch, st));
    if (int rc = finish(h, st)) return rc;
    K2Y_CUDA_CHECK(cudaStreamSynchronize(st));
    return K2Y_OK;
}

extern "C" int k2y_coco_reset(k2y_coco *h, void *stream) {
    if (!h) {
        set_error("k2y_coco_reset: null handle");
        return K2Y_ERR_INVALID;
    }
    DeviceGuard g(h->device);
    cudaStream_t st = (cudaStream_t)stream;
    if (int rc = begin(h, st)) return rc;
    if (int rc = coco_clear(h, st)) return rc;
    return finish(h, st);
}
