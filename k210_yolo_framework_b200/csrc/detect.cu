// Fused decode + per-class greedy NMS, both dialects of the reference:
//   KERAS    keras_inference.py:94-135 (+ tools/utils.py:524-547, keras_inference.py:32-72)
//   REGION_C yolo3_frame_test_public/region_layer.c:121-283
// KERAS, two kernels:
//   detect_scan_kernel  CTA = 64-box slab of one image.  The slab's records ([box][5+C] floats, contiguous in the NHWC head)
//                       are staged in shared memory with coalesced loads, so every head value is read from HBM exactly once;
//                       sigmoid(conf) is evaluated once per box, every box is decoded once (tf_xywh_to_all + correct_box)
//                       into a per-image box table, and every (box, class) with score >= obj_thresh appends its sort key
//                       (score bits << 32 | ~index) to the class's candidate list.
//   detect_nms_kernel   CTA = one (image, class), 512 threads: the class's greedy NMS in one of three tiers, chosen from its
//                       candidate count (the rule is stated above the kernel):
//                         chunked  <= 256 candidates: rank sort, then 32-candidate chunks resolved warp by warp;
//                         rounds   keys in registers, decoded boxes in shared memory (4 or 8 slots per thread), then
//                                  <= max_per_class rounds of "best live candidate (CTA-wide arg-max, no sort) -> keep ->
//                                  every thread tests its candidates against it";
//                         global   the same rounds with keys, boxes and liveness bits in global memory.
// REGION_C: one CTA per image (softmax + decode by all threads, then one warp per class).
//
// Arithmetic is float32 in the reference's operation order with explicit round-to-nearest intrinsics where FMA
// contraction would change a rounding.  exp() is DEFINED, for the KERAS dialect, as the correctly rounded float32
// exponential (computed in double and rounded once; oracle/decode_ref.py does the same), so scores, their order and
// therefore the survivor sets are bit-identical to the oracle's on identical head tensors.  The REGION_C dialect calls
// glibc's expf in the reference; expf_glibc() below restates that algorithm (table + cubic in double) bit for bit.
#include <cmath>
#include <cstdlib>
#include <vector>

#include "common.h"

namespace k2y {

namespace {

constexpr int DET_THREADS = 1024;
constexpr unsigned FULL = 0xffffffffu;

// correctly rounded float32 exp: double-precision exp (<= 1 ulp of double) rounded once to float
__device__ __forceinline__ float exp_cr(float x) { return __double2float_rn(exp((double)x)); }
__device__ __forceinline__ float sigmoidf_ref(float x) { return __fdiv_rn(1.0f, __fadd_rn(1.0f, exp_cr(-x))); }

// glibc >= 2.28 expf (sysdeps/ieee754/flt-32/e_expf.c, EXP2F_TABLE_BITS = 5): exp(x) = 2^(k/32) * 2^(r/32) with
// k = round(x * 32/ln2), the second factor a cubic in r, all in double, one final rounding to float.  The x86-64 build
// selects the FMA variant on every CPU of this decade, hence the explicit fma()s.  Overflow/underflow limits as glibc's.
__constant__ unsigned long long EXP2F_TAB[32] = {
    0x3ff0000000000000ull, 0x3fefd9b0d3158574ull, 0x3fefb5586cf9890full, 0x3fef9301d0125b51ull,
    0x3fef72b83c7d517bull, 0x3fef54873168b9aaull, 0x3fef387a6e756238ull, 0x3fef1e9df51fdee1ull,
    0x3fef06fe0a31b715ull, 0x3feef1a7373aa9cbull, 0x3feedea64c123422ull, 0x3feece086061892dull,
    0x3feebfdad5362a27ull, 0x3feeb42b569d4f82ull, 0x3feeab07dd485429ull, 0x3feea47eb03a5585ull,
    0x3feea09e667f3bcdull, 0x3fee9f75e8ec5f74ull, 0x3feea11473eb0187ull, 0x3feea589994cce13ull,
    0x3feeace5422aa0dbull, 0x3feeb737b0cdc5e5ull, 0x3feec49182a3f090ull, 0x3feed503b23e255dull,
    0x3feee89f995ad3adull, 0x3feeff76f2fb5e47ull, 0x3fef199bdd85529cull, 0x3fef3720dcef9069ull,
    0x3fef5818dcfba487ull, 0x3fef7c97337b9b5full, 0x3fefa4afa2a490daull, 0x3fefd0765b6e4540ull,
};
__device__ __forceinline__ float expf_glibc(float x) {
    if (!(x == x)) return x + x;
    if (x > 88.72283172607421875f) return __int_as_float(0x7f800000);   // 0x1.62e42ep6f
    if (x < -103.97207641601562500f) return 0.0f;                       // -0x1.9fe368p6f
    const double z = __dmul_rn(0x1.71547652b82fep+5, (double)x);         // 32/ln2
    double kd = __dadd_rn(z, 6755399441055744.0);                        // + 0x1.8p52: round to nearest integer
    const unsigned long long ki = (unsigned long long)__double_as_longlong(kd);
    kd = __dsub_rn(kd, 6755399441055744.0);
    const double r = __dsub_rn(z, kd);
    const unsigned long long t = EXP2F_TAB[ki & 31ull] + (ki << 47);
    const double s = __longlong_as_double((long long)t);
    const double zz = __fma_rn(0x1.c6af84b912394p-20, r, 0x1.ebfce50fac4f3p-13);
    const double r2 = __dmul_rn(r, r);
    double y = __fma_rn(0x1.62e42ff0c52d6p-6, r, 1.0);
    y = __fma_rn(zz, r2, y);
    return __double2float_rn(__dmul_rn(y, s));
}
__device__ __forceinline__ float sigmoidf_glibc(float x) { return __fdiv_rn(1.0f, __fadd_rn(1.0f, expf_glibc(-x))); }

__device__ __forceinline__ unsigned long long pack_key(float score, int idx) {
    // scores are > 0 here, so the IEEE bit pattern is monotonic; larger key == earlier in the order
    return ((unsigned long long)__float_as_uint(score) << 32) | (unsigned long long)(0xffffffffu - (unsigned)idx);
}
__device__ __forceinline__ int key_index(unsigned long long k) { return (int)(0xffffffffu - (unsigned)(k & 0xffffffffull)); }
__device__ __forceinline__ float key_score(unsigned long long k) { return __uint_as_float((unsigned)(k >> 32)); }

// The rounds tier's key also carries the candidate's position in shared memory: (score bits << 32) | ((0xFFFFF - index) << 12)
// | position.  The low 12 bits never decide a comparison (the (score, index) pair is unique), so ONE 64-bit maximum yields the
// winner AND where its decoded box sits.  Needs index < 2^20 - 1 and position < 4096.
__device__ __forceinline__ unsigned long long pack_pos_key(unsigned long long key, int pos) {
    return (key & 0xffffffff00000000ull) | ((unsigned long long)(0xFFFFFu - (unsigned)key_index(key)) << 12) | (unsigned long long)pos;
}
__device__ __forceinline__ int pos_key_index(unsigned long long k) { return (int)(0xFFFFFu - (unsigned)((k >> 12) & 0xFFFFFull)); }
__device__ __forceinline__ int pos_key_position(unsigned long long k) { return (int)(k & 0xFFFull); }

// Sort (descending) n <= 32 keys held one per lane (lanes >= n hold 0).
__device__ __forceinline__ unsigned long long warp_sort_desc(unsigned long long key, int lane) {
#pragma unroll
    for (int k = 2; k <= 32; k <<= 1) {
#pragma unroll
        for (int j = k >> 1; j > 0; j >>= 1) {
            const unsigned long long other = __shfl_xor_sync(FULL, key, j);
            const bool up = ((lane & k) == 0);      // this k-block sorts descending
            const bool lower = ((lane & j) == 0);   // this lane keeps the "first" element
            const bool take_max = (up == lower);
            key = take_max ? (key > other ? key : other) : (key < other ? key : other);
        }
    }
    return key;
}

// Bitonic sort (descending) of P (power of two) keys in memory by one warp.
__device__ __forceinline__ void warp_sort_desc_mem(unsigned long long *keys, int P, int lane) {
    for (int k = 2; k <= P; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = lane; i < P; i += 32) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const unsigned long long a = keys[i], b = keys[ixj];
                    const bool desc = ((i & k) == 0);
                    if (desc ? (a < b) : (a > b)) {
                        keys[i] = b;
                        keys[ixj] = a;
                    }
                }
            }
            __syncwarp();
        }
    }
}

// tf.image.non_max_suppression's test `IoU(a, b) > thr` on (ymin,xmin,ymax,xmax) boxes (zero-area boxes -> IoU 0), without
// the division in the common case: inter/uni > thr  <=>  inter > thr*uni (uni > 0).  The product form is only trusted
// outside a 1e-6 relative margin, and only where that margin argument holds: thr and t = fl(thr*uni) both normal floats
// (>= 2^-126) and t < 2^126.  Then t and fl(t * 1.000001f) each carry one relative rounding <= 2^-24, so inter above it
// puts the exact quotient above thr * (1 + 8e-7), past the next float after thr (a normal thr's ulp is <= 2^-23 * thr), and
// fl(inter/uni) > thr; the lower side likewise.  Outside that range the exact IEEE division decides:
//   - thr == +-0: inter > 0 does NOT imply fl(inter/uni) > 0 — a denormal-area box inside a large one has a quotient
//     below 2^-150 that rounds to 0 (IoU 0, kept by the reference);
//   - a subnormal thr or t: their rounding error is absolute (2^-150), not relative, and exceeds the margin;
//   - uni infinite or NaN (boxes decoded from exp overflow): t is inf or NaN;
//   - thr < 0: IoU >= 0 > thr is the division's own answer, and a NaN IoU (two infinite boxes) is not > thr.
// So the boolean is bit-identical to the reference's `iou > iou_threshold` for every float input.  Boxes are (min,max)-normalised with their areas
// cached (once per box instead of once per pair).  One body computes the intersection and union; two control-flow forms decide
// the same boolean from them:
//   iou_norm_gt     straight-line (selects, the exact division only under a rarely-taken branch).  The chunked tier tests up to
//                   eight independent pairs per thread in a row, and with early-outs the compiler serialises those chains
//                   (~190 cycles each) instead of interleaving them.
//   iou_norm_gt_eo  early returns.  The rounds tiers and the operator NMS test one pair per live candidate under its own liveness
//                   branch; there the early-out form measured faster (on an H100 at 700 W the 8-slot rounds tier ran ~9 %
//                   slower with the straight-line form).
__device__ __forceinline__ float4 norm_box(const float4 a, float &area) {
    float4 n;
    n.x = fminf(a.x, a.z);
    n.y = fminf(a.y, a.w);
    n.z = fmaxf(a.x, a.z);
    n.w = fmaxf(a.y, a.w);
    area = __fmul_rn(__fsub_rn(n.z, n.x), __fsub_rn(n.w, n.y));
    return n;
}
__device__ __forceinline__ float2 iou_terms(const float4 a, float area_a, const float4 b, float area_b) {
    const float iy = fmaxf(__fsub_rn(fminf(a.z, b.z), fmaxf(a.x, b.x)), 0.f);
    const float ix = fmaxf(__fsub_rn(fminf(a.w, b.w), fmaxf(a.y, b.y)), 0.f);
    const float inter = __fmul_rn(iy, ix);
    return make_float2(inter, __fsub_rn(__fadd_rn(area_a, area_b), inter));
}
__device__ __forceinline__ bool product_form_usable(float thr, float t) {
    return thr >= 0x1p-126f && t >= 0x1p-126f && t < 0x1p126f;   // false for NaN
}
__device__ __forceinline__ bool iou_norm_gt(const float4 a, float area_a, const float4 b, float area_b, float thr) {
    const float2 iu = iou_terms(a, area_a, b, area_b);
    const float inter = iu.x, uni = iu.y;
    const float t = __fmul_rn(thr, uni);
    const bool usable = product_form_usable(thr, t);
    const bool gt = usable && inter > __fmul_rn(t, 1.000001f);
    const bool lt = usable && inter < __fmul_rn(t, 0.999999f);
    bool res = gt;
    if (!(gt || lt)) res = __fdiv_rn(inter, uni) > thr;                 // inside the margin (or degenerate): exact IEEE division
    const bool degenerate = area_a <= 0.f || area_b <= 0.f;             // zero-area boxes: IoU 0
    return degenerate ? (0.f > thr) : res;
}
__device__ __forceinline__ bool iou_norm_gt_eo(const float4 a, float area_a, const float4 b, float area_b, float thr) {
    if (area_a <= 0.f || area_b <= 0.f) return 0.f > thr;
    const float2 iu = iou_terms(a, area_a, b, area_b);
    const float inter = iu.x, uni = iu.y;
    const float t = __fmul_rn(thr, uni);
    if (product_form_usable(thr, t)) {
        if (inter > __fmul_rn(t, 1.000001f)) return true;
        if (inter < __fmul_rn(t, 0.999999f)) return false;
    }
    return __fdiv_rn(inter, uni) > thr;
}

// region_layer.c box_iou on centre-form (x,y,w,h) boxes (:228-254).
__device__ __forceinline__ float overlap_c(float x1, float w1, float x2, float w2) {
    const float l1 = __fsub_rn(x1, __fmul_rn(w1, 0.5f));
    const float l2 = __fsub_rn(x2, __fmul_rn(w2, 0.5f));
    const float left = l1 > l2 ? l1 : l2;
    const float r1 = __fadd_rn(x1, __fmul_rn(w1, 0.5f));
    const float r2 = __fadd_rn(x2, __fmul_rn(w2, 0.5f));
    const float right = r1 < r2 ? r1 : r2;
    return __fsub_rn(right, left);
}
__device__ __forceinline__ float iou_center(const float4 a, const float4 b) {
    const float w = overlap_c(a.x, a.z, b.x, b.z);
    const float h = overlap_c(a.y, a.w, b.y, b.w);
    const float inter = (w < 0.f || h < 0.f) ? 0.f : __fmul_rn(w, h);
    const float uni = __fsub_rn(__fadd_rn(__fmul_rn(a.z, a.w), __fmul_rn(b.z, b.w)), inter);
    return __fdiv_rn(inter, uni);
}

struct KerasParams {
    const float *heads[3];
    int lh[3], lw[3], loff[4];
    int n_layers, A, C, nbox, P;
    float anchors[48];
    float in_h, in_w;
    float obj, iou;
    float logit_min;                  // a logit below this cannot give a sigmoid >= obj (with a wide margin); -inf = no shortcut
    unsigned long long c_magic;       // ceil(2^32 / C) = (2^32 + e) / C, 0 <= e < C, up to 2^32 (C == 1): it / C == (it * c_magic) >> 32
                                      // exactly while it * e < 2^32, i.e. for the it < 64 C items of a slab at every C < 8192 (the
                                      // scan's shared memory takes C <= 377)
    int maxk;
    const float *image_hw;
    k2y_det *dets;
    int *counts;
    long long det_stride, cnt_stride;  // per-image strides of dets / counts in 32-bit words (dense: C*maxk*6 and C)
    // workspace
    float4 *boxes;                    // [B][nbox] decoded (ymin,xmin,ymax,xmax) of every box
    unsigned long long *keys;         // [B][C][P] candidate sort keys
    int *ncand;                       // [B][C] candidates per (image, class); zeroed before the scan
    unsigned *alive;                  // [B][C][alive_stride] liveness words (only when a class has more candidates than fit shared memory)
    int alive_stride;
    int cap;                          // candidates the NMS kernel can hold in shared memory (key 8 B + decoded box 16 B each)
};

// Collects the candidates of one class (score > thr) in index order, sorts them.
// Returns n; on return either `rkey` holds the sorted keys (n <= 32) or keys[0..n) does.
__device__ __forceinline__ int gather_sorted(const float *sc, int nbox, float thr, unsigned long long *keys, int lane,
                                             unsigned long long &rkey) {
    int n = 0;
    for (int base = 0; base < nbox; base += 32) {
        const int i = base + lane;
        const float s = (i < nbox) ? sc[i] : -1.f;
        const bool pass = (i < nbox) && s > thr;
        const unsigned m = __ballot_sync(FULL, pass);
        if (pass) keys[n + __popc(m & ((1u << lane) - 1u))] = pack_key(s, i);
        n += __popc(m);
    }
    __syncwarp();
    rkey = 0ull;
    if (n <= 32) {
        if (lane < n) rkey = keys[lane];
        rkey = warp_sort_desc(rkey, lane);
    } else {
        int P = 64;
        while (P < n) P <<= 1;
        for (int i = n + lane; i < P; i += 32) keys[i] = 0ull;
        __syncwarp();
        warp_sort_desc_mem(keys, P, lane);
    }
    return n;
}

// The box decode, shared by the fused scan kernel and the operator kernels (xywh_to_all_kernel, correct_box_kernel), so
// that both give the same bits.

// correct_box's letterbox constants of one image (keras_inference.py:53-58)
struct BoxXform {
    float img_h, img_w, off_y, off_x, sc_y, sc_x;
};
__device__ __forceinline__ BoxXform letterbox(float in_h, float in_w, float img_h, float img_w) {
    BoxXform x;
    x.img_h = img_h;
    x.img_w = img_w;
    const float r = fminf(__fdiv_rn(in_h, img_h), __fdiv_rn(in_w, img_w));
    const float new_h = rintf(__fmul_rn(img_h, r)), new_w = rintf(__fmul_rn(img_w, r));
    x.off_y = __fdiv_rn(__fdiv_rn(__fsub_rn(in_h, new_h), 2.0f), in_h);
    x.off_x = __fdiv_rn(__fdiv_rn(__fsub_rn(in_w, new_w), 2.0f), in_w);
    x.sc_y = __fdiv_rn(in_h, new_h);
    x.sc_x = __fdiv_rn(in_w, new_w);
    return x;
}

// tf_xywh_to_all (tools/utils.py:545-546) for one box, given sigmoid(tx), sigmoid(ty), exp(tw), exp(th), its cell (col, row)
// of a W x H layer and its anchor (aw, ah): (x, y, w, h) as fractions of the network input
__device__ __forceinline__ float4 xywh_to_all(float sx, float sy, float ew, float eh, int col, int row, int W, int H, float aw,
                                              float ah) {
    float4 r;
    r.x = __fdiv_rn(__fadd_rn(sx, (float)col), (float)W);
    r.y = __fdiv_rn(__fadd_rn(sy, (float)row), (float)H);
    r.z = __fmul_rn(ew, aw);
    r.w = __fmul_rn(eh, ah);
    return r;
}

// correct_box (keras_inference.py:59-71) for one box: (x, y, w, h) relative to the letterboxed input -> (ymin, xmin, ymax, xmax)
// in pixels of the original image
__device__ __forceinline__ float4 to_corners(const BoxXform &x, const float4 b) {
    const float cy = __fmul_rn(__fsub_rn(b.y, x.off_y), x.sc_y), cx = __fmul_rn(__fsub_rn(b.x, x.off_x), x.sc_x);
    const float hh2 = __fdiv_rn(__fmul_rn(b.w, x.sc_y), 2.0f), ww2 = __fdiv_rn(__fmul_rn(b.z, x.sc_x), 2.0f);
    float4 r;
    r.x = __fmul_rn(__fsub_rn(cy, hh2), x.img_h);
    r.y = __fmul_rn(__fsub_rn(cx, ww2), x.img_w);
    r.z = __fmul_rn(__fadd_rn(cy, hh2), x.img_h);
    r.w = __fmul_rn(__fadd_rn(cx, ww2), x.img_w);
    return r;
}

// ---- pass 1: scan.  grid = (ceil(nbox / 64), B) ----------------------------------------------------------------------
constexpr int SCAN_THREADS = 256;
constexpr int SCAN_BOXES = 64;

__global__ void __launch_bounds__(SCAN_THREADS) detect_scan_kernel(const KerasParams p) {
    extern __shared__ __align__(16) float s_scan[];  // [SCAN_BOXES][E] records, then [SCAN_BOXES] sigmoid(conf)
    const int b = blockIdx.y, box0 = blockIdx.x * SCAN_BOXES, tid = threadIdx.x;
    const int nb = min(SCAN_BOXES, p.nbox - box0);
    const int E = 5 + p.C;
    float *s_rec = s_scan, *s_conf = s_scan + SCAN_BOXES * E;
    pdl_wait();  // the heads belong to the previous kernel
    // the boxes of a layer are contiguous [cell][anchor] records of the NHWC head: a slab is one run per layer it touches
    for (int l = 0; l < p.n_layers; ++l) {
        const int lo = max(box0, p.loff[l]), hi = min(box0 + nb, p.loff[l + 1]);
        if (lo >= hi) continue;
        const float *src = p.heads[l] + ((size_t)b * (p.loff[l + 1] - p.loff[l]) + (lo - p.loff[l])) * E;
        float *dst = s_rec + (lo - box0) * E;
        const int cnt = (hi - lo) * E;
        // four loads in flight per thread before the first store: the slab is cold (HBM / L2), a load-store-load chain would
        // pay the full latency once per element
        for (int i0 = 0; i0 < cnt; i0 += 4 * SCAN_THREADS) {
            float v[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int i = i0 + u * SCAN_THREADS + tid;
                v[u] = i < cnt ? __ldg(src + i) : 0.f;
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int i = i0 + u * SCAN_THREADS + tid;
                if (i < cnt) dst[i] = v[u];
            }
        }
    }
    __syncthreads();
    float *s_thr = s_conf + SCAN_BOXES;
    // The five transcendentals of a box — sigmoid(tx), sigmoid(ty), exp(tw), exp(th), sigmoid(conf), each a correctly rounded
    // (double precision) exponential — are spread over ALL threads (5 * nb items), written back in place of the raw values; with
    // one thread per box the two warps doing the decode were the critical path of the CTA.
    for (int it = tid; it < 5 * nb; it += SCAN_THREADS) {
        const int i = it / 5, k = it - 5 * i;
        float *e = s_rec + i * E + k;
        const float t = *e;
        float r;
        if (k == 4) r = (t < p.logit_min) ? 0.f : sigmoidf_ref(t);   // 0 marks "no class can pass" (obj > 0 whenever the shortcut is on)
        else if (k < 2) r = sigmoidf_ref(t);
        else r = exp_cr(t);
        *e = r;
    }
    __syncthreads();
    if (tid < nb) {
        // score = sigmoid(cls) * sigmoid(conf) <= sigmoid(conf): a box whose objectness is below the threshold has no candidate
        // in any class.  For the other boxes a class can only pass if sigmoid(cls) >= obj / sigmoid(conf), i.e. cls >=
        // logit(obj / sc): a per-box logit bound (with a margin of 2e-3 (+0.2 %), thousands of float ulps of the sigmoid)
        // rejects most (box, class) pairs with ONE comparison instead of a correctly rounded exponential.
        const float sc = s_rec[tid * E + 4];
        s_conf[tid] = sc;
        float thr = p.logit_min;
        if (p.logit_min > -__int_as_float(0x7f800000) && sc >= p.obj) {
            const float q = __fdividef(p.obj, sc);
            if (q < 0.999f) {   // 1 - q >= 1e-3: the margin below is > 1e-5 of the sigmoid, the float roundings involved < 1e-6
                const float lg = __logf(__fdividef(q, 1.0f - q));
                thr = fmaxf(thr, lg - 2e-3f - 2e-3f * fabsf(lg));
            }
        }
        s_thr[tid] = thr;
    } else if (tid >= SCAN_BOXES && tid < SCAN_BOXES + nb) {
        // the record's first four entries hold sigmoid(tx), sigmoid(ty), exp(tw), exp(th) now
        const int i = tid - SCAN_BOXES;
        const BoxXform x = letterbox(p.in_h, p.in_w, p.image_hw[2 * b], p.image_hw[2 * b + 1]);
        const float *e = s_rec + i * E;
        const int box = box0 + i;
        int l = 0;
        if (p.n_layers > 1 && box >= p.loff[1]) l = 1;
        if (p.n_layers > 2 && box >= p.loff[2]) l = 2;
        const int local = box - p.loff[l];
        const int a = local % p.A, cell = local / p.A;
        const int W = p.lw[l];
        const float4 xywh = xywh_to_all(e[0], e[1], e[2], e[3], cell % W, cell / W, W, p.lh[l], p.anchors[(l * p.A + a) * 2],
                                        p.anchors[(l * p.A + a) * 2 + 1]);
        p.boxes[(size_t)b * p.nbox + box0 + i] = to_corners(x, xywh);
    }
    __syncthreads();
    const bool shortcut = p.logit_min > -__int_as_float(0x7f800000);
    // (box, class) pairs, four per thread at a time: scores first, then the list-slot atomics back to back (independent, so
    // their L2 round trips overlap), then the keys
    const int n_items = nb * p.C;
    for (int it0 = 0; it0 < n_items; it0 += 4 * SCAN_THREADS) {
        float sc4[4];
        int cls[4], bi[4];
        bool pass[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int it = it0 + u * SCAN_THREADS + tid;
            pass[u] = false;
            sc4[u] = 0.f;
            cls[u] = bi[u] = 0;
            if (it < n_items) {
                const int i = (int)(((unsigned long long)(unsigned)it * p.c_magic) >> 32), c = it - i * p.C;
                const float t = s_rec[i * E + 5 + c];
                if (!(t < s_thr[i])) {
                    const float sc = s_conf[i];
                    if (!shortcut || sc >= p.obj) {
                        const float s = __fmul_rn(sigmoidf_ref(t), sc);
                        pass[u] = s >= p.obj;
                        sc4[u] = s;
                        cls[u] = c;
                        bi[u] = box0 + i;
                    }
                }
            }
        }
        int pos[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) pos[u] = pass[u] ? atomicAdd(p.ncand + b * p.C + cls[u], 1) : 0;
#pragma unroll
        for (int u = 0; u < 4; ++u)
            if (pass[u]) p.keys[((size_t)b * p.C + cls[u]) * p.P + pos[u]] = pack_key(sc4[u], bi[u]);
    }
}

// ---- pass 2: greedy NMS.  grid = (C, B), one CTA of NMS_THREADS per (image, class) ---------------------------------------
// tf.image.non_max_suppression visits candidates in descending score and keeps one iff no box kept earlier overlaps it by
// more than the threshold.  The rounds tiers restate this as: repeat { take the best candidate still alive, keep it, kill
// everything it overlaps } — at most max_per_class rounds, with NO sort: a round is an arg-max over the live candidates
// (warp-reduce instructions on the key + one shared-memory exchange) followed by one IoU test per live candidate, all
// candidates spread over the CTA's threads.  The selection order is exactly the order of the sorted keys (score descending,
// index ascending), so the records equal the sequential algorithm's.
constexpr int NMS_THREADS = 512;
constexpr int NMS_WARPS = NMS_THREADS / 32;

__device__ __forceinline__ void write_det(k2y_det *out, int slot, const float4 box, float score, int index) {
    k2y_det d;
    d.ymin = box.x;
    d.xmin = box.y;
    d.ymax = box.z;
    d.xmax = box.w;
    d.score = score;
    d.index = index;
    out[slot] = d;
}

// Global-memory rounds (n > cap): keys and decoded boxes are read from the global candidate lists, the liveness bits live in
// global memory.  Candidate `pos` belongs to thread pos % NMS_THREADS; its liveness is bit (pos / NMS_THREADS) % 32 of the
// thread's word (pos / NMS_THREADS) / 32.
__device__ __forceinline__ int nms_rounds(const KerasParams &p, int n, const unsigned long long *keys, const float4 *gboxes,
                                          unsigned *alive_g, k2y_det *out, int (*s_red)[NMS_WARPS][3]) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int slots = n > tid ? (n - tid + NMS_THREADS - 1) / NMS_THREADS : 0;
    const int nwords = (slots + 31) >> 5;
    for (int w = 0; w < nwords; ++w) {
        const int left = slots - w * 32;
        alive_g[(size_t)w * NMS_THREADS + tid] = left >= 32 ? 0xffffffffu : ((1u << left) - 1u);
    }
    int nsel = 0, par = 0;
    // best live candidate of this thread; afterwards maintained by the kill pass of each round
    unsigned long long best = 0ull;
    int bpos = -1;
    for (int w = 0; w < nwords; ++w) {
        for (unsigned m = alive_g[(size_t)w * NMS_THREADS + tid]; m;) {
            const int q = __ffs(m) - 1;
            m &= m - 1u;
            const int pos = tid + (w * 32 + q) * NMS_THREADS;
            const unsigned long long k = keys[pos];
            if (bpos < 0 || k > best) {
                best = k;
                bpos = pos;
            }
        }
    }
    while (nsel < p.maxk) {
        // ---- arg-max over the CTA: (score bits, ~index) lexicographic; keys are unique, so the winner is ----
        const unsigned hi = bpos >= 0 ? (unsigned)(best >> 32) : 0u;
        const unsigned mhi = __reduce_max_sync(FULL, hi);
        const unsigned lo = (bpos >= 0 && hi == mhi) ? (unsigned)best : 0u;
        const unsigned mlo = __reduce_max_sync(FULL, lo);
        const int cpos = (bpos >= 0 && hi == mhi && lo == mlo) ? bpos : 0x7fffffff;
        const int mpos = __reduce_min_sync(FULL, cpos);
        if (lane == 0) {
            s_red[par][warp][0] = (int)mhi;
            s_red[par][warp][1] = (int)mlo;
            s_red[par][warp][2] = mpos;
        }
        __syncthreads();
        // every warp reduces the per-warp winners again (lane w holds warp w's entry): no second barrier needed
        unsigned whi = 0u, wlo = 0u;
        int wpos = 0x7fffffff;
        {
            const int ent = lane < NMS_WARPS ? lane : 0;
            const int p2 = lane < NMS_WARPS ? s_red[par][ent][2] : 0x7fffffff;
            const unsigned h2 = p2 != 0x7fffffff ? (unsigned)s_red[par][ent][0] : 0u;
            const unsigned l2 = p2 != 0x7fffffff ? (unsigned)s_red[par][ent][1] : 0u;
            whi = __reduce_max_sync(FULL, h2);
            wlo = __reduce_max_sync(FULL, (p2 != 0x7fffffff && h2 == whi) ? l2 : 0u);
            wpos = __reduce_min_sync(FULL, (p2 != 0x7fffffff && h2 == whi && l2 == wlo) ? p2 : 0x7fffffff);
        }
        par ^= 1;
        if (wpos == 0x7fffffff) break;   // nothing alive
        const unsigned long long wkey = ((unsigned long long)whi << 32) | wlo;
        const float4 ob = gboxes[key_index(wkey)];
        float ka;
        const float4 kb = norm_box(ob, ka);
        if (tid == 0) write_det(out, nsel, ob, key_score(wkey), key_index(wkey));
        // ---- the kept box kills what it overlaps (and itself); the same pass finds this thread's best survivor ----
        best = 0ull;
        bpos = -1;
        for (int w = 0; w < nwords; ++w) {
            unsigned word = alive_g[(size_t)w * NMS_THREADS + tid];
            for (unsigned m = word; m;) {
                const int q = __ffs(m) - 1;
                m &= m - 1u;
                const int pos = tid + (w * 32 + q) * NMS_THREADS;
                bool kill = pos == wpos;
                const unsigned long long k = keys[pos];
                if (!kill) {
                    float ar;
                    const float4 cb = norm_box(gboxes[key_index(k)], ar);
                    kill = iou_norm_gt_eo(kb, ka, cb, ar, p.iou);
                }
                if (kill) {
                    word &= ~(1u << q);
                } else if (bpos < 0 || k > best) {
                    best = k;
                    bpos = pos;
                }
            }
            alive_g[(size_t)w * NMS_THREADS + tid] = word;
        }
        ++nsel;
    }
    return nsel;
}

// Shared-memory rounds (n <= cap <= 4096): every thread keeps the position-carrying keys (pack_pos_key) of its candidates in
// registers — position t + s * NMS_THREADS in slot s; their boxes stay in shared memory (the register budget decides how many
// CTAs fit an SM).  A round: per-warp maximum (two warp-reduce instructions) -> shared memory -> barrier -> every warp reduces
// the per-warp maxima again -> winner's box from shared memory -> IoU tests of the thread's own live candidates.
// Work-efficient (maxk x n IoU tests), but maxk barrier-separated rounds.
template <int SLOTS>
__device__ __forceinline__ int nms_rounds_smem(const KerasParams &p, int n, const unsigned long long *s_keys, const float4 *s_box,
                                               k2y_det *out, unsigned long long *s_best) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    unsigned long long pk[SLOTS];
    unsigned alive = 0u;
    unsigned long long tbest = 0ull;
#pragma unroll
    for (int s = 0; s < SLOTS; ++s) {
        const int pos = tid + s * NMS_THREADS;
        pk[s] = 0ull;
        if (pos < n) {
            pk[s] = pack_pos_key(s_keys[pos], pos);
            alive |= 1u << s;
            tbest = pk[s] > tbest ? pk[s] : tbest;
        }
    }
    int nsel = 0, par = 0;
    while (nsel < p.maxk) {
        unsigned long long wmax = 0ull;
        if (__ballot_sync(FULL, alive != 0u) != 0u) {   // warps whose candidates are all dead only keep the barrier company
            const unsigned hi = (unsigned)(tbest >> 32);
            const unsigned mhi = __reduce_max_sync(FULL, hi);
            const unsigned lo = (alive != 0u && hi == mhi) ? (unsigned)tbest : 0u;
            const unsigned mlo = __reduce_max_sync(FULL, lo);
            wmax = ((unsigned long long)mhi << 32) | mlo;
        }
        if (lane == 0) s_best[par * NMS_WARPS + warp] = wmax;
        __syncthreads();
        const unsigned long long mine = lane < NMS_WARPS ? s_best[par * NMS_WARPS + lane] : 0ull;
        par ^= 1;
        const unsigned whi = __reduce_max_sync(FULL, (unsigned)(mine >> 32));
        const unsigned wlo = __reduce_max_sync(FULL, (unsigned)(mine >> 32) == whi ? (unsigned)mine : 0u);
        const unsigned long long w = ((unsigned long long)whi << 32) | wlo;
        if (w == 0ull) break;   // nothing alive (a live key is never 0: its index field is non-zero)
        const float4 ob = s_box[pos_key_position(w)];   // as decoded (the record keeps these); every thread normalises its own copy
        float ka;
        const float4 kb = norm_box(ob, ka);
        if (tid == 0) write_det(out, nsel, ob, key_score(w), pos_key_index(w));
        tbest = 0ull;
#pragma unroll
        for (int s = 0; s < SLOTS; ++s) {
            if ((alive >> s) & 1u) {
                float ar;
                const float4 bx = norm_box(s_box[tid + s * NMS_THREADS], ar);   // from shared memory: 2 registers per slot, not 7
                if (pk[s] == w || iou_norm_gt_eo(kb, ka, bx, ar, p.iou)) alive &= ~(1u << s);
                else tbest = pk[s] > tbest ? pk[s] : tbest;
            }
        }
        ++nsel;
    }
    return nsel;
}

// Chunked tier (n <= CHUNK_MAX = 256 candidates, maxk <= CHUNK_MAXK): the usual case.  Greedy NMS keeps a candidate iff no
// EARLIER KEPT candidate (in (score desc, index asc) order) overlaps it by more than the threshold, so with the candidates in
// that order the serial dependence is between 32-candidate chunks, not between survivors:
//   1. rank sort: two lanes per candidate (l, l ^ 16 of one warp) count the keys <= its own, half of the list each — broadcast
//      16-byte shared-memory reads, three carry-chain integer instructions per 64-bit compare — add their counts with one
//      shuffle and scatter key / decoded + normalised box to that position: O(n^2) compares, trivial at n <= 256, and no
//      barrier-separated sort passes;
//   2. chunk c = sorted positions 32c .. 32c+31 belongs to warps c and 8+c, one member per lane.  Every unordered pair of a
//      chunk is tested ONCE (the predicate is symmetric bit for bit: min/max/+ commute): member q meets q+1 .. q+16 (mod 32),
//      warp c the distances 1-8, warp 8+c 9-16; one vote per distance hands every lane the hits of the whole warp, from which
//      it assembles its own row ("whom do I suppress": later members only).  Warp 8+c passes its half through shared memory
//      (a 64-thread named barrier per chunk) and leaves;
//   3. chunk steps c = 0 .. ceil(n/32)-1 on warp c: starting from the members already removed by earlier chunks, repeatedly
//      keep the first member still standing and remove its row (one find-first-set + one shuffle per SURVIVOR, <= maxk over
//      the whole class); the kept boxes go to a shared list, the warp ARRIVES at the step's named barrier and leaves; the
//      later warps wait on it and test their candidate against the newly kept boxes only (four independent tests at a time).
//      Every candidate still meets each survivor at most once (work n x maxk + 16 n tests), but the barrier count drops from
//      maxk (30) to n/32 (<= 8) and finished warps stop paying.
// Its IoU test (iou_norm_gt) decides the same booleans as the rounds tiers' (iou_norm_gt_eo): same terms, same decision rule.
constexpr int CHUNK_MAX = 256;
constexpr int CHUNK_MAXK = 64;
static_assert(NMS_THREADS == 2 * CHUNK_MAX, "the chunked tier runs two lanes per candidate");
struct __align__(16) ChunkShared {
    unsigned long long skey[CHUNK_MAX];   // sorted keys
    float4 sobox[CHUNK_MAX];              // sorted boxes as decoded
    float4 snbox[CHUNK_MAX];              // ... (min,max)-normalised
    float sarea[CHUNK_MAX];
    unsigned rows[CHUNK_MAX];             // warp 8+c's half of the rows of chunk c
    float4 kbox[CHUNK_MAXK];              // survivors so far, normalised
    float karea[CHUNK_MAXK];
    int cnt[CHUNK_MAX / 32];              // survivors after chunk c
};
constexpr size_t CHUNK_SMEM_BYTES = (CHUNK_MAX + 4) * sizeof(unsigned long long) + sizeof(ChunkShared);   // arrival keys (padded to x4), tables

// r += (a >= b) for 64-bit keys given as 32-bit halves: the borrow chain of a - b, its final carry added to r
__device__ __forceinline__ void count_ge(unsigned &r, unsigned alo, unsigned ahi, unsigned blo, unsigned bhi) {
    asm("{\n\t.reg .u32 t;\n\tsub.cc.u32 t, %1, %3;\n\tsubc.cc.u32 t, %2, %4;\n\taddc.u32 %0, %0, 0;\n\t}" : "+r"(r) : "r"(alo), "r"(ahi), "r"(blo), "r"(bhi));
}

// named barriers with immediate ids (a register id makes ptxas reserve all 16 barriers for the CTA)
#define K2Y_BAR_CASE(op, i) case i: asm volatile(op " " #i ", %0;" ::"r"(count) : "memory"); break;
#define K2Y_BAR_SWITCH(op)                                                                                                  \
    switch (id) {                                                                                                           \
        K2Y_BAR_CASE(op, 1) K2Y_BAR_CASE(op, 2) K2Y_BAR_CASE(op, 3) K2Y_BAR_CASE(op, 4) K2Y_BAR_CASE(op, 5) K2Y_BAR_CASE(op, 6) \
        K2Y_BAR_CASE(op, 7) K2Y_BAR_CASE(op, 8) K2Y_BAR_CASE(op, 9) K2Y_BAR_CASE(op, 10) K2Y_BAR_CASE(op, 11)                   \
        default: break;                                                                                                     \
    }
__device__ __forceinline__ void named_sync(int id, int count) { K2Y_BAR_SWITCH("bar.sync") }
__device__ __forceinline__ void named_arrive(int id, int count) { K2Y_BAR_SWITCH("bar.arrive") }

__device__ __forceinline__ void nms_chunked(const KerasParams &p, int n, const unsigned long long *gkeys, const float4 *gboxes,
                                            k2y_det *out, int *count_out, unsigned long long *s_arrival, ChunkShared &cs) {
    constexpr int HW = CHUNK_MAX / 32;   // warps 0..7 own the chunks, warps 8..15 help with the pair tests
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nchunks = (n + 31) >> 5;
    // phase 1: warp w, lanes l and l ^ 16 <-> candidate 16 w + (l & 15)
    const int half = lane >> 4, ci = warp * 16 + (lane & 15);
    const bool cvalid = ci < n;
    const int L = (n + 3) & ~3;   // arrival list padded with zero keys (below every real key) to a multiple of four
    {
        unsigned long long kt = 0ull;
        float4 ob = make_float4(0.f, 0.f, 0.f, 0.f);
        if (cvalid) {
            kt = gkeys[ci];
            if (half) ob = gboxes[key_index(kt)];
        }
        if (!half && ci < L) s_arrival[ci] = kt;
        __syncthreads();
        const bool ranks = warp * 16 < n, pairs_too = (warp < HW ? warp : warp - HW) < nchunks;
        if (!ranks && !pairs_too) return;   // (warp-uniform) the named barrier below counts the warps that stay
        if (ranks) {
            // keys <= own among entries [j0, j0 + L/2); sorted position = L - (count of both halves): pads and the key itself count
            const int j0 = half ? (L >> 1) : 0;
            const ulonglong2 *pairs = reinterpret_cast<const ulonglong2 *>(s_arrival + j0);
            const unsigned klo = (unsigned)kt, khi = (unsigned)(kt >> 32);
            unsigned cnt = 0u;
#pragma unroll 4
            for (int j = 0; j < (L >> 2); ++j) {
                const ulonglong2 v = pairs[j];
                count_ge(cnt, klo, khi, (unsigned)v.x, (unsigned)(v.x >> 32));
                count_ge(cnt, klo, khi, (unsigned)v.y, (unsigned)(v.y >> 32));
            }
            cnt += __shfl_xor_sync(FULL, cnt, 16);
            const int r = L - (int)cnt;
            if (cvalid) {
                if (half) {
                    float ar;
                    const float4 nb = norm_box(ob, ar);
                    cs.sobox[r] = ob;
                    cs.snbox[r] = nb;
                    cs.sarea[r] = ar;
                } else {
                    cs.skey[r] = kt;
                }
            }
        }
        int staying = 0;
        for (int w = 0; w < 2 * HW; ++w) staying += (w * 16 < n || (w < HW ? w : w - HW) < nchunks) ? 32 : 0;
        named_sync(1, staying);
    }
    // phase 2: warps c and 8+c, lane q <-> sorted candidate 32 c + q
    const int c_own = warp < HW ? warp : warp - HW;
    if (c_own >= nchunks) return;
    const int si = 32 * c_own + lane;
    const bool valid = si < n;
    float4 nb = make_float4(0.f, 0.f, 0.f, 0.f);
    float ar = 0.f;
    if (valid) {
        nb = cs.snbox[si];
        ar = cs.sarea[si];
    }
    unsigned myrow = 0u;   // later members of the chunk that this one suppresses
    {
        const int d0 = warp < HW ? 0 : 8;
#pragma unroll
        for (int u = 1; u <= 8; ++u) {
            const int d = d0 + u, b = (lane + d) & 31;
            bool hit = iou_norm_gt(cs.snbox[32 * c_own + b], cs.sarea[32 * c_own + b], nb, ar, p.iou);
            hit = hit && valid && 32 * c_own + b < n && !(d == 16 && lane >= 16);   // distance 16: from the lower member only
            const unsigned T = __ballot_sync(FULL, hit);   // bit q: members q and (q + d) & 31 overlap
            if (lane + d < 32) myrow |= ((T >> lane) & 1u) << (lane + d);   // my own test, partner above me
            if (lane < d) myrow |= T & (1u << (lane + 32 - d));              // the test of member lane + 32 - d wrapped around to me
        }
    }
    if (warp >= HW) {
        cs.rows[si] = myrow;
        __threadfence_block();
        named_arrive(4 + c_own, 64);
        return;
    }
    named_sync(4 + c_own, 64);
    myrow |= cs.rows[si];
    // phase 3
    bool removed = !valid;
    int base = 0;
    for (int c = 0; c < nchunks; ++c) {
        const int nthr = (nchunks - c) * 32;   // warps c .. nchunks-1 meet at this step's barrier (ids alternate: the count changes)
        if (warp == c) {
            unsigned R = __ballot_sync(FULL, removed), K = 0u;
            const int room = p.maxk - base;
            int count = 0;
            while (R != FULL && count < room) {
                const int b = __ffs(~R) - 1;   // first member still standing: kept; it removes its row
                K |= 1u << b;
                ++count;
                R |= (1u << b) | __shfl_sync(FULL, myrow, b);
            }
            const bool kept = (K >> lane) & 1u;
            const int slot = __popc(K & ((1u << lane) - 1u));
            const int total = base + count;
            if (kept) {
                cs.kbox[base + slot] = nb;
                cs.karea[base + slot] = ar;
            }
            if (lane == 0) cs.cnt[c] = total;
            if (c < nchunks - 1) {
                __threadfence_block();
                named_arrive(2 + (c & 1), nthr);
            }
            if (kept) {
                const unsigned long long k = cs.skey[si];
                write_det(out, base + slot, cs.sobox[si], key_score(k), key_index(k));
            }
            if (lane == 0 && (c == nchunks - 1 || total >= p.maxk)) *count_out = total;
            return;
        }
        named_sync(2 + (c & 1), nthr);
        const int total = cs.cnt[c];
        if (!removed) {
            // against the survivors of chunk c, four independent straight-line tests at a time; past the end the last survivor is
            // tested again (never an entry >= total: the next chunk's warp may be writing those already)
            for (int k = base; k < total; k += 4) {
                bool hit = false;
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int kk = min(k + u, total - 1);
                    hit |= iou_norm_gt(cs.kbox[kk], cs.karea[kk], nb, ar, p.iou);
                }
                if (hit) {
                    removed = true;
                    break;
                }
            }
        }
        base = total;
        if (base >= p.maxk) return;
    }
}

// The tier of one (image, class) follows from its candidate count n, max_per_class (maxk) and cap = min(round_up(nbox, 256),
// 4096), the number of candidates whose keys and decoded boxes the shared memory holds (0 when nbox >= 2^20 - 1):
//   - chunked:                       n <= 256 (CHUNK_MAX) and maxk <= 64 (CHUNK_MAXK);
//   - shared-memory rounds, 4 slots: not chunked, n <= cap and cap <= 2048;
//   - shared-memory rounds, 8 slots: not chunked, n <= cap and cap > 2048;
//   - global-memory rounds:          not chunked and n > cap.
// SLOTS is chosen on the host from cap (NMS_THREADS x SLOTS >= cap), one instantiation each, so that the common grids are not
// compiled at the register count of the largest.
template <int SLOTS>
__global__ void __launch_bounds__(NMS_THREADS, 2) detect_nms_kernel(const KerasParams p) {
    extern __shared__ __align__(16) unsigned char s_nms[];
    __shared__ int s_red[2][NMS_WARPS][3];
    __shared__ unsigned long long s_best[2 * NMS_WARPS];
    const int c = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    pdl_wait();
    const int n = p.ncand[b * p.C + c];
    k2y_det *out = reinterpret_cast<k2y_det *>(reinterpret_cast<int *>(p.dets) + (size_t)b * p.det_stride) + (size_t)c * p.maxk;
    int *count_out = p.counts + (size_t)b * p.cnt_stride + c;
    if (n == 0) {
        if (tid == 0) *count_out = 0;
        return;
    }
    const unsigned long long *gkeys = p.keys + ((size_t)b * p.C + c) * p.P;
    const float4 *gboxes = p.boxes + (size_t)b * p.nbox;

    int nsel;
    if (n <= CHUNK_MAX && p.maxk <= CHUNK_MAXK) {
        // dynamic region = [CHUNK_MAX + 4] arrival-order keys, then the chunk tables (the launch provides at least CHUNK_SMEM_BYTES)
        nms_chunked(p, n, gkeys, gboxes, out, count_out, reinterpret_cast<unsigned long long *>(s_nms),
                    *reinterpret_cast<ChunkShared *>(s_nms + (CHUNK_MAX + 4) * sizeof(unsigned long long)));
        return;
    }
    if (n <= p.cap) {
        // keys and decoded boxes of all candidates in shared memory (arrival order: no sort needed)
        unsigned long long *s_keys = reinterpret_cast<unsigned long long *>(s_nms);
        float4 *s_box = reinterpret_cast<float4 *>(s_nms + (size_t)p.cap * 8);
        for (int i = tid; i < n; i += NMS_THREADS) {
            const unsigned long long k = gkeys[i];
            s_keys[i] = k;
            s_box[i] = gboxes[key_index(k)];
        }
        __syncthreads();
        nsel = nms_rounds_smem<SLOTS>(p, n, s_keys, s_box, out, s_best);
    } else {
        unsigned *alive_g = p.alive + ((size_t)b * p.C + c) * (size_t)p.alive_stride;
        nsel = nms_rounds(p, n, gkeys, gboxes, alive_g, out, s_red);
    }
    if (tid == 0) *count_out = nsel;
}

struct RegionParams {
    const float *in;
    float *out;                 // may be null
    float *probs;               // [B][N][C+1]
    float4 *boxes;              // [B][N]
    float *scores;              // ws [B][C][N]
    unsigned long long *keys;   // ws [B][C][P]
    int *kept;                  // ws [B][C][N]
    int W, H, A, C, N, P;
    float anchors[16];
    float thr, nms;
    double dx, dy, sxw, syh;    // correct_region_boxes constants (region_layer.c:158-159)
    float wscale, hscale;       // (:160-161)
};

__global__ void __launch_bounds__(DET_THREADS) region_kernel(const RegionParams p) {
    const int b = blockIdx.x, tid = threadIdx.x;
    const int wh = p.W * p.H, E = 5 + p.C;
    const float *in = p.in + (size_t)b * p.A * E * wh;
    float *outp = p.out ? p.out + (size_t)b * p.A * E * wh : nullptr;
    float *probs = p.probs + (size_t)b * p.N * (p.C + 1);
    float4 *boxes = p.boxes + (size_t)b * p.N;
    float *scores = p.scores + (size_t)b * p.C * p.N;

    // ---- phase 1: forward_region_layer + get_region_boxes + correct_region_boxes ----
    for (int index = tid; index < p.N; index += DET_THREADS) {
        const int a = index / wh, loc = index - a * wh;
        const int row = loc / p.W, col = loc - row * p.W;
        const float *e = in + (size_t)a * E * wh + loc;
        const float sx = sigmoidf_glibc(__ldg(e)), sy = sigmoidf_glibc(__ldg(e + wh));
        const float tw = __ldg(e + 2 * wh), th = __ldg(e + 3 * wh);
        const float conf = sigmoidf_glibc(__ldg(e + 4 * wh));
        float largest = __ldg(e + 5 * wh);
        for (int j = 1; j < p.C; ++j) largest = fmaxf(largest, __ldg(e + (5 + j) * wh));
        float sum = 0.f;
        for (int j = 0; j < p.C; ++j) sum = __fadd_rn(sum, expf_glibc(__fsub_rn(__ldg(e + (5 + j) * wh), largest)));
        float mx = 0.f;
        for (int j = 0; j < p.C; ++j) {
            const float sm = __fdiv_rn(expf_glibc(__fsub_rn(__ldg(e + (5 + j) * wh), largest)), sum);
            const float prob = __fmul_rn(conf, sm);
            const float kept = (prob > p.thr) ? prob : 0.f;
            probs[(size_t)index * (p.C + 1) + j] = kept;
            scores[(size_t)j * p.N + index] = kept;
            if (prob > mx) mx = prob;
            if (outp) outp[(size_t)a * E * wh + (5 + j) * wh + loc] = sm;
        }
        probs[(size_t)index * (p.C + 1) + p.C] = mx;
        if (outp) {
            float *o = outp + (size_t)a * E * wh + loc;
            o[0] = sx;
            o[wh] = sy;
            o[2 * wh] = tw;
            o[3 * wh] = th;
            o[4 * wh] = conf;
        }
        const float bx = __fdiv_rn(__fadd_rn((float)col, sx), (float)p.W);
        const float by = __fdiv_rn(__fadd_rn((float)row, sy), (float)p.H);
        const float bw = __fmul_rn(expf_glibc(tw), p.anchors[2 * a]);
        const float bh = __fmul_rn(expf_glibc(th), p.anchors[2 * a + 1]);
        float4 bb;
        bb.x = (float)__ddiv_rn(__dsub_rn((double)bx, p.dx), p.sxw);
        bb.y = (float)__ddiv_rn(__dsub_rn((double)by, p.dy), p.syh);
        bb.z = __fmul_rn(bw, p.wscale);
        bb.w = __fmul_rn(bh, p.hscale);
        boxes[index] = bb;
    }
    __syncthreads();

    // ---- phase 2: do_nms_sort, one warp per class, no output cap ----
    const int warp = tid >> 5, lane = tid & 31, nwarps = DET_THREADS >> 5;
    for (int k = warp; k < p.C; k += nwarps) {
        unsigned long long *keys = p.keys + ((size_t)b * p.C + k) * p.P;
        int *kept = p.kept + ((size_t)b * p.C + k) * p.N;
        unsigned long long rkey;
        const int n = gather_sorted(scores + (size_t)k * p.N, p.N, 0.f, keys, lane, rkey);
        float4 mybox = make_float4(0.f, 0.f, 0.f, 0.f);
        int nsel = 0;
        for (int i = 0; i < n; ++i) {
            const unsigned long long key = (n <= 32) ? __shfl_sync(FULL, rkey, i) : keys[i];
            const int idx = key_index(key);
            const float4 cb = boxes[idx];
            // box_iou(a = kept, b = candidate) — argument order as in the reference loop
            bool sup = (lane < nsel) && (iou_center(mybox, cb) > p.nms);
            bool any = __ballot_sync(FULL, sup) != 0u;
            for (int base = 32; !any && base < nsel; base += 32) {
                const int j = base + lane;
                sup = (j < nsel) && (iou_center(boxes[kept[j]], cb) > p.nms);
                any = __ballot_sync(FULL, sup) != 0u;
            }
            if (any) {
                if (lane == 0) probs[(size_t)idx * (p.C + 1) + k] = 0.f;
            } else {
                if (lane == nsel) mybox = cb;
                if (lane == 0) kept[nsel] = idx;
                ++nsel;
                __syncwarp();
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Operator-level entry points of the reference's decode loop (keras_inference.py:94-135), for callers that keep that loop
// and replace one operator at a time.  They call the fused path's decode helpers and IoU terms, so they give its bits.
// ---------------------------------------------------------------------------------------------------------------------
struct OpsAnchors {
    float wh[16];  // (w, h) pairs of one layer, A <= 8
};

// tf_xywh_to_all (tools/utils.py:524-547): raw [.., h, w, A, 2] xy / wh head slices -> xy in [0, 1], wh as input fraction.
__global__ void __launch_bounds__(256) xywh_to_all_kernel(const float2 *__restrict__ pred_xy, const float2 *__restrict__ pred_wh,
                                                          float2 *__restrict__ xy, float2 *__restrict__ wh, long long total, int H,
                                                          int W, int A, const OpsAnchors anc) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int a = (int)(i % A);
    const int cell = (int)((i / A) % ((long long)H * W));
    const float2 t = pred_xy[i], u = pred_wh[i];
    const float4 o = xywh_to_all(sigmoidf_ref(t.x), sigmoidf_ref(t.y), exp_cr(u.x), exp_cr(u.y), cell % W, cell / W, W, H,
                                 anc.wh[2 * a], anc.wh[2 * a + 1]);
    xy[i] = make_float2(o.x, o.y);
    wh[i] = make_float2(o.z, o.w);
}

// correct_box (keras_inference.py:32-72): (xy, wh) relative to the letterboxed input -> (ymin, xmin, ymax, xmax) in pixels
// of the original image.
__global__ void __launch_bounds__(256) correct_box_kernel(const float2 *__restrict__ xy, const float2 *__restrict__ wh,
                                                          float4 *__restrict__ boxes, long long total, float in_h, float in_w,
                                                          float img_h, float img_w) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const float2 c = xy[i], s = wh[i];
    boxes[i] = to_corners(letterbox(in_h, in_w, img_h, img_w), make_float4(c.x, c.y, s.x, s.y));
}

// tf.image.non_max_suppression(boxes, scores, max_output_size, iou_threshold) (score_threshold = -inf): one warp sorts
// every box by (score desc, index asc) and runs the greedy selection, lanes testing the kept boxes in parallel.
__device__ __forceinline__ unsigned long long pack_key_any(float score, int idx) {
    unsigned u = __float_as_uint(score);
    u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);  // total order of finite floats and infinities as unsigned
    return ((unsigned long long)u << 32) | (unsigned long long)(0xffffffffu - (unsigned)idx);
}

__global__ void __launch_bounds__(32) nms_boxes_kernel(const float4 *__restrict__ boxes, const float *__restrict__ scores, int n, int P,
                                                       int max_out, float thr, unsigned long long *keys, float4 *kept, float *kept_area,
                                                       int *__restrict__ out_idx, int *__restrict__ out_count) {
    const int lane = threadIdx.x;
    for (int i = lane; i < P; i += 32) keys[i] = i < n ? pack_key_any(scores[i], i) : 0ull;
    __syncwarp();
    warp_sort_desc_mem(keys, P, lane);
    int nsel = 0;
    for (int t = 0; t < n && nsel < max_out; ++t) {
        const int idx = key_index(keys[t]);
        float area;
        const float4 c = norm_box(boxes[idx], area);
        bool hit = false;
        for (int j = lane; j < nsel; j += 32) hit = hit || iou_norm_gt_eo(c, area, kept[j], kept_area[j], thr);
        if (!__any_sync(FULL, hit)) {
            if (lane == 0) {
                kept[nsel] = c;
                kept_area[nsel] = area;
                out_idx[nsel] = idx;
            }
            ++nsel;
            __syncwarp();
        }
    }
    if (lane == 0) *out_count = nsel;
}

// ---- merge of views.  grid = (C, rows), one CTA of MERGE_THREADS per (image, class) ---------------------------------------
// An image detected as V views (view 0 the whole image, the others windows of it, k2y_letterbox_u8_views) has V record lists
// per class, each in the window's own coordinates.  The merge moves them into image coordinates (one float32 add of the
// window's origin per coordinate), renumbers them (index = view * nbox + index) and runs the detector's greedy NMS once more
// over their union in (score descending, view ascending, index ascending) order.  The union is at most MERGE_MAX records, all
// in shared memory: keys (pack_key of the score and the new index) sorted by warp 0, every record's box scattered to its key's
// rank (binary search; the keys are unique), then rounds of "first candidate still alive -> keep -> every thread tests its own
// two candidates against it", one barrier per round, liveness exchanged as one ballot word per 32 candidates.
//
// k2y_merge_views_ex generalises it (k2y_merge_views is its case of uniform ranges and the defaults):
//   view ranges   image b owns views [off[b], off[b+1]) of the per-view blocks (at most V of them); view numbers stay per image.
//   border drop   with a border m >= 0, a record of a view is dropped while it is loaded if it lies within m pixels of one of
//                 the view's interior sides (a side bit per view, computed on the host), in the window's own coordinates:
//                 fminf / fmaxf of its two y (x) fields against m and fl(th - m) (fl(tw - m)).  Dropped records become
//                 zero keys, which sort behind every real one; the CTA counts them with a shared atomic.
//   MATCH         template: MATCH_IOU is the detector's test above, MATCH_IOS is inter / fminf(area_a, area_b) > thr with the
//                 same inter (a box of area <= 0 has metric 0), by the exact IEEE division.
//   UNION         template: the kept record's box becomes the field-wise union (min of ymin / xmin, max of ymax / xmax) of the
//                 records that die in its round, itself included.  Each warp reduces the four extrema of its dying candidates
//                 as order-preserving integer keys (union_key: -0.0 below +0.0, NaN fields skipped), one shared word per
//                 warp and field, double-buffered like the liveness words; warp 0 folds the 16 warps' words behind the next
//                 round's barrier and writes the record then, so a round still costs one barrier (plus one after the loop
//                 when it ends at max_per_class).
// k2y_merge_views_mirror adds mirrored views (the window flipped left to right, k2y_letterbox_u8_views_mirror), whose records
// are in mirrored window coordinates: the load maps them back, xmin = fl(fl(tw - xmax) + x0), xmax = fl(fl(tw - xmin) + x0),
// and the border drop, which tests the record as it comes, swaps the window's left and right side bits (2 and 8).
constexpr int MERGE_THREADS = 512;
constexpr int MERGE_MAX = 2 * MERGE_THREADS;   // records of one (image, class) over all views
constexpr int MERGE_WARPS = MERGE_THREADS / 32;
static_assert(MERGE_MAX == 1024, "one liveness word per lane: 32 words of 32 candidates");
enum { MATCH_IOU = 0, MATCH_IOS = 1 };

struct MergeParams {
    const k2y_det *vdets;   // [N][C][K] records of every view
    const int *vcounts;     // [N][C]
    const float *view_yx;   // [N][2] (y0, x0)
    const int *off;         // [n + 1] first view of image b; null: b * V (uniform ranges)
    const int *sides;       // [N] interior-side bits (1 top, 2 left, 4 bottom, 8 right); null: no border drop
    const int *mirror;      // [N] nonzero: view mirrored left to right; null: none is
    const float *view_hw;   // [N][2] (th, tw), read with `sides` or `mirror`
    float border;
    int n, V, C, K, nbox;
    float iou;
    k2y_det *dets;
    int *counts;
    long long det_stride, cnt_stride;
};

__device__ __forceinline__ bool ios_norm_gt(const float4 a, float area_a, const float4 b, float area_b, float thr) {
    if (area_a <= 0.f || area_b <= 0.f) return 0.f > thr;
    return __fdiv_rn(iou_terms(a, area_a, b, area_b).x, fminf(area_a, area_b)) > thr;
}
template <int MATCH>
__device__ __forceinline__ bool merge_match(const float4 a, float area_a, const float4 b, float area_b, float thr) {
    if constexpr (MATCH == MATCH_IOS) return ios_norm_gt(a, area_a, b, area_b, thr);
    else return iou_norm_gt_eo(a, area_a, b, area_b, thr);
}

// order-preserving key of a non-NaN float (-0.0 below +0.0); a NaN gets the identity `nan_key` of the reduction it enters
__device__ __forceinline__ unsigned union_key(float f, unsigned nan_key) {
    const unsigned u = __float_as_uint(f);
    return f != f ? nan_key : (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float union_field(unsigned key, unsigned nan_key, float own) {
    return key == nan_key ? own : __uint_as_float((key & 0x80000000u) ? (key & 0x7fffffffu) : ~key);
}

// UNION: warp 0 writes record `slot`, the kept candidate `o` / `key`, with the union of the extrema its group left in `ext`
__device__ __forceinline__ void merge_write_union(k2y_det *out, int slot, const float4 o, unsigned long long key, const uint4 *ext,
                                                  int lane) {
    const uint4 e = lane < MERGE_WARPS ? ext[lane] : make_uint4(0xffffffffu, 0xffffffffu, 0u, 0u);
    const unsigned ymin = __reduce_min_sync(FULL, e.x), xmin = __reduce_min_sync(FULL, e.y);
    const unsigned ymax = __reduce_max_sync(FULL, e.z), xmax = __reduce_max_sync(FULL, e.w);
    if (lane == 0)
        write_det(out, slot, make_float4(union_field(ymin, 0xffffffffu, o.x), union_field(xmin, 0xffffffffu, o.y),
                                         union_field(ymax, 0u, o.z), union_field(xmax, 0u, o.w)), key_score(key), key_index(key));
}

template <int MATCH, bool UNION>
__global__ void __launch_bounds__(MERGE_THREADS) merge_views_kernel(const MergeParams p) {
    __shared__ unsigned long long s_keys[MERGE_MAX];   // arrival order (view, then position in the view's list), then sorted
    __shared__ float4 s_box[MERGE_MAX];                // shifted boxes in sorted order
    __shared__ int s_off[MERGE_MAX + 1];               // first arrival position of view v (V <= MERGE_MAX)
    __shared__ unsigned s_alive[2][32];
    __shared__ uint4 s_ext[UNION ? 2 : 1][MERGE_WARPS];   // UNION: per warp the extrema keys of the round's dying candidates
    __shared__ int s_drop;
    const int c = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    k2y_det *out = reinterpret_cast<k2y_det *>(reinterpret_cast<int *>(p.dets) + (size_t)b * p.det_stride) + (size_t)c * p.K;
    int *count_out = p.counts + (size_t)b * p.cnt_stride + c;
    if (b >= p.n) {
        if (tid == 0) *count_out = 0;
        return;
    }
    const size_t view0 = p.off ? (size_t)p.off[b] : (size_t)b * p.V;
    const int V = p.off ? min(max(p.off[b + 1] - p.off[b], 0), p.V) : p.V;
    for (int v = tid; v < V; v += MERGE_THREADS) s_off[v + 1] = min(max(p.vcounts[(view0 + v) * p.C + c], 0), p.K);
    if (tid == 0) s_drop = 0;
    __syncthreads();
    if (tid == 0) {
        s_off[0] = 0;
        for (int v = 0; v < V; ++v) s_off[v + 1] += s_off[v];
    }
    __syncthreads();
    const int loaded = s_off[V];
    if (loaded == 0) {
        if (tid == 0) *count_out = 0;
        return;
    }
    // slot i = v * K + k of the per-view lists: at most two per thread (V * K <= MERGE_MAX), kept in registers until the sort is done
    unsigned long long mykey[2] = {0ull, 0ull};
    float4 mybox[2];
#pragma unroll
    for (int s = 0; s < 2; ++s) {
        const int i = tid + s * MERGE_THREADS, v = i / p.K, k = i - v * p.K;
        if (v >= V || k >= s_off[v + 1] - s_off[v]) continue;
        const k2y_det d = p.vdets[((view0 + v) * p.C + c) * p.K + k];
        const bool mirrored = p.mirror && p.mirror[view0 + v];
        if (p.sides) {
            int side = p.sides[view0 + v];
            if (mirrored) side = (side & 5) | ((side & 2) << 2) | ((side & 8) >> 2);   // the window's left edge is the view's right
            const float m = p.border;
            const bool drop = ((side & 1) && fminf(d.ymin, d.ymax) < m) || ((side & 2) && fminf(d.xmin, d.xmax) < m) ||
                              ((side & 4) && fmaxf(d.ymin, d.ymax) > __fsub_rn(p.view_hw[2 * (view0 + v)], m)) ||
                              ((side & 8) && fmaxf(d.xmin, d.xmax) > __fsub_rn(p.view_hw[2 * (view0 + v) + 1], m));
            if (drop) {
                s_keys[s_off[v] + k] = 0ull;
                atomicAdd(&s_drop, 1);
                continue;
            }
        }
        const float y0 = p.view_yx[2 * (view0 + v)], x0 = p.view_yx[2 * (view0 + v) + 1];
        float xmin = d.xmin, xmax = d.xmax;
        if (mirrored) {
            const float tw = p.view_hw[2 * (view0 + v) + 1];
            xmin = __fsub_rn(tw, d.xmax);
            xmax = __fsub_rn(tw, d.xmin);
        }
        mybox[s] = make_float4(__fadd_rn(d.ymin, y0), __fadd_rn(xmin, x0), __fadd_rn(d.ymax, y0), __fadd_rn(xmax, x0));
        s_keys[s_off[v] + k] = mykey[s] = pack_key(d.score, v * p.nbox + d.index);
    }
    int P = 32;
    while (P < loaded) P <<= 1;
    for (int i = loaded + tid; i < P; i += MERGE_THREADS) s_keys[i] = 0ull;
    __syncthreads();
    const int n = loaded - s_drop;   // dropped records are zero keys, sorted behind the n real ones
    if (n == 0) {
        if (tid == 0) *count_out = 0;
        return;
    }
    if (warp == 0) {
        if (P == 32) s_keys[lane] = warp_sort_desc(s_keys[lane], lane);   // every key, dropped ones included, is in s_keys[0, P)
        else warp_sort_desc_mem(s_keys, P, lane);
    }
    __syncthreads();
#pragma unroll
    for (int s = 0; s < 2; ++s) {
        if (mykey[s] == 0ull) continue;   // a real key is never 0: its index field is inverted
        int lo = 0, hi = n - 1;           // descending, unique: the rank of a key is the number of keys above it
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (s_keys[mid] > mykey[s]) lo = mid + 1;
            else hi = mid;
        }
        s_box[lo] = mybox[s];
    }
    __syncthreads();
    // candidate tid + s * MERGE_THREADS is this thread's slot s; liveness word w covers candidates 32 w .. 32 w + 31
    float4 nb[2];
    float ar[2];
    bool alive[2];
#pragma unroll
    for (int s = 0; s < 2; ++s) {
        const int pos = tid + s * MERGE_THREADS;
        alive[s] = pos < n;
        nb[s] = norm_box(alive[s] ? s_box[pos] : make_float4(0.f, 0.f, 0.f, 0.f), ar[s]);
    }
    int nsel = 0, par = 0, prev = -1;
    while (nsel < p.K) {
#pragma unroll
        for (int s = 0; s < 2; ++s) {
            const unsigned m = __ballot_sync(FULL, alive[s]);
            if (lane == 0) s_alive[par][warp + s * (MERGE_THREADS / 32)] = m;
        }
        __syncthreads();
        const unsigned word = s_alive[par][lane];
        if constexpr (UNION) {
            if (warp == 0 && prev >= 0) merge_write_union(out, nsel - 1, s_box[prev], s_keys[prev], s_ext[par], lane);
        }
        par ^= 1;
        const unsigned any = __ballot_sync(FULL, word != 0u);
        if (any == 0u) break;
        const int w = __ffs(any) - 1;
        const int best = 32 * w + __ffs(__shfl_sync(FULL, word, w)) - 1;   // first in the order still alive: kept
        const float4 ob = s_box[best];
        float ka;
        const float4 kb = norm_box(ob, ka);
        if constexpr (!UNION) {
            if (tid == 0) {
                const unsigned long long k = s_keys[best];
                write_det(out, nsel, ob, key_score(k), key_index(k));
            }
        }
        unsigned died = 0u;
#pragma unroll
        for (int s = 0; s < 2; ++s) {
            if (alive[s] && (tid + s * MERGE_THREADS == best || merge_match<MATCH>(kb, ka, nb[s], ar[s], p.iou))) {
                alive[s] = false;
                died |= 1u << s;
            }
        }
        if constexpr (UNION) {
            uint4 e = make_uint4(0xffffffffu, 0xffffffffu, 0u, 0u);
#pragma unroll
            for (int s = 0; s < 2; ++s) {
                if (died & (1u << s)) {
                    const float4 r = s_box[tid + s * MERGE_THREADS];
                    e.x = min(e.x, union_key(r.x, 0xffffffffu));
                    e.y = min(e.y, union_key(r.y, 0xffffffffu));
                    e.z = max(e.z, union_key(r.z, 0u));
                    e.w = max(e.w, union_key(r.w, 0u));
                }
            }
            e.x = __reduce_min_sync(FULL, e.x);
            e.y = __reduce_min_sync(FULL, e.y);
            e.z = __reduce_max_sync(FULL, e.z);
            e.w = __reduce_max_sync(FULL, e.w);
            if (lane == 0) s_ext[par][warp] = e;   // read behind the next round's barrier
            prev = best;
        }
        ++nsel;
    }
    if constexpr (UNION) {
        if (nsel == p.K) {   // the loop ended at max_per_class, not at a barrier: the last round's extrema need one
            __syncthreads();
            if (warp == 0) merge_write_union(out, nsel - 1, s_box[prev], s_keys[prev], s_ext[par], lane);
        }
    }
    if (tid == 0) *count_out = nsel;
}

inline int next_pow2(int v) {
    int p = 64;
    while (p < v) p <<= 1;
    return p;
}
inline size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

}  // namespace

}  // namespace k2y

using namespace k2y;

namespace {
constexpr int NMS_SMEM_CAP = 4096;  // candidates of one class held in shared memory (24 bytes each); more -> global-memory path

struct DetectLayout {
    size_t nbox, P, boxes_off, keys_off, ncand_off, alive_off, alive_stride, total;
    int cap;
};
// workspace: [boxes B*nbox float4][keys B*C*P u64][ncand B*C int][alive B*C*P/32 u32]
DetectLayout detect_layout(const k2y_detect_cfg *cfg, int batch) {
    DetectLayout L;
    L.nbox = 0;
    for (int l = 0; l < cfg->n_layers; ++l) L.nbox += (size_t)cfg->layer_h[l] * cfg->layer_w[l] * cfg->anchor_num;
    L.P = (size_t)next_pow2((int)L.nbox);
    L.cap = (int)(L.nbox < (size_t)NMS_SMEM_CAP ? ((L.nbox + 255) / 256 * 256) : (size_t)NMS_SMEM_CAP);
    if (L.nbox >= 0xFFFFFu) L.cap = 0;  // the shared-memory path packs the box index into 20 bits of its sort key
    const size_t BC = (size_t)batch * cfg->class_num;
    size_t off = 256;  // alignment slack
    L.boxes_off = off;
    off += align256((size_t)batch * L.nbox * sizeof(float4));
    L.keys_off = off;
    off += align256(BC * L.P * sizeof(unsigned long long));
    L.ncand_off = off;
    off += align256(BC * sizeof(int));
    L.alive_off = off;
    L.alive_stride = (L.P / 32 + 511) / 512 * 512 + 512;   // whole words per thread, 512 threads at most
    off += L.nbox > (size_t)L.cap ? align256(BC * L.alive_stride * sizeof(unsigned)) : 0;
    L.total = off;
    return L;
}
}  // namespace

extern "C" int k2y_detect_workspace_bytes(const k2y_detect_cfg *cfg, int batch, size_t *bytes) {
    if (!cfg || !bytes || batch <= 0 || cfg->n_layers < 1 || cfg->n_layers > 3 || cfg->anchor_num < 1 || cfg->class_num < 1) {
        set_error("k2y_detect_workspace_bytes: bad arguments");
        return K2Y_ERR_INVALID;
    }
    *bytes = detect_layout(cfg, batch).total;
    return K2Y_OK;
}

extern "C" int k2y_detect_keras(const k2y_detect_cfg *cfg, const float *const *heads_dev, int batch,
                                const float *image_hw_dev, k2y_det *dets_dev, int32_t *counts_dev, void *workspace,
                                size_t workspace_bytes, void *stream) {
    if (!cfg) {
        set_error("k2y_detect_keras: cfg is NULL");
        return K2Y_ERR_INVALID;
    }
    return k2y_detect_keras_strided(cfg, heads_dev, batch, image_hw_dev, dets_dev, counts_dev,
                                    (long long)cfg->class_num * cfg->max_per_class * 6, (long long)cfg->class_num, workspace,
                                    workspace_bytes, stream);
}

extern "C" int k2y_detect_keras_strided(const k2y_detect_cfg *cfg, const float *const *heads_dev, int batch,
                                        const float *image_hw_dev, k2y_det *dets_dev, int32_t *counts_dev,
                                        long long det_image_stride_words, long long count_image_stride_words, void *workspace,
                                        size_t workspace_bytes, void *stream) {
    size_t need = 0;
    int rc = k2y_detect_workspace_bytes(cfg, batch, &need);
    if (rc != K2Y_OK) return rc;
    if (!heads_dev || !image_hw_dev || !dets_dev || !counts_dev || !workspace || workspace_bytes < need) {
        set_error("k2y_detect_keras: null pointer or workspace too small (%zu < %zu)", workspace_bytes, need);
        return K2Y_ERR_INVALID;
    }
    if (cfg->anchor_num > 8 || cfg->max_per_class < 1) {
        set_error("k2y_detect_keras: anchor_num must be 1..8, class_num and max_per_class >= 1");
        return K2Y_ERR_INVALID;
    }
    if (det_image_stride_words < (long long)cfg->class_num * cfg->max_per_class * 6 || count_image_stride_words < cfg->class_num) {
        set_error("k2y_detect_keras: image strides smaller than one image's records / counts");
        return K2Y_ERR_INVALID;
    }
    const DetectLayout L = detect_layout(cfg, batch);
    KerasParams p;
    p.n_layers = cfg->n_layers;
    p.A = cfg->anchor_num;
    p.C = cfg->class_num;
    int off = 0;
    for (int l = 0; l < 3; ++l) {
        p.heads[l] = l < cfg->n_layers ? heads_dev[l] : nullptr;
        p.lh[l] = l < cfg->n_layers ? cfg->layer_h[l] : 0;
        p.lw[l] = l < cfg->n_layers ? cfg->layer_w[l] : 0;
        p.loff[l] = off;
        off += p.lh[l] * p.lw[l] * p.A;
    }
    p.loff[3] = off;
    p.nbox = off;
    p.P = (int)L.P;
    for (int i = 0; i < 48; ++i) p.anchors[i] = 0.f;
    for (int i = 0; i < cfg->n_layers * cfg->anchor_num * 2; ++i) p.anchors[i] = cfg->anchors[i];
    p.in_h = (float)cfg->in_h;
    p.in_w = (float)cfg->in_w;
    p.obj = cfg->obj_thresh;
    p.iou = cfg->iou_thresh;
    // sigmoid(t) >= obj needs t >= logit(obj); the scan skips the transcendental for logits below that with a margin of
    // 1e-3 (+0.1 %) — about 1e4 float ulps of the sigmoid, so no candidate can be lost to it
    p.logit_min = -__builtin_huge_valf();
    if (cfg->obj_thresh > 0.f && cfg->obj_thresh < 1.f) {
        const double lg = std::log((double)cfg->obj_thresh / (1.0 - (double)cfg->obj_thresh));
        p.logit_min = (float)(lg - 1e-3 - 1e-3 * std::fabs(lg));
    }
    p.maxk = cfg->max_per_class;
    p.image_hw = image_hw_dev;
    p.dets = dets_dev;
    p.counts = counts_dev;
    p.det_stride = det_image_stride_words;
    p.cnt_stride = count_image_stride_words;
    char *ws = reinterpret_cast<char *>(((uintptr_t)workspace + 255) & ~(uintptr_t)255) - 256;  // layout offsets start at 256
    p.boxes = reinterpret_cast<float4 *>(ws + L.boxes_off);
    p.keys = reinterpret_cast<unsigned long long *>(ws + L.keys_off);
    p.ncand = reinterpret_cast<int *>(ws + L.ncand_off);
    p.alive = reinterpret_cast<unsigned *>(ws + L.alive_off);
    p.cap = L.cap;
    p.alive_stride = (int)L.alive_stride;
    const size_t scan_smem = (size_t)SCAN_BOXES * (5 + p.C + 2) * sizeof(float);
    p.c_magic = (0x100000000ull + (unsigned long long)p.C - 1ull) / (unsigned long long)p.C;
    const size_t nms_smem = std::max((size_t)p.cap * 24, CHUNK_SMEM_BYTES);  // keys + decoded boxes | the chunked tier's tables
    int dev = 0;
    K2Y_CUDA_CHECK(cudaGetDevice(&dev));
    static bool attr_set[64] = {false};  // per device: opt-in shared memory is a per-device function attribute
    if (dev >= 0 && dev < 64 && !attr_set[dev]) {
        K2Y_CUDA_CHECK(cudaFuncSetAttribute(detect_nms_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, NMS_SMEM_CAP * 24));
        K2Y_CUDA_CHECK(cudaFuncSetAttribute(detect_nms_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, NMS_SMEM_CAP * 24));
        K2Y_CUDA_CHECK(cudaFuncSetAttribute(detect_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
        attr_set[dev] = true;
    }
    if (scan_smem > 96 * 1024) {
        set_error("k2y_detect_keras: class_num %d too large for the scan kernel's shared-memory slab", p.C);
        return K2Y_ERR_INVALID;
    }
    cudaStream_t st = (cudaStream_t)stream;
    K2Y_CUDA_CHECK(cudaMemsetAsync(p.ncand, 0, (size_t)batch * p.C * sizeof(int), st));
    dim3 sgrid((p.nbox + SCAN_BOXES - 1) / SCAN_BOXES, batch);
    detect_scan_kernel<<<sgrid, SCAN_THREADS, scan_smem, st>>>(p);  // follows a memset: plain stream order
    K2Y_CUDA_CHECK(cudaGetLastError());
    if (p.cap <= 2048) launch_k(detect_nms_kernel<4>, dim3(p.C, batch), dim3(NMS_THREADS), nms_smem, st, p);
    else launch_k(detect_nms_kernel<8>, dim3(p.C, batch), dim3(NMS_THREADS), nms_smem, st, p);
    K2Y_CUDA_CHECK(cudaGetLastError());
    return K2Y_OK;
}

extern "C" int k2y_merge_views_max_records(void) { return MERGE_MAX; }

namespace {
int merge_views_launch(const char *fn, const k2y_det *view_dets_dev, const int32_t *view_counts_dev, const float *view_yx_dev,
                       const int32_t *view_offsets_dev, const int32_t *view_sides_dev, const int32_t *view_mirror_dev,
                       const float *view_hw_dev, float border, int match, int merge, int n_images, int rows, int max_views,
                       int n_boxes, int class_num, int max_per_class, float thresh, k2y_det *dets_dev, int32_t *counts_dev,
                       long long det_image_stride_words, long long count_image_stride_words, void *stream) {
    if (!view_dets_dev || !view_counts_dev || !view_yx_dev || !dets_dev || !counts_dev || n_images < 0 || rows < 1 || rows < n_images ||
        max_views < 1 || n_boxes < 1 || class_num < 1 || class_num > 65535 || max_per_class < 1) {
        set_error("%s: null pointer, or not 0 <= n_images <= rows, rows, views, n_boxes, max_per_class >= 1, class_num 1..65535", fn);
        return K2Y_ERR_INVALID;
    }
    if ((match != K2Y_MATCH_IOU && match != K2Y_MATCH_IOS) || (merge != K2Y_MERGE_SUPPRESS && merge != K2Y_MERGE_UNION)) {
        set_error("%s: unknown match metric %d or merge action %d", fn, match, merge);
        return K2Y_ERR_INVALID;
    }
    if (view_sides_dev && (!view_hw_dev || !(border >= 0.f))) {
        set_error("%s: a border drop needs the views' sizes and a border >= 0 (got %g)", fn, (double)border);
        return K2Y_ERR_INVALID;
    }
    if (view_mirror_dev && !view_hw_dev) {
        set_error("%s: mirrored views need the views' sizes", fn);
        return K2Y_ERR_INVALID;
    }
    if ((long long)max_views * max_per_class > MERGE_MAX) {
        set_error("%s: %d views x %d records per class exceed the %d records one merge holds", fn, max_views, max_per_class, MERGE_MAX);
        return K2Y_ERR_INVALID;
    }
    if ((long long)max_views * n_boxes > 0x7fffffffLL) {
        set_error("%s: view * n_boxes + index does not fit the record's int32 index (%d views x %d boxes)", fn, max_views, n_boxes);
        return K2Y_ERR_INVALID;
    }
    if (det_image_stride_words < (long long)class_num * max_per_class * 6 || count_image_stride_words < class_num) {
        set_error("%s: image strides smaller than one image's records / counts", fn);
        return K2Y_ERR_INVALID;
    }
    MergeParams p;
    p.vdets = view_dets_dev;
    p.vcounts = view_counts_dev;
    p.view_yx = view_yx_dev;
    p.off = view_offsets_dev;
    p.sides = view_sides_dev;
    p.mirror = view_mirror_dev;
    p.view_hw = view_hw_dev;
    p.border = border;
    p.n = n_images;
    p.V = max_views;
    p.C = class_num;
    p.K = max_per_class;
    p.nbox = n_boxes;
    p.iou = thresh;
    p.dets = dets_dev;
    p.counts = counts_dev;
    p.det_stride = det_image_stride_words;
    p.cnt_stride = count_image_stride_words;
    const dim3 grid(class_num, rows);
    cudaStream_t st = (cudaStream_t)stream;
    if (match == K2Y_MATCH_IOU && merge == K2Y_MERGE_SUPPRESS) merge_views_kernel<MATCH_IOU, false><<<grid, MERGE_THREADS, 0, st>>>(p);
    else if (match == K2Y_MATCH_IOU) merge_views_kernel<MATCH_IOU, true><<<grid, MERGE_THREADS, 0, st>>>(p);
    else if (merge == K2Y_MERGE_SUPPRESS) merge_views_kernel<MATCH_IOS, false><<<grid, MERGE_THREADS, 0, st>>>(p);
    else merge_views_kernel<MATCH_IOS, true><<<grid, MERGE_THREADS, 0, st>>>(p);
    K2Y_CUDA_CHECK(cudaGetLastError());
    return K2Y_OK;
}
}  // namespace

extern "C" int k2y_merge_views_mirror(const k2y_det *view_dets_dev, const int32_t *view_counts_dev, const float *view_yx_dev,
                                      const int32_t *view_offsets_dev, const int32_t *view_sides_dev, const int32_t *view_mirror_dev,
                                      const float *view_hw_dev, float border, int match, int merge, int n_images, int rows,
                                      int max_views, int n_boxes, int class_num, int max_per_class, float thresh, k2y_det *dets_dev,
                                      int32_t *counts_dev, long long det_image_stride_words, long long count_image_stride_words,
                                      void *stream) {
    return merge_views_launch("k2y_merge_views_mirror", view_dets_dev, view_counts_dev, view_yx_dev, view_offsets_dev, view_sides_dev,
                              view_mirror_dev, view_hw_dev, border, match, merge, n_images, rows, max_views, n_boxes, class_num,
                              max_per_class, thresh, dets_dev, counts_dev, det_image_stride_words, count_image_stride_words, stream);
}

extern "C" int k2y_merge_views_ex(const k2y_det *view_dets_dev, const int32_t *view_counts_dev, const float *view_yx_dev,
                                  const int32_t *view_offsets_dev, const int32_t *view_sides_dev, const float *view_hw_dev,
                                  float border, int match, int merge, int n_images, int rows, int max_views, int n_boxes,
                                  int class_num, int max_per_class, float thresh, k2y_det *dets_dev, int32_t *counts_dev,
                                  long long det_image_stride_words, long long count_image_stride_words, void *stream) {
    return merge_views_launch("k2y_merge_views_ex", view_dets_dev, view_counts_dev, view_yx_dev, view_offsets_dev, view_sides_dev,
                              nullptr, view_hw_dev, border, match, merge, n_images, rows, max_views, n_boxes, class_num, max_per_class, thresh,
                              dets_dev, counts_dev, det_image_stride_words, count_image_stride_words, stream);
}

extern "C" int k2y_merge_views(const k2y_det *view_dets_dev, const int32_t *view_counts_dev, const float *view_yx_dev, int n_images,
                               int rows, int views, int n_boxes, int class_num, int max_per_class, float iou_thresh, k2y_det *dets_dev,
                               int32_t *counts_dev, long long det_image_stride_words, long long count_image_stride_words,
                               void *stream) {
    return merge_views_launch("k2y_merge_views", view_dets_dev, view_counts_dev, view_yx_dev, nullptr, nullptr, nullptr, nullptr, -1.f,
                              K2Y_MATCH_IOU,
                              K2Y_MERGE_SUPPRESS, n_images, rows, views, n_boxes, class_num, max_per_class, iou_thresh, dets_dev,
                              counts_dev, det_image_stride_words, count_image_stride_words, stream);
}

// Parity hook: the two pinned float32 exponentials, element-wise on device arrays.
__global__ void __launch_bounds__(256) expf_eval_kernel(const float *__restrict__ x, float *__restrict__ y, long long n, int mode) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) y[i] = mode == 0 ? k2y::exp_cr(x[i]) : k2y::expf_glibc(x[i]);
}
extern "C" int k2y_expf_eval(int mode, const float *x_dev, float *y_dev, long long n, void *stream) {
    if ((mode != 0 && mode != 1) || !x_dev || !y_dev || n < 0) {
        set_error("k2y_expf_eval: mode must be 0 (correctly rounded) or 1 (glibc expf algorithm); non-null pointers");
        return K2Y_ERR_INVALID;
    }
    if (n == 0) return K2Y_OK;
    expf_eval_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x_dev, y_dev, n, mode);
    K2Y_CUDA_CHECK(cudaGetLastError());
    return K2Y_OK;
}

extern "C" int k2y_region_workspace_bytes(const k2y_region_cfg *cfg, int batch, size_t *bytes) {
    if (!cfg || !bytes || batch <= 0) {
        set_error("k2y_region_workspace_bytes: bad arguments");
        return K2Y_ERR_INVALID;
    }
    const size_t N = (size_t)cfg->layer_w * cfg->layer_h * cfg->anchor_num;
    const size_t P = next_pow2((int)N);
    *bytes = align256((size_t)batch * cfg->classes * N * sizeof(float)) +
             align256((size_t)batch * cfg->classes * P * sizeof(unsigned long long)) +
             align256((size_t)batch * cfg->classes * N * sizeof(int));
    return K2Y_OK;
}

extern "C" int k2y_region_run(const k2y_region_cfg *cfg, const float *in_dev, int batch, float *out_dev,
                              float *probs_dev, float *boxes_dev, void *workspace, size_t workspace_bytes,
                              void *stream) {
    size_t need = 0;
    int rc = k2y_region_workspace_bytes(cfg, batch, &need);
    if (rc != K2Y_OK) return rc;
    if (!in_dev || !probs_dev || !boxes_dev || !workspace || workspace_bytes < need) {
        set_error("k2y_region_run: null pointer or workspace too small (%zu < %zu)", workspace_bytes, need);
        return K2Y_ERR_INVALID;
    }
    if (cfg->anchor_num < 1 || cfg->anchor_num > 8 || cfg->classes < 1) {
        set_error("k2y_region_run: anchor_num must be 1..8 and classes >= 1");
        return K2Y_ERR_INVALID;
    }
    RegionParams p;
    p.in = in_dev;
    p.out = out_dev;
    p.probs = probs_dev;
    p.boxes = (float4 *)boxes_dev;
    p.W = cfg->layer_w;
    p.H = cfg->layer_h;
    p.A = cfg->anchor_num;
    p.C = cfg->classes;
    p.N = p.W * p.H * p.A;
    p.P = next_pow2(p.N);
    for (int i = 0; i < 16; ++i) p.anchors[i] = i < 2 * p.A ? cfg->anchors[i] : 0.f;
    p.thr = cfg->threshold;
    p.nms = cfg->nms_value;
    // correct_region_boxes (region_layer.c:139-164) — same C types and evaluation order.
    {
        const uint32_t net_width = (uint32_t)cfg->net_w, net_height = (uint32_t)cfg->net_h;
        const uint32_t image_width = (uint32_t)cfg->image_w, image_height = (uint32_t)cfg->image_h;
        int new_w = 0, new_h = 0;
        if (((float)net_width / image_width) < ((float)net_height / image_height)) {
            new_w = (int)net_width;
            new_h = (int)((image_height * net_width) / image_width);
        } else {
            new_h = (int)net_height;
            new_w = (int)((image_width * net_height) / image_height);
        }
        p.dx = (net_width - new_w) / 2. / net_width;
        p.dy = (net_height - new_h) / 2. / net_height;
        p.sxw = (double)((float)new_w / net_width);
        p.syh = (double)((float)new_h / net_height);
        p.wscale = (float)net_width / new_w;
        p.hscale = (float)net_height / new_h;
    }
    char *ws = (char *)workspace;
    p.scores = (float *)ws;
    ws += align256((size_t)batch * p.C * p.N * sizeof(float));
    p.keys = (unsigned long long *)ws;
    ws += align256((size_t)batch * p.C * p.P * sizeof(unsigned long long));
    p.kept = (int *)ws;
    region_kernel<<<batch, DET_THREADS, 0, (cudaStream_t)stream>>>(p);
    K2Y_CUDA_CHECK(cudaGetLastError());
    return K2Y_OK;
}

extern "C" int k2y_xywh_to_all(const float *pred_xy_dev, const float *pred_wh_dev, long long n_boxes, int layer_h, int layer_w,
                               int anchor_num, const float *anchors_wh_host, float *xy_dev, float *wh_dev, void *stream) {
    if (!pred_xy_dev || !pred_wh_dev || !xy_dev || !wh_dev || !anchors_wh_host || n_boxes <= 0 || layer_h <= 0 || layer_w <= 0 ||
        anchor_num < 1 || anchor_num > 8 || (n_boxes % ((long long)layer_h * layer_w * anchor_num)) != 0) {
        set_error("k2y_xywh_to_all: bad arguments (n_boxes must be a multiple of layer_h*layer_w*anchor_num, anchor_num 1..8)");
        return K2Y_ERR_INVALID;
    }
    OpsAnchors anc;
    memset(&anc, 0, sizeof(anc));
    for (int i = 0; i < 2 * anchor_num; ++i) anc.wh[i] = anchors_wh_host[i];
    xywh_to_all_kernel<<<(unsigned)((n_boxes + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const float2 *>(pred_xy_dev), reinterpret_cast<const float2 *>(pred_wh_dev), reinterpret_cast<float2 *>(xy_dev),
        reinterpret_cast<float2 *>(wh_dev), n_boxes, layer_h, layer_w, anchor_num, anc);
    K2Y_CUDA_CHECK(cudaGetLastError());
    return K2Y_OK;
}

extern "C" int k2y_correct_box(const float *xy_dev, const float *wh_dev, long long n_boxes, float in_h, float in_w, float image_h,
                               float image_w, float *boxes_dev, void *stream) {
    if (!xy_dev || !wh_dev || !boxes_dev || n_boxes <= 0 || !(in_h > 0.f) || !(in_w > 0.f) || !(image_h > 0.f) || !(image_w > 0.f)) {
        set_error("k2y_correct_box: bad arguments");
        return K2Y_ERR_INVALID;
    }
    correct_box_kernel<<<(unsigned)((n_boxes + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const float2 *>(xy_dev), reinterpret_cast<const float2 *>(wh_dev), reinterpret_cast<float4 *>(boxes_dev), n_boxes,
        in_h, in_w, image_h, image_w);
    K2Y_CUDA_CHECK(cudaGetLastError());
    return K2Y_OK;
}

extern "C" int k2y_nms_workspace_bytes(int n_boxes, int max_output_size, size_t *bytes) {
    if (!bytes || n_boxes < 0 || max_output_size < 0) {
        set_error("k2y_nms_workspace_bytes: bad arguments");
        return K2Y_ERR_INVALID;
    }
    const size_t P = (size_t)next_pow2(n_boxes);
    const size_t keep = (size_t)(max_output_size < n_boxes ? max_output_size : n_boxes);
    *bytes = align256(P * sizeof(unsigned long long)) + align256(keep * sizeof(float4)) + align256(keep * sizeof(float)) + 256;
    return K2Y_OK;
}

extern "C" int k2y_nms_boxes(const float *boxes_dev, const float *scores_dev, int n_boxes, int max_output_size, float iou_threshold,
                             int32_t *indices_dev, int32_t *count_dev, void *workspace, size_t workspace_bytes, void *stream) {
    size_t need = 0;
    int rc = k2y_nms_workspace_bytes(n_boxes, max_output_size, &need);
    if (rc != K2Y_OK) return rc;
    if (!count_dev || !workspace || workspace_bytes < need || (n_boxes > 0 && (!boxes_dev || !scores_dev)) ||
        (n_boxes > 0 && max_output_size > 0 && !indices_dev) || (((uintptr_t)boxes_dev) & 15) != 0) {
        set_error("k2y_nms_boxes: null / misaligned pointer or workspace too small (%zu < %zu)", workspace_bytes, need);
        return K2Y_ERR_INVALID;
    }
    const int P = next_pow2(n_boxes);
    const size_t keep = (size_t)(max_output_size < n_boxes ? max_output_size : n_boxes);
    char *w = reinterpret_cast<char *>(workspace);
    unsigned long long *keys = reinterpret_cast<unsigned long long *>(w);
    float4 *kept = reinterpret_cast<float4 *>(w + align256((size_t)P * sizeof(unsigned long long)));
    float *kept_area = reinterpret_cast<float *>(reinterpret_cast<char *>(kept) + align256(keep * sizeof(float4)));
    nms_boxes_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4 *>(boxes_dev), scores_dev, n_boxes, P,
                                                         (int)keep, iou_threshold, keys, kept, kept_area, indices_dev, count_dev);
    K2Y_CUDA_CHECK(cudaGetLastError());
    return K2Y_OK;
}
