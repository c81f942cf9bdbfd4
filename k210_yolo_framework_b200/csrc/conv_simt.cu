// fp32 CUDA-core convolution kernels (K2Y_MATH_FP32_SIMT): implicit-GEMM dense conv with
// fused concat / nearest-upsample loader and BN+activation(+residual) epilogue, depthwise 3x3,
// 2x2 max-pool.  These are the exact-fp32 GPU path every tensor-core kernel is validated
// against, and the path for shapes the tensor-core kernels do not cover (Cin = 3 first conv).
//
// Replaces the TF ops the reference reaches through keras predict (keras_inference.py:88):
// Conv2D / DepthwiseConv2dNative / FusedBatchNorm / LeakyRelu / Relu(6) / ResizeNearestNeighbor /
// ConcatV2 / MaxPool / Add, as composed by models/yolonet.py and models/keras_mobilenet*.py.
#include <cstdlib>

#include "common.h"

namespace k2y {

bool pdl_enabled() { return getenv("K2Y_NO_PDL") == nullptr; }


namespace {

constexpr int BN_T = 64;
constexpr int BK_T = 16;

__device__ __forceinline__ const float *src_ptr(const ConvArgs &a, int b, int iy, int ix, int ci) {
    // (iy, ix) are in-bounds logical coordinates; ci indexes the concatenated channel axis.
    if (ci < a.C0) {
        if (a.up0) {
            const int h2 = a.H >> 1, w2 = a.W >> 1;
            return a.src0 + ((size_t)(b * h2 + (iy >> 1)) * w2 + (ix >> 1)) * a.C0 + ci;
        }
        return a.src0 + ((size_t)(b * a.H + iy) * a.W + ix) * a.C0 + ci;
    }
    return a.src1 + ((size_t)(b * a.H + iy) * a.W + ix) * a.C1 + (ci - a.C0);
}

template <int TM, bool VEC>
__global__ void __launch_bounds__(256) conv_igemm_simt_kernel(const ConvArgs a) {
    pdl_wait();
    constexpr int BM = 16 * TM;
    constexpr int A_PER_T = VEC ? (BM / 64) : (BM / 16);  // float4s or scalars of A per thread per k-tile
    __shared__ __align__(16) float As[BK_T][BM + 4];
    __shared__ __align__(16) float Bs[BK_T][BN_T];

    const int tid = threadIdx.x;
    const int M = a.B * a.OH * a.OW;
    const int Cin = a.C0 + a.C1;
    const int K = a.kh * a.kw * Cin;
    const int m0 = blockIdx.x * BM;
    const int n0 = blockIdx.y * BN_T;

    // Per-thread A-load coordinates (fixed over the K loop).
    int pb[A_PER_T], py[A_PER_T], px[A_PER_T];
#pragma unroll
    for (int i = 0; i < A_PER_T; ++i) {
        const int m_l = VEC ? ((tid >> 2) + 64 * i) : ((tid >> 4) + 16 * i);
        const int m = m0 + m_l;
        if (m < M) {
            const int ox = m % a.OW;
            const int t = m / a.OW;
            const int oy = t % a.OH;
            pb[i] = t / a.OH;
            py[i] = oy * a.stride - a.pad_t;
            px[i] = ox * a.stride - a.pad_l;
        } else {
            pb[i] = -1;
            py[i] = 0;
            px[i] = 0;
        }
    }
    const int ak = VEC ? ((tid & 3) * 4) : (tid & 15);  // k offset inside the tile
    const int bk = tid >> 4;                            // B tile: row
    const int bn = (tid & 15) * 4;                      // B tile: first col
    const bool n_vec = (a.N & 3) == 0;

    float4 ra[VEC ? A_PER_T : 1];
    float rs[VEC ? 1 : A_PER_T];
    float4 rb;

    auto load_tiles = [&](int k0) {
        // ---- A ----
        const int k = k0 + ak;
        int ky = 0, kx = 0, ci = 0;
        const bool kin = k < K;
        if (kin) {
            const int tap = k / Cin;
            ci = k - tap * Cin;
            ky = tap / a.kw;
            kx = tap - ky * a.kw;
        }
#pragma unroll
        for (int i = 0; i < A_PER_T; ++i) {
            const int iy = py[i] + ky, ix = px[i] + kx;
            const bool ok = kin && pb[i] >= 0 && iy >= 0 && iy < a.H && ix >= 0 && ix < a.W;
            if (VEC) {
                ra[VEC ? i : 0] = ok ? __ldg(reinterpret_cast<const float4 *>(src_ptr(a, pb[i], iy, ix, ci)))
                                     : make_float4(0.f, 0.f, 0.f, 0.f);
            } else {
                rs[VEC ? 0 : i] = ok ? __ldg(src_ptr(a, pb[i], iy, ix, ci)) : 0.f;
            }
        }
        // ---- B ----
        const int kk = k0 + bk;
        const int n = n0 + bn;
        if (kk < K && n_vec && n + 3 < a.N) {
            rb = __ldg(reinterpret_cast<const float4 *>(a.w + (size_t)kk * a.N + n));
        } else {
            float t[4] = {0.f, 0.f, 0.f, 0.f};
            if (kk < K) {
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if (n + j < a.N) t[j] = __ldg(a.w + (size_t)kk * a.N + n + j);
            }
            rb = make_float4(t[0], t[1], t[2], t[3]);
        }
    };
    auto store_tiles = [&]() {
#pragma unroll
        for (int i = 0; i < A_PER_T; ++i) {
            if (VEC) {
                const int m_l = (tid >> 2) + 64 * i;
                const float4 v = ra[VEC ? i : 0];
                As[ak + 0][m_l] = v.x;
                As[ak + 1][m_l] = v.y;
                As[ak + 2][m_l] = v.z;
                As[ak + 3][m_l] = v.w;
            } else {
                const int m_l = (tid >> 4) + 16 * i;
                As[ak][m_l] = rs[VEC ? 0 : i];
            }
        }
        *reinterpret_cast<float4 *>(&Bs[bk][bn]) = rb;
    };

    float acc[TM][4];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    const int ty = tid >> 4, tx = tid & 15;
    load_tiles(0);
    store_tiles();
    __syncthreads();
    for (int k0 = 0; k0 < K; k0 += BK_T) {
        const bool more = k0 + BK_T < K;
        if (more) load_tiles(k0 + BK_T);
#pragma unroll
        for (int kk = 0; kk < BK_T; ++kk) {
            float av[TM];
#pragma unroll
            for (int i = 0; i < TM; i += 4) {
                const float4 v = *reinterpret_cast<const float4 *>(&As[kk][ty * TM + i]);
                av[i] = v.x;
                av[i + 1] = v.y;
                av[i + 2] = v.z;
                av[i + 3] = v.w;
            }
            const float4 bv = *reinterpret_cast<const float4 *>(&Bs[kk][tx * 4]);
#pragma unroll
            for (int i = 0; i < TM; ++i) {
                acc[i][0] = fmaf(av[i], bv.x, acc[i][0]);
                acc[i][1] = fmaf(av[i], bv.y, acc[i][1]);
                acc[i][2] = fmaf(av[i], bv.z, acc[i][2]);
                acc[i][3] = fmaf(av[i], bv.w, acc[i][3]);
            }
        }
        __syncthreads();
        if (more) {
            store_tiles();
            __syncthreads();
        }
    }

    // ---- epilogue: folded BN / bias, activation, residual ----
    const int n = n0 + tx * 4;
    float sc[4], sh[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        sc[j] = (n + j < a.N) ? __ldg(a.scale + n + j) : 0.f;
        sh[j] = (n + j < a.N) ? __ldg(a.shift + n + j) : 0.f;
    }
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        const int m = m0 + ty * TM + i;
        if (m >= M) continue;
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = apply_act(fmaf(acc[i][j], sc[j], sh[j]), a.act, a.alpha);
        float *out = a.dst + (size_t)m * a.N + n;
        if (n_vec && n + 3 < a.N) {
            if (a.residual) {
                const float4 r = __ldg(reinterpret_cast<const float4 *>(a.residual + (size_t)m * a.N + n));
                v[0] += r.x;
                v[1] += r.y;
                v[2] += r.z;
                v[3] += r.w;
            }
            *reinterpret_cast<float4 *>(out) = make_float4(v[0], v[1], v[2], v[3]);
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (n + j < a.N) {
                    float r = a.residual ? __ldg(a.residual + (size_t)m * a.N + n + j) : 0.f;
                    out[j] = v[j] + r;
                }
        }
    }
}

// Depthwise 3x3, NHWC fp32: one thread = 4 channels x (TY rows x TX columns) of output pixels.  The 9 per-channel taps
// live in registers; every input row is loaded once per thread and feeds up to 3 output rows, every input column up to 3
// output columns, so the L2 -> SM read amplification drops from 9x (one thread per output) to
// ((TY-1)*S+3)*((TX-1)*S+3) / (TY*TX)  (3x for stride 1 with 2x4 outputs).  grid = (ceil(XT*C4 / 128), B*ceil(OH/TY)).
template <int STRIDE, int TX, int TY>
__global__ void __launch_bounds__(128) dwconv3x3_kernel(const DwArgs a) {
    pdl_wait();
    constexpr int NCOL = (TX - 1) * STRIDE + 3;
    constexpr int NROW = (TY - 1) * STRIDE + 3;
    const int c4n = a.C >> 2;
    const int xt_n = (a.OW + TX - 1) / TX;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= xt_n * c4n) return;
    const int c = (idx % c4n) * 4;
    const int ox0 = (idx / c4n) * TX;
    const int yt_n = (a.OH + TY - 1) / TY;
    const int b = blockIdx.y / yt_n;
    const int oy0 = (blockIdx.y - b * yt_n) * TY;
    const int iy0 = oy0 * STRIDE - a.pad_t, ix0 = ox0 * STRIDE - a.pad_l;

    float4 w[9];
#pragma unroll
    for (int t = 0; t < 9; ++t) w[t] = __ldg(reinterpret_cast<const float4 *>(a.w + t * a.C + c));
    float4 acc[TY][TX];
#pragma unroll
    for (int r = 0; r < TY; ++r)
#pragma unroll
        for (int i = 0; i < TX; ++i) acc[r][i] = make_float4(0.f, 0.f, 0.f, 0.f);

#pragma unroll
    for (int ry = 0; ry < NROW; ++ry) {
        const int iy = iy0 + ry;
        if (iy < 0 || iy >= a.H) continue;
        const float *rowp = a.src + ((size_t)(b * a.H + iy) * a.W) * a.C + c;
        float4 col[NCOL];
#pragma unroll
        for (int j = 0; j < NCOL; ++j) {
            const int ix = ix0 + j;
            col[j] = (ix >= 0 && ix < a.W) ? __ldg(reinterpret_cast<const float4 *>(rowp + (size_t)ix * a.C))
                                           : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int r = 0; r < TY; ++r) {
            const int ky = ry - r * STRIDE;  // compile-time after unrolling
            if (ky < 0 || ky > 2) continue;
#pragma unroll
            for (int i = 0; i < TX; ++i) {
#pragma unroll
                for (int kx = 0; kx < 3; ++kx) {
                    const float4 v = col[i * STRIDE + kx];
                    const float4 ww = w[ky * 3 + kx];
                    acc[r][i].x = fmaf(v.x, ww.x, acc[r][i].x);
                    acc[r][i].y = fmaf(v.y, ww.y, acc[r][i].y);
                    acc[r][i].z = fmaf(v.z, ww.z, acc[r][i].z);
                    acc[r][i].w = fmaf(v.w, ww.w, acc[r][i].w);
                }
            }
        }
    }
    const float4 sc = __ldg(reinterpret_cast<const float4 *>(a.scale + c));
    const float4 sh = __ldg(reinterpret_cast<const float4 *>(a.shift + c));
#pragma unroll
    for (int r = 0; r < TY; ++r) {
        const int oy = oy0 + r;
        if (oy >= a.OH) break;
        float *outp = a.dst + ((size_t)(b * a.OH + oy) * a.OW) * a.C + c;
#pragma unroll
        for (int i = 0; i < TX; ++i) {
            const int ox = ox0 + i;
            if (ox >= a.OW) break;
            float4 o;
            o.x = apply_act(fmaf(acc[r][i].x, sc.x, sh.x), a.act, a.alpha);
            o.y = apply_act(fmaf(acc[r][i].y, sc.y, sh.y), a.act, a.alpha);
            o.z = apply_act(fmaf(acc[r][i].z, sc.z, sh.z), a.act, a.alpha);
            o.w = apply_act(fmaf(acc[r][i].w, sc.w, sh.w), a.act, a.alpha);
            *reinterpret_cast<float4 *>(outp + (size_t)ox * a.C) = o;
        }
    }
}

// First convolution of every network: 3x3, Cin = 3, Cout in {16, 24, 32}.  One thread = one output pixel, all output
// channels.  The 27 x COUT weights and the folded BN constants travel BY VALUE in the kernel parameters, i.e. in the
// constant bank: every FFMA takes its weight as a constant operand and no load instruction is issued for it (with the
// weights in shared memory the 162 warp-wide LDS.128 broadcasts per pixel — 4 data-path cycles each — made the kernel
// L1/shared-pipe bound at 87 %).  A CTA owns 128 consecutive pixels of the
// flattened [B*OH*OW] output, one contiguous 128*COUT*4-byte block: results are staged in shared memory and written
// with fully coalesced 16-byte stores.
template <int COUT>
struct FirstConvConsts {
    float w[27 * COUT];  // [(ky,kx,ci)][n]
    float scale[COUT], shift[COUT];
};

template <int COUT, bool U8, int ACT>  // ACT: compile-time activation (ACT_LEAKY / ACT_RELU6), -1 = read a.act at run time
__global__ void __launch_bounds__(128) first_conv3x3_kernel(const ConvArgs a, const FirstConvConsts<COUT> cw) {
    constexpr int PITCH = COUT + 4;  // floats; conflict-free float4 rows
    __shared__ __align__(16) float stage[128 * PITCH];
    __shared__ float lut[U8 ? 512 : 1];  // u8 -> u8 / max(image) (IEEE division, as the reference's float32 cast implies) for the
                                         // two images a CTA's pixel range can touch
    const int per_img = a.OH * a.OW;
    const long long total = (long long)a.B * per_img;
    const long long p0 = (long long)blockIdx.x * 128;
    const int b0 = (int)(p0 / per_img);
    pdl_wait();  // the image maximum / input / output below belong to the stream order
    if (U8) {
        const float mx0 = (float)a.img_max[b0];
        const float mx1 = (float)a.img_max[min(b0 + 1, a.B - 1)];
        for (int v = threadIdx.x; v < 256; v += blockDim.x) {
            lut[v] = __fdiv_rn((float)v, mx0);
            lut[256 + v] = __fdiv_rn((float)v, mx1);
        }
        __syncthreads();
    }
    const long long pix = p0 + threadIdx.x;
    if (pix < total) {
        const int b = (int)(pix / per_img);
        const int rem = (int)(pix - (long long)b * per_img);
        const int oy = rem / a.OW, ox = rem - oy * a.OW;
        const int iy0 = oy * a.stride - a.pad_t, ix0 = ox * a.stride - a.pad_l;
        const bool far = U8 && b - b0 > 1;  // images smaller than 128 output pixels: divide directly
        const float mxf = far ? (float)a.img_max[b] : 1.f;
        const float *lt = lut + (far ? 0 : (b - b0) * 256);
        float in[27];
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
            const int iy = iy0 + ky;
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                const int ix = ix0 + kx;
                const bool ok = iy >= 0 && iy < a.H && ix >= 0 && ix < a.W;
                if (U8) {
                    const unsigned char *p8 = a.src_u8 + ((size_t)(b * a.H + iy) * a.W + ix) * 3;
#pragma unroll
                    for (int ci = 0; ci < 3; ++ci) {
                        const int v = ok ? (int)__ldg(p8 + ci) : 0;
                        in[(ky * 3 + kx) * 3 + ci] = !ok ? 0.f : (far ? __fdiv_rn((float)v, mxf) : lt[v]);
                    }
                } else {
                    const float *p = a.src0 + ((size_t)(b * a.H + iy) * a.W + ix) * 3;
#pragma unroll
                    for (int ci = 0; ci < 3; ++ci) in[(ky * 3 + kx) * 3 + ci] = ok ? __ldg(p + ci) : 0.f;
                }
            }
        }
        float acc[COUT];
#pragma unroll
        for (int n = 0; n < COUT; ++n) acc[n] = 0.f;
#pragma unroll
        for (int k = 0; k < 27; ++k) {
#pragma unroll
            for (int n = 0; n < COUT; ++n) acc[n] = fmaf(in[k], cw.w[k * COUT + n], acc[n]);
        }
        const int act = ACT >= 0 ? ACT : a.act;
#pragma unroll
        for (int n = 0; n < COUT; n += 4) {
            float4 o;
            o.x = apply_act(fmaf(acc[n], cw.scale[n], cw.shift[n]), act, a.alpha);
            o.y = apply_act(fmaf(acc[n + 1], cw.scale[n + 1], cw.shift[n + 1]), act, a.alpha);
            o.z = apply_act(fmaf(acc[n + 2], cw.scale[n + 2], cw.shift[n + 2]), act, a.alpha);
            o.w = apply_act(fmaf(acc[n + 3], cw.scale[n + 3], cw.shift[n + 3]), act, a.alpha);
            *reinterpret_cast<float4 *>(&stage[threadIdx.x * PITCH + n]) = o;
        }
    }
    __syncthreads();
    constexpr int Q = COUT / 4;  // float4 per pixel
    const long long valid = (total - p0 < 128 ? total - p0 : 128) * Q;
    float4 *outp = reinterpret_cast<float4 *>(a.dst + (size_t)p0 * COUT);
#pragma unroll
    for (int j = 0; j < Q; ++j) {
        const int e = threadIdx.x + 128 * j;
        if (e < valid) outp[e] = *reinterpret_cast<const float4 *>(&stage[(e / Q) * PITCH + (e % Q) * 4]);
    }
}

template <int COUT>
cudaError_t launch_first_conv(const ConvArgs &a, cudaStream_t st) {
    if (!a.w_host || !a.scale_host || !a.shift_host) return cudaErrorInvalidValue;
    FirstConvConsts<COUT> cw;
    memcpy(cw.w, a.w_host, sizeof(cw.w));
    memcpy(cw.scale, a.scale_host, sizeof(cw.scale));
    memcpy(cw.shift, a.shift_host, sizeof(cw.shift));
    const dim3 grid((unsigned)(((long long)a.B * a.OH * a.OW + 127) / 128));
#define K2Y_FIRST(U8V, ACTV) launch_k(first_conv3x3_kernel<COUT, U8V, ACTV>, grid, dim3(128), 0, st, a, cw)
    if (a.src_u8) {
        if (a.act == ACT_LEAKY) return K2Y_FIRST(true, ACT_LEAKY);
        if (a.act == ACT_RELU6) return K2Y_FIRST(true, ACT_RELU6);
        return K2Y_FIRST(true, -1);
    }
    if (a.act == ACT_LEAKY) return K2Y_FIRST(false, ACT_LEAKY);
    if (a.act == ACT_RELU6) return K2Y_FIRST(false, ACT_RELU6);
    return K2Y_FIRST(false, -1);
#undef K2Y_FIRST
}

// Per-image maximum of a uint8 batch (np.max(img) of tools/utils.py:405): grid = (chunks, B), atomicMax into int[B].
__global__ void __launch_bounds__(256) image_max_u8_kernel(const unsigned char *__restrict__ x, size_t bytes_per_image,
                                                           int *__restrict__ max_out) {
    const unsigned char *img = x + (size_t)blockIdx.y * bytes_per_image;
    const size_t n16 = bytes_per_image / 16;
    unsigned m = 0u;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (size_t)gridDim.x * blockDim.x) {
        const uint4 v = __ldg(reinterpret_cast<const uint4 *>(img) + i);
        m = __vmaxu4(m, __vmaxu4(__vmaxu4(v.x, v.y), __vmaxu4(v.z, v.w)));
    }
    for (size_t i = n16 * 16 + (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < bytes_per_image; i += (size_t)gridDim.x * blockDim.x)
        m = max(m, (unsigned)img[i]);
    unsigned r = max(max(m & 0xffu, (m >> 8) & 0xffu), max((m >> 16) & 0xffu, m >> 24));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) r = max(r, __shfl_xor_sync(0xffffffffu, r, o));
    if ((threadIdx.x & 31) == 0 && r > 0) atomicMax(max_out + blockIdx.y, (int)r);
}

__global__ void __launch_bounds__(256) maxpool2x2_kernel(const PoolArgs a) {
    pdl_wait();
    const int c4n = a.C >> 2;
    const size_t total = (size_t)a.B * a.OH * a.OW * c4n;
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int c = (int)(idx % c4n) * 4;
    size_t p = idx / c4n;
    const int ox = (int)(p % a.OW);
    p /= a.OW;
    const int oy = (int)(p % a.OH);
    const int b = (int)(p / a.OH);
    const float ninf = -__int_as_float(0x7f800000);
    float4 m = make_float4(ninf, ninf, ninf, ninf);
#pragma unroll
    for (int ky = 0; ky < 2; ++ky) {
        const int iy = oy * a.stride + ky;
        if (iy >= a.H) continue;
#pragma unroll
        for (int kx = 0; kx < 2; ++kx) {
            const int ix = ox * a.stride + kx;
            if (ix >= a.W) continue;
            const float4 v = __ldg(reinterpret_cast<const float4 *>(a.src + ((size_t)(b * a.H + iy) * a.W + ix) * a.C + c));
            m.x = fmaxf(m.x, v.x);
            m.y = fmaxf(m.y, v.y);
            m.z = fmaxf(m.z, v.z);
            m.w = fmaxf(m.w, v.w);
        }
    }
    *reinterpret_cast<float4 *>(a.dst + ((size_t)(b * a.OH + oy) * a.OW + ox) * a.C + c) = m;
}

}  // namespace

// SM count of the current device (cached per device ordinal)
static int device_sms() {
    static int cache[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    if (cache[dev] == 0) {
        int n = 0;
        cache[dev] = (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0) ? n : 132;
    }
    return cache[dev];
}

cudaError_t launch_conv_simt(const ConvArgs &a, cudaStream_t st) {
    const int M = a.B * a.OH * a.OW;
    if (a.kh == 3 && a.kw == 3 && a.C0 == 3 && a.C1 == 0 && !a.up0 && !a.residual && (a.N == 16 || a.N == 24 || a.N == 32)) {
        cudaError_t fe = a.N == 16 ? launch_first_conv<16>(a, st) : (a.N == 24 ? launch_first_conv<24>(a, st) : launch_first_conv<32>(a, st));
        if (fe != cudaSuccess) return fe;
        return cudaGetLastError();
    }
    const bool vec = (a.C0 % 4 == 0) && (a.C1 % 4 == 0);
    const int gy = (a.N + BN_T - 1) / BN_T;
    // Small-M layers (7x10 / 14x20 grids) use 64-row tiles when 128-row tiles would give fewer than two CTAs per SM.
    const bool small = ((M + 127) / 128) * gy < 2 * device_sms();
    if (small) {
        dim3 grid((M + 63) / 64, gy);
        if (vec)
            launch_k(conv_igemm_simt_kernel<4, true>, grid, dim3(256), 0, st, a);
        else
            launch_k(conv_igemm_simt_kernel<4, false>, grid, dim3(256), 0, st, a);
    } else {
        dim3 grid((M + 127) / 128, gy);
        if (vec)
            launch_k(conv_igemm_simt_kernel<8, true>, grid, dim3(256), 0, st, a);
        else
            launch_k(conv_igemm_simt_kernel<8, false>, grid, dim3(256), 0, st, a);
    }
    return cudaGetLastError();
}

cudaError_t launch_dwconv(const DwArgs &a, cudaStream_t st) {
    constexpr int TX = 4;
    const int per_row = ((a.OW + TX - 1) / TX) * (a.C / 4);
    if (a.stride == 1) {  // two output rows per thread (each input row loaded once for both); stride 2 uses one
        dim3 grid((per_row + 127) / 128, a.B * ((a.OH + 1) / 2));
        launch_k(dwconv3x3_kernel<1, TX, 2>, grid, dim3(128), 0, st, a);
    } else {
        dim3 grid((per_row + 127) / 128, a.B * a.OH);
        launch_k(dwconv3x3_kernel<2, TX, 1>, grid, dim3(128), 0, st, a);
    }
    return cudaGetLastError();
}

cudaError_t launch_image_max_u8(const unsigned char *x, int batch, size_t bytes_per_image, int *max_out, cudaStream_t st) {
    cudaError_t e = cudaMemsetAsync(max_out, 0, (size_t)batch * sizeof(int), st);
    if (e != cudaSuccess) return e;
    dim3 grid(64, batch);
    image_max_u8_kernel<<<grid, 256, 0, st>>>(x, bytes_per_image, max_out);  // follows a memset: plain stream order
    return cudaGetLastError();
}

cudaError_t launch_maxpool(const PoolArgs &a, cudaStream_t st) {
    const size_t total = (size_t)a.B * a.OH * a.OW * (a.C / 4);
    launch_k(maxpool2x2_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, st, a);
    return cudaGetLastError();
}

}  // namespace k2y
