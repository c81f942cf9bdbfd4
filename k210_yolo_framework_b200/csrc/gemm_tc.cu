// Hopper (sm_90a) tensor-core convolution: 1x1 and 3x3 dense convs as (implicit) GEMMs
//   D[M,N] = A[M,K] * W[N,K]^T,  M = B*OH*OW pixels, K = kh*kw*Cin, N = Cout
// with fp32 NHWC storage in HBM, tf32 or bf16 warpgroup MMAs (wgmma) and fp32 accumulators in registers.
//
// One persistent CTA per SM walks the (k-slice, m-tile, n-tile) work list; a tile is 128 GEMM rows x BN columns.
//   warpgroup 0  producers   one elected lane of warp 0 issues the TMA loads of the weight tile (hi/lo planes) every
//                            k-block, and of the A tile too when the conv is a plain 1x1 (A is then the [M,K] row-major
//                            activation matrix).  Otherwise all 128 threads gather the A tile of a 3x3 / strided / concat /
//                            nearest-upsample input with cp.async (zero-fill = padding).  A is stored as fp32 in the
//                            128B-swizzled K-major layout, 128 rows x 128 bytes per 16 KB sub-tile.
//   warpgroups 1-2  consumers  64 rows each: read their A rows from shared memory into the wgmma A register fragment,
//                            split them into hi/lo planes (3xTF32: hi = tf32(a), lo = tf32(a - hi); bf16x3: hi = bf16(a),
//                            mid = bf16(a - hi); the weights were split on the host), so that lo*hi + hi*lo + hi*hi
//                            recovers fp32-class accuracy from the tensor cores; B comes from shared memory.  A k-block's
//                            MMAs are one committed wgmma group; while it runs, the next k-block's A is read and split
//                            into a second fragment buffer, and a stage is released once its group has completed.  After
//                            the last k-block of a tile they apply folded BN, activation and residual and store to HBM:
//                            in the plain 1x1 kernels through two 8 KB shared-memory chunk buffers per warpgroup and TMA
//                            stores, which drain while the warpgroup moves on to the next tile's MMAs (the register
//                            epilogue remains where the output is no legal tensor map: N % 4 != 0 or an unaligned dst);
//                            in the gather kernels with direct global stores from the accumulator registers.
// mbarrier ring per stage: full_b (TMA tx) / full_a (cp.async arrivals) -> [consumers] -> empty.
//
// Replaces the TF Conv2D + FusedBatchNorm + LeakyRelu/Relu6 (+ ResizeNearestNeighbor/ConcatV2/Add) ops that
// models/yolonet.py:244-260 and models/keras_mobilenet*.py compose.
#include <cuda.h>
#include <cuda_runtime.h>

#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "gemm_tc.h"
#include "tc_ptx.cuh"

namespace k2y {

namespace {

constexpr int BM = 128;                    // rows per tile (two consumer warpgroups x 64)
constexpr int BK = 32;                     // fp32 per A sub-tile row = 128 bytes = one SWIZZLE_128B row
constexpr int A_TILE_BYTES = BM * BK * 4;  // 16 KB
constexpr int MAX_BN = 128;                // accumulators: BN / 2 registers per consumer thread
constexpr int NUM_THREADS = 3 * 128;
constexpr int MAX_STAGES = 8;

using namespace ptx;

struct TcParams {
    // gather-mode A source (also used for the shape arithmetic in both modes)
    const float *src0, *src1;
    int H, W, C0, C1, up0;          // logical input extent (after upsampling src0)
    int OH, OW, kh, kw, stride, pad_t, pad_l;
    // epilogue
    float *dst;
    const float *residual, *scale, *shift;
    int M, N, K;
    int BN, n_tiles, m_tiles, nkb, stages;
    int k_splits, kb_per_split;     // split-K: work item = (m-tile, n-tile, k-slice); partials go to a scratch buffer
    int partial;                    // 1: raw accumulators to dst (split-K scratch, row pitch N, rows of slice ks at ks * m_tiles * 128)
    int tma_store;                  // plain 1x1: results leave through shared-memory chunks and TMA stores (map_c / map_c16)
    int half_taps;                  // gather: Cin is half a k-block (16 with tf32, 32 with bf16 k-blocks), a k-block holds TWO consecutive taps
    float act_slope, act_clamp;     // branch-free activation parameters
};

struct __align__(8) Barriers {
    uint64_t full_b[MAX_STAGES], full_a[MAX_STAGES], empty[MAX_STAGES];
};
// dynamic smem besides the stage ring: alignment slack + barriers
constexpr size_t FIXED_SMEM = 1024 + 1024;
// TMA-A (plain 1x1) kernels also hold the output staging: per consumer warpgroup two buffers of one 64-row x 32-column fp32
// chunk (8 KB each), written by the warpgroup while TMA stores the other one
constexpr int CHUNK_BYTES = 64 * 32 * 4;
constexpr size_t STAGING_SMEM = 2 * 2 * CHUNK_BYTES;

// one fp32 element of the 128B-swizzled A sub-tile: row r, column k (0..31)
__device__ __forceinline__ uint32_t a_addr(uint32_t box, int r, int k) {
    return box + (uint32_t)r * 128u + ((uint32_t)((k >> 2) ^ (r & 7)) << 4) + (uint32_t)(k & 3) * 4u;
}

// Register budget of the warp-specialised kernel: the consumers, which hold the accumulators and two k-blocks of A fragments,
// rise to CONSUMER_REGS (the least with no spills in every instantiation) and the producers give up the difference
// (128 x 152 + 256 x 176 = 384 x 168, the launch's share).  The gather producers run measurably slower at smaller budgets.
constexpr int PRODUCER_REGS = 152;
constexpr int CONSUMER_REGS = 176;

// Attribution builds (scripts/bench_conv_tc.py), never the shipped library: K2Y_TC_ABLATE = 1 drops the epilogue's stores to
// global memory, 2 skips the MMAs (loads, splits and barriers stay), 3 skips the A split (the raw bits are the hi plane, lo
// is zero), 4 stops loading B after a CTA's first `stages` k-blocks (the MMAs read stale weight tiles: no B traffic from L2).
// Results are wrong in every variant; only the time means something.
#ifndef K2Y_TC_ABLATE
#define K2Y_TC_ABLATE 0
#endif
constexpr int ABLATE = K2Y_TC_ABLATE;

template <int I>
struct Buf {
    static constexpr int value = I;
};

// The MMAs of one k-block for one consumer warpgroup, NKS k-steps of it (the rest of the k-block is K padding), as one batch:
// a fence, the wgmmas, one commit.  Per k-step the split schemes issue lo*hi, hi*lo, hi*hi, each one MMA over the whole tile
// width (N columns are independent, so every accumulator sees the same sequence of MMAs as with narrower instructions; 16-
// column MMAs for the tail of a tile that was no multiple of 64 wide left the tensor pipe mostly idle).
template <int MODE, int BNT, int NKS>
__device__ __forceinline__ void mma_ksteps(float (&acc)[BNT / 2], const uint32_t (&ahi)[4][4], const uint32_t (&alo)[4][4],
                                           uint64_t dhi, uint64_t dlo, uint32_t accumulate) {
    using W = Wgmma<BNT>;  // the whole tile width in one MMA
    wgmma_fence();
    if constexpr (ABLATE == 2) {
#pragma unroll
        for (int kk = 0; kk < NKS; ++kk)
#pragma unroll
            for (int j = 0; j < 4; ++j) asm volatile("" ::"r"(ahi[kk][j]), "r"(alo[kk][j]));  // keep the split alive
        wgmma_commit();
        return;
    }
#pragma unroll
    for (int kk = 0; kk < NKS; ++kk) {
        const uint64_t o = (uint64_t)((kk * 32) >> 4);  // 32 bytes of B per k-step inside the 128 B swizzle row
        const uint32_t first = kk == 0 ? accumulate : 1u;
        if constexpr (MODE == K2Y_MATH_TC_BF16X3) {
            W::bf16(acc, alo[kk], dhi + o, first);
            W::bf16(acc, ahi[kk], dlo + o, 1u);
            W::bf16(acc, ahi[kk], dhi + o, 1u);
        } else if constexpr (MODE == K2Y_MATH_TC_3XTF32) {
            W::tf32(acc, alo[kk], dhi + o, first);
            W::tf32(acc, ahi[kk], dlo + o, 1u);
            W::tf32(acc, ahi[kk], dhi + o, 1u);
        } else {
            W::tf32(acc, ahi[kk], dhi + o, first);
        }
    }
    wgmma_commit();
}

// BNT = the tile width p.BN and MODE = the math mode (K2Y_MATH_TC_*), compile-time constants so that every accumulator
// register and every wgmma of the consumers is fixed at compile time and a k-block's MMAs are one branch-free batch (a
// runtime-sliced accumulator made ptxas serialise the wgmma pipeline; a runtime mode test split the batch into groups).
// STAGED (plain 1x1 only) selects the shared-memory + TMA-store epilogue; a runtime choice between the two epilogues made
// several consumer instantiations spill.
template <bool GATHER, int BNT, int MODE, bool STAGED>
__global__ void __launch_bounds__(NUM_THREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_bhi,
               const __grid_constant__ CUtensorMap map_blo, const __grid_constant__ CUtensorMap map_c,
               const __grid_constant__ CUtensorMap map_c16, const TcParams p) {
    constexpr bool BF16 = MODE == K2Y_MATH_TC_BF16X3;       // operands are bf16 (hi, mid) planes, 64 k per k-block
    constexpr bool THREE_X = MODE != K2Y_MATH_TC_TF32;      // split scheme: 3 MMAs per k-step; else one tf32 pass, 32 k per k-block
    constexpr int A_BOXES = BF16 ? 2 : 1;                   // 16 KB sub-tiles of raw fp32 A per stage
    constexpr int KBK = A_BOXES * BK;                       // k values per k-block
    constexpr int KSTEP = BF16 ? 16 : 8;                    // k values per wgmma
    static_assert(KBK / KSTEP == 4, "a k-block is four k-steps");
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // carve: [stages] x { A (raw fp32) A_BOXES x 16K | B_hi BN*128 | B_lo BN*128 (3x) }, output staging (TMA A only), barriers
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t b_bytes = (uint32_t)p.BN * 128u;
    const uint32_t a_bytes = (uint32_t)A_TILE_BYTES * (uint32_t)A_BOXES;
    const uint32_t stage_bytes = a_bytes + b_bytes * (THREE_X ? 2u : 1u);
    const uint32_t stage_c = smem_base + (uint32_t)p.stages * stage_bytes;  // 1024-aligned: stage_bytes is a multiple of 2 KB
    uint8_t *smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
    Barriers *bars = reinterpret_cast<Barriers *>(smem_gen + (size_t)p.stages * stage_bytes + (GATHER ? 0 : STAGING_SMEM));
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        for (int s = 0; s < p.stages; ++s) {
            mbar_init(smem_u32(&bars->full_b[s]), 1);
            mbar_init(smem_u32(&bars->full_a[s]), 128);
            mbar_init(smem_u32(&bars->empty[s]), 8);  // every consumer warp releases the stage
        }
        fence_barrier_init();
        if (!GATHER) prefetch_tmap(&map_a);
        if (STAGED) prefetch_tmap(&map_c);
        prefetch_tmap(&map_bhi);
        if (THREE_X) prefetch_tmap(&map_blo);
    }
    __syncthreads();
    pdl_wait();  // barrier set-up and descriptor prefetch overlap the previous kernel's tail; activations do not

    const int num_tiles = p.m_tiles * p.n_tiles * p.k_splits;
    auto stage_a = [&](int s) { return smem_base + (uint32_t)s * stage_bytes; };
    auto stage_b_hi = [&](int s) { return smem_base + (uint32_t)s * stage_bytes + a_bytes; };
    auto stage_b_lo = [&](int s) { return stage_b_hi(s) + b_bytes; };

    if (warp < 4) {
        // ================= producers =================
        setmaxnreg_dec<PRODUCER_REGS>();
        const int r = threadIdx.x;  // GEMM row inside the tile (gather), or producer thread index
        int s = 0;
        uint32_t ph = 0;
        const uint32_t tx = b_bytes * (THREE_X ? 2u : 1u) + (GATHER ? 0u : a_bytes);
        constexpr int bk_elems = BF16 ? 64 : 32;  // k-block extent in elements of the weight map (bf16 or fp32)
        int kb_done = 0;                          // ABLATE 4: k-blocks this CTA has loaded so far
        if (!GATHER && warp != 0) return;
        const int Cin = p.C0 + p.C1;
        const int wrow0 = warp * 32;  // first tile row of this warp
        for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
            const int ks = t % p.k_splits, tt = t / p.k_splits;
            const int mt = tt / p.n_tiles, nt = tt - mt * p.n_tiles;
            const int kb0 = ks * p.kb_per_split, kb1 = min(p.nkb, kb0 + p.kb_per_split);
            const int m = mt * BM + r;
            int b = -1, iy0 = 0, ix0 = 0;
            if (GATHER && m < p.M) {
                const int ox = m % p.OW;
                const int q = m / p.OW;
                const int oy = q % p.OH;
                b = q / p.OH;
                iy0 = oy * p.stride - p.pad_t;
                ix0 = ox * p.stride - p.pad_l;
            }
            for (int kb = kb0; kb < kb1; ++kb) {
                mbar_wait(smem_u32(&bars->empty[s]), ph ^ 1u);
                if (warp == 0) {
                    const bool load_b = ABLATE != 4 || kb_done < p.stages;
                    if (elect_one_sync()) {
                        const uint32_t fb = smem_u32(&bars->full_b[s]);
                        mbar_arrive_expect_tx(fb, load_b ? tx : (GATHER ? 0u : a_bytes));
                        if (!GATHER) {
                            for (int bx = 0; bx < A_BOXES; ++bx)
                                tma_load_2d(stage_a(s) + (uint32_t)bx * A_TILE_BYTES, &map_a, fb, kb * KBK + bx * BK, mt * BM);
                        }
                        if (load_b) {
                            tma_load_2d(stage_b_hi(s), &map_bhi, fb, kb * bk_elems, nt * p.BN);
                            if (THREE_X) tma_load_2d(stage_b_lo(s), &map_blo, fb, kb * bk_elems, nt * p.BN);
                        }
                    }
                    __syncwarp();
                    ++kb_done;
                }
                if (GATHER) {
                    // Each k-block is KBK consecutive channels of one filter tap, i.e. one contiguous run per output pixel.
                    // Thread r computes the source address of GEMM row r; the addresses are exchanged with warp shuffles so
                    // that 8 (tf32) or 16 (bf16) consecutive lanes copy one row's run with 16-byte cp.async.
                    const int k = kb * KBK;
                    const int tap = k / Cin;
                    const int ci = k - tap * Cin;
                    const int ky = tap / p.kw, kx = tap - ky * p.kw;
                    const int iy = iy0 + ky, ix = ix0 + kx;
                    const bool ok = b >= 0 && iy >= 0 && iy < p.H && ix >= 0 && ix < p.W;
                    unsigned long long pr = 0ull;   // 0 = zero-fill (padding / rows beyond M)
                    unsigned long long pr2 = 0ull;  // half_taps: the second tap of the k-block (upper half of its channels)
                    if (p.half_taps) {
                        // k-block kb = taps 2 kb and 2 kb + 1, C0 channels each; tap kh*kw (K padding) stays zero
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const int tp = 2 * kb + h;
                            const int ky2 = tp / p.kw, kx2 = tp - ky2 * p.kw;
                            const int iy2 = iy0 + ky2, ix2 = ix0 + kx2;
                            const bool ok2 = b >= 0 && tp < p.kh * p.kw && iy2 >= 0 && iy2 < p.H && ix2 >= 0 && ix2 < p.W;
                            const unsigned long long a2 =
                                ok2 ? (unsigned long long)(p.src0 + ((size_t)(b * p.H + iy2) * p.W + ix2) * p.C0) : 0ull;
                            if (h == 0) pr = a2;
                            else pr2 = a2;
                        }
                    } else if (ok) {
                        const float *src;
                        if (ci < p.C0) {
                            if (p.up0)
                                src = p.src0 + ((size_t)(b * (p.H >> 1) + (iy >> 1)) * (p.W >> 1) + (ix >> 1)) * p.C0 + ci;
                            else
                                src = p.src0 + ((size_t)(b * p.H + iy) * p.W + ix) * p.C0 + ci;
                        } else {
                            src = p.src1 + ((size_t)(b * p.H + iy) * p.W + ix) * p.C1 + (ci - p.C0);
                        }
                        pr = (unsigned long long)src;
                    }
                    const uint32_t stg_a = stage_a(s);
                    if constexpr (A_BOXES == 2) {
                        const int cjj = lane & 15;
                        const uint32_t dcol = (uint32_t)(cjj >> 3) * A_TILE_BYTES;
#pragma unroll
                        for (int i = 0; i < 16; ++i) {
                            const int lr = 2 * i + (lane >> 4);
                            const unsigned long long q0 = __shfl_sync(0xffffffffu, pr, lr);
                            const unsigned long long q1 = __shfl_sync(0xffffffffu, pr2, lr);
                            // half taps: sub-tile 0 = first tap's 32 channels, sub-tile 1 = second tap's
                            const unsigned long long q = (p.half_taps && (cjj & 8)) ? q1 : q0;
                            const unsigned long long off = (unsigned long long)(p.half_taps ? (cjj & 7) : cjj) * 16ull;
                            const int row = wrow0 + lr;
                            cp_async_16(stg_a + dcol + (uint32_t)row * 128u + (uint32_t)(((cjj & 7) ^ (row & 7)) << 4),
                                        q ? (const void *)(q + off) : (const void *)p.src0, q ? 16u : 0u);
                        }
                    } else {
                        const int cjj = lane & 7;
#pragma unroll
                        for (int i = 0; i < 8; ++i) {
                            const int lr = 4 * i + (lane >> 3);
                            const unsigned long long q0 = __shfl_sync(0xffffffffu, pr, lr);
                            const unsigned long long q1 = __shfl_sync(0xffffffffu, pr2, lr);
                            // half taps: chunks 0-3 = first tap, 4-7 = second tap
                            const unsigned long long q = (p.half_taps && (cjj & 4)) ? q1 : q0;
                            const unsigned long long off = (unsigned long long)(p.half_taps ? (cjj & 3) : cjj) * 16ull;
                            const int row = wrow0 + lr;
                            cp_async_16(stg_a + (uint32_t)row * 128u + (uint32_t)((cjj ^ (row & 7)) << 4),
                                        q ? (const void *)(q + off) : (const void *)p.src0, q ? 16u : 0u);
                        }
                    }
                    cp_async_mbar_arrive_noinc(smem_u32(&bars->full_a[s]));
                }
                if (++s == p.stages) {
                    s = 0;
                    ph ^= 1u;
                }
            }
        }
        return;
    }

    // ================= consumers: warpgroup cg owns tile rows [64 cg, 64 cg + 64) =================
    setmaxnreg_inc<CONSUMER_REGS>();
    const int cw = warp - 4;                 // 0..7
    const int cg = cw >> 2, wq = cw & 3;     // warpgroup, warp inside it
    const int g = lane >> 2, tq = lane & 3;  // fragment row / column group
    const int r0 = cg * 64 + wq * 16 + g;    // this thread's two tile rows: r0, r0 + 8
    int s = 0;
    uint32_t ph = 0;
    // A fragments of two k-blocks (4 k-steps x 4 registers, hi and lo planes): the MMAs of one k-block read their buffer
    // while the next k-block's A is read from shared memory and split into the other
    uint32_t ahi[2][4][4], alo[2][4][4];
    // wait for stage s, read this thread's A elements of it and split them into the (hi, lo) planes
    auto load_a = [&](uint32_t (&hi)[4][4], uint32_t (&lo)[4][4]) {
        mbar_wait(smem_u32(&bars->full_b[s]), ph);
        if (GATHER) mbar_wait(smem_u32(&bars->full_a[s]), ph);
        const uint32_t sa = stage_a(s);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            if constexpr (BF16) {
                // k-step kk = 16 bf16 columns: sub-tile kk/2, columns (kk&1)*16 + {2tq, 2tq+1} and + 8
                float v[4][2];  // fragment element j: row r0 + 8*(j&1), columns (lo, hi) of the pair
                const uint32_t box = sa + (uint32_t)(kk >> 1) * A_TILE_BYTES;
                const int c0 = (kk & 1) * 16 + 2 * tq;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int row = r0 + 8 * (j & 1), col = c0 + 8 * (j >> 1);
                    const float2 x = ld_shared_v2(a_addr(box, row, col));
                    v[j][0] = x.x;
                    v[j][1] = x.y;
                }
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    if constexpr (ABLATE == 3) {
                        hi[kk][j] = __byte_perm(__float_as_uint(v[j][0]), __float_as_uint(v[j][1]), 0x7632);
                        lo[kk][j] = 0u;
                        continue;
                    }
                    const uint32_t h = pack_bf16x2(v[j][0], v[j][1]);
                    hi[kk][j] = h;
                    lo[kk][j] = pack_bf16x2(v[j][0] - __uint_as_float(h << 16), v[j][1] - __uint_as_float(h & 0xffff0000u));
                }
            } else {
                // k-step kk = 8 tf32 columns: (row r0 / r0+8) x (column 8kk + tq / 8kk + tq + 4)
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float x = ld_shared_f32(a_addr(sa, r0 + 8 * (j & 1), kk * 8 + tq + 4 * (j >> 1)));
                    if constexpr (ABLATE == 3) {
                        hi[kk][j] = __float_as_uint(x);
                        lo[kk][j] = 0u;
                        continue;
                    }
                    const float h = to_tf32_rna(x);
                    hi[kk][j] = __float_as_uint(THREE_X ? h : x);
                    if (THREE_X) lo[kk][j] = __float_as_uint(to_tf32_rna(x - h));
                }
            }
        }
    };
    auto release = [&](int stage) {
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(&bars->empty[stage]));
    };
    // staged epilogue: one thread of the warpgroup issues (and waits for) its TMA stores
    const bool lead = (threadIdx.x & 127) == 0;
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const int ks = t % p.k_splits, tt = t / p.k_splits;
        const int mt = tt / p.n_tiles, nt = tt - mt * p.n_tiles;
        const int kb0 = ks * p.kb_per_split, kb1 = min(p.nkb, kb0 + p.kb_per_split);
        float acc[BNT / 2];
#pragma unroll
        for (int i = 0; i < BNT / 2; ++i) acc[i] = 0.f;
        load_a(ahi[0], alo[0]);
        int kb = kb0, prev = 0;
        // k-block kb from fragment buffer B: issue its MMAs, retire the previous k-block's (freeing its stage and the other
        // buffer), then load the next k-block into the other buffer while these run.  false after the tile's last k-block.
        auto kblock = [&](auto buf) -> bool {
            constexpr int B = decltype(buf)::value;
            const uint64_t dhi = make_desc_sw128(stage_b_hi(s)), dlo = make_desc_sw128(stage_b_lo(s));
            const uint32_t accumulate = kb == kb0 ? 0u : 1u;
            // only the k-steps that hold real K: past it A and B are zero-filled
            const int k_left = p.K - kb * KBK;
            if (k_left > 3 * KSTEP) mma_ksteps<MODE, BNT, 4>(acc, ahi[B], alo[B], dhi, dlo, accumulate);
            else if (k_left > 2 * KSTEP) mma_ksteps<MODE, BNT, 3>(acc, ahi[B], alo[B], dhi, dlo, accumulate);
            else if (k_left > KSTEP) mma_ksteps<MODE, BNT, 2>(acc, ahi[B], alo[B], dhi, dlo, accumulate);
            else mma_ksteps<MODE, BNT, 1>(acc, ahi[B], alo[B], dhi, dlo, accumulate);
            wgmma_wait<1>();
            if (kb > kb0) release(prev);
            prev = s;
            if (++s == p.stages) {
                s = 0;
                ph ^= 1u;
            }
            if (++kb < kb1) {
                load_a(ahi[B ^ 1], alo[B ^ 1]);
                return true;
            }
            wgmma_wait<0>();
            release(prev);
            return false;
        };
        while (kblock(Buf<0>{}) && kblock(Buf<1>{})) {
        }
#pragma unroll
        for (int i = 0; i < BNT / 2; ++i) reg_fence(acc[i]);
        if constexpr (STAGED) {
            // ---- staged epilogue: folded BN + activation (+ residual), or the raw split-K partial, one 64-row x 32-column
            // chunk of the warpgroup's rows at a time into a staging buffer, then one TMA store per chunk.  TMA clips rows >= M
            // and columns >= N.  The stores run on while the warpgroup fills the other buffer and then starts the next tile's
            // MMAs; before a buffer is rewritten, the store that read it has finished (wait_group.read before the barrier of
            // the chunk in between).  A tile width that is an odd multiple of 16 ends with a 16-column chunk (map_c16).
            const int row0 = (p.partial ? ks * p.m_tiles * BM : 0) + mt * BM + cg * 64;
            constexpr int CHUNKS = (BNT + 31) / 32;
            // chunks this warpgroup stored before this tile: the staging buffers alternate over them (derived from t rather
            // than counted, which kept one more register live through the mainloop)
            const uint32_t chunk0 = (uint32_t)(t - (int)blockIdx.x) / gridDim.x * (uint32_t)CHUNKS;
#pragma unroll
            for (int j = 0; j < CHUNKS; ++j) {
                const bool full = 32 * j + 32 <= BNT;
                const uint32_t buf = stage_c + (uint32_t)(cg * 2 + ((chunk0 + j) & 1u)) * CHUNK_BYTES;
                // (a half-warp's 8-byte stores hit each bank twice; trading column groups between threads to avoid that
                // made the bn-96 bf16x3 consumers spill)
#pragma unroll
                for (int q = 0; q < (full ? 4 : 2); ++q) {
                    const int c = 4 * j + q;  // accumulator column group
                    const int n = nt * BNT + 8 * c + 2 * tq;
                    float sc0 = 0.f, sh0 = 0.f, sc1 = 0.f, sh1 = 0.f;
                    if (!p.partial && n < p.N) {  // N % 4 == 0: n + 1 < N too
                        sc0 = __ldg(p.scale + n), sh0 = __ldg(p.shift + n);
                        sc1 = __ldg(p.scale + n + 1), sh1 = __ldg(p.shift + n + 1);
                    }
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        float o0 = acc[4 * c + 2 * h], o1 = acc[4 * c + 2 * h + 1];
                        const int row = wq * 16 + g + 8 * h;  // inside the warpgroup's 64 rows
                        if (!p.partial) {
                            o0 = act_bf(fmaf(o0, sc0, sh0), p.act_slope, p.act_clamp);
                            o1 = act_bf(fmaf(o1, sc1, sh1), p.act_slope, p.act_clamp);
                            const int mloc = mt * BM + cg * 64 + row;
                            if (p.residual && mloc < p.M && n < p.N) {
                                const float2 rr = __ldg(reinterpret_cast<const float2 *>(p.residual + (size_t)mloc * p.N + n));
                                o0 += rr.x, o1 += rr.y;
                            }
                        }
                        const int col = 8 * q + 2 * tq;
                        st_shared_v2(full ? a_addr(buf, row, col) : buf + (uint32_t)(row * 64 + col * 4), o0, o1);
                    }
                }
                fence_proxy_async_smem();
                if (lead) bulk_wait_group_0<true>();
                named_bar_sync(1 + cg, 128);
                if (lead && ABLATE != 1) {
                    tma_store_2d(full ? &map_c : &map_c16, buf, nt * BNT + 32 * j, row0);
                    bulk_commit_group();
                }
            }
            continue;
        }
        // ---- epilogue: folded BN + activation (+ residual) straight from the accumulator registers ----
        if constexpr (ABLATE == 1) continue;
        const int n_base = nt * BNT + 2 * tq;
        if (p.partial) {
            // split-K partial of slice ks: raw sums, rows [ks * m_tiles * 128, ...) of the scratch tensor (N % 4 == 0)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float *out = p.dst + ((size_t)ks * p.m_tiles * BM + mt * BM + r0 + 8 * h) * p.N;
#pragma unroll
                for (int c = 0; c < BNT / 8; ++c) {
                    const int n = n_base + 8 * c;
                    if (n >= p.N) continue;
                    *reinterpret_cast<float2 *>(out + n) = make_float2(acc[4 * c + 2 * h], acc[4 * c + 2 * h + 1]);
                }
            }
            continue;
        }
        const bool vec = (p.N & 1) == 0;
#pragma unroll
        for (int c = 0; c < BNT / 8; ++c) {
            const int n = n_base + 8 * c;
            if (n >= p.N) continue;
            // the column pair's BN constants, once for both row halves (n + 1 < N whenever N is even)
            const bool two = n + 1 < p.N;
            const float sc0 = __ldg(p.scale + n), sh0 = __ldg(p.shift + n);
            const float sc1 = two ? __ldg(p.scale + n + 1) : 0.f, sh1 = two ? __ldg(p.shift + n + 1) : 0.f;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int mloc = mt * BM + r0 + 8 * h;
                if (mloc >= p.M) continue;
                float *out = p.dst + (size_t)mloc * p.N;
                const float *res = p.residual ? p.residual + (size_t)mloc * p.N : nullptr;
                float o0 = act_bf(fmaf(acc[4 * c + 2 * h], sc0, sh0), p.act_slope, p.act_clamp);
                if (vec) {
                    float o1 = act_bf(fmaf(acc[4 * c + 2 * h + 1], sc1, sh1), p.act_slope, p.act_clamp);
                    if (res) {
                        const float2 rr = __ldg(reinterpret_cast<const float2 *>(res + n));
                        o0 += rr.x, o1 += rr.y;
                    }
                    *reinterpret_cast<float2 *>(out + n) = make_float2(o0, o1);
                } else {
                    if (res) o0 += __ldg(res + n);
                    out[n] = o0;
                    if (two) {
                        float o1 = act_bf(fmaf(acc[4 * c + 2 * h + 1], sc1, sh1), p.act_slope, p.act_clamp);
                        if (res) o1 += __ldg(res + n + 1);
                        out[n + 1] = o1;
                    }
                }
            }
        }
    }
    // the outputs are complete before the CTA exits (and before a PDL successor reads them)
    if (STAGED && lead) bulk_wait_group_0<false>();
}

// Split-K reduction + epilogue: out[m,n] = act(scale[n] * sum_s partial[s][m][n] + shift[n]) (+ residual).
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const float *__restrict__ part, float *__restrict__ dst,
                                                            const float *__restrict__ residual, const float *__restrict__ scale,
                                                            const float *__restrict__ shift, int M, int N, int splits,
                                                            size_t split_stride, float slope, float clamp) {
    pdl_wait();
    const int n4 = N >> 2;
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (size_t)M * n4) return;
    const int n = (int)(idx % n4) * 4;
    const size_t m = idx / n4;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int s = 0; s < splits; ++s) {
        const float4 v = __ldg(reinterpret_cast<const float4 *>(part + (size_t)s * split_stride + m * N + n));
        acc.x += v.x, acc.y += v.y, acc.z += v.z, acc.w += v.w;
    }
    const float4 sc = __ldg(reinterpret_cast<const float4 *>(scale + n));
    const float4 sh = __ldg(reinterpret_cast<const float4 *>(shift + n));
    float4 o;
    o.x = act_bf(fmaf(acc.x, sc.x, sh.x), slope, clamp);
    o.y = act_bf(fmaf(acc.y, sc.y, sh.y), slope, clamp);
    o.z = act_bf(fmaf(acc.z, sc.z, sh.z), slope, clamp);
    o.w = act_bf(fmaf(acc.w, sc.w, sh.w), slope, clamp);
    if (residual) {
        const float4 r = __ldg(reinterpret_cast<const float4 *>(residual + m * N + n));
        o.x += r.x, o.y += r.y, o.z += r.z, o.w += r.w;
    }
    *reinterpret_cast<float4 *>(dst + m * N + n) = o;
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

// 2-D row-major [rows][cols] tensor (fp32 or bf16), box = [box_rows][128 bytes of columns], 128B swizzle, OOB -> 0.
bool make_map_2d(CUtensorMap *map, const void *base, uint64_t rows, uint64_t cols, uint32_t box_rows, uint64_t pitch_elems = 0,
                 bool bf16 = false) {
    EncodeTiledFn enc = get_encode();
    if (!enc) return false;
    const size_t esz = bf16 ? 2 : 4;
    cuuint64_t dims[2] = {cols, rows};
    cuuint64_t strides[1] = {(pitch_elems ? pitch_elems : cols) * esz};
    cuuint32_t box[2] = {(cuuint32_t)(128 / esz), box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(map, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void *>(base), dims,
                     strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

// fp32 output [rows][cols] of the staged epilogue (row pitch cols, a multiple of 4): box = 64 rows x box_cols, 128B
// swizzle for the 32-column chunks (the staging layout), none for the 16-column ones
bool make_out_map(CUtensorMap *map, void *base, uint64_t rows, uint64_t cols, uint32_t box_cols) {
    EncodeTiledFn enc = get_encode();
    if (!enc) return false;
    cuuint64_t dims[2] = {cols, rows};
    cuuint64_t strides[1] = {cols * 4};
    cuuint32_t box[2] = {box_cols, 64};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     box_cols == 32 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

float __int_as_float_host(uint32_t u) {
    float f;
    memcpy(&f, &u, 4);
    return f;
}

uint16_t bf16_rne_host(float x) {
    uint32_t u;
    memcpy(&u, &x, 4);
    return (uint16_t)((u + 0x7fffu + ((u >> 16) & 1u)) >> 16);
}
float bf16_to_float_host(uint16_t b) {
    const uint32_t u = (uint32_t)b << 16;
    float f;
    memcpy(&f, &u, 4);
    return f;
}

float tf32_rna_host(float x) {
    uint32_t u;
    memcpy(&u, &x, 4);
    if ((u & 0x7f800000u) == 0x7f800000u) return x;
    u = (u + 0x1000u) & 0xffffe000u;
    float y;
    memcpy(&y, &u, 4);
    return y;
}



// Tile width BN and split-K factor from a rough cost model (SM cycles): a work item costs  kb * max(MMA time, shared-memory
// time, pipeline latency / depth) + epilogue + fixed, the layer costs ceil(items / SMs) item times (+ the reduction pass when
// K is split).  A is re-read once per n-tile, so ties go to the wider tile; BN is a multiple of 16 and at most 128 (the
// accumulators live in the consumer threads' registers).
int g_num_sms = 0;        // SM count / opt-in shared memory of the first device initialised (the planner's view of the GPU)
size_t g_max_smem = 0;
constexpr int DEFAULT_SMS = 132;              // H100 SXM, when no device has been initialised (host-only planner queries)
constexpr size_t DEFAULT_SMEM = 232448;       // 227 KB opt-in shared memory per block
constexpr int ID_LEN = 4096;
constexpr size_t DEFAULT_SCRATCH_BYTES = (size_t)64 << 20;
// Per-device state: function attributes (opt-in shared memory) are per device, and so are the allocations.  A net brings
// its own split-K scratch (ConvArgs::tc_scratch), so nets on different streams never share partials; the per-device
// default scratch below only serves the single-layer test hook (k2y_conv2d).
struct DevState {
    bool init = false;
    float *scratch = nullptr;      // split-K partials [splits][m_tiles*128][N]
    size_t scratch_bytes = 0;
};
constexpr int MAX_DEVICES = 64;
DevState g_dev[MAX_DEVICES];
DevState *cur_dev() {
    int d = -1;
    if (cudaGetDevice(&d) != cudaSuccess || d < 0 || d >= MAX_DEVICES) return nullptr;
    return &g_dev[d];
}

// SMs a conv may plan for: the device's, or the caller's budget (even, >= 8) when it asks for less
int budget_sms(int sm_limit) {
    const int all = g_num_sms > 0 ? g_num_sms : DEFAULT_SMS;
    if (sm_limit <= 0 || sm_limit >= all) return all;
    return (sm_limit < 8 ? 8 : sm_limit) & ~1;
}

size_t stage_bytes_of(int bn, bool three_x, bool bf16) {
    return (size_t)A_TILE_BYTES * (bf16 ? 2 : 1) + (size_t)bn * 128 * (three_x ? 2 : 1);
}
// shared memory besides the stage ring: the plain 1x1 (TMA A) kernels also hold the output staging
size_t fixed_smem_of(bool gather) { return FIXED_SMEM + (gather ? 0 : STAGING_SMEM); }
int stages_for(int bn, bool three_x, bool bf16, bool gather) {
    int st = (int)(((g_max_smem ? g_max_smem : DEFAULT_SMEM) - fixed_smem_of(gather)) / stage_bytes_of(bn, three_x, bf16));
    return st > MAX_STAGES ? MAX_STAGES : st;
}

void pick_tile(int M, int N, int nkb, bool three_x, bool bf16, bool gather, size_t scratch_limit, int sms, int *bn_out,
               int *splits_out) {
    if (scratch_limit == 0) scratch_limit = DEFAULT_SCRATCH_BYTES;
    const int n16 = (N + 15) / 16 * 16;
    const int m_tiles = (M + BM - 1) / BM;
    const char *force = getenv("K2Y_TC_SPLITK");
    int best = 16, best_s = 1;
    double best_cost = 1e30;
    for (int bn = 16; bn <= MAX_BN; bn += 16) {
        if (bn > n16) break;
        const int stages = stages_for(bn, three_x, bf16, gather);
        if (stages < 2) continue;
        const int n_tiles = (n16 + bn - 1) / bn;
        // per k-block (32 k for tf32, 64 k for bf16): tensor time (a 64 x bn x 8 tf32 or 64 x bn x 16 bf16 wgmma per warpgroup
        // and k-step), shared-memory reads (A fragments + B per pass), and the load -> mma -> free round trip over the stages
        const double passes = three_x ? 3.0 : 1.0;
        const double mma = passes * 4.0 * (bn < 64 ? 32.0 : bn / 2.0);
        const double smem_t = ((double)A_TILE_BYTES * (bf16 ? 2 : 1) + passes * 2.0 * bn * 128.0) / 128.0;
        const double lat = (gather ? 4000.0 : 2500.0) / stages;
        double kbt = mma > lat ? mma : lat;
        if (smem_t > kbt) kbt = smem_t;
        const double waste = (double)(n_tiles * bn) / n16;  // zero-padded columns still cost MMA time
        for (int sp = 1; sp <= 8; ++sp) {
            if (force && sp != atoi(force) && !(atoi(force) < 1 && sp == 1)) continue;
            if (sp > 1) {
                if ((N & 3) != 0 || N > ID_LEN || nkb / sp < 12) continue;
                if ((size_t)sp * m_tiles * BM * N * sizeof(float) > scratch_limit) continue;
            }
            const int kb = (nkb + sp - 1) / sp;
            const long items = (long)m_tiles * n_tiles * sp;
            const double item = kb * kbt + bn * 20.0 + 2000.0;
            double cost = (double)((items + sms - 1) / sms) * item * (0.9 + 0.1 * waste) + n_tiles * 40.0;
            if (sp > 1) cost += 7000.0 + (double)sp * M * N * 4.0 / 1500.0;  // reduce pass: launch + partial traffic
            if (cost < best_cost) {
                best_cost = cost;
                best = bn;
                best_s = sp;
            }
        }
    }
    *bn_out = best;
    *splits_out = best_s;
}

using ConvKernel = decltype(&conv_tc_kernel<false, 16, K2Y_MATH_TC_TF32, false>);

// the instantiation for tile width bn (a multiple of 16 up to MAX_BN)
template <bool G, bool S, int MODE>
ConvKernel conv_kernel_bn(int bn) {
    switch (bn) {
        case 16: return conv_tc_kernel<G, 16, MODE, S>;
        case 32: return conv_tc_kernel<G, 32, MODE, S>;
        case 48: return conv_tc_kernel<G, 48, MODE, S>;
        case 64: return conv_tc_kernel<G, 64, MODE, S>;
        case 80: return conv_tc_kernel<G, 80, MODE, S>;
        case 96: return conv_tc_kernel<G, 96, MODE, S>;
        case 112: return conv_tc_kernel<G, 112, MODE, S>;
        case 128: return conv_tc_kernel<G, 128, MODE, S>;
        default: return nullptr;
    }
}
// the instantiation for a gather / TMA A operand, a tensor-core math mode (K2Y_MATH_TC_*) and tile width bn
template <bool G, bool S>
ConvKernel conv_kernel_for(int mode, int bn) {
    switch (mode) {
        case K2Y_MATH_TC_TF32: return conv_kernel_bn<G, S, K2Y_MATH_TC_TF32>(bn);
        case K2Y_MATH_TC_3XTF32: return conv_kernel_bn<G, S, K2Y_MATH_TC_3XTF32>(bn);
        case K2Y_MATH_TC_BF16X3: return conv_kernel_bn<G, S, K2Y_MATH_TC_BF16X3>(bn);
        default: return nullptr;
    }
}
constexpr int TC_MODES[] = {K2Y_MATH_TC_TF32, K2Y_MATH_TC_3XTF32, K2Y_MATH_TC_BF16X3};

int tc_init() {
    int dev = 0;
    K2Y_CUDA_CHECK(cudaGetDevice(&dev));
    if (dev < 0 || dev >= MAX_DEVICES) {
        set_error("tc_init: device ordinal %d out of range", dev);
        return K2Y_ERR_INVALID;
    }
    DevState &ds = g_dev[dev];
    if (ds.init) return K2Y_OK;
    cudaDeviceProp prop;
    K2Y_CUDA_CHECK(cudaGetDeviceProperties(&prop, dev));
    for (int mode : TC_MODES)
        for (int bn = 16; bn <= MAX_BN; bn += 16) {
            K2Y_CUDA_CHECK(cudaFuncSetAttribute(conv_kernel_for<false, false>(mode, bn), cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                (int)prop.sharedMemPerBlockOptin));
            K2Y_CUDA_CHECK(cudaFuncSetAttribute(conv_kernel_for<false, true>(mode, bn), cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                (int)prop.sharedMemPerBlockOptin));
            K2Y_CUDA_CHECK(cudaFuncSetAttribute(conv_kernel_for<true, false>(mode, bn), cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                (int)prop.sharedMemPerBlockOptin));
        }
    if (g_num_sms == 0) {
        g_max_smem = prop.sharedMemPerBlockOptin;
        g_num_sms = prop.multiProcessorCount;
    }
    ds.init = true;
    return K2Y_OK;
}

}  // namespace

int tc_pack(TcWeights &w, const float *kernel_kn, int K, int N) {
    tc_free(w);
    int rc = tc_init();
    if (rc != K2Y_OK) return rc;
    w.K = K;
    w.N = N;
    w.Kpad = (K + BK - 1) / BK * BK;
    w.Npad = (N + 15) / 16 * 16;  // tiles wider than the remainder are zero-filled by TMA
    std::vector<float> hi((size_t)w.Npad * w.Kpad, 0.f), lo((size_t)w.Npad * w.Kpad, 0.f);
    for (int k = 0; k < K; ++k)
        for (int n = 0; n < N; ++n) {
            const float v = kernel_kn[(size_t)k * N + n];
            const float h = tf32_rna_host(v);
            hi[(size_t)n * w.Kpad + k] = h;
            lo[(size_t)n * w.Kpad + k] = tf32_rna_host(v - h);
        }
    K2Y_CUDA_CHECK(cudaMalloc(&w.d_hi, hi.size() * sizeof(float)));
    K2Y_CUDA_CHECK(cudaMalloc(&w.d_lo, lo.size() * sizeof(float)));
    K2Y_CUDA_CHECK(cudaMemcpy(w.d_hi, hi.data(), hi.size() * sizeof(float), cudaMemcpyHostToDevice));
    K2Y_CUDA_CHECK(cudaMemcpy(w.d_lo, lo.data(), lo.size() * sizeof(float), cudaMemcpyHostToDevice));
    // bf16x3 planes
    w.Kpad64 = (K + 63) / 64 * 64;
    std::vector<uint16_t> bh((size_t)w.Npad * w.Kpad64, 0), bm((size_t)w.Npad * w.Kpad64, 0);
    for (int k = 0; k < K; ++k)
        for (int n = 0; n < N; ++n) {
            const float v = kernel_kn[(size_t)k * N + n];
            const uint16_t h = bf16_rne_host(v);
            bh[(size_t)n * w.Kpad64 + k] = h;
            bm[(size_t)n * w.Kpad64 + k] = bf16_rne_host(v - bf16_to_float_host(h));
        }
    K2Y_CUDA_CHECK(cudaMalloc(&w.d_bh, bh.size() * sizeof(uint16_t)));
    K2Y_CUDA_CHECK(cudaMalloc(&w.d_bm, bm.size() * sizeof(uint16_t)));
    K2Y_CUDA_CHECK(cudaMemcpy(w.d_bh, bh.data(), bh.size() * sizeof(uint16_t), cudaMemcpyHostToDevice));
    K2Y_CUDA_CHECK(cudaMemcpy(w.d_bm, bm.data(), bm.size() * sizeof(uint16_t), cudaMemcpyHostToDevice));
    return K2Y_OK;
}

void tc_free(TcWeights &w) {
    cudaFree(w.d_hi);
    cudaFree(w.d_lo);
    cudaFree(w.d_bh);
    cudaFree(w.d_bm);
    w = TcWeights();
}

static bool is_plain_1x1(const ConvArgs &a) {
    return a.kh == 1 && a.kw == 1 && a.stride == 1 && a.src1 == nullptr && !a.up0 && a.pad_t == 0 && a.pad_l == 0;
}
// Gather convs over ONE plain source whose channel count is HALF a k-block: the k-block then holds two consecutive taps —
// 16 channels with the 32-wide tf32 k-blocks (tiny_yolo's 16->32 conv), 32 channels with the 64-wide bf16 k-blocks (the
// 32-channel 3x3 convs of Darknet-53 and tiny_yolo), where each tap fills exactly one 16 KB sub-tile of the stage.
static bool is_half_taps(const ConvArgs &a, int channels) {
    return !is_plain_1x1(a) && a.C0 == channels && a.C1 == 0 && a.src1 == nullptr && !a.up0;
}
// bf16x3 needs whole 64-channel k-blocks per tap in the gather path; layers that do not fit run as 3xTF32
static int effective_mode(const ConvArgs &a, int math_mode) {
    if (math_mode != K2Y_MATH_TC_BF16X3) return math_mode;
    // K <= 32 fits one 32-wide tf32 k-block: half the A bytes staged and converted per tile of the 64-wide bf16 k-block; same
    // error class
    if (is_plain_1x1(a)) return (a.C0 + a.C1 <= 32) ? K2Y_MATH_TC_3XTF32 : math_mode;
    const int Cin = a.C0 + a.C1;
    if ((Cin % 64) == 0 && (a.C0 % 64) == 0) return math_mode;
    return is_half_taps(a, 32) ? math_mode : K2Y_MATH_TC_3XTF32;
}

bool tc_supported(const ConvArgs &a, const TcWeights &w) {
    if (!w.d_hi || !get_encode()) return false;
    const int Cin = a.C0 + a.C1;
    if (is_plain_1x1(a)) return (Cin % 4) == 0 && (((uintptr_t)a.src0) & 15) == 0;  // TMA: 16-byte row pitch
    // gather path: every k-block is one 128-byte channel run of one tap of one source ...
    if ((Cin % BK) == 0 && (a.C0 % BK) == 0)
        return (((uintptr_t)a.src0) & 15) == 0 && (a.src1 == nullptr || (((uintptr_t)a.src1) & 15) == 0);
    // ... or two 64-byte runs of two consecutive taps (Cin == 16, one plain source; runs as 3xTF32: effective_mode)
    return is_half_taps(a, 16) && (((uintptr_t)a.src0) & 15) == 0;
}

// The tile plan of one conv with K = kh*kw*Cin: what the launch, the launch count and the host-only planner view all read.
struct TcPlan {
    int mode;                   // effective math mode (effective_mode)
    bool gather;                // A gathered by the producer warpgroup; false: TMA loads of a plain 1x1 conv's [M,K] rows
    int nkb;                    // k-blocks: 64 k each with bf16x3, 32 k otherwise
    int bn, stages;
    int k_splits, kb_per_split;
    int m_tiles, n_tiles, grid;  // grid: persistent CTAs, at most the SM budget
};

static TcPlan plan_conv(const ConvArgs &a, int K, int math_mode) {
    TcPlan pl;
    pl.mode = effective_mode(a, math_mode);
    const bool bf = pl.mode == K2Y_MATH_TC_BF16X3, three_x = pl.mode != K2Y_MATH_TC_TF32;
    pl.gather = !is_plain_1x1(a);
    pl.nkb = bf ? (K + 63) / 64 : (K + BK - 1) / BK;
    const int M = a.B * a.OH * a.OW, sms = budget_sms(a.sm_limit);
    pick_tile(M, a.N, pl.nkb, three_x, bf, pl.gather, a.tc_scratch ? a.tc_scratch_bytes : 0, sms, &pl.bn, &pl.k_splits);
    pl.kb_per_split = (pl.nkb + pl.k_splits - 1) / pl.k_splits;
    pl.k_splits = (pl.nkb + pl.kb_per_split - 1) / pl.kb_per_split;  // no empty slices
    pl.stages = stages_for(pl.bn, three_x, bf, pl.gather);
    pl.m_tiles = (M + BM - 1) / BM;
    pl.n_tiles = ((a.N + 15) / 16 * 16 + pl.bn - 1) / pl.bn;
    const int tiles = pl.m_tiles * pl.n_tiles * pl.k_splits;
    pl.grid = tiles < sms ? tiles : sms;
    return pl;
}

cudaError_t launch_conv_tc(const ConvArgs &a, const TcWeights &w, int math_mode, cudaStream_t st) {
    DevState *ds = cur_dev();
    if (!ds) return cudaErrorInvalidDevice;
    if (!ds->init && tc_init() != K2Y_OK) return cudaErrorNotReady;  // first launch on this device: attributes
    TcParams p;
    memset(&p, 0, sizeof(p));
    p.src0 = a.src0;
    p.src1 = a.src1;
    p.H = a.H;
    p.W = a.W;
    p.C0 = a.C0;
    p.C1 = a.C1;
    p.up0 = a.up0;
    p.OH = a.OH;
    p.OW = a.OW;
    p.kh = a.kh;
    p.kw = a.kw;
    p.stride = a.stride;
    p.pad_t = a.pad_t;
    p.pad_l = a.pad_l;
    p.dst = a.dst;
    p.residual = a.residual;
    p.scale = a.scale;
    p.shift = a.shift;
    p.act_slope = a.act == ACT_NONE ? 1.f : (a.act == ACT_LEAKY ? a.alpha : 0.f);
    p.act_clamp = a.act == ACT_RELU6 ? 6.f : __int_as_float_host(0x7f800000);
    p.M = a.B * a.OH * a.OW;
    p.N = a.N;
    p.K = w.K;
    const TcPlan pl = plan_conv(a, w.K, math_mode);
    const bool bf16 = pl.mode == K2Y_MATH_TC_BF16X3, three_x = pl.mode != K2Y_MATH_TC_TF32;
    p.half_taps = is_half_taps(a, bf16 ? 32 : 16) ? 1 : 0;
    p.nkb = pl.nkb;
    p.BN = pl.bn;
    p.n_tiles = pl.n_tiles;
    p.m_tiles = pl.m_tiles;
    p.kb_per_split = pl.kb_per_split;
    p.k_splits = pl.k_splits;
    p.stages = pl.stages;
    if (p.stages < 2) return cudaErrorInvalidConfiguration;
    const size_t smem = fixed_smem_of(pl.gather) + (size_t)p.stages * stage_bytes_of(p.BN, three_x, bf16);

    CUtensorMap map_a, map_bhi, map_blo, map_c, map_c16;
    memset(&map_a, 0, sizeof(map_a));
    memset(&map_c, 0, sizeof(map_c));
    memset(&map_c16, 0, sizeof(map_c16));
    const size_t mpad = (size_t)p.m_tiles * BM;
    float *scratch = a.tc_scratch;
    if (p.k_splits > 1) {
        if (!scratch) {  // no caller-owned scratch (k2y_conv2d): the device's default one, created on first use
            if (!ds->scratch) {
                cudaError_t me = cudaMalloc(&ds->scratch, DEFAULT_SCRATCH_BYTES);
                if (me != cudaSuccess) return me;
                ds->scratch_bytes = DEFAULT_SCRATCH_BYTES;
            }
            scratch = ds->scratch;
        }
        // partial pass: raw accumulators -> scratch, the reduce pass applies BN, activation and residual
        p.partial = 1;
        p.dst = scratch;
        p.residual = nullptr;
    }
    if (!pl.gather && !make_map_2d(&map_a, a.src0, (uint64_t)p.M, (uint64_t)(a.C0 + a.C1), BM)) return cudaErrorInvalidValue;
    // plain 1x1: TMA stores of the output (or of the split-K partials, whose scratch always qualifies) where the output is a
    // legal tensor map — 16-byte row pitch and base; otherwise (the 75-channel head outputs) the register epilogue
    p.tma_store = !pl.gather && (p.partial || ((a.N & 3) == 0 && ((uintptr_t)a.dst & 15) == 0)) ? 1 : 0;
    if (p.tma_store) {
        const uint64_t rows = p.partial ? (uint64_t)p.k_splits * mpad : (uint64_t)p.M;
        if (!make_out_map(&map_c, p.dst, rows, (uint64_t)p.N, 32) || !make_out_map(&map_c16, p.dst, rows, (uint64_t)p.N, 16))
            return cudaErrorInvalidValue;
    }
    if (bf16) {
        if (!make_map_2d(&map_bhi, w.d_bh, (uint64_t)w.Npad, (uint64_t)w.Kpad64, (uint32_t)p.BN, 0, true)) return cudaErrorInvalidValue;
        if (!make_map_2d(&map_blo, w.d_bm, (uint64_t)w.Npad, (uint64_t)w.Kpad64, (uint32_t)p.BN, 0, true)) return cudaErrorInvalidValue;
    } else {
        if (!make_map_2d(&map_bhi, w.d_hi, (uint64_t)w.Npad, (uint64_t)w.Kpad, (uint32_t)p.BN)) return cudaErrorInvalidValue;
        if (!make_map_2d(&map_blo, w.d_lo, (uint64_t)w.Npad, (uint64_t)w.Kpad, (uint32_t)p.BN)) return cudaErrorInvalidValue;
    }

    // null for a tile width or math mode that has no instantiation
    const ConvKernel kern = pl.gather      ? conv_kernel_for<true, false>(pl.mode, p.BN)
                            : p.tma_store ? conv_kernel_for<false, true>(pl.mode, p.BN)
                                          : conv_kernel_for<false, false>(pl.mode, p.BN);
    if (!kern) return cudaErrorInvalidConfiguration;
    const dim3 g((unsigned)pl.grid), b(NUM_THREADS);
    cudaError_t le = launch_k(kern, g, b, smem, st, map_a, map_bhi, map_blo, map_c, map_c16, p);
    if (le != cudaSuccess) return le;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    if (p.k_splits > 1) {
        const size_t total = (size_t)p.M * (a.N / 4);
        launch_k(splitk_reduce_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, st, (const float *)scratch, a.dst, a.residual,
                 a.scale, a.shift, p.M, a.N, p.k_splits, mpad * a.N, p.act_slope, p.act_clamp);
        e = cudaGetLastError();
    }
    return e;
}

int tc_launch_count(const ConvArgs &a, const TcWeights &w, int math_mode) {
    return plan_conv(a, w.K, math_mode).k_splits > 1 ? 2 : 1;
}

// Upper bound of the split-K scratch a conv of this shape can ask for (8 slices of [m_tiles*128][N] partials, capped at the
// planner's default limit); 0 when the shape is never split.  A net sizes its own scratch with the maximum over its layers.
size_t tc_scratch_bound(const ConvArgs &a, const TcWeights &w) {
    const int M = a.B * a.OH * a.OW;
    if ((a.N & 3) != 0 || a.N > ID_LEN || w.Kpad / BK < 24) return 0;
    const size_t need = (size_t)8 * ((M + BM - 1) / BM) * BM * a.N * sizeof(float);
    return need < DEFAULT_SCRATCH_BYTES ? need : DEFAULT_SCRATCH_BYTES;
}

}  // namespace k2y

// Host-only view of the tile planner (no GPU needed: without a device it assumes an H100 SXM — 132 SMs, 227 KB of shared
// memory): which tile width, split-K factor and pipeline depth a dense conv of this GEMM shape gets.  `cluster` is always 1
// (kept in the ABI: every CTA loads its own weight tiles).
extern "C" int k2y_tc_plan_budget(int M, int N, int K, int ksize, int math_mode, int sm_limit, int *bn, int *k_splits, int *stages,
                                  int *cluster, int *effective_math, int *grid);

extern "C" int k2y_tc_plan(int M, int N, int K, int ksize, int math_mode, int *bn, int *k_splits, int *stages, int *cluster,
                           int *effective_math) {
    int grid = 0;
    return k2y_tc_plan_budget(M, N, K, ksize, math_mode, 0, bn, k_splits, stages, cluster, effective_math, &grid);
}

// The same view under an SM budget (k2y_net_set_sm_limit): also reports the persistent grid size.
extern "C" int k2y_tc_plan_budget(int M, int N, int K, int ksize, int math_mode, int sm_limit, int *bn, int *k_splits, int *stages,
                                  int *cluster, int *effective_math, int *grid) {
    using namespace k2y;
    if (M <= 0 || N <= 0 || K <= 0 || (ksize != 1 && ksize != 3) || !bn || !k_splits || !stages || !cluster || !effective_math ||
        (math_mode != K2Y_MATH_TC_3XTF32 && math_mode != K2Y_MATH_TC_TF32 && math_mode != K2Y_MATH_TC_BF16X3) || sm_limit < 0 || !grid) {
        set_error("k2y_tc_plan: bad arguments");
        return K2Y_ERR_INVALID;
    }
    // the GEMM as a conv: M output pixels in one row, ksize x ksize taps over K / ksize^2 channels of one plain source
    ConvArgs a{};
    a.B = a.H = a.OH = 1;
    a.W = a.OW = M;
    a.kh = a.kw = ksize;
    a.stride = 1;
    a.C0 = K / (ksize * ksize);
    a.N = N;
    a.sm_limit = sm_limit;
    const TcPlan pl = plan_conv(a, K, math_mode);
    *bn = pl.bn;
    *k_splits = pl.k_splits;
    *stages = pl.stages;
    *cluster = 1;
    *effective_math = pl.mode;
    *grid = pl.grid;
    return K2Y_OK;
}
