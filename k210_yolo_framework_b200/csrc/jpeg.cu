// Baseline JPEG decoding on the GPU, bit-exact with libjpeg-turbo as PIL runs it on x86-64 (the reference reads every image
// with skimage.io.imread, tools/utils.py:339-355, i.e. PIL / libjpeg-turbo underneath): the x86 SIMD JDCT_ISLOW integer IDCT,
// fancy upsampling, ycc_rgb_convert.  The pixels land in the packed uint8 HWC buffer k2y_letterbox_u8_batch reads.
//
// Host side: a marker walker classifies each file (GPU-decodable, valid but not for the GPU, malformed) and builds one
// descriptor blob per batch (JpegBlobHeader, JpegImg[n], JpegSeg[segments], JpegHuff[2 * components per image]).  The caller
// puts the blob next to the compressed bytes in pinned memory, so one H2D copy moves both.
//
// Device side, one launch per stage whatever the image count:
//   1. jpeg_unstuff_kernel   (CTA per image)   drops the 0x00 after each 0xFF, cuts the entropy data at RSTn markers and
//                            checks their numbers (the k-th between intervals must be RST(k mod 8)); a marker past the
//                            last interval ends the data
//   2. jpeg_huffman_kernel   (CTA per segment) self-synchronising Huffman decode (Weissenberger & Schmidt): each thread owns
//                            a fixed-length subsequence of the segment's bits, decodes it from a guessed state, then restarts
//                            from its left neighbour's exact end state until its own end state stops changing; an exclusive
//                            scan of completed blocks gives each thread its first block, and a last pass writes int16
//                            coefficients in natural order (DC as differences)
//   3. jpeg_dc_kernel        (CTA per segment) per-component scan of the DC differences in decode order
//   4. jpeg_idct_kernel      dequantise + libjpeg-turbo's x86 SIMD islow (jidctint-avx2.asm / -sse2.asm, 16-bit lanes)
//                            -> uint8 component planes at the MCU-padded size
//   5. jpeg_color_kernel     libjpeg-turbo's upsampler dispatch (fancy on) + ycc_rgb_convert, cropped, HWC RGB out
#include "jpeg_common.cuh"

#include <vector>

namespace k2y {
namespace {

constexpr uint32_t JPEG_BLOB_MAGIC = 0x4a504731u;   // "JPG1"

constexpr int SYNC_THREADS = 256;                    // subsequences per window of one segment
constexpr int SUBSEQ_BITS = 512;                     // bits per subsequence
constexpr int UNSTUFF_THREADS = 512;
constexpr int UNSTUFF_BYTES = 16;                    // source bytes per thread per tile
constexpr int DC_THREADS = 256;


struct alignas(16) JpegImg {
    long long src_offset;       // first entropy-coded byte in the source buffer
    long long src_end;          // end of the file in the source buffer
    long long dst_offset;       // HWC RGB output
    long long unstuff_offset;   // workspace: unstuffed entropy bytes
    long long seg_offset;       // workspace: int32 [nseg + 1] segment starts in the unstuffed bytes
    long long coef_offset;      // workspace: int16 coefficients, bytes
    long long plane_offset;     // workspace: uint8 component planes, bytes
    int32_t h, w, ncomp, upsample;
    int32_t mcux, mcuy, bpm, nseg;
    int32_t restart_mcus, seg_first, huff_first, blocks;   // MCUs per segment, global index of segment 0 / table 0, blocks
    int32_t bw[3], bh[3];       // component planes in blocks (MCU-padded)
    int32_t dw[3], dh[3];       // libjpeg downsampled_width / downsampled_height
    int32_t hs[3], vs[3];
    int32_t coef_block[3];      // first block of each component
    int32_t plane_byte[3];      // byte offset of each component plane
    uint8_t mcu_comp[MAX_BLOCKS_PER_MCU], mcu_bx[MAX_BLOCKS_PER_MCU], mcu_by[MAX_BLOCKS_PER_MCU];
    uint8_t pad_[2];
    uint16_t qt[3][64];         // natural order
};

struct alignas(16) JpegSeg {
    int32_t image, index, first_mcu, mcus;
};

struct alignas(16) JpegBlobHeader {
    uint32_t magic;
    int32_t n, nseg, max_blocks;
    long long max_pixels;
    long long img_off, seg_off, huff_off, blob_bytes;
    long long ws_unstuff, ws_seg, ws_coef, ws_plane, ws_bytes;
};


struct ImgPlan {
    Parsed p;
    int nseg = 0;
};

// ---------------------------------------------------------------------------------------------------------------------
// Device helpers
// ---------------------------------------------------------------------------------------------------------------------
// Exclusive scan over the CTA (blockDim.x a multiple of 32, <= 1024); `sh` holds 32 ints.
__device__ __forceinline__ int block_excl_scan(int v, int &total, int *sh) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) sh[warp] = x;
    __syncthreads();
    if (warp == 0) {
        int s = lane < nw ? sh[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += y;
        }
        sh[lane] = s;
    }
    __syncthreads();
    const int before = warp > 0 ? sh[warp - 1] : 0;
    total = sh[nw - 1];
    __syncthreads();
    return before + x - v;
}

// MSB-first bit reader over one segment's unstuffed bytes; zeros past its end (as libjpeg inserts on a premature end).
struct BitReader {
    const uint8_t *u;
    int len, pos, nb;
    uint64_t buf;
    __device__ __forceinline__ void fill() {
        while (nb <= 56) {
            const uint64_t b = pos < len ? (uint64_t)__ldg(u + pos) : 0ull;
            buf |= b << (56 - nb);
            nb += 8;
            ++pos;
        }
    }
    __device__ __forceinline__ void init(const uint8_t *base, int bytes, unsigned bit) {
        u = base;
        len = bytes;
        pos = (int)(bit >> 3);
        nb = 0;
        buf = 0;
        fill();
        buf <<= (bit & 7);
        nb -= (bit & 7);
    }
    __device__ __forceinline__ unsigned get(int n) {   // 1 <= n <= 16, nb >= n
        const unsigned v = (unsigned)(buf >> (64 - n));
        buf <<= n;
        nb -= n;
        return v;
    }
};

// Decoder state at a codeword boundary: bit position, block within the MCU, zig-zag index (0 = DC next).
__device__ __forceinline__ unsigned long long pack_state(unsigned p, int c, int z) {
    return (unsigned long long)p | ((unsigned long long)c << 32) | ((unsigned long long)z << 40);
}

struct SegCtx {
    const JpegHuff *tab;    // shared memory: DC, AC table of each component
    const uint8_t *comp;    // shared memory: component of each block of the MCU
    int bpm;
};

struct WriteCtx {
    int16_t *coef;          // the image's coefficients
    const JpegImg *im;
    int first_mcu;
    int seg_blocks;
};

// Decodes codewords starting in [state.p, limit); returns the state after the last one, counts completed blocks.
// WRITE: also stores the coefficients of blocks first_block.. (segment-relative) below seg_blocks, and reports a bad code there.
template <bool WRITE>
__device__ unsigned long long decode_run(const uint8_t *u, int bytes, unsigned long long st, unsigned limit, const SegCtx &cx,
                                         int &blocks, const WriteCtx *wc, int first_block, bool &bad_out) {
    unsigned p = (unsigned)st;
    int c = (int)((st >> 32) & 255), z = (int)((st >> 40) & 255);
    BitReader br;
    br.init(u, bytes, p);
    int nblk = 0;
    int blk = first_block;
    int16_t *dstb = nullptr;
    int mcu = 0;
    if (WRITE) {
        mcu = wc->first_mcu + blk / cx.bpm;
    }
    auto block_ptr = [&]() -> int16_t * {
        const JpegImg *im = wc->im;
        const int comp = im->mcu_comp[c];
        const int mx = mcu % im->mcux, my = mcu / im->mcux;
        const int bx = mx * im->hs[comp] + im->mcu_bx[c], by = my * im->vs[comp] + im->mcu_by[c];
        return wc->coef + ((long long)im->coef_block[comp] + (long long)by * im->bw[comp] + bx) * 64;
    };
    if (WRITE && blk < wc->seg_blocks) dstb = block_ptr();
    bool bad = false;
    while (p < limit) {
        br.fill();
        int used = 0;
        bool badc = false;
        if (z == 0) {
            const int s = huff_decode(br, cx.tab[2 * cx.comp[c]], used, badc);
            int v = 0;
            if (s) {
                v = huff_extend(br.get(s), s);
                used += s;
            }
            if (WRITE && dstb) dstb[0] = (int16_t)v;
            z = 1;
        } else {
            const int rs = huff_decode(br, cx.tab[2 * cx.comp[c] + 1], used, badc);
            const int r = rs >> 4, s = rs & 15;
            if (s) {
                z += r;
                const int v = huff_extend(br.get(s), s);
                used += s;
                if (WRITE && dstb) dstb[c_natural[z > 63 ? 63 : z]] = (int16_t)v;
                z = z > 63 ? 64 : z + 1;
            } else if (r == 15) {
                z += 16;
            } else {
                z = 64;   // EOB
            }
        }
        if (WRITE && badc && blk < wc->seg_blocks) bad = true;
        p += used;
        if (z >= 64) {
            z = 0;
            ++nblk;
            if (++c == cx.bpm) c = 0;
            if (WRITE) {
                ++blk;
                if (c == 0) ++mcu;
                dstb = blk < wc->seg_blocks ? block_ptr() : nullptr;
            }
        }
    }
    blocks = nblk;
    bad_out = bad;
    return pack_state(p, c, z);
}

// ---------------------------------------------------------------------------------------------------------------------
// Kernels
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ const JpegBlobHeader &hdr(const uint8_t *blob) { return *reinterpret_cast<const JpegBlobHeader *>(blob); }
__device__ __forceinline__ const JpegImg *imgs(const uint8_t *blob) { return reinterpret_cast<const JpegImg *>(blob + hdr(blob).img_off); }

__global__ void __launch_bounds__(UNSTUFF_THREADS) jpeg_unstuff_kernel(const uint8_t *__restrict__ blob, const uint8_t *__restrict__ src,
                                                                       uint8_t *__restrict__ ws, int *__restrict__ status) {
    __shared__ int sh[32];
    __shared__ int s_term, s_last, s_order;
    const JpegImg &im = imgs(blob)[blockIdx.x];
    const uint8_t *s = src + im.src_offset;
    const long long n = im.src_end - im.src_offset;
    uint8_t *u = ws + hdr(blob).ws_unstuff + im.unstuff_offset;
    int *seg = reinterpret_cast<int *>(ws + hdr(blob).ws_seg + im.seg_offset);
    const int nseg = im.nseg;
    long long term = n;
    int out_total = 0, rst_total = 0;
    const int tile = UNSTUFF_THREADS * UNSTUFF_BYTES;
    if (threadIdx.x == 0) {
        s_last = 0x7fffffff;
        s_order = 0;
    }
    for (long long base = 0; base < term; base += tile) {
        const long long b0 = base + (long long)threadIdx.x * UNSTUFF_BYTES;
        const long long b1 = min(b0 + UNSTUFF_BYTES, n);
        if (threadIdx.x == 0) s_term = 0x7fffffff;
        __syncthreads();
        // the first marker that is neither a stuffed zero, a fill byte nor RSTn ends the entropy-coded data
        for (long long q = b0; q < b1; ++q) {
            if (s[q] == 0xFF) {
                const int nx = q + 1 < n ? s[q + 1] : 0xD9;
                if (!(nx == 0x00 || nx == 0xFF || (nx >= 0xD0 && nx <= 0xD7))) {
                    atomicMin(&s_term, (int)(q - base));
                    break;
                }
            }
        }
        __syncthreads();
        if (s_term != 0x7fffffff) term = min(term, base + s_term);
        const long long e = min(b1, term);
        int kept = 0, rst = 0;
        for (long long q = b0; q < e; ++q) {
            const int cur = s[q], prev = q > 0 ? s[q - 1] : 0;
            if (cur == 0xFF) {
                kept += (q + 1 < n && s[q + 1] == 0x00);
            } else if (prev == 0xFF && (cur == 0x00 || (cur >= 0xD0 && cur <= 0xD7))) {
                rst += cur != 0x00;
            } else {
                ++kept;
            }
        }
        int kept_total, rst_sum;
        int ko = block_excl_scan(kept, kept_total, sh);
        int ro = block_excl_scan(rst, rst_sum, sh);
        int o = out_total + ko, r = rst_total + ro;
        for (long long q = b0; q < e; ++q) {
            const int cur = s[q], prev = q > 0 ? s[q - 1] : 0;
            if (cur == 0xFF) {
                if (q + 1 < n && s[q + 1] == 0x00) u[o++] = 0xFF;
            } else if (prev == 0xFF && (cur == 0x00 || (cur >= 0xD0 && cur <= 0xD7))) {
                if (cur != 0x00) {
                    ++r;
                    if (r < nseg) {
                        seg[r] = o;
                        if ((cur & 7) != ((r - 1) & 7)) s_order = 1;
                    } else if (r == nseg) {
                        s_last = o;
                    }
                }
            } else {
                u[o++] = (uint8_t)cur;
            }
        }
        out_total += kept_total;
        rst_total += rst_sum;
        __syncthreads();
    }
    // segments whose RSTn never came are empty (the decode reports the premature end)
    for (int k = rst_total + 1 + threadIdx.x; k < nseg; k += blockDim.x) seg[k] = out_total;
    if (threadIdx.x == 0) {
        seg[0] = 0;
        // a marker past the last interval (or any with no restart interval) ends the data, where libjpeg stops reading it
        seg[nseg] = min(out_total, s_last);
        // a marker between intervals out of sequence: libjpeg-turbo resynchronises, which this decode does not model
        if (s_order) atomicOr(status + 4 * blockIdx.x, 4);
    }
}

// status words per image: [0] error bits (1 bad Huffman code, 2 premature end of data, 4 a restart marker between intervals
// out of sequence), [1] max sync rounds of a window,
// [2] sum of sync rounds over windows, [3] windows
__global__ void __launch_bounds__(SYNC_THREADS) jpeg_huffman_kernel(const uint8_t *__restrict__ blob, uint8_t *__restrict__ ws,
                                                                    int *__restrict__ status) {
    __shared__ JpegHuff s_tab[6];
    __shared__ unsigned long long s_end[SYNC_THREADS];
    __shared__ int sh[32];
    const JpegBlobHeader &H = hdr(blob);
    const JpegSeg &sg = reinterpret_cast<const JpegSeg *>(blob + H.seg_off)[blockIdx.x];
    const JpegImg &im = imgs(blob)[sg.image];
    const JpegHuff *tabs = reinterpret_cast<const JpegHuff *>(blob + H.huff_off) + im.huff_first;
    const int ntab = 2 * im.ncomp;
    {
        const int4 *srcv = reinterpret_cast<const int4 *>(tabs);
        int4 *dstv = reinterpret_cast<int4 *>(s_tab);
        for (int k = threadIdx.x; k < ntab * (int)(sizeof(JpegHuff) / 16); k += blockDim.x) dstv[k] = srcv[k];
    }
    __shared__ uint8_t s_comp[MAX_BLOCKS_PER_MCU];
    if (threadIdx.x < MAX_BLOCKS_PER_MCU) s_comp[threadIdx.x] = im.mcu_comp[threadIdx.x];
    SegCtx cx;
    cx.tab = s_tab;
    cx.comp = s_comp;
    cx.bpm = im.bpm;
    const int *seg = reinterpret_cast<const int *>(ws + H.ws_seg + im.seg_offset);
    const int sbeg = seg[sg.index], send = max(seg[sg.index + 1], sbeg);
    const uint8_t *u = ws + H.ws_unstuff + im.unstuff_offset + sbeg;
    const int bytes = send - sbeg;
    const unsigned L = (unsigned)bytes * 8u;
    WriteCtx wc;
    wc.coef = reinterpret_cast<int16_t *>(ws + H.ws_coef + im.coef_offset);
    wc.im = &im;
    wc.first_mcu = sg.first_mcu;
    wc.seg_blocks = sg.mcus * im.bpm;
    __syncthreads();

    unsigned long long exact = pack_state(0, 0, 0);
    int done = 0, max_rounds = 0, sum_rounds = 0, windows = 0;
    bool bad_any = false;
    for (unsigned w0 = 0; w0 < L && done < wc.seg_blocks; w0 += SYNC_THREADS * SUBSEQ_BITS) {
        const unsigned k0 = w0 + threadIdx.x * SUBSEQ_BITS;
        const bool active = k0 < L;
        const unsigned lim = min(k0 + SUBSEQ_BITS, L);
        unsigned long long start = threadIdx.x == 0 ? exact : pack_state(k0, 0, 0);   // guess: a block starts here
        unsigned long long end = start;
        int nb = 0;
        bool bad;
        if (active) end = decode_run<false>(u, bytes, start, lim, cx, nb, nullptr, 0, bad);
        s_end[threadIdx.x] = end;
        __syncthreads();
        int rounds = 0;
        for (;;) {   // restart from the left neighbour's end state until no subsequence's start changes
            const unsigned long long left = threadIdx.x > 0 ? s_end[threadIdx.x - 1] : start;
            __syncthreads();
            const bool redo = active && left != start;
            if (redo) {
                start = left;
                end = decode_run<false>(u, bytes, start, lim, cx, nb, nullptr, 0, bad);
                s_end[threadIdx.x] = end;
            }
            if (!__syncthreads_or(redo)) break;
            ++rounds;
        }
        int total;
        const int first = done + block_excl_scan(active ? nb : 0, total, sh);
        if (active) {
            int nb2;
            decode_run<true>(u, bytes, start, lim, cx, nb2, &wc, first, bad);
            bad_any |= bad;
        }
        done += total;
        const int last = min((int)((L - 1 - w0) / SUBSEQ_BITS), SYNC_THREADS - 1);
        exact = s_end[last];
        max_rounds = max(max_rounds, rounds);
        sum_rounds += rounds;
        ++windows;
        __syncthreads();
    }
    int *st = status + 4 * sg.image;
    if (__syncthreads_or(bad_any) && threadIdx.x == 0) atomicOr(st, 1);
    if (threadIdx.x == 0) {
        if (done < wc.seg_blocks) atomicOr(st, 2);
        atomicMax(st + 1, max_rounds);
        atomicAdd(st + 2, sum_rounds);
        atomicAdd(st + 3, windows);
    }
}

__device__ __forceinline__ int16_t *dc_ptr(int16_t *coef, const JpegImg &im, int mcu, int c) {
    const int comp = im.mcu_comp[c];
    const int mx = mcu % im.mcux, my = mcu / im.mcux;
    const int bx = mx * im.hs[comp] + im.mcu_bx[c], by = my * im.vs[comp] + im.mcu_by[c];
    return coef + ((long long)im.coef_block[comp] + (long long)by * im.bw[comp] + bx) * 64;
}

// DC differences -> absolute values: per component, in decode order, from zero at each restart.
__global__ void __launch_bounds__(DC_THREADS) jpeg_dc_kernel(const uint8_t *__restrict__ blob, uint8_t *__restrict__ ws) {
    __shared__ int sh[32];
    const JpegBlobHeader &H = hdr(blob);
    const JpegSeg &sg = reinterpret_cast<const JpegSeg *>(blob + H.seg_off)[blockIdx.x];
    const JpegImg &im = imgs(blob)[sg.image];
    int16_t *coef = reinterpret_cast<int16_t *>(ws + H.ws_coef + im.coef_offset);
    int carry[3] = {0, 0, 0};
    for (int base = 0; base < sg.mcus; base += DC_THREADS) {
        const bool active = base + (int)threadIdx.x < sg.mcus;
        const int mcu = sg.first_mcu + base + threadIdx.x;
        int d[MAX_BLOCKS_PER_MCU];
        int sum[3] = {0, 0, 0};
        for (int c = 0; c < im.bpm; ++c) {
            d[c] = active ? *dc_ptr(coef, im, mcu, c) : 0;
            sum[im.mcu_comp[c]] += d[c];
        }
        int run[3];
        for (int k = 0; k < im.ncomp; ++k) {
            int total;
            run[k] = carry[k] + block_excl_scan(sum[k], total, sh);
            carry[k] += total;
        }
        if (active) {
            for (int c = 0; c < im.bpm; ++c) {
                const int k = im.mcu_comp[c];
                run[k] += d[c];
                *dc_ptr(coef, im, mcu, c) = (int16_t)run[k];
            }
        }
    }
}

// Dequantise + IDCT (jpeg_common.cuh): one thread per 8x8 block; grid (block tiles, image).
__global__ void __launch_bounds__(IDCT_THREADS) jpeg_idct_kernel(const uint8_t *__restrict__ blob, uint8_t *__restrict__ ws) {
    __shared__ int s_q[3][64];
    const JpegBlobHeader &H = hdr(blob);
    const JpegImg &im = imgs(blob)[blockIdx.y];
    idct_image(im, ws + H.ws_coef + im.coef_offset, ws + H.ws_plane + im.plane_offset, s_q);
}

// Upsample + colour convert (jpeg_common.cuh): one thread per output pixel; grid (pixel tiles, image).
__global__ void __launch_bounds__(COLOR_THREADS) jpeg_color_kernel(const uint8_t *__restrict__ blob, const uint8_t *__restrict__ ws,
                                                                   uint8_t *__restrict__ dst) {
    const JpegBlobHeader &H = hdr(blob);
    const JpegImg &im = imgs(blob)[blockIdx.y];
    color_image(im, ws + H.ws_plane + im.plane_offset, dst + im.dst_offset);
}

}  // namespace
}  // namespace k2y

using namespace k2y;

extern "C" int k2y_jpeg_inspect(const unsigned char *data, size_t size, k2y_jpeg_info *info) {
    if (!data || !info) {
        set_error("k2y_jpeg_inspect: bad arguments");
        return K2Y_ERR_INVALID;
    }
    Parsed p;
    const int rc = parse_jpeg(data, size, p, "k2y_jpeg_inspect");
    if (rc != K2Y_OK) return rc;
    memset(info, 0, sizeof(*info));
    info->height = p.h;
    info->width = p.w;
    info->components = p.ncomp;
    for (int c = 0; c < 4; ++c) {
        info->h_samp[c] = c < p.ncomp ? p.hs[c] : 0;
        info->v_samp[c] = c < p.ncomp ? p.vs[c] : 0;
    }
    info->restart_interval = p.restart;
    info->precision = p.precision;
    info->sof_marker = p.sof;
    info->gpu_decodable = p.gpu ? 1 : 0;
    info->entropy_offset = p.gpu ? (int32_t)p.entropy : 0;
    snprintf(info->reason, sizeof(info->reason), "%s", p.gpu ? "" : p.reason);
    return K2Y_OK;
}

extern "C" int k2y_jpeg_plan(const unsigned char *const *files, const size_t *sizes, int n, const long long *src_offsets,
                             const long long *dst_offsets, void *blob, size_t blob_capacity, size_t *blob_bytes) {
    if (!files || !sizes || n <= 0 || !blob_bytes || (blob && (!src_offsets || !dst_offsets))) {
        set_error("k2y_jpeg_plan: bad arguments");
        return K2Y_ERR_INVALID;
    }
    std::vector<ImgPlan> plans(n);
    long long nseg = 0, ntab = 0;
    for (int i = 0; i < n; ++i) {
        char who[48];
        snprintf(who, sizeof(who), "k2y_jpeg_plan: image %d", i);
        Parsed &p = plans[i].p;
        if (!files[i]) {
            set_error("%s: null file pointer", who);
            return K2Y_ERR_INVALID;
        }
        const int rc = parse_jpeg(files[i], sizes[i], p, who);
        if (rc != K2Y_OK) return rc;
        if (!p.gpu) {
            set_error("%s: not decodable on the GPU: %s", who, p.reason);
            return K2Y_ERR_INVALID;
        }
        int hmax = 1, vmax = 1;
        if (p.ncomp == 3)
            for (int c = 0; c < 3; ++c) {
                hmax = std::max(hmax, p.hs[c]);
                vmax = std::max(vmax, p.vs[c]);
            }
        const long long mcus = (long long)((p.w + 8 * hmax - 1) / (8 * hmax)) * ((p.h + 8 * vmax - 1) / (8 * vmax));
        plans[i].nseg = p.restart ? (int)((mcus + p.restart - 1) / p.restart) : 1;
        nseg += plans[i].nseg;
        ntab += 2 * p.ncomp;
    }
    const long long img_off = align16(sizeof(JpegBlobHeader));
    const long long seg_off = img_off + (long long)sizeof(JpegImg) * n;
    const long long huff_off = align16(seg_off + (long long)sizeof(JpegSeg) * nseg);
    const long long total = huff_off + (long long)sizeof(JpegHuff) * ntab;
    *blob_bytes = (size_t)total;
    if (!blob) return K2Y_OK;
    if (blob_capacity < (size_t)total || ((uintptr_t)blob & 15)) {
        set_error("k2y_jpeg_plan: the blob needs %lld bytes at a 16-byte aligned address, got %zu", total, blob_capacity);
        return K2Y_ERR_INVALID;
    }
    uint8_t *B = static_cast<uint8_t *>(blob);
    memset(B, 0, (size_t)total);
    JpegBlobHeader &H = *reinterpret_cast<JpegBlobHeader *>(B);
    JpegImg *I = reinterpret_cast<JpegImg *>(B + img_off);
    JpegSeg *S = reinterpret_cast<JpegSeg *>(B + seg_off);
    JpegHuff *T = reinterpret_cast<JpegHuff *>(B + huff_off);
    long long unstuff = 0, segw = 0, coef = 0, plane = 0, max_pixels = 0;
    int max_blocks = 0, sg = 0, tb = 0;
    for (int i = 0; i < n; ++i) {
        const Parsed &p = plans[i].p;
        JpegImg &im = I[i];
        im.src_offset = src_offsets[i] + p.entropy;
        im.src_end = src_offsets[i] + (long long)sizes[i];
        im.dst_offset = dst_offsets[i];
        im.h = p.h;
        im.w = p.w;
        im.ncomp = p.ncomp;
        int hs[3] = {1, 1, 1}, vs[3] = {1, 1, 1}, hmax = 1, vmax = 1;
        if (p.ncomp == 3)
            for (int c = 0; c < 3; ++c) {
                hs[c] = p.hs[c];
                vs[c] = p.vs[c];
                hmax = std::max(hmax, hs[c]);
                vmax = std::max(vmax, vs[c]);
            }
        im.mcux = (p.w + 8 * hmax - 1) / (8 * hmax);
        im.mcuy = (p.h + 8 * vmax - 1) / (8 * vmax);
        int blocks = 0, pbytes = 0;
        for (int c = 0; c < p.ncomp; ++c) {
            im.hs[c] = hs[c];
            im.vs[c] = vs[c];
            im.bw[c] = im.mcux * hs[c];
            im.bh[c] = im.mcuy * vs[c];
            im.dw[c] = (int)(((long long)p.w * hs[c] + hmax - 1) / hmax);
            im.dh[c] = (int)(((long long)p.h * vs[c] + vmax - 1) / vmax);
            im.coef_block[c] = blocks;
            im.plane_byte[c] = pbytes;
            blocks += im.bw[c] * im.bh[c];
            pbytes += (int)align16((long long)im.bw[c] * 8 * im.bh[c] * 8);
            for (int k = 0; k < 64; ++k) im.qt[c][k] = p.scan_qt[c][k];
        }
        for (int c = p.ncomp; c < 3; ++c) im.coef_block[c] = blocks;
        im.blocks = blocks;
        int bpm = 0;
        for (int k = 0; k < p.ns; ++k) {
            const int f = p.scan_comp[k];
            for (int by = 0; by < vs[f]; ++by)
                for (int bx = 0; bx < hs[f]; ++bx) {
                    im.mcu_comp[bpm] = (uint8_t)f;
                    im.mcu_bx[bpm] = (uint8_t)bx;
                    im.mcu_by[bpm] = (uint8_t)by;
                    ++bpm;
                }
        }
        im.bpm = bpm;
        if (p.ncomp == 1) {
            im.upsample = UP_GRAY;
        } else {
            const int h0 = hs[0], v0 = vs[0], dw = im.dw[1];
            im.upsample = h0 == 1 && v0 == 1 ? UP_FULL
                          : h0 == 2 && v0 == 1 ? (dw > 2 ? UP_H2V1_FANCY : UP_H2V1_BOX)
                          : h0 == 1 && v0 == 2 ? UP_H1V2_FANCY
                          : h0 == 2 && v0 == 2 ? (dw > 2 ? UP_H2V2_FANCY : UP_H2V2_BOX)
                                               : UP_H4V1_BOX;
        }
        const int total_mcus = im.mcux * im.mcuy;
        im.nseg = plans[i].nseg;
        im.restart_mcus = p.restart ? p.restart : total_mcus;
        im.seg_first = sg;
        for (int k = 0; k < im.nseg; ++k, ++sg) {
            S[sg].image = i;
            S[sg].index = k;
            S[sg].first_mcu = k * im.restart_mcus;
            S[sg].mcus = std::min(im.restart_mcus, total_mcus - k * im.restart_mcus);
        }
        im.huff_first = tb;
        for (int c = 0; c < p.ncomp; ++c) {
            int k = 0;
            while (p.scan_comp[k] != c) ++k;
            if (!derive_huff(p.dc[p.td[k]], T[tb + 2 * c]) || !derive_huff(p.ac[p.ta[k]], T[tb + 2 * c + 1])) {
                set_error("k2y_jpeg_plan: image %d: bad Huffman table (code lengths overflow)", i);
                return K2Y_ERR_INVALID;
            }
        }
        tb += 2 * p.ncomp;
        im.unstuff_offset = unstuff;
        unstuff += align16((long long)sizes[i] - p.entropy);
        im.seg_offset = segw;
        segw += align16(4LL * (im.nseg + 1));
        im.coef_offset = coef;
        coef += (long long)blocks * 128;
        im.plane_offset = plane;
        plane += pbytes;
        max_blocks = std::max(max_blocks, blocks);
        max_pixels = std::max(max_pixels, (long long)p.h * p.w);
    }
    H.magic = JPEG_BLOB_MAGIC;
    H.n = n;
    H.nseg = (int)nseg;
    H.max_blocks = max_blocks;
    H.max_pixels = max_pixels;
    H.img_off = img_off;
    H.seg_off = seg_off;
    H.huff_off = huff_off;
    H.blob_bytes = total;
    H.ws_coef = 0;
    H.ws_plane = H.ws_coef + coef;
    H.ws_unstuff = H.ws_plane + align16(plane);
    H.ws_seg = H.ws_unstuff + unstuff;
    H.ws_bytes = H.ws_seg + segw;
    return K2Y_OK;
}

static const JpegBlobHeader *check_blob(const void *blob_host, const char *fn) {
    const JpegBlobHeader *H = static_cast<const JpegBlobHeader *>(blob_host);
    if (!H || H->magic != JPEG_BLOB_MAGIC || H->n <= 0) {
        set_error("%s: not a descriptor blob made by k2y_jpeg_plan", fn);
        return nullptr;
    }
    return H;
}

extern "C" int k2y_jpeg_workspace_bytes(const void *blob_host, size_t *bytes) {
    const JpegBlobHeader *H = check_blob(blob_host, "k2y_jpeg_workspace_bytes");
    if (!H || !bytes) {
        if (H) set_error("k2y_jpeg_workspace_bytes: bad arguments");
        return K2Y_ERR_INVALID;
    }
    *bytes = (size_t)H->ws_bytes;
    return K2Y_OK;
}

extern "C" int k2y_jpeg_decode(const void *blob_host, const void *blob_dev, const unsigned char *src_dev, unsigned char *dst_dev,
                               void *workspace_dev, size_t workspace_bytes, int32_t *status_dev, void *stream) {
    const JpegBlobHeader *H = check_blob(blob_host, "k2y_jpeg_decode");
    if (!H) return K2Y_ERR_INVALID;
    if (!blob_dev || !src_dev || !dst_dev || !workspace_dev || !status_dev || ((uintptr_t)blob_dev & 15) ||
        ((uintptr_t)workspace_dev & 15) || workspace_bytes < (size_t)H->ws_bytes) {
        set_error("k2y_jpeg_decode: bad arguments (16-byte aligned blob and workspace of %lld bytes needed, got %zu)", H->ws_bytes,
                  workspace_bytes);
        return K2Y_ERR_INVALID;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const uint8_t *blob = static_cast<const uint8_t *>(blob_dev);
    uint8_t *ws = static_cast<uint8_t *>(workspace_dev);
    K2Y_CUDA_CHECK(cudaMemsetAsync(status_dev, 0, sizeof(int32_t) * 4 * (size_t)H->n, st));
    K2Y_CUDA_CHECK(cudaMemsetAsync(ws + H->ws_coef, 0, (size_t)(H->ws_plane - H->ws_coef), st));
    jpeg_unstuff_kernel<<<H->n, UNSTUFF_THREADS, 0, st>>>(blob, src_dev, ws, status_dev);
    jpeg_huffman_kernel<<<H->nseg, SYNC_THREADS, 0, st>>>(blob, ws, status_dev);
    jpeg_dc_kernel<<<H->nseg, DC_THREADS, 0, st>>>(blob, ws);
    jpeg_idct_kernel<<<dim3((unsigned)((H->max_blocks + IDCT_THREADS - 1) / IDCT_THREADS), H->n), IDCT_THREADS, 0, st>>>(blob, ws);
    jpeg_color_kernel<<<dim3((unsigned)((H->max_pixels + COLOR_THREADS - 1) / COLOR_THREADS), H->n), COLOR_THREADS, 0, st>>>(blob, ws,
                                                                                                                          dst_dev);
    K2Y_CUDA_CHECK(cudaGetLastError());
    return K2Y_OK;
}
