// Baseline JPEG encoding on the GPU, byte-identical to PIL's `Image.fromarray(rgb).save(f, "JPEG", quality=q)` (libjpeg-turbo
// underneath): JFIF APP0, two DQT, SOF0 with 4:2:0 sampling, the four standard Huffman tables, one interleaved scan without
// restart markers, EOI.  The arithmetic follows libjpeg-turbo's compressor step by step: rgb_ycc_convert's fixed-point
// tables, edge replication to the MCU size (jcprepct.c / jcsample.c), h2v2_downsample's alternating 1/2 bias,
// jpeg_fdct_islow, jcdctmgr.c's reciprocal quantisation, the dummy blocks of jccoefct.c's compress_data, and jchuff.c's
// Huffman coding with 0xFF stuffing and 1-bit padding.
//
// Host side: k2y_jpeg_encode_plan builds one descriptor blob per batch (per image: size, offsets, the marker segments up to
// and including SOS, the quantisation divisors; once: the Huffman code tables).  The caller copies it to the device.
//
// Device side, one launch per stage whatever the image count:
//   1. enc_dct_kernel      (thread per 8x8 block)  colour convert + downsample + FDCT + quantise -> int16 zigzag coefficients
//   2. enc_len_kernel      (thread per block)      Huffman code length of the block in bits (DC predicted per component)
//   3. enc_scan_kernel     (CTA per image)         exclusive scan of the lengths -> bit offsets; clears the image's bit
//                                                  buffer and sets the 1-bit padding of its last byte
//   4. enc_emit_kernel     (thread per block)      writes the block's bits at its offset (atomicOr into big-endian words)
//   5. enc_ffcount_kernel  (CTA per chunk)         0xFF bytes of each chunk of the unstuffed stream
//   6. enc_ffscan_kernel   (CTA per image)         exclusive scan of the chunk counts; the image's file length
//   7. enc_pack_kernel     (CTA per chunk)         headers, stuffed entropy bytes and EOI, the images back to back
#include "common.h"
#include "jpeg_std_huff.cuh"

#include <algorithm>
#include <vector>

namespace k2y {
namespace {

constexpr uint32_t ENC_BLOB_MAGIC = 0x4a504531u;   // "JPE1"
constexpr int ENC_THREADS = 128;
constexpr int SCAN_THREADS = 1024;
constexpr int CHUNK_THREADS = 512;
constexpr int CHUNK_BYTES = CHUNK_THREADS * 16;     // unstuffed bytes per chunk
// Most bits one block can take: DC category code (<= 9 bits) + 11 magnitude bits, 63 AC codes of <= 16 + 10 bits.
constexpr long long MAX_BLOCK_BITS = 20 + 63 * 26;

struct alignas(16) EncImg {
    long long src_offset;      // packed HWC RGB input
    long long block_first;     // first block of the image in the batch's block numbering (MCU order, 6 blocks per MCU)
    long long bits_offset;     // workspace: uint32 words of the unstuffed stream
    long long chunk_first;     // first chunk of the image (stuffing counts)
    int32_t h, w, mcux, mcuy;
    int32_t ywb, yhb;          // luma width / height in blocks (libjpeg width_in_blocks / height_in_blocks)
    int32_t header_off, header_len;   // marker segments SOI .. SOS inside the blob
    int32_t max_chunks, pad_;
    uint16_t recip[2][64];     // jcdctmgr.c divisors, natural order: luma, chroma
    uint16_t corr[2][64];
    uint8_t shift[2][64];      // total right shift of (|x| + corr) * recip
};

struct alignas(16) EncBlobHeader {
    uint32_t magic;
    int32_t n;
    long long blocks, chunks, max_image_blocks;
    long long img_off, blob_bytes;
    long long ws_coef, ws_len, ws_off, ws_bits, ws_chunk, ws_nbytes, ws_total;
    long long out_capacity;    // bytes every image takes at most, summed
    uint32_t ehufco[4][256];   // DC0, AC0, DC1, AC1
    uint8_t ehufsi[4][256];
};

const uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                             41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                             30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
__constant__ uint8_t c_zigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                     41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                     30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// jcparam.c std_luminance_quant_tbl / std_chrominance_quant_tbl (ITU T.81 Annex K), natural order
const uint16_t kStdQuant[2][64] = {
    {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,  14, 13, 16, 24, 40,  57,  69,  56,
     14, 17, 22, 29, 51,  87,  80,  62,  18, 22, 37, 56, 68,  109, 103, 77,  24, 35, 55, 64, 81,  104, 113, 92,
     49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99},
    {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99,
     99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
     99, 99, 99, 99, 99, 99, 99, 99}};

// ---------------------------------------------------------------------------------------------------------------------
// Host: headers, divisors, Huffman codes
// ---------------------------------------------------------------------------------------------------------------------
// jcparam.c jpeg_quality_scaling + jpeg_add_quant_table(force_baseline = TRUE)
void quant_table(int quality, int which, uint16_t out[64]) {
    const int scale = quality < 50 ? 5000 / quality : 200 - quality * 2;
    for (int i = 0; i < 64; ++i) {
        long t = ((long)kStdQuant[which][i] * scale + 50L) / 100L;
        out[i] = (uint16_t)std::min(255L, std::max(1L, t));
    }
}

// jcdctmgr.c compute_reciprocal (the divisor is quantval << 3 for the islow DCT, so never 1)
void compute_reciprocal(uint16_t divisor, uint16_t &recip, uint16_t &corr, uint8_t &shift) {
    int b = 0;
    while ((1u << (b + 1)) <= divisor) ++b;   // flss(divisor) - 1
    int r = 16 + b;
    uint32_t fq = (uint32_t)((1ull << r) / divisor);
    const uint32_t fr = (uint32_t)((1ull << r) % divisor);
    uint32_t c = divisor / 2;
    if (fr == 0) {
        fq >>= 1;
        --r;
    } else if (fr <= divisor / 2u) {
        ++c;
    } else {
        ++fq;
    }
    recip = (uint16_t)fq;
    corr = (uint16_t)c;
    shift = (uint8_t)r;
}

// jchuff.c jpeg_make_c_derived_tbl for the standard tables
void derive_codes(int t, uint32_t code_out[256], uint8_t size_out[256]) {
    memset(code_out, 0, 256 * sizeof(uint32_t));
    memset(size_out, 0, 256);
    const uint8_t *vals = huff_vals(t);
    uint32_t code = 0;
    int k = 0;
    for (int l = 1; l <= 16; ++l) {
        for (int i = 0; i < kHuffBits[t][l - 1]; ++i, ++k) {
            code_out[vals[k]] = code++;
            size_out[vals[k]] = (uint8_t)l;
        }
        code <<= 1;
    }
}

void put16(std::vector<uint8_t> &v, int x) {
    v.push_back((uint8_t)(x >> 8));
    v.push_back((uint8_t)x);
}

// SOI, JFIF APP0 (version 1.01, no units, density 1:1), DQT x2, SOF0 (4:2:0), DHT x4, SOS: what jcmarker.c writes for PIL's
// defaults.
std::vector<uint8_t> build_header(int h, int w, const uint16_t qt[2][64]) {
    std::vector<uint8_t> v;
    const uint8_t app0[] = {0xFF, 0xD8, 0xFF, 0xE0, 0, 16, 'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0};
    v.insert(v.end(), app0, app0 + sizeof(app0));
    for (int t = 0; t < 2; ++t) {
        const uint8_t m[] = {0xFF, 0xDB, 0, 67, (uint8_t)t};
        v.insert(v.end(), m, m + sizeof(m));
        for (int k = 0; k < 64; ++k) v.push_back((uint8_t)qt[t][kZigzag[k]]);
    }
    v.push_back(0xFF);
    v.push_back(0xC0);
    put16(v, 17);
    v.push_back(8);
    put16(v, h);
    put16(v, w);
    const uint8_t comps[] = {3, 1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1};
    v.insert(v.end(), comps, comps + sizeof(comps));
    const uint8_t classes[4] = {0x00, 0x10, 0x01, 0x11};
    for (int t = 0; t < 4; ++t) {
        int nv = 0;
        for (int l = 0; l < 16; ++l) nv += kHuffBits[t][l];
        v.push_back(0xFF);
        v.push_back(0xC4);
        put16(v, 2 + 1 + 16 + nv);
        v.push_back(classes[t]);
        v.insert(v.end(), kHuffBits[t], kHuffBits[t] + 16);
        v.insert(v.end(), huff_vals(t), huff_vals(t) + nv);
    }
    const uint8_t sos[] = {0xFF, 0xDA, 0, 12, 3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0};
    v.insert(v.end(), sos, sos + sizeof(sos));
    return v;
}

// ---------------------------------------------------------------------------------------------------------------------
// Per-block arithmetic, shared by the kernels (and usable on the host)
// ---------------------------------------------------------------------------------------------------------------------
#define ENC_FIX(x) ((int32_t)((x) * 65536.0 + 0.5))

// jccolor.c rgb_ycc_convert: the sums of its per-channel tables (ONE_HALF / CBCR_OFFSET + ONE_HALF - 1 folded in)
__host__ __device__ inline int rgb_to_ycc(int r, int g, int b, int comp) {
    if (comp == 0) return (ENC_FIX(0.29900) * r + ENC_FIX(0.58700) * g + ENC_FIX(0.11400) * b + (1 << 15)) >> 16;
    if (comp == 1) return (-ENC_FIX(0.16874) * r - ENC_FIX(0.33126) * g + ENC_FIX(0.5) * b + (128 << 16) + (1 << 15) - 1) >> 16;
    return (ENC_FIX(0.5) * r - ENC_FIX(0.41869) * g - ENC_FIX(0.08131) * b + (128 << 16) + (1 << 15) - 1) >> 16;
}

__host__ __device__ inline int pixel_comp(const uint8_t *img, int w, int y, int x, int comp) {
    const uint8_t *p = img + ((long long)y * w + x) * 3;
    return rgb_to_ycc(p[0], p[1], p[2], comp);
}

// The 8x8 samples of block (by, bx) of component `comp`, as libjpeg's compressor sees them.  Luma: rows and columns past the
// image repeat the last one.  Chroma: the full-resolution plane's columns are extended to the MCU width (expand_right_edge)
// and its rows paired with the last row repeated (a row group of 2), h2v2_downsample averages each 2x2 with bias 1, 2, 1,
// 2, ... along a row, and downsampled rows past the last real one repeat it (the bottom pad to the iMCU height).
__host__ __device__ inline void load_block(const uint8_t *img, int h, int w, int comp, int by, int bx, int32_t s[64]) {
    if (comp == 0) {
        for (int r = 0; r < 8; ++r) {
            const int y = min(by * 8 + r, h - 1);
            for (int c = 0; c < 8; ++c) s[r * 8 + c] = pixel_comp(img, w, y, min(bx * 8 + c, w - 1), 0);
        }
        return;
    }
    const int last_row = (h + 1) / 2 - 1;
    for (int r = 0; r < 8; ++r) {
        const int oy = min(by * 8 + r, last_row);
        const int y0 = min(2 * oy, h - 1), y1 = min(2 * oy + 1, h - 1);
        for (int c = 0; c < 8; ++c) {
            const int ox = bx * 8 + c;
            const int x0 = min(2 * ox, w - 1), x1 = min(2 * ox + 1, w - 1);
            const int sum = pixel_comp(img, w, y0, x0, comp) + pixel_comp(img, w, y0, x1, comp) + pixel_comp(img, w, y1, x0, comp) +
                            pixel_comp(img, w, y1, x1, comp);
            s[r * 8 + c] = (sum + 1 + (ox & 1)) >> 2;
        }
    }
}

// jfdctint.c jpeg_fdct_islow on samples - 128; the output is scaled up by 8
__host__ __device__ inline void fdct_islow(int32_t d[64]) {
    constexpr int CB = 13, P1 = 2;
    for (int pass = 0; pass < 2; ++pass) {
        const int stride = pass == 0 ? 8 : 1, step = pass == 0 ? 1 : 8;
        const int sh = pass == 0 ? CB - P1 : CB + P1;
        for (int i = 0; i < 8; ++i) {
            int32_t *p = d + i * stride;
            const int32_t tmp0 = p[0] + p[7 * step], tmp7 = p[0] - p[7 * step];
            const int32_t tmp1 = p[step] + p[6 * step], tmp6 = p[step] - p[6 * step];
            const int32_t tmp2 = p[2 * step] + p[5 * step], tmp5 = p[2 * step] - p[5 * step];
            const int32_t tmp3 = p[3 * step] + p[4 * step], tmp4 = p[3 * step] - p[4 * step];
            const int32_t tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
            if (pass == 0) {
                p[0] = (tmp10 + tmp11) * (1 << P1);
                p[4 * step] = (tmp10 - tmp11) * (1 << P1);
            } else {
                p[0] = (tmp10 + tmp11 + (1 << (P1 - 1))) >> P1;
                p[4 * step] = (tmp10 - tmp11 + (1 << (P1 - 1))) >> P1;
            }
            const int32_t rnd = 1 << (sh - 1);
            int32_t z1 = (tmp12 + tmp13) * 4433;
            p[2 * step] = (z1 + tmp13 * 6270 + rnd) >> sh;
            p[6 * step] = (z1 + tmp12 * -15137 + rnd) >> sh;
            z1 = tmp4 + tmp7;
            int32_t z2 = tmp5 + tmp6, z3 = tmp4 + tmp6, z4 = tmp5 + tmp7;
            const int32_t z5 = (z3 + z4) * 9633;
            const int32_t t4 = tmp4 * 2446, t5 = tmp5 * 16819, t6 = tmp6 * 25172, t7 = tmp7 * 12299;
            z1 *= -7373;
            z2 *= -20995;
            z3 = z3 * -16069 + z5;
            z4 = z4 * -3196 + z5;
            p[7 * step] = (t4 + z1 + z3 + rnd) >> sh;
            p[5 * step] = (t5 + z2 + z4 + rnd) >> sh;
            p[3 * step] = (t6 + z2 + z3 + rnd) >> sh;
            p[step] = (t7 + z1 + z4 + rnd) >> sh;
        }
    }
}

// jcdctmgr.c quantize: sign(x) * (((|x| + corr) * recip) >> shift), in the 16-bit arithmetic of its SIMD form
__host__ __device__ inline int quantize(int32_t x, uint16_t recip, uint16_t corr, uint8_t shift) {
    const uint32_t a = (uint32_t)(uint16_t)((x < 0 ? -x : x) + corr);
    const int q = (int)((a * (uint32_t)recip) >> shift);
    return x < 0 ? -q : q;
}

// Where block `b` of an image lies: component and block coordinates; dummy blocks (past the luma plane's blocks inside the
// last MCU column / row) get the coordinates of the block whose DC they repeat (jccoefct.c compress_data).
__host__ __device__ inline void block_place(const EncImg &im, long long b, int &comp, int &by, int &bx, bool &dummy) {
    const long long mcu = b / 6;
    const int k = (int)(b - mcu * 6);
    const int my = (int)(mcu / im.mcux), mx = (int)(mcu - (long long)my * im.mcux);
    dummy = false;
    if (k >= 4) {
        comp = k - 3;
        by = my;
        bx = mx;
        return;
    }
    comp = 0;
    by = my * 2 + (k >> 1);
    bx = mx * 2 + (k & 1);
    if (by >= im.yhb) {   // a row of dummies repeats the DC of the last block of the MCU's first row
        dummy = true;
        by -= 1;
        bx = min(mx * 2 + 1, im.ywb - 1);
    } else if (bx >= im.ywb) {
        dummy = true;
        bx = im.ywb - 1;
    }
}

// Quantised coefficients of one block in zigzag order
__host__ __device__ inline void encode_block(const EncImg &im, const uint8_t *img, long long b, int16_t out[64]) {
    int comp, by, bx;
    bool dummy;
    block_place(im, b, comp, by, bx, dummy);
    int32_t s[64];
    load_block(img, im.h, im.w, comp, by, bx, s);
    const int t = comp == 0 ? 0 : 1;
    if (dummy) {   // DC only: the FDCT's DC output is the sum of the centred samples
        int32_t sum = 0;
        for (int i = 0; i < 64; ++i) sum += s[i] - 128;
        out[0] = (int16_t)quantize(sum, im.recip[t][0], im.corr[t][0], im.shift[t][0]);
        for (int i = 1; i < 64; ++i) out[i] = 0;
        return;
    }
    for (int i = 0; i < 64; ++i) s[i] -= 128;
    fdct_islow(s);
    for (int k = 0; k < 64; ++k) {
#ifdef __CUDA_ARCH__
        const int nat = c_zigzag[k];
#else
        const int nat = kZigzag[k];
#endif
        out[k] = (int16_t)quantize(s[nat], im.recip[t][nat], im.corr[t][nat], im.shift[t][nat]);
    }
}

// The block of the same component coded before block b (MCU order), or -1 for the first one
__host__ __device__ inline long long prev_same_comp(long long b) {
    const long long mcu = b / 6;
    const int k = (int)(b - mcu * 6);
    if (k >= 1 && k <= 3) return b - 1;
    if (mcu == 0) return -1;
    return k == 0 ? b - 3 : b - 6;
}

__host__ __device__ inline int nbits_of(int v) {
    int n = 0;
    while (v) {
        ++n;
        v >>= 1;
    }
    return n;
}

// jchuff.c encode_one_block through an emitter: put(code, size)
template <typename Put>
__host__ __device__ inline void huff_block(const int16_t *coef, int last_dc, int comp, const uint32_t (*co)[256],
                                           const uint8_t (*si)[256], Put &put) {
    const int dct = comp == 0 ? 0 : 2, act = dct + 1;
    int temp = coef[0] - last_dc, temp2 = temp;
    if (temp < 0) {
        temp = -temp;
        --temp2;
    }
    int nb = nbits_of(temp);
    put(co[dct][nb], si[dct][nb]);
    if (nb) put((uint32_t)temp2 & ((1u << nb) - 1), nb);
    int r = 0;
    for (int k = 1; k < 64; ++k) {
        temp = coef[k];
        if (temp == 0) {
            ++r;
            continue;
        }
        while (r > 15) {
            put(co[act][0xF0], si[act][0xF0]);
            r -= 16;
        }
        temp2 = temp;
        if (temp < 0) {
            temp = -temp;
            --temp2;
        }
        nb = nbits_of(temp);
        const int i = (r << 4) + nb;
        put(co[act][i], si[act][i]);
        put((uint32_t)temp2 & ((1u << nb) - 1), nb);
        r = 0;
    }
    if (r > 0) put(co[act][0], si[act][0]);
}

struct CountBits {
    uint32_t n = 0;
    __host__ __device__ void operator()(uint32_t, int size) { n += size; }
};

// Big-endian bit writer into uint32 words shared with the neighbouring blocks (atomicOr on the device)
struct WriteBits {
    uint32_t *words;
    long long wi;
    int nb;
    uint64_t buf;
    __device__ WriteBits(uint32_t *w, unsigned long long bitpos) : words(w), wi((long long)(bitpos >> 5)), nb((int)(bitpos & 31)), buf(0) {}
    __device__ void operator()(uint32_t code, int size) {
        buf = (buf << size) | code;
        nb += size;
        if (nb >= 32) {
            nb -= 32;
            atomicOr(words + wi++, (uint32_t)(buf >> nb));
            buf &= (1ull << nb) - 1;
        }
    }
    __device__ void flush() {
        if (nb > 0) atomicOr(words + wi, (uint32_t)(buf << (32 - nb)));
    }
};

// ---------------------------------------------------------------------------------------------------------------------
// Kernels
// ---------------------------------------------------------------------------------------------------------------------
struct EncPtrs {
    const EncBlobHeader *hdr;
    const EncImg *img;
    const uint8_t *blob;
    const uint8_t *src;
    uint8_t *dst;
    long long *lengths;
    int16_t *coef;
    uint32_t *len;
    unsigned long long *off;
    uint32_t *bits;
    uint32_t *chunk;       // 0xFF count per chunk, then its exclusive scan
    long long *nbytes;     // unstuffed bytes per image (padded)
};

__device__ inline int image_of_block(const EncImg *img, int n, long long b) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (img[mid].block_first <= b) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(ENC_THREADS) enc_dct_kernel(EncPtrs p, int n, long long blocks) {
    const long long g = (long long)blockIdx.x * ENC_THREADS + threadIdx.x;
    if (g >= blocks) return;
    const EncImg &im = p.img[image_of_block(p.img, n, g)];
    int16_t out[64];
    encode_block(im, p.src + im.src_offset, g - im.block_first, out);
    int4 *dst = reinterpret_cast<int4 *>(p.coef + g * 64);
#pragma unroll
    for (int i = 0; i < 8; ++i) dst[i] = reinterpret_cast<const int4 *>(out)[i];
}

__device__ inline void load_coef(const int16_t *src, int16_t out[64]) {
    const int4 *s = reinterpret_cast<const int4 *>(src);
#pragma unroll
    for (int i = 0; i < 8; ++i) reinterpret_cast<int4 *>(out)[i] = s[i];
}

__global__ void __launch_bounds__(ENC_THREADS) enc_len_kernel(EncPtrs p, int n, long long blocks) {
    const long long g = (long long)blockIdx.x * ENC_THREADS + threadIdx.x;
    if (g >= blocks) return;
    const EncImg &im = p.img[image_of_block(p.img, n, g)];
    const long long b = g - im.block_first;
    const long long pb = prev_same_comp(b);
    const int last_dc = pb < 0 ? 0 : p.coef[(im.block_first + pb) * 64];
    int16_t c[64];
    load_coef(p.coef + g * 64, c);
    CountBits cnt;
    const int k = (int)(b % 6);
    huff_block(c, last_dc, k < 4 ? 0 : k - 3, p.hdr->ehufco, p.hdr->ehufsi, cnt);
    p.len[g] = cnt.n;
}

__device__ inline unsigned long long block_scan_u64(unsigned long long v, unsigned long long *warp_sums, unsigned long long &total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    unsigned long long x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warp_sums[wid] = x;
    __syncthreads();
    if (wid == 0) {
        unsigned long long s = lane < nw ? warp_sums[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long y = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += y;
        }
        if (lane < nw) warp_sums[lane] = s;
    }
    __syncthreads();
    const unsigned long long excl = x - v + (wid > 0 ? warp_sums[wid - 1] : 0);
    total = warp_sums[nw - 1];
    __syncthreads();
    return excl;
}

__global__ void __launch_bounds__(SCAN_THREADS) enc_scan_kernel(EncPtrs p) {
    __shared__ unsigned long long warp_sums[32];
    const EncImg &im = p.img[blockIdx.x];
    const long long nblk = (long long)im.mcux * im.mcuy * 6;
    unsigned long long carry = 0;
    for (long long t0 = 0; t0 < nblk; t0 += SCAN_THREADS) {
        const long long b = t0 + threadIdx.x;
        const unsigned long long v = b < nblk ? p.len[im.block_first + b] : 0;
        unsigned long long total;
        const unsigned long long ex = block_scan_u64(v, warp_sums, total);
        if (b < nblk) p.off[im.block_first + b] = carry + ex;
        carry += total;
    }
    const unsigned long long nbits = carry, nbytes = (nbits + 7) / 8;
    uint32_t *words = p.bits + im.bits_offset;
    const long long nwords = (long long)((nbytes + 3) / 4);
    for (long long i = threadIdx.x; i < nwords; i += SCAN_THREADS) words[i] = 0;
    __syncthreads();
    if (threadIdx.x == 0) {
        const int pad = (int)(nbytes * 8 - nbits);   // flush_bits: 1-bits up to the byte boundary
        if (pad) {
            const unsigned long long pos = nbits;
            const uint32_t ones = ((1u << pad) - 1) << (32 - (int)(pos & 31) - pad);
            words[pos >> 5] |= ones;
        }
        p.nbytes[blockIdx.x] = (long long)nbytes;
    }
}

__global__ void __launch_bounds__(ENC_THREADS) enc_emit_kernel(EncPtrs p, int n, long long blocks) {
    const long long g = (long long)blockIdx.x * ENC_THREADS + threadIdx.x;
    if (g >= blocks) return;
    const EncImg &im = p.img[image_of_block(p.img, n, g)];
    const long long b = g - im.block_first;
    const long long pb = prev_same_comp(b);
    const int last_dc = pb < 0 ? 0 : p.coef[(im.block_first + pb) * 64];
    int16_t c[64];
    load_coef(p.coef + g * 64, c);
    WriteBits wr(p.bits + im.bits_offset, p.off[g]);
    const int k = (int)(b % 6);
    huff_block(c, last_dc, k < 4 ? 0 : k - 3, p.hdr->ehufco, p.hdr->ehufsi, wr);
    wr.flush();
}

__device__ inline uint8_t stream_byte(const uint32_t *words, long long i) {
    return (uint8_t)(words[i >> 2] >> (24 - 8 * (int)(i & 3)));
}

// grid (max_chunks, n)
__global__ void __launch_bounds__(CHUNK_THREADS) enc_ffcount_kernel(EncPtrs p) {
    const EncImg &im = p.img[blockIdx.y];
    if ((int)blockIdx.x >= im.max_chunks) return;
    const long long nbytes = p.nbytes[blockIdx.y];
    const long long c0 = (long long)blockIdx.x * CHUNK_BYTES;
    int cnt = 0;
    if (c0 < nbytes) {
        const uint32_t *words = p.bits + im.bits_offset;
        const long long b0 = c0 + threadIdx.x * 16;
        for (int i = 0; i < 16; ++i)
            if (b0 + i < nbytes && stream_byte(words, b0 + i) == 0xFF) ++cnt;
    }
    __shared__ int s;
    if (threadIdx.x == 0) s = 0;
    __syncthreads();
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(&s, cnt);
    __syncthreads();
    if (threadIdx.x == 0) p.chunk[im.chunk_first + blockIdx.x] = (uint32_t)s;
}

// CTA per image: exclusive scan of the chunk counts in place; the image's file length
__global__ void __launch_bounds__(SCAN_THREADS) enc_ffscan_kernel(EncPtrs p) {
    __shared__ unsigned long long warp_sums[32];
    const EncImg &im = p.img[blockIdx.x];
    unsigned long long carry = 0;
    for (int t0 = 0; t0 < im.max_chunks; t0 += SCAN_THREADS) {
        const int c = t0 + threadIdx.x;
        const unsigned long long v = c < im.max_chunks ? p.chunk[im.chunk_first + c] : 0;
        unsigned long long total;
        const unsigned long long ex = block_scan_u64(v, warp_sums, total);
        if (c < im.max_chunks) p.chunk[im.chunk_first + c] = (uint32_t)(carry + ex);
        carry += total;
    }
    if (threadIdx.x == 0) p.lengths[blockIdx.x] = im.header_len + p.nbytes[blockIdx.x] + (long long)carry + 2;
}

// grid (max_chunks + 1, n): chunk c < max_chunks writes its stuffed bytes, the last x writes the headers and EOI
__global__ void __launch_bounds__(CHUNK_THREADS) enc_pack_kernel(EncPtrs p, int n) {
    __shared__ long long s_off;
    __shared__ long long s_part[CHUNK_THREADS / 32];
    const int i = blockIdx.y;
    const EncImg &im = p.img[i];
    const int c = blockIdx.x;
    const bool tail = c == (int)gridDim.x - 1;
    if (!tail && c >= im.max_chunks) return;
    const long long nbytes = p.nbytes[i];
    const long long c0 = (long long)c * CHUNK_BYTES;
    if (!tail && c0 >= nbytes) return;
    long long part = 0;   // where image i starts in the output: the lengths of the images before it
    for (int j = threadIdx.x; j < i; j += CHUNK_THREADS) part += p.lengths[j];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = part;
    __syncthreads();
    if (threadIdx.x == 0) {
        long long t = 0;
        for (int w = 0; w < CHUNK_THREADS / 32; ++w) t += s_part[w];
        s_off = t;
    }
    __syncthreads();
    uint8_t *out = p.dst + s_off;
    if (tail) {
        const uint8_t *hdr = p.blob + im.header_off;
        for (int k = threadIdx.x; k < im.header_len; k += CHUNK_THREADS) out[k] = hdr[k];
        if (threadIdx.x == 0) {
            const long long end = p.lengths[i];
            out[end - 2] = 0xFF;
            out[end - 1] = 0xD9;
        }
        return;
    }
    const uint32_t *words = p.bits + im.bits_offset;
    const long long b0 = c0 + threadIdx.x * 16;
    uint8_t v[16];
    int ff = 0;
#pragma unroll
    for (int k = 0; k < 16; ++k) {
        v[k] = b0 + k < nbytes ? stream_byte(words, b0 + k) : 0;
        ff += (b0 + k < nbytes && v[k] == 0xFF);
    }
    // exclusive scan of the 0xFF counts across the CTA
    __shared__ int s_warp[CHUNK_THREADS / 32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int x = ff;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) s_warp[wid] = x;
    __syncthreads();
    int before = x - ff;
    for (int w = 0; w < wid; ++w) before += s_warp[w];
    long long o = im.header_len + b0 + p.chunk[im.chunk_first + c] + before;
    for (int k = 0; k < 16 && b0 + k < nbytes; ++k) {
        out[o++] = v[k];
        if (v[k] == 0xFF) out[o++] = 0;
    }
}

}  // namespace
}  // namespace k2y

using namespace k2y;

extern "C" int k2y_jpeg_encode_plan(int n, const int *hw_host, const long long *src_offsets_host, int quality, void *blob,
                                    size_t blob_capacity, size_t *blob_bytes) {
    if (n <= 0 || !hw_host || !src_offsets_host || !blob_bytes) {
        set_error("k2y_jpeg_encode_plan: bad arguments");
        return K2Y_ERR_INVALID;
    }
    if (quality < 1 || quality > 100) {
        set_error("k2y_jpeg_encode_plan: quality %d is outside 1..100", quality);
        return K2Y_ERR_INVALID;
    }
    for (int i = 0; i < n; ++i) {
        const int h = hw_host[2 * i], w = hw_host[2 * i + 1];
        if (h < 1 || h > JPEG_MAX_DIMENSION || w < 1 || w > JPEG_MAX_DIMENSION) {
            set_error("k2y_jpeg_encode_plan: image %d is %dx%d; JPEG files have 1..%d rows and columns (libjpeg's limit)", i, h, w, JPEG_MAX_DIMENSION);
            return K2Y_ERR_INVALID;
        }
        if (src_offsets_host[i] < 0) {
            set_error("k2y_jpeg_encode_plan: image %d has a negative source offset", i);
            return K2Y_ERR_INVALID;
        }
    }
    uint16_t qt[2][64];
    quant_table(quality, 0, qt[0]);
    quant_table(quality, 1, qt[1]);
    const long long img_off = (long long)sizeof(EncBlobHeader);
    long long pos = img_off + (long long)n * sizeof(EncImg);
    std::vector<std::vector<uint8_t>> headers(n);
    std::vector<long long> header_at(n);
    for (int i = 0; i < n; ++i) {
        headers[i] = build_header(hw_host[2 * i], hw_host[2 * i + 1], qt);
        header_at[i] = pos;
        pos += (long long)headers[i].size();
    }
    const long long total = (pos + 15) & ~15LL;
    *blob_bytes = (size_t)total;
    if (!blob) return K2Y_OK;
    if (blob_capacity < (size_t)total || ((uintptr_t)blob & 15)) {
        set_error("k2y_jpeg_encode_plan: the blob needs %lld bytes, 16-byte aligned", total);
        return K2Y_ERR_INVALID;
    }
    uint8_t *base = (uint8_t *)blob;
    memset(base, 0, (size_t)total);
    EncBlobHeader &hd = *(EncBlobHeader *)base;
    EncImg *img = (EncImg *)(base + img_off);
    hd.magic = ENC_BLOB_MAGIC;
    hd.n = n;
    hd.img_off = img_off;
    hd.blob_bytes = total;
    for (int t = 0; t < 4; ++t) derive_codes(t, hd.ehufco[t], hd.ehufsi[t]);
    uint16_t recip[2][64], corr[2][64];
    uint8_t shift[2][64];
    for (int t = 0; t < 2; ++t)
        for (int k = 0; k < 64; ++k) compute_reciprocal((uint16_t)(qt[t][k] << 3), recip[t][k], corr[t][k], shift[t][k]);
    long long blocks = 0, words = 0, chunks = 0, out = 0, max_blocks = 0;
    for (int i = 0; i < n; ++i) {
        EncImg &m = img[i];
        m.h = hw_host[2 * i];
        m.w = hw_host[2 * i + 1];
        m.mcux = (m.w + 15) / 16;
        m.mcuy = (m.h + 15) / 16;
        m.ywb = (m.w + 7) / 8;
        m.yhb = (m.h + 7) / 8;
        m.src_offset = src_offsets_host[i];
        m.header_off = (int32_t)header_at[i];
        m.header_len = (int32_t)headers[i].size();
        memcpy(base + header_at[i], headers[i].data(), headers[i].size());
        memcpy(m.recip, recip, sizeof(recip));
        memcpy(m.corr, corr, sizeof(corr));
        memcpy(m.shift, shift, sizeof(shift));
        const long long nb = (long long)m.mcux * m.mcuy * 6;
        const long long max_bytes = (nb * MAX_BLOCK_BITS + 7) / 8;
        m.block_first = blocks;
        m.bits_offset = words;
        m.chunk_first = chunks;
        m.max_chunks = (int32_t)((max_bytes + CHUNK_BYTES - 1) / CHUNK_BYTES);
        blocks += nb;
        words += (max_bytes + 3) / 4 + 1;
        chunks += m.max_chunks;
        out += m.header_len + 2 * max_bytes + 2;
        max_blocks = std::max(max_blocks, nb);
    }
    hd.blocks = blocks;
    hd.chunks = chunks;
    hd.max_image_blocks = max_blocks;
    hd.out_capacity = out;
    long long ws = 0;
    auto take = [&ws](long long bytes) {
        const long long at = ws;
        ws += (bytes + 255) & ~255LL;
        return at;
    };
    hd.ws_coef = take(blocks * 64 * 2);
    hd.ws_len = take(blocks * 4);
    hd.ws_off = take(blocks * 8);
    hd.ws_bits = take(words * 4);
    hd.ws_chunk = take(chunks * 4);
    hd.ws_nbytes = take((long long)n * 8);
    hd.ws_total = ws;
    return K2Y_OK;
}

extern "C" int k2y_jpeg_encode_header(int h, int w, int quality, unsigned char *out, size_t capacity, size_t *length) {
    if (h < 1 || h > JPEG_MAX_DIMENSION || w < 1 || w > JPEG_MAX_DIMENSION || quality < 1 || quality > 100 || !length) {
        set_error("k2y_jpeg_encode_header: %dx%d at quality %d (1..%d rows and columns, quality 1..100)", h, w, quality,
                  JPEG_MAX_DIMENSION);
        return K2Y_ERR_INVALID;
    }
    uint16_t qt[2][64];
    quant_table(quality, 0, qt[0]);
    quant_table(quality, 1, qt[1]);
    const std::vector<uint8_t> v = build_header(h, w, qt);
    *length = v.size();
    if (out) {
        if (capacity < v.size()) {
            set_error("k2y_jpeg_encode_header: %zu bytes needed", v.size());
            return K2Y_ERR_INVALID;
        }
        memcpy(out, v.data(), v.size());
    }
    return K2Y_OK;
}

static const EncBlobHeader *enc_header(const void *blob_host) {
    const EncBlobHeader *h = (const EncBlobHeader *)blob_host;
    if (!h || h->magic != ENC_BLOB_MAGIC) {
        set_error("not a k2y_jpeg_encode_plan blob");
        return nullptr;
    }
    return h;
}

static long long enc_workspace(const EncBlobHeader *h) { return h->ws_total; }

extern "C" int k2y_jpeg_encode_workspace_bytes(const void *blob_host, size_t *workspace_bytes, size_t *output_capacity) {
    const EncBlobHeader *h = enc_header(blob_host);
    if (!h) return K2Y_ERR_INVALID;
    if (workspace_bytes) *workspace_bytes = (size_t)enc_workspace(h);
    if (output_capacity) *output_capacity = (size_t)h->out_capacity;
    return K2Y_OK;
}

extern "C" int k2y_jpeg_encode(const void *blob_host, const void *blob_dev, const unsigned char *src_dev, unsigned char *dst_dev,
                               long long *lengths_dev, void *workspace_dev, size_t workspace_bytes, void *stream) {
    const EncBlobHeader *h = enc_header(blob_host);
    if (!h) return K2Y_ERR_INVALID;
    if (!blob_dev || !src_dev || !dst_dev || !lengths_dev || !workspace_dev || ((uintptr_t)blob_dev & 15) ||
        ((uintptr_t)workspace_dev & 15)) {
        set_error("k2y_jpeg_encode: bad arguments");
        return K2Y_ERR_INVALID;
    }
    if ((long long)workspace_bytes < enc_workspace(h)) {
        set_error("k2y_jpeg_encode: workspace of %zu bytes, %lld needed", workspace_bytes, enc_workspace(h));
        return K2Y_ERR_INVALID;
    }
    const EncImg *img_host = (const EncImg *)((const uint8_t *)blob_host + h->img_off);
    int max_chunks = 0;
    for (int i = 0; i < h->n; ++i) max_chunks = std::max(max_chunks, (int)img_host[i].max_chunks);
    uint8_t *ws = (uint8_t *)workspace_dev;
    EncPtrs p;
    p.hdr = (const EncBlobHeader *)blob_dev;
    p.img = (const EncImg *)((const uint8_t *)blob_dev + h->img_off);
    p.blob = (const uint8_t *)blob_dev;
    p.src = src_dev;
    p.dst = dst_dev;
    p.lengths = lengths_dev;
    p.coef = (int16_t *)(ws + h->ws_coef);
    p.len = (uint32_t *)(ws + h->ws_len);
    p.off = (unsigned long long *)(ws + h->ws_off);
    p.bits = (uint32_t *)(ws + h->ws_bits);
    p.chunk = (uint32_t *)(ws + h->ws_chunk);
    p.nbytes = (long long *)(ws + h->ws_nbytes);
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned grid = (unsigned)((h->blocks + ENC_THREADS - 1) / ENC_THREADS);
    enc_dct_kernel<<<grid, ENC_THREADS, 0, st>>>(p, h->n, h->blocks);
    enc_len_kernel<<<grid, ENC_THREADS, 0, st>>>(p, h->n, h->blocks);
    enc_scan_kernel<<<h->n, SCAN_THREADS, 0, st>>>(p);
    enc_emit_kernel<<<grid, ENC_THREADS, 0, st>>>(p, h->n, h->blocks);
    enc_ffcount_kernel<<<dim3(max_chunks, h->n), CHUNK_THREADS, 0, st>>>(p);
    enc_ffscan_kernel<<<h->n, SCAN_THREADS, 0, st>>>(p);
    enc_pack_kernel<<<dim3(max_chunks + 1, h->n), CHUNK_THREADS, 0, st>>>(p, h->n);
    K2Y_CUDA_CHECK(cudaGetLastError());
    return K2Y_OK;
}
