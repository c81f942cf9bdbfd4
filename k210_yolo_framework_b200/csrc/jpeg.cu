// Baseline JPEG decoding on the GPU, bit-exact with libjpeg-turbo as PIL runs it on x86-64 (the reference reads every image
// with skimage.io.imread, tools/utils.py:339-355, i.e. PIL / libjpeg-turbo underneath): the x86 SIMD JDCT_ISLOW integer IDCT,
// fancy upsampling, ycc_rgb_convert.  The pixels land in the packed uint8 HWC buffer k2y_letterbox_u8_batch reads.
//
// Host side: a marker walker classifies each file (GPU-decodable, valid but not for the GPU, malformed) and builds one
// descriptor blob per batch (JpegBlobHeader, JpegImg[n], JpegSeg[segments], JpegHuff[2 * components per image]).  The caller
// puts the blob next to the compressed bytes in pinned memory, so one H2D copy moves both.
//
// Device side, one launch per stage whatever the image count:
//   1. jpeg_unstuff_kernel   (CTA per image)   drops the 0x00 after each 0xFF, cuts the entropy data at RSTn markers
//   2. jpeg_huffman_kernel   (CTA per segment) self-synchronising Huffman decode (Weissenberger & Schmidt): each thread owns
//                            a fixed-length subsequence of the segment's bits, decodes it from a guessed state, then restarts
//                            from its left neighbour's exact end state until its own end state stops changing; an exclusive
//                            scan of completed blocks gives each thread its first block, and a last pass writes int16
//                            coefficients in natural order (DC as differences)
//   3. jpeg_dc_kernel        (CTA per segment) per-component scan of the DC differences in decode order
//   4. jpeg_idct_kernel      dequantise + libjpeg-turbo's x86 SIMD islow (jidctint-avx2.asm / -sse2.asm, 16-bit lanes)
//                            -> uint8 component planes at the MCU-padded size
//   5. jpeg_color_kernel     libjpeg-turbo's upsampler dispatch (fancy on) + ycc_rgb_convert, cropped, HWC RGB out
#include "common.h"

#include <algorithm>
#include <cstdarg>
#include <vector>

namespace k2y {
namespace {

constexpr uint32_t JPEG_BLOB_MAGIC = 0x4a504731u;   // "JPG1"
constexpr int HUFF_LOOKAHEAD = 9;
constexpr int MAX_BLOCKS_PER_MCU = 6;                // luma 4x1 or 2x2 + two 1x1 chroma

constexpr int SYNC_THREADS = 256;                    // subsequences per window of one segment
constexpr int SUBSEQ_BITS = 512;                     // bits per subsequence
constexpr int UNSTUFF_THREADS = 512;
constexpr int UNSTUFF_BYTES = 16;                    // source bytes per thread per tile
constexpr int DC_THREADS = 256;
constexpr int IDCT_THREADS = 128;
constexpr int COLOR_THREADS = 256;

enum Upsample : int { UP_FULL = 0, UP_H2V1_FANCY, UP_H2V1_BOX, UP_H1V2_FANCY, UP_H2V2_FANCY, UP_H2V2_BOX, UP_H4V1_BOX, UP_GRAY };

// Huffman decode table, lookup form: codes of up to HUFF_LOOKAHEAD bits through `lut` ((length << 8) | symbol, 0 = longer);
// longer ones through libjpeg's maxcode / valoffset arrays.
struct alignas(16) JpegHuff {
    uint16_t lut[1 << HUFF_LOOKAHEAD];
    int32_t maxcode[18];
    int32_t valoffset[18];
    uint8_t huffval[256];
};

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

__host__ __device__ inline long long align16(long long v) { return (v + 15) & ~15LL; }

const uint8_t kNatural[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                              41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                              30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
__constant__ uint8_t c_natural[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                      41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                      30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// ---------------------------------------------------------------------------------------------------------------------
// Host: marker walker
// ---------------------------------------------------------------------------------------------------------------------
struct HuffSpec {
    bool defined = false;
    uint8_t bits[17] = {};
    uint8_t vals[256] = {};
};

struct Parsed {
    int sof = -1, precision = 0, h = 0, w = 0, ncomp = 0;
    int id[4] = {}, hs[4] = {}, vs[4] = {}, tq[4] = {};
    uint16_t qt[4][64] = {};
    bool qt_defined[4] = {};
    HuffSpec dc[4], ac[4];
    int restart = 0;
    bool jfif = false, adobe = false;
    int adobe_transform = -1;
    int ns = 0, scan_comp[4] = {}, td[4] = {}, ta[4] = {}, ss = 0, se = 0, ah = 0, al = 0;
    uint16_t scan_qt[4][64] = {};   // quant tables as latched at the scan
    long long entropy = -1;
    bool gpu = false;
    char reason[64] = {};
};

void set_reason(Parsed &p, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(p.reason, sizeof(p.reason), fmt, ap);
    va_end(ap);
}

bool derive_huff(const HuffSpec &hs, JpegHuff &t);

// Files the decoder's 32-bit bit positions and plane offsets cover; larger (valid) files are left to the host.
constexpr long long JPEG_MAX_FILE_BYTES = 1LL << 28;
constexpr long long JPEG_MAX_PLANE_BYTES = 1LL << 30;

// Returns K2Y_OK (p filled up to the first SOS; p.gpu / p.reason classify it) or K2Y_ERR_INVALID with the marker in the error.
int parse_jpeg(const uint8_t *d, size_t n, Parsed &p, const char *who) {
    if (n < 4 || d[0] != 0xFF || d[1] != 0xD8) {
        set_error("%s: not a JPEG file (no SOI marker)", who);
        return K2Y_ERR_INVALID;
    }
    size_t i = 2;
    bool saw_sof = false;
    for (;;) {
        while (i < n && d[i] != 0xFF) ++i;   // libjpeg skips extraneous bytes before a marker
        while (i < n && d[i] == 0xFF) ++i;   // fill bytes
        if (i >= n) {
            set_error("%s: truncated before SOS (offset %zu)", who, i);
            return K2Y_ERR_INVALID;
        }
        const int m = d[i++];
        const size_t at = i - 2;
        if (m == 0xD8) {
            set_error("%s: second SOI marker at offset %zu", who, at);
            return K2Y_ERR_INVALID;
        }
        if (m == 0xD9) {
            set_error("%s: EOI marker at offset %zu before any SOS", who, at);
            return K2Y_ERR_INVALID;
        }
        if ((m >= 0xD0 && m <= 0xD7) || m == 0x01) continue;   // parameterless markers outside a scan (libjpeg ignores them)
        if (i + 2 > n) {
            set_error("%s: truncated length of marker 0x%02X at offset %zu", who, m, at);
            return K2Y_ERR_INVALID;
        }
        const size_t len = ((size_t)d[i] << 8) | d[i + 1];
        if (len < 2 || i + len > n) {
            set_error("%s: marker 0x%02X at offset %zu has length %zu, %zu bytes left", who, m, at, len, n - i);
            return K2Y_ERR_INVALID;
        }
        const uint8_t *s = d + i + 2;
        const size_t sl = len - 2;
        const size_t next = i + len;
        if (m >= 0xE0 && m <= 0xEF) {
            if (m == 0xE0 && sl >= 14 && memcmp(s, "JFIF\0", 5) == 0) p.jfif = true;
            if (m == 0xEE && sl >= 12 && memcmp(s, "Adobe", 5) == 0) {
                p.adobe = true;
                p.adobe_transform = s[11];
            }
        } else if (m == 0xFE || m == 0xCC) {
            // COM; DAC (arithmetic conditioning, the SOF already says arithmetic)
        } else if (m == 0xDB) {
            size_t k = 0;
            while (k < sl) {
                const int pq = s[k] >> 4, tq = s[k] & 15;
                const size_t need = 1 + 64 * (pq ? 2 : 1);
                if (pq > 1 || tq > 3 || k + need > sl) {
                    set_error("%s: bad DQT marker at offset %zu (precision %d, table %d)", who, at, pq, tq);
                    return K2Y_ERR_INVALID;
                }
                for (int z = 0; z < 64; ++z)
                    p.qt[tq][kNatural[z]] = pq ? (uint16_t)((s[k + 1 + 2 * z] << 8) | s[k + 2 + 2 * z]) : s[k + 1 + z];
                p.qt_defined[tq] = true;
                k += need;
            }
        } else if (m == 0xC4) {
            size_t k = 0;
            while (k < sl) {
                if (k + 17 > sl) {
                    set_error("%s: truncated DHT marker at offset %zu", who, at);
                    return K2Y_ERR_INVALID;
                }
                const int tc = s[k] >> 4, th = s[k] & 15;
                int count = 0;
                for (int l = 1; l <= 16; ++l) count += s[k + l];
                if (tc > 1 || th > 3 || count > 256 || k + 17 + count > sl) {
                    set_error("%s: bad DHT marker at offset %zu (class %d, table %d, %d symbols)", who, at, tc, th, count);
                    return K2Y_ERR_INVALID;
                }
                HuffSpec &hs = tc ? p.ac[th] : p.dc[th];
                hs.defined = true;
                hs.bits[0] = 0;
                for (int l = 1; l <= 16; ++l) hs.bits[l] = s[k + l];
                memset(hs.vals, 0, sizeof(hs.vals));
                memcpy(hs.vals, s + k + 17, count);
                k += 17 + count;
            }
        } else if (m == 0xDD) {
            if (sl < 2) {
                set_error("%s: bad DRI marker at offset %zu", who, at);
                return K2Y_ERR_INVALID;
            }
            p.restart = (s[0] << 8) | s[1];
        } else if (m >= 0xC0 && m <= 0xCF && m != 0xC4 && m != 0xC8 && m != 0xCC) {
            if (saw_sof) {
                set_error("%s: second SOF marker 0x%02X at offset %zu", who, m, at);
                return K2Y_ERR_INVALID;
            }
            saw_sof = true;
            if (sl < 6) {
                set_error("%s: truncated SOF marker 0x%02X at offset %zu", who, m, at);
                return K2Y_ERR_INVALID;
            }
            p.sof = m;
            p.precision = s[0];
            p.h = (s[1] << 8) | s[2];
            p.w = (s[3] << 8) | s[4];
            p.ncomp = s[5];
            if (p.ncomp < 1 || p.ncomp > 4 || sl < 6 + 3 * (size_t)p.ncomp || p.w == 0) {
                set_error("%s: bad SOF marker 0x%02X at offset %zu (%d components, width %d)", who, m, at, p.ncomp, p.w);
                return K2Y_ERR_INVALID;
            }
            for (int c = 0; c < p.ncomp; ++c) {
                p.id[c] = s[6 + 3 * c];
                p.hs[c] = s[7 + 3 * c] >> 4;
                p.vs[c] = s[7 + 3 * c] & 15;
                p.tq[c] = s[8 + 3 * c];
                if (p.hs[c] < 1 || p.hs[c] > 4 || p.vs[c] < 1 || p.vs[c] > 4 || p.tq[c] > 3) {
                    set_error("%s: bad SOF marker 0x%02X at offset %zu (component %d sampling %dx%d, table %d)", who, m, at, c,
                              p.hs[c], p.vs[c], p.tq[c]);
                    return K2Y_ERR_INVALID;
                }
            }
            // anything but 8-bit sequential Huffman is valid JPEG the GPU path does not take: stop at the frame header
            const char *kind = nullptr;
            if (m == 0xC2 || m == 0xC6) kind = "progressive";
            else if (m == 0xC3 || m == 0xC7) kind = "lossless";
            else if (m == 0xC5) kind = "hierarchical";
            else if (m >= 0xC9) kind = "arithmetic coding";
            if (kind) {
                set_reason(p, "%s (SOF 0x%02X)", kind, m);
                return K2Y_OK;
            }
            if (p.precision != 8) {
                set_reason(p, "%d-bit samples", p.precision);
                return K2Y_OK;
            }
            if (p.h == 0) {
                set_reason(p, "height from a DNL marker");
                return K2Y_OK;
            }
        } else if (m == 0xDA) {
            if (!saw_sof) {
                set_error("%s: SOS marker at offset %zu before any SOF", who, at);
                return K2Y_ERR_INVALID;
            }
            p.ns = sl >= 1 ? s[0] : 0;
            if (p.ns < 1 || p.ns > 4 || sl != 4 + 2 * (size_t)p.ns) {
                set_error("%s: bad SOS marker at offset %zu (%d components, length %zu)", who, at, p.ns, len);
                return K2Y_ERR_INVALID;
            }
            for (int k = 0; k < p.ns; ++k) {
                const int cid = s[1 + 2 * k];
                int f = -1;
                for (int c = 0; c < p.ncomp; ++c)
                    if (p.id[c] == cid) f = c;
                if (f < 0) {
                    set_error("%s: SOS marker at offset %zu names component id %d the frame does not have", who, at, cid);
                    return K2Y_ERR_INVALID;
                }
                // T.81 B.2.3: a scan lists its components in frame order; libjpeg-turbo refuses the file otherwise
                if (k > 0 && f <= p.scan_comp[k - 1]) {
                    set_error("%s: SOS marker at offset %zu lists component id %d out of frame order", who, at, cid);
                    return K2Y_ERR_INVALID;
                }
                p.scan_comp[k] = f;
                p.td[k] = s[2 + 2 * k] >> 4;
                p.ta[k] = s[2 + 2 * k] & 15;
                if (p.td[k] > 3 || p.ta[k] > 3) {
                    set_error("%s: SOS marker at offset %zu selects Huffman table %d/%d", who, at, p.td[k], p.ta[k]);
                    return K2Y_ERR_INVALID;
                }
            }
            p.ss = s[1 + 2 * p.ns];
            p.se = s[2 + 2 * p.ns];
            p.ah = s[3 + 2 * p.ns] >> 4;
            p.al = s[3 + 2 * p.ns] & 15;
            for (int c = 0; c < p.ncomp; ++c) {
                if (!p.qt_defined[p.tq[c]]) {
                    set_error("%s: quantisation table %d of component %d is not defined at the SOS marker (offset %zu)", who,
                              p.tq[c], c, at);
                    return K2Y_ERR_INVALID;
                }
                memcpy(p.scan_qt[c], p.qt[p.tq[c]], sizeof(p.scan_qt[c]));
            }
            p.entropy = (long long)next;
            break;
        } else {
            set_error("%s: unsupported marker 0x%02X at offset %zu", who, m, at);
            return K2Y_ERR_INVALID;
        }
        i = next;
    }
    // classification of an 8-bit sequential Huffman file
    // jdinput.c initial_setup: libjpeg-turbo refuses a larger frame at the first SOS, so PIL cannot read the file
    if (p.h > JPEG_MAX_DIMENSION || p.w > JPEG_MAX_DIMENSION)
        return set_reason(p, "%dx%d exceeds libjpeg's %d-pixel limit", p.w, p.h, JPEG_MAX_DIMENSION), K2Y_OK;
    if (p.ncomp == 2) return set_reason(p, "2 components"), K2Y_OK;
    if (p.ncomp == 4) return set_reason(p, "4 components (CMYK/YCCK)"), K2Y_OK;
    if (p.ncomp == 3 && !p.jfif) {   // libjpeg's default_decompress_parms
        if (p.adobe && p.adobe_transform == 0) return set_reason(p, "RGB colour space (Adobe transform 0)"), K2Y_OK;
        if (!p.adobe && p.id[0] == 'R' && p.id[1] == 'G' && p.id[2] == 'B') return set_reason(p, "RGB colour space (component ids R, G, B)"), K2Y_OK;
    }
    if (p.ns != p.ncomp) return set_reason(p, "multi-scan sequential"), K2Y_OK;
    if (p.ss != 0 || p.se != 63 || p.ah != 0 || p.al != 0) return set_reason(p, "scan parameters Ss=%d Se=%d Ah=%d Al=%d", p.ss, p.se, p.ah, p.al), K2Y_OK;
    if (p.ncomp == 3) {
        const int h0 = p.hs[0], v0 = p.vs[0];
        const bool chroma11 = p.hs[1] == 1 && p.vs[1] == 1 && p.hs[2] == 1 && p.vs[2] == 1;
        const bool luma_ok = (h0 == 1 && v0 == 1) || (h0 == 2 && v0 == 1) || (h0 == 1 && v0 == 2) || (h0 == 2 && v0 == 2) || (h0 == 4 && v0 == 1);
        if (!chroma11 || !luma_ok)
            return set_reason(p, "sampling %dx%d,%dx%d,%dx%d", p.hs[0], p.vs[0], p.hs[1], p.vs[1], p.hs[2], p.vs[2]), K2Y_OK;
    }
    for (int k = 0; k < p.ns; ++k) {
        if (!p.dc[p.td[k]].defined || !p.ac[p.ta[k]].defined)
            return set_reason(p, "Huffman table not defined before the scan"), K2Y_OK;
        for (int v = 0; v < 256; ++v) {   // jpeg_make_d_derived_tbl: DC symbols above 15 are an error
            int count = 0;
            for (int l = 1; l <= 16; ++l) count += p.dc[p.td[k]].bits[l];
            if (v < count && p.dc[p.td[k]].vals[v] > 15) {
                set_error("%s: DHT DC table %d has symbol %d", who, p.td[k], p.dc[p.td[k]].vals[v]);
                return K2Y_ERR_INVALID;
            }
        }
        // jpeg_make_d_derived_tbl: code lengths that overflow their bit count are an error (libjpeg refuses the file)
        JpegHuff t;
        if (!derive_huff(p.dc[p.td[k]], t) || !derive_huff(p.ac[p.ta[k]], t)) {
            set_error("%s: DHT table %d/%d of the SOS marker has more codes than its code lengths allow", who, p.td[k], p.ta[k]);
            return K2Y_ERR_INVALID;
        }
    }
    {
        int hmax = 1, vmax = 1;
        for (int c = 0; c < p.ncomp; ++c) {
            hmax = std::max(hmax, p.ncomp == 1 ? 1 : p.hs[c]);
            vmax = std::max(vmax, p.ncomp == 1 ? 1 : p.vs[c]);
        }
        const long long luma = (long long)((p.w + 8 * hmax - 1) / (8 * hmax)) * 8 * hmax * ((p.h + 8 * vmax - 1) / (8 * vmax)) * 8 * vmax;
        if ((long long)n > JPEG_MAX_FILE_BYTES || 3 * luma > JPEG_MAX_PLANE_BYTES)
            return set_reason(p, "too large for the GPU decoder (%zu bytes, %dx%d)", n, p.w, p.h), K2Y_OK;
    }
    p.gpu = true;
    return K2Y_OK;
}

// jpeg_make_d_derived_tbl
bool derive_huff(const HuffSpec &hs, JpegHuff &t) {
    memset(&t, 0, sizeof(t));
    int huffsize[257], huffcode[257];
    int p = 0;
    for (int l = 1; l <= 16; ++l)
        for (int i = 0; i < hs.bits[l]; ++i) huffsize[p++] = l;
    huffsize[p] = 0;
    const int numsymbols = p;
    int code = 0, si = huffsize[0];
    p = 0;
    while (huffsize[p]) {
        while (huffsize[p] == si) huffcode[p++] = code++;
        if (code >= (1 << si)) return false;
        code <<= 1;
        ++si;
    }
    p = 0;
    for (int l = 1; l <= 16; ++l) {
        if (hs.bits[l]) {
            t.valoffset[l] = p - huffcode[p];
            p += hs.bits[l];
            t.maxcode[l] = huffcode[p - 1];
        } else {
            t.maxcode[l] = -1;
        }
    }
    t.maxcode[17] = 0x7fffffff;
    memcpy(t.huffval, hs.vals, 256);
    p = 0;
    for (int l = 1; l <= HUFF_LOOKAHEAD; ++l) {
        for (int i = 0; i < hs.bits[l]; ++i, ++p) {
            int look = huffcode[p] << (HUFF_LOOKAHEAD - l);
            for (int c = 0; c < (1 << (HUFF_LOOKAHEAD - l)); ++c) t.lut[look++] = (uint16_t)((l << 8) | hs.vals[p]);
        }
    }
    (void)numsymbols;
    return true;
}

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

// One Huffman symbol; sets `bad` (and returns 0 after 16 bits, as libjpeg does) on a code no table entry matches.
__device__ __forceinline__ int huff_decode(BitReader &br, const JpegHuff &t, int &used, bool &bad) {
    const unsigned look = (unsigned)(br.buf >> 48);
    const unsigned e = t.lut[look >> (16 - HUFF_LOOKAHEAD)];
    if (e) {
        const int l = e >> 8;
        br.buf <<= l;
        br.nb -= l;
        used = l;
        return e & 255;
    }
    for (int l = HUFF_LOOKAHEAD + 1; l <= 16; ++l) {
        const int code = (int)(look >> (16 - l));
        if (code <= t.maxcode[l]) {
            br.buf <<= l;
            br.nb -= l;
            used = l;
            return t.huffval[(code + t.valoffset[l]) & 255];
        }
    }
    bad = true;
    br.buf <<= 16;
    br.nb -= 16;
    used = 16;
    return 0;
}

__device__ __forceinline__ int huff_extend(unsigned x, int s) {
    return (int)x < (1 << (s - 1)) ? (int)x + (int)(~0u << s) + 1 : (int)x;
}

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
                                                                       uint8_t *__restrict__ ws) {
    __shared__ int sh[32];
    __shared__ int s_term;
    const JpegImg &im = imgs(blob)[blockIdx.x];
    const uint8_t *s = src + im.src_offset;
    const long long n = im.src_end - im.src_offset;
    uint8_t *u = ws + hdr(blob).ws_unstuff + im.unstuff_offset;
    int *seg = reinterpret_cast<int *>(ws + hdr(blob).ws_seg + im.seg_offset);
    const int nseg = im.nseg;
    long long term = n;
    int out_total = 0, rst_total = 0;
    const int tile = UNSTUFF_THREADS * UNSTUFF_BYTES;
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
                    if (r < nseg) seg[r] = o;
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
        seg[nseg] = out_total;
    }
}

// status words per image: [0] error bits (1 bad Huffman code, 2 premature end of data), [1] max sync rounds of a window,
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

// libjpeg-turbo's x86 SIMD islow (jidctint-avx2.asm, jidctint-sse2.asm), the IDCT PIL runs on x86-64.  Same 13-bit
// constants and 2 pass bits as jidctint.c, but on 16-bit lanes: the dequantised product keeps its low 16 bits (pmullw); the
// sums feeding a multiply (in0 +- in4, in7 + in3, in5 + in1) wrap to 16 bits (paddw); products and the other sums are 32-bit
// (pmaddwd; they stay below 2^31 for 16-bit inputs); pass 1 saturates its results to int16 (packssdw), pass 2 to int16 and
// then int8 before adding 128 (packssdw, packsswb).  When rows 1-7 of the whole block are zero, pass 1 is row 0 shifted left
// by 2 in 16 bits (psllw, wrapping).  On the coefficients an 8-bit encoder writes this equals jidctint.c; outside them it
// does not, and jidctint.c's masked range-limit table gives other pixels.
#define FIX_0_298631336 2446
#define FIX_0_390180644 3196
#define FIX_0_541196100 4433
#define FIX_0_765366865 6270
#define FIX_0_899976223 7373
#define FIX_1_175875602 9633
#define FIX_1_501321110 12299
#define FIX_1_847759065 15137
#define FIX_1_961570560 16069
#define FIX_2_053119869 16819
#define FIX_2_562915447 20995
#define FIX_3_072711026 25172

__device__ __forceinline__ int wrap16(int x) { return (int)(int16_t)x; }

// One 1-D pass on int16 inputs: pass 1 -> int16 (saturated), pass 2 -> the sample value (saturated to [-128, 127], + 128).
template <int PASS>
__device__ __forceinline__ void idct_1d(int i0, int i1, int i2, int i3, int i4, int i5, int i6, int i7, int *o) {
    const int tmp3 = i2 * (FIX_0_541196100 + FIX_0_765366865) + i6 * FIX_0_541196100;
    const int tmp2 = i2 * FIX_0_541196100 + i6 * (FIX_0_541196100 - FIX_1_847759065);
    const int tmp0 = wrap16(i0 + i4) * (1 << 13);
    const int tmp1 = wrap16(i0 - i4) * (1 << 13);
    const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    const int z3 = wrap16(i7 + i3), z4 = wrap16(i5 + i1);
    const int z3p = z3 * (FIX_1_175875602 - FIX_1_961570560) + z4 * FIX_1_175875602;
    const int z4p = z3 * FIX_1_175875602 + z4 * (FIX_1_175875602 - FIX_0_390180644);
    const int o0 = i7 * (FIX_0_298631336 - FIX_0_899976223) - i1 * FIX_0_899976223 + z3p;
    const int o3 = -i7 * FIX_0_899976223 + i1 * (FIX_1_501321110 - FIX_0_899976223) + z4p;
    const int o1 = i5 * (FIX_2_053119869 - FIX_2_562915447) - i3 * FIX_2_562915447 + z4p;
    const int o2 = -i5 * FIX_2_562915447 + i3 * (FIX_3_072711026 - FIX_2_562915447) + z3p;
    constexpr int sh = PASS == 1 ? 13 - 2 : 13 + 2 + 3;
    constexpr int rnd = 1 << (sh - 1);
    constexpr int lo = PASS == 1 ? -32768 : -128, hi = PASS == 1 ? 32767 : 127, add = PASS == 1 ? 0 : 128;
    o[0] = min(max((tmp10 + o3 + rnd) >> sh, lo), hi) + add;
    o[7] = min(max((tmp10 - o3 + rnd) >> sh, lo), hi) + add;
    o[1] = min(max((tmp11 + o2 + rnd) >> sh, lo), hi) + add;
    o[6] = min(max((tmp11 - o2 + rnd) >> sh, lo), hi) + add;
    o[2] = min(max((tmp12 + o1 + rnd) >> sh, lo), hi) + add;
    o[5] = min(max((tmp12 - o1 + rnd) >> sh, lo), hi) + add;
    o[3] = min(max((tmp13 + o0 + rnd) >> sh, lo), hi) + add;
    o[4] = min(max((tmp13 - o0 + rnd) >> sh, lo), hi) + add;
}

// One thread per 8x8 block; grid (block tiles, image).
__global__ void __launch_bounds__(IDCT_THREADS) jpeg_idct_kernel(const uint8_t *__restrict__ blob, uint8_t *__restrict__ ws) {
    __shared__ int s_q[3][64];
    const JpegBlobHeader &H = hdr(blob);
    const JpegImg &im = imgs(blob)[blockIdx.y];
    for (int k = threadIdx.x; k < 3 * 64; k += blockDim.x) s_q[k / 64][k % 64] = (int16_t)im.qt[k / 64][k % 64];
    __syncthreads();
    const int b = blockIdx.x * IDCT_THREADS + threadIdx.x;
    if (b >= im.blocks) return;
    const int comp = im.ncomp == 1 ? 0 : (b < im.coef_block[1] ? 0 : (b < im.coef_block[2] ? 1 : 2));
    const int local = b - im.coef_block[comp];
    const int bx = local % im.bw[comp], by = local / im.bw[comp];
    const int4 *cp = reinterpret_cast<const int4 *>(ws + H.ws_coef + im.coef_offset) + (long long)b * 8;
    int ws_[64];
    int ac_rows = 0;   // any coefficient of rows 1-7
#pragma unroll
    for (int r = 0; r < 8; ++r) {
        const int4 q = cp[r];
        const int v[4] = {q.x, q.y, q.z, q.w};
        if (r > 0) ac_rows |= q.x | q.y | q.z | q.w;
#pragma unroll
        for (int j = 0; j < 4; ++j) {   // the low 16 bits of the product
            ws_[r * 8 + 2 * j] = wrap16((int)(int16_t)(v[j] & 0xffff) * s_q[comp][r * 8 + 2 * j]);
            ws_[r * 8 + 2 * j + 1] = wrap16((int)(int16_t)((unsigned)v[j] >> 16) * s_q[comp][r * 8 + 2 * j + 1]);
        }
    }
    // pass 1: columns
    if (ac_rows == 0) {
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const int dc = wrap16(ws_[c] * 4);
#pragma unroll
            for (int r = 0; r < 8; ++r) ws_[r * 8 + c] = dc;
        }
    } else {
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            int o[8];
            idct_1d<1>(ws_[c], ws_[8 + c], ws_[16 + c], ws_[24 + c], ws_[32 + c], ws_[40 + c], ws_[48 + c], ws_[56 + c], o);
#pragma unroll
            for (int r = 0; r < 8; ++r) ws_[r * 8 + c] = o[r];
        }
    }
    const int stride = im.bw[comp] * 8;
    uint8_t *out = ws + H.ws_plane + im.plane_offset + im.plane_byte[comp] + (long long)by * 8 * stride + bx * 8;
    // pass 2: rows
#pragma unroll
    for (int r = 0; r < 8; ++r) {
        int o[8];
        idct_1d<2>(ws_[r * 8], ws_[r * 8 + 1], ws_[r * 8 + 2], ws_[r * 8 + 3], ws_[r * 8 + 4], ws_[r * 8 + 5], ws_[r * 8 + 6],
                   ws_[r * 8 + 7], o);
        uint2 pk;
        pk.x = o[0] | (o[1] << 8) | (o[2] << 16) | ((unsigned)o[3] << 24);
        pk.y = o[4] | (o[5] << 8) | (o[6] << 16) | ((unsigned)o[7] << 24);
        *reinterpret_cast<uint2 *>(out + (long long)r * stride) = pk;
    }
}

// One thread per output pixel; grid (pixel tiles, image).  Chroma follows jdsample.c (fancy upsampling on); the context rows
// above the first and below the last downsampled row replicate those rows, as jdmainct.c sets them up.
__global__ void __launch_bounds__(COLOR_THREADS) jpeg_color_kernel(const uint8_t *__restrict__ blob, const uint8_t *__restrict__ ws,
                                                                   uint8_t *__restrict__ dst) {
    const JpegBlobHeader &H = hdr(blob);
    const JpegImg &im = imgs(blob)[blockIdx.y];
    const long long idx = (long long)blockIdx.x * COLOR_THREADS + threadIdx.x;
    if (idx >= (long long)im.h * im.w) return;
    const int y = (int)(idx / im.w), x = (int)(idx % im.w);
    const uint8_t *planes = ws + H.ws_plane + im.plane_offset;
    const int ys = im.bw[0] * 8;
    const int Y = planes[(long long)y * ys + x];
    uint8_t *o = dst + im.dst_offset + idx * 3;
    if (im.upsample == UP_GRAY) {
        o[0] = o[1] = o[2] = (uint8_t)Y;
        return;
    }
    const int cs = im.bw[1] * 8, dw = im.dw[1], dh = im.dh[1];
    int ch[2];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        const uint8_t *pl = planes + im.plane_byte[1 + k];
        int v;
        switch (im.upsample) {
            case UP_FULL: v = pl[(long long)y * cs + x]; break;
            case UP_H2V1_FANCY: {
                const int j = x >> 1, jn = (x & 1) ? min(j + 1, dw - 1) : max(j - 1, 0);
                const uint8_t *row = pl + (long long)y * cs;
                v = (3 * row[j] + row[jn] + 1 + (x & 1)) >> 2;
                break;
            }
            case UP_H2V1_BOX: v = pl[(long long)y * cs + (x >> 1)]; break;
            case UP_H1V2_FANCY: {
                const int i = y >> 1, in = (y & 1) ? min(i + 1, dh - 1) : max(i - 1, 0);
                v = (3 * pl[(long long)i * cs + x] + pl[(long long)in * cs + x] + 1 + (y & 1)) >> 2;
                break;
            }
            case UP_H2V2_FANCY: {
                const int i = y >> 1, in = (y & 1) ? min(i + 1, dh - 1) : max(i - 1, 0);
                const int j = x >> 1, jn = (x & 1) ? min(j + 1, dw - 1) : max(j - 1, 0);
                const uint8_t *r0 = pl + (long long)i * cs, *r1 = pl + (long long)in * cs;
                const int c0 = 3 * r0[j] + r1[j], c1 = 3 * r0[jn] + r1[jn];
                v = (3 * c0 + c1 + 8 - (x & 1)) >> 4;
                break;
            }
            case UP_H2V2_BOX: v = pl[(long long)(y >> 1) * cs + (x >> 1)]; break;
            default: v = pl[(long long)y * cs + (x >> 2)]; break;   // UP_H4V1_BOX (int_upsample)
        }
        ch[k] = v;
    }
    // jdcolor.c ycc_rgb_convert: 16 scale bits, ONE_HALF rounding, sample range limit
    const int cb = ch[0] - 128, cr = ch[1] - 128;
    const int r = Y + ((91881 * cr + 32768) >> 16);
    const int g = Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16);
    const int b = Y + ((116130 * cb + 32768) >> 16);
    o[0] = (uint8_t)min(max(r, 0), 255);
    o[1] = (uint8_t)min(max(g, 0), 255);
    o[2] = (uint8_t)min(max(b, 0), 255);
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
    jpeg_unstuff_kernel<<<H->n, UNSTUFF_THREADS, 0, st>>>(blob, src_dev, ws);
    jpeg_huffman_kernel<<<H->nseg, SYNC_THREADS, 0, st>>>(blob, ws, status_dev);
    jpeg_dc_kernel<<<H->nseg, DC_THREADS, 0, st>>>(blob, ws);
    jpeg_idct_kernel<<<dim3((unsigned)((H->max_blocks + IDCT_THREADS - 1) / IDCT_THREADS), H->n), IDCT_THREADS, 0, st>>>(blob, ws);
    jpeg_color_kernel<<<dim3((unsigned)((H->max_pixels + COLOR_THREADS - 1) / COLOR_THREADS), H->n), COLOR_THREADS, 0, st>>>(blob, ws,
                                                                                                                          dst_dev);
    K2Y_CUDA_CHECK(cudaGetLastError());
    return K2Y_OK;
}
