// Pieces the baseline (jpeg.cu) and progressive (jpeg_progressive.cu) JPEG decoders share: the marker walker, Huffman
// tables in lookup form, the Huffman symbol decoder, and the back end (libjpeg-turbo's x86 SIMD islow IDCT, fancy upsampling
// and ycc_rgb_convert) as device functions over an image descriptor with the same field names in both decoders.
#pragma once
#include "common.h"
#include "jpeg_std_huff.cuh"

#include <algorithm>
#include <cstdarg>

namespace k2y {
namespace {

constexpr int HUFF_LOOKAHEAD = 9;
constexpr int MAX_BLOCKS_PER_MCU = 6;                // luma 4x1 or 2x2 + two 1x1 chroma
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

// What the progressive decoder adds to the walk.  Without a hook the walk stops at the first SOS (a baseline file).  With one,
// an SOF2 frame is the GPU kind, each SOS goes to scan() with p's scan fields filled, which latches the quantisation tables
// and returns where the marker walk resumes (after the scan's entropy-coded data), and the walk ends at EOI, or at the end of
// the data after at least one scan; finish() then classifies the script.
struct ScanHook {
    virtual int scan(const uint8_t *d, size_t n, Parsed &p, size_t sos_at, size_t data_at, size_t &resume, const char *who) = 0;
    virtual int finish(Parsed &p, bool eoi, const char *who) = 0;
    virtual bool any() const = 0;
};

// Returns K2Y_OK (p filled up to the first SOS; p.gpu / p.reason classify it) or K2Y_ERR_INVALID with the marker in the error.
int parse_jpeg(const uint8_t *d, size_t n, Parsed &p, const char *who, ScanHook *hook = nullptr) {
    if (n < 4 || d[0] != 0xFF || d[1] != 0xD8) {
        set_error("%s: not a JPEG file (no SOI marker)", who);
        return K2Y_ERR_INVALID;
    }
    size_t i = 2;
    bool saw_sof = false, eoi = false;
    for (;;) {
        while (i < n && d[i] != 0xFF) ++i;   // libjpeg skips extraneous bytes before a marker
        while (i < n && d[i] == 0xFF) ++i;   // fill bytes
        if (i >= n) {
            if (hook && hook->any()) break;
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
            if (hook && hook->any()) {
                eoi = true;
                break;
            }
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
            // anything but the decoder's own kind (8-bit sequential Huffman, or progressive Huffman with a hook) is valid JPEG
            // the GPU path does not take: stop at the frame header
            const char *kind = nullptr;
            if (m == 0xC2 || m == 0xC6) kind = "progressive";
            else if (m == 0xC3 || m == 0xC7) kind = "lossless";
            else if (m == 0xC5) kind = "hierarchical";
            else if (m >= 0xC9) kind = "arithmetic coding";
            if (hook) kind = m == 0xC2 ? nullptr : m == 0xC0 || m == 0xC1 ? "sequential" : m == 0xC6 ? "differential progressive" : kind;
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
            if (hook) {
                size_t resume = next;
                const int rc = hook->scan(d, n, p, at, next, resume, who);
                if (rc != K2Y_OK) return rc;
                i = resume;
                continue;
            }
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
    // classification of an 8-bit sequential (or, with a hook, progressive) Huffman file
    // jdinput.c initial_setup: libjpeg-turbo refuses a larger frame at the first SOS, so PIL cannot read the file
    if (p.h > JPEG_MAX_DIMENSION || p.w > JPEG_MAX_DIMENSION)
        return set_reason(p, "%dx%d exceeds libjpeg's %d-pixel limit", p.w, p.h, JPEG_MAX_DIMENSION), K2Y_OK;
    if (p.ncomp == 2) return set_reason(p, "2 components"), K2Y_OK;
    if (p.ncomp == 4) return set_reason(p, "4 components (CMYK/YCCK)"), K2Y_OK;
    if (p.ncomp == 3 && !p.jfif) {   // libjpeg's default_decompress_parms
        if (p.adobe && p.adobe_transform == 0) return set_reason(p, "RGB colour space (Adobe transform 0)"), K2Y_OK;
        if (!p.adobe && p.id[0] == 'R' && p.id[1] == 'G' && p.id[2] == 'B') return set_reason(p, "RGB colour space (component ids R, G, B)"), K2Y_OK;
    }
    if (!hook) {
        if (p.ns != p.ncomp) return set_reason(p, "multi-scan sequential"), K2Y_OK;
        if (p.ss != 0 || p.se != 63 || p.ah != 0 || p.al != 0) return set_reason(p, "scan parameters Ss=%d Se=%d Ah=%d Al=%d", p.ss, p.se, p.ah, p.al), K2Y_OK;
    }
    if (p.ncomp == 3) {
        const int h0 = p.hs[0], v0 = p.vs[0];
        const bool chroma11 = p.hs[1] == 1 && p.vs[1] == 1 && p.hs[2] == 1 && p.vs[2] == 1;
        const bool luma_ok = (h0 == 1 && v0 == 1) || (h0 == 2 && v0 == 1) || (h0 == 1 && v0 == 2) || (h0 == 2 && v0 == 2) || (h0 == 4 && v0 == 1);
        if (!chroma11 || !luma_ok)
            return set_reason(p, "sampling %dx%d,%dx%d,%dx%d", p.hs[0], p.vs[0], p.hs[1], p.vs[1], p.hs[2], p.vs[2]), K2Y_OK;
    }
    if (hook) {
        const int rc = hook->finish(p, eoi, who);
        if (rc != K2Y_OK || p.reason[0]) return rc;
    }
    // jdhuff.c jinit_huff_decoder -> std_huff_tables: a sequential scan's DC / AC slots 0 and 1 that no DHT defined take the
    // Annex K.3 tables, each slot on its own (Motion-JPEG frames leave them out); an undefined slot 2 or 3 stays an error
    for (int s = 0; !hook && s < 2; ++s)
        for (int ac = 0; ac < 2; ++ac) {
            HuffSpec &hs = ac ? p.ac[s] : p.dc[s];
            if (hs.defined) continue;
            const int t = 2 * s + ac;
            int count = 0;
            hs.defined = true;
            hs.bits[0] = 0;
            for (int l = 1; l <= 16; ++l) count += hs.bits[l] = kHuffBits[t][l - 1];
            memset(hs.vals, 0, sizeof(hs.vals));
            memcpy(hs.vals, huff_vals(t), count);
        }
    for (int k = 0; !hook && k < p.ns; ++k) {
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

// ---------------------------------------------------------------------------------------------------------------------
// Device: Huffman symbols
// ---------------------------------------------------------------------------------------------------------------------
// One Huffman symbol from a bit reader holding at least 16 bits MSB-first in `buf` (count `nb`); sets `bad` (and returns 0
// after 16 bits, as libjpeg does) on a code no table entry matches.
template <class Reader>
__device__ __forceinline__ int huff_decode(Reader &br, const JpegHuff &t, int &used, bool &bad) {
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

// ---------------------------------------------------------------------------------------------------------------------
// Device: back end.  `Img` has h, w, ncomp, upsample, blocks, bw, dw, dh, coef_block, plane_byte and qt (natural order).
// ---------------------------------------------------------------------------------------------------------------------
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

// The body of an IDCT kernel: one thread per 8x8 block, grid (block tiles, image); `coef` and `planes` are the image's
// coefficients and component planes, `s_q` shared memory for its quantisation tables.
template <class Img>
__device__ __forceinline__ void idct_image(const Img &im, const uint8_t *coef, uint8_t *planes, int (*s_q)[64]) {
    for (int k = threadIdx.x; k < 3 * 64; k += blockDim.x) s_q[k / 64][k % 64] = (int16_t)im.qt[k / 64][k % 64];
    __syncthreads();
    const int b = blockIdx.x * IDCT_THREADS + threadIdx.x;
    if (b >= im.blocks) return;
    const int comp = im.ncomp == 1 ? 0 : (b < im.coef_block[1] ? 0 : (b < im.coef_block[2] ? 1 : 2));
    const int local = b - im.coef_block[comp];
    const int bx = local % im.bw[comp], by = local / im.bw[comp];
    const int4 *cp = reinterpret_cast<const int4 *>(coef) + (long long)b * 8;
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
    uint8_t *out = planes + im.plane_byte[comp] + (long long)by * 8 * stride + bx * 8;
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

// The body of a colour kernel: one thread per output pixel, grid (pixel tiles, image); `planes` are the image's component
// planes, `o_img` its HWC RGB output.  Chroma follows jdsample.c (fancy upsampling on); the context rows above the first and
// below the last downsampled row replicate those rows, as jdmainct.c sets them up.
template <class Img>
__device__ __forceinline__ void color_image(const Img &im, const uint8_t *planes, uint8_t *o_img) {
    const long long idx = (long long)blockIdx.x * COLOR_THREADS + threadIdx.x;
    if (idx >= (long long)im.h * im.w) return;
    const int y = (int)(idx / im.w), x = (int)(idx % im.w);
    const int ys = im.bw[0] * 8;
    const int Y = planes[(long long)y * ys + x];
    uint8_t *o = o_img + idx * 3;
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
