// Progressive Huffman JPEG decoding on the GPU, bit-exact with libjpeg-turbo as PIL runs it (jdphuff.c for the entropy
// decode, then the baseline decoder's back end: the x86 SIMD islow IDCT, fancy upsampling and ycc_rgb_convert).
//
// Host side: the baseline marker walker (jpeg_common.cuh) with a ScanHook walks every marker to EOI.  Each SOS is checked as
// jdphuff.c start_pass_phuff_decoder checks it (a bad progression is K2Y_ERR_INVALID naming the scan); the walker skips the
// scan's entropy-coded data, cutting it at RSTn into restart segments, and keeps the Huffman tables and restart interval in
// force at the scan.  Quantisation tables are latched at each component's first scan, as jdinput.c latches them.  A file
// stays on the host when libjpeg-turbo would decode it with a JWRN_BOGUS_PROGRESSION warning, when its script leaves
// libjpeg-turbo to block-smooth the output (jdcoefct.c smoothing_ok: a component's DC is known but one of its zig-zag
// coefficients 1..9 is not fully known), when it has more than PROG_MAX_SCANS scans, or when a scan's restart markers are
// out of sequence (the k-th marker between its intervals not RST(k mod 8), too few of them, or any with no restart interval:
// libjpeg-turbo's resynchronisation then drops or rereads data, which the decoder does not model).
//
// The descriptor blob (ProgBlobHeader, ProgImg[n], ProgScan[scans], ProgSeg[segments], JpegHuff[tables]) lists every
// (scan, restart interval) segment with its byte range in the file.  Each scan gets a level from the (component,
// coefficient) pairs it may write: 0 when no earlier scan may write any of them, else one more than the highest level of
// those that may.  A scan may write past its band: jdphuff.c indexes the natural order (whose last sixteen entries are 63)
// at k after a run, so an AC first scan may write zig-zag Ss..min(63, Se + 15) and an AC refinement Ss..min(63, Se + 1).
// Scans that may write a common coefficient thus decode in file order, and scans of one level write disjoint coefficients
// and read none another scan of the level writes, so they decode concurrently; the segments are sorted by level.
//
// Device side:
//   1. prog_entropy_kernel  one launch per level (a default libjpeg script has four), one thread per segment in a CTA of
//                           its own, decoding the segment serially from its bytes as they lie in the file (stuffing and
//                           fill bytes dropped on the fly): DC first (prediction in the unshifted domain, stored as
//                           (JCOEF)((unsigned)v << Al)), DC refine (one raw bit per block), AC first (EOB runs across
//                           blocks) and AC refine (correction bits, new +-1 << Al coefficients, EOB runs).  A segment
//                           is a restart interval, so the DC predictors and the EOB run start from zero in each.
//   2. prog_idct_kernel     dequantise + islow IDCT (jpeg_common.cuh)
//   3. prog_color_kernel    upsample + colour convert (jpeg_common.cuh)
// The entropy decode is serial within a segment: an AC refinement's bit count depends on which coefficients earlier scans
// made nonzero, so a decoder started at a guessed bit position cannot place itself.  Parallelism comes from images,
// components, scans of one level and restart intervals only.
#include "jpeg_common.cuh"

#include <climits>
#include <vector>

namespace k2y {
namespace {

constexpr uint32_t PROG_BLOB_MAGIC = 0x4a504732u;   // "JPG2"
constexpr int PROG_MAX_SCANS = 64;                  // per file; more stay on the host
constexpr int DC_REFINE_GROUP = 16;                 // blocks whose DC a refinement scan loads at once

struct alignas(16) ProgImg {
    long long src_offset;       // the file in the source buffer (a multiple of 16)
    long long dst_offset;       // HWC RGB output
    long long coef_offset;      // workspace: int16 coefficients, bytes
    long long plane_offset;     // workspace: uint8 component planes, bytes
    int32_t h, w, ncomp, upsample;
    int32_t blocks, pad_[3];
    int32_t bw[3], bh[3];       // component planes in blocks (MCU-padded)
    int32_t dw[3], dh[3];       // libjpeg downsampled_width / downsampled_height
    int32_t coef_block[3];      // first block of each component
    int32_t plane_byte[3];      // byte offset of each component plane
    uint16_t qt[3][64];         // natural order, as latched at the component's first scan (zero if it has none)
};

struct alignas(16) ProgScan {
    int32_t image, ss, se, ah, al;
    int32_t mcux, bpm, huff_first, ntab;   // MCUs per row, blocks per MCU; the scan's tables in the blob
    int32_t hs[3], vs[3];                  // blocks per MCU of each frame component (1 x 1 in a one-component scan)
    uint8_t mcu_comp[MAX_BLOCKS_PER_MCU], mcu_bx[MAX_BLOCKS_PER_MCU], mcu_by[MAX_BLOCKS_PER_MCU];
    uint8_t mcu_tab[MAX_BLOCKS_PER_MCU];   // table of each block within the scan's tables
};

struct alignas(16) ProgSeg {
    long long begin, end;       // entropy-coded bytes from the file's start, stuffing included
    int32_t scan, first_mcu, mcus, level;
};

struct alignas(16) ProgBlobHeader {
    uint32_t magic;
    int32_t n, nscan, nseg;
    int32_t ntab, nlevel, max_blocks, pad_;
    long long max_pixels;
    long long img_off, scan_off, seg_off, huff_off, blob_bytes;
    long long ws_coef, ws_plane, ws_bytes;
    int32_t level_seg[PROG_MAX_SCANS + 1];   // first segment of each level; level_seg[nlevel] = nseg
};

// ---------------------------------------------------------------------------------------------------------------------
// Host: the scan walk
// ---------------------------------------------------------------------------------------------------------------------
struct ScanRec {
    int ns = 0, comp[4] = {}, ss = 0, se = 0, ah = 0, al = 0, restart = 0, level = 0;
    HuffSpec tab[4];                 // DC first: the DC table of each component; AC scans: tab[0] is the AC table
    int ntab = 0;
    std::vector<long long> bounds;   // restart segment k of the data is [bounds[2k], bounds[2k + 1])
};

struct ProgHook : ScanHook {
    std::vector<ScanRec> scans;
    int nscans = 0;
    int coef_bits[4][64];            // jdphuff.c coef_bits: -1 never sent, else the Al of the last scan that sent it
    int last_level[4][64];           // highest level of a scan that touched the coefficient, -1 none
    bool latched[4] = {};
    uint16_t qt[4][64] = {};
    char bogus[64] = {};
    int nlevel = 0;

    ProgHook() {
        for (int c = 0; c < 4; ++c)
            for (int k = 0; k < 64; ++k) coef_bits[c][k] = last_level[c][k] = -1;
    }
    bool any() const override { return nscans > 0; }

    int scan(const uint8_t *d, size_t n, Parsed &p, size_t sos_at, size_t data_at, size_t &resume, const char *who) override {
        const int si = nscans++;
        // jdinput.c latch_quant_tables: at a component's first scan
        for (int k = 0; k < p.ns; ++k) {
            const int c = p.scan_comp[k];
            if (latched[c]) continue;
            if (!p.qt_defined[p.tq[c]]) {
                set_error("%s: scan %d (SOS at offset %zu): quantisation table %d of component %d is not defined", who, si, sos_at,
                          p.tq[c], c);
                return K2Y_ERR_INVALID;
            }
            memcpy(qt[c], p.qt[p.tq[c]], sizeof(qt[c]));
            latched[c] = true;
        }
        // jdphuff.c start_pass_phuff_decoder: JERR_BAD_PROGRESSION
        const bool dc = p.ss == 0;
        const char *bad = nullptr;
        if (dc && p.se != 0) bad = "a DC scan with Se != 0";
        if (!dc && (p.ss > p.se || p.se > 63)) bad = "an AC scan with Ss > Se or Se > 63";
        if (!dc && p.ns != 1) bad = "an AC scan of more than one component";
        if (p.ah != 0 && p.al != p.ah - 1) bad = "a refinement with Al != Ah - 1";
        if (p.al > 13) bad = "Al > 13";
        if (bad) {
            set_error("%s: scan %d (SOS at offset %zu) is %s (Ss=%d Se=%d Ah=%d Al=%d)", who, si, sos_at, bad, p.ss, p.se, p.ah,
                      p.al);
            return K2Y_ERR_INVALID;
        }
        ScanRec r;
        r.ns = p.ns;
        r.ss = p.ss;
        r.se = p.se;
        r.ah = p.ah;
        r.al = p.al;
        r.restart = p.restart;
        // the tables the scan decodes with (a DC refinement needs none); jpeg_make_d_derived_tbl's errors refuse the file
        if (!(dc && p.ah != 0)) {
            r.ntab = dc ? p.ns : 1;
            for (int k = 0; k < r.ntab; ++k) {
                const HuffSpec &hs = dc ? p.dc[p.td[k]] : p.ac[p.ta[0]];
                const int t = dc ? p.td[k] : p.ta[0];
                if (!hs.defined) {
                    if (!bogus[0]) snprintf(bogus, sizeof(bogus), "Huffman table not defined before scan %d", si);
                    continue;
                }
                int count = 0;
                for (int l = 1; l <= 16; ++l) count += hs.bits[l];
                for (int v = 0; dc && v < count; ++v)
                    if (hs.vals[v] > 15) {
                        set_error("%s: scan %d: DHT DC table %d has symbol %d", who, si, t, hs.vals[v]);
                        return K2Y_ERR_INVALID;
                    }
                JpegHuff tmp;
                if (!derive_huff(hs, tmp)) {
                    set_error("%s: scan %d: DHT table %d has more codes than its code lengths allow", who, si, t);
                    return K2Y_ERR_INVALID;
                }
                r.tab[k] = hs;
            }
        }
        // the progression as jdphuff.c tracks it: scripts it warns about (JWRN_BOGUS_PROGRESSION) stay on the host, and so
        // does a first scan of a coefficient that was already sent
        for (int k = 0; k < p.ns; ++k) {
            const int c = p.scan_comp[k];
            r.comp[k] = c;
            if (!dc && coef_bits[c][0] < 0 && !bogus[0])
                snprintf(bogus, sizeof(bogus), "scan %d: AC of component %d before its DC", si, c);
            for (int z = p.ss; z <= p.se; ++z) {
                if (p.ah == 0 && coef_bits[c][z] >= 0 && !bogus[0])
                    snprintf(bogus, sizeof(bogus), "scan %d: coefficient %d of component %d sent twice", si, z, c);
                if (p.ah != 0 && p.ah != coef_bits[c][z] && !bogus[0])
                    snprintf(bogus, sizeof(bogus), "scan %d: refinement Ah=%d of coefficient %d of component %d", si, p.ah, z, c);
                coef_bits[c][z] = p.al;
            }
        }
        // the level, from the coefficients the scan may write rather than its band: jdphuff.c writes a run that ends past Se
        // through the natural order's trailing 63s, up to Se + 15 in an AC first scan and Se + 1 in an AC refinement
        const int reach = dc ? 0 : std::min(63, p.se + (p.ah == 0 ? 15 : 1));
        int level = 0;
        for (int k = 0; k < p.ns; ++k)
            for (int z = p.ss; z <= reach; ++z) level = std::max(level, last_level[r.comp[k]][z] + 1);
        for (int k = 0; k < p.ns; ++k)
            for (int z = p.ss; z <= reach; ++z) last_level[r.comp[k]][z] = level;
        r.level = level;
        nlevel = std::max(nlevel, level + 1);
        // restart intervals the scan needs; libjpeg-turbo resynchronises on a marker out of sequence, which the decoder does
        // not model, so such a file stays on the host
        long long mcus = 0;
        {
            int hmax = 1, vmax = 1;
            for (int c = 0; c < p.ncomp && p.ncomp > 1; ++c) {
                hmax = std::max(hmax, p.hs[c]);
                vmax = std::max(vmax, p.vs[c]);
            }
            if (p.ns == 1) {
                const int c = r.comp[0], hc = p.ncomp > 1 ? p.hs[c] : 1, vc = p.ncomp > 1 ? p.vs[c] : 1;
                const long long dw = ((long long)p.w * hc + hmax - 1) / hmax, dh = ((long long)p.h * vc + vmax - 1) / vmax;
                mcus = ((dw + 7) / 8) * ((dh + 7) / 8);
            } else {
                mcus = (long long)((p.w + 8 * hmax - 1) / (8 * hmax)) * ((p.h + 8 * vmax - 1) / (8 * vmax));
            }
        }
        const long long need = p.restart && mcus > 0 ? (mcus + p.restart - 1) / p.restart - 1 : 0;   // markers between intervals
        long long seen = 0;
        // the entropy-coded data: up to the first marker that is neither a stuffed zero, a fill byte nor RSTn
        size_t j = data_at;
        r.bounds.push_back((long long)j);
        for (;;) {
            const void *f = j < n ? memchr(d + j, 0xFF, n - j) : nullptr;
            if (!f) {
                j = n;
                break;
            }
            j = (size_t)(static_cast<const uint8_t *>(f) - d);
            if (j + 1 >= n) {
                j = n;
                break;
            }
            const int nx = d[j + 1];
            if (nx == 0x00) {
                j += 2;
            } else if (nx == 0xFF) {
                j += 1;
            } else if (nx >= 0xD0 && nx <= 0xD7) {
                if (!p.restart && !bogus[0])
                    snprintf(bogus, sizeof(bogus), "scan %d: RST%d with no restart interval", si, nx - 0xD0);
                else if (seen < need && nx - 0xD0 != (int)(seen % 8) && !bogus[0])
                    snprintf(bogus, sizeof(bogus), "scan %d: restart marker %lld is RST%d, not RST%d", si, seen, nx - 0xD0,
                             (int)(seen % 8));
                ++seen;
                r.bounds.push_back((long long)j);
                r.bounds.push_back((long long)j + 2);
                j += 2;
            } else {
                break;
            }
        }
        if (seen < need && !bogus[0]) snprintf(bogus, sizeof(bogus), "scan %d: %lld restart markers of %lld", si, seen, need);
        r.bounds.push_back((long long)j);
        resume = j;
        if (si < PROG_MAX_SCANS) scans.push_back(std::move(r));
        return K2Y_OK;
    }

    int finish(Parsed &p, bool eoi, const char *) override {
        if (!eoi) return set_reason(p, "file ends before its EOI marker"), K2Y_OK;
        if (bogus[0]) return set_reason(p, "%s", bogus), K2Y_OK;
        if (nscans > PROG_MAX_SCANS) return set_reason(p, "%d scans, more than %d", nscans, PROG_MAX_SCANS), K2Y_OK;
        // jdcoefct.c smoothing_ok: every component latched, its quantisers of zig-zag 0..9 nonzero and its DC sent, and then
        // some coefficient 1..9 of some component not fully known
        bool ok = true;
        int sc = -1, sz = -1;
        for (int c = 0; c < p.ncomp && ok; ++c) {
            if (!latched[c] || coef_bits[c][0] < 0) ok = false;
            for (int z = 0; z < 10 && ok; ++z)
                if (qt[c][kNatural[z]] == 0) ok = false;
            for (int z = 1; z < 10 && ok && sc < 0; ++z)
                if (coef_bits[c][z] != 0) sc = c, sz = z;
        }
        if (ok && sc >= 0) {
            if (coef_bits[sc][sz] < 0) return set_reason(p, "block smoothing: coefficient %d of component %d never sent", sz, sc), K2Y_OK;
            return set_reason(p, "block smoothing: coefficient %d of component %d known to bit %d", sz, sc, coef_bits[sc][sz]), K2Y_OK;
        }
        for (int c = 0; c < p.ncomp; ++c) memcpy(p.scan_qt[c], qt[c], sizeof(qt[c]));
        return K2Y_OK;
    }
};

// ---------------------------------------------------------------------------------------------------------------------
// Device
// ---------------------------------------------------------------------------------------------------------------------
// MSB-first bit reader over one segment's bytes as they lie in the file: drops the 0x00 after a stuffed 0xFF and fill bytes
// (an 0xFF not followed by 0x00), reads aligned 16-byte words of the file (its slot is readable up to its size rounded up
// to 16), and past the segment's end reads zeros and counts them.
struct StuffedReader {
    const uint8_t *base;
    long long pos, end, word_at;
    uint4 word;
    uint64_t buf;
    int nb, pad;
    __device__ __forceinline__ void init(const uint8_t *file, long long begin, long long stop) {
        base = file;
        pos = begin;
        end = stop;
        word_at = -1;
        buf = 0;
        nb = 0;
        pad = 0;
    }
    __device__ __forceinline__ unsigned byte_at(long long q) {
        const long long a = q & ~15LL;
        if (a != word_at) {
            word = __ldg(reinterpret_cast<const uint4 *>(base + a));
            word_at = a;
        }
        const unsigned w = (q & 8) ? ((q & 4) ? word.w : word.z) : ((q & 4) ? word.y : word.x);
        return (w >> ((q & 3) * 8)) & 255;
    }
    __device__ __forceinline__ void fill() {
        while (nb <= 56) {
            unsigned b = 0;
            if (pos < end) {
                b = byte_at(pos++);
                if (b == 0xFF) {
                    if (pos < end && byte_at(pos) == 0) ++pos;
                    else continue;   // a fill byte
                }
            } else {
                ++pad;
            }
            buf |= (uint64_t)b << (56 - nb);
            nb += 8;
        }
    }
    __device__ __forceinline__ unsigned get(int n) {   // 1 <= n <= 16
        if (nb < n) fill();
        const unsigned v = (unsigned)(buf >> (64 - n));
        buf <<= n;
        nb -= n;
        return v;
    }
    __device__ __forceinline__ bool overrun() const { return pad * 8 > nb; }   // a bit past the segment's end was used
};

__device__ __forceinline__ const ProgBlobHeader &phdr(const uint8_t *blob) { return *reinterpret_cast<const ProgBlobHeader *>(blob); }
__device__ __forceinline__ const ProgImg *pimgs(const uint8_t *blob) { return reinterpret_cast<const ProgImg *>(blob + phdr(blob).img_off); }

__device__ __forceinline__ int16_t *scan_block(int16_t *coef, const ProgImg &im, const ProgScan &sc, int mcu, int c) {
    const int comp = sc.mcu_comp[c];
    const int mx = mcu % sc.mcux, my = mcu / sc.mcux;
    const int bx = mx * sc.hs[comp] + sc.mcu_bx[c], by = my * sc.vs[comp] + sc.mcu_by[c];
    return coef + ((long long)im.coef_block[comp] + (long long)by * im.bw[comp] + bx) * 64;
}

// status words per image: [0] error bits (1 bad Huffman code, 2 premature end of data, 4 a DC value outside int, which
// libjpeg refuses), [1] and [2] zero (no synchronisation rounds: the decode does not speculate), [3] segments decoded
__global__ void __launch_bounds__(1) prog_entropy_kernel(const uint8_t *__restrict__ blob, const uint8_t *__restrict__ src,
                                                         uint8_t *__restrict__ ws, int *__restrict__ status, int seg0) {
    __shared__ JpegHuff s_tab[3];
    __shared__ int4 s_blk4[8];
    const ProgBlobHeader &H = phdr(blob);
    const ProgSeg &sg = reinterpret_cast<const ProgSeg *>(blob + H.seg_off)[seg0 + blockIdx.x];
    const ProgScan &sc = reinterpret_cast<const ProgScan *>(blob + H.scan_off)[sg.scan];
    const ProgImg &im = pimgs(blob)[sc.image];
    {
        const int4 *srcv = reinterpret_cast<const int4 *>(reinterpret_cast<const JpegHuff *>(blob + H.huff_off) + sc.huff_first);
        int4 *dstv = reinterpret_cast<int4 *>(s_tab);
        for (int k = 0; k < sc.ntab * (int)(sizeof(JpegHuff) / 16); ++k) dstv[k] = srcv[k];
    }
    int16_t *coef = reinterpret_cast<int16_t *>(ws + H.ws_coef + im.coef_offset);
    StuffedReader br;
    br.init(src + im.src_offset, sg.begin, sg.end);
    int err = 0;
    const int ss = sc.ss, se = sc.se, al = sc.al;
    if (ss == 0 && sc.ah == 0) {   // DC first
        long long pred0 = 0, pred1 = 0, pred2 = 0;   // per component, in registers
        for (int m = 0; m < sg.mcus; ++m) {
            for (int c = 0; c < sc.bpm; ++c) {
                br.fill();
                int used;
                bool bad = false;
                const int s = huff_decode(br, s_tab[sc.mcu_tab[c]], used, bad);
                const int v = s ? huff_extend(br.get(s), s) : 0;
                const int comp = sc.mcu_comp[c];
                const long long pred = (comp == 0 ? pred0 : comp == 1 ? pred1 : pred2) + v;
                if (comp == 0) pred0 = pred;
                else if (comp == 1) pred1 = pred;
                else pred2 = pred;
                if (pred > INT_MAX || pred < INT_MIN) err |= 4;
                if (bad) err |= 1;
                *scan_block(coef, im, sc, sg.first_mcu + m, c) = (int16_t)((unsigned)pred << al);
            }
        }
    } else if (ss == 0) {          // DC refine: one bit per block, ORed in; the blocks' DC words are loaded a group at a time
        const int p1 = 1 << al;
        const int total = sg.mcus * sc.bpm;
        for (int b0 = 0; b0 < total; b0 += DC_REFINE_GROUP) {
            int16_t *ptr[DC_REFINE_GROUP];
            int16_t val[DC_REFINE_GROUP];
#pragma unroll
            for (int g = 0; g < DC_REFINE_GROUP; ++g) {
                if (b0 + g < total) {
                    ptr[g] = scan_block(coef, im, sc, sg.first_mcu + (b0 + g) / sc.bpm, (b0 + g) % sc.bpm);
                    val[g] = *ptr[g];
                }
            }
#pragma unroll
            for (int g = 0; g < DC_REFINE_GROUP; ++g)
                if (b0 + g < total && br.get(1)) *ptr[g] = (int16_t)(val[g] | p1);
        }
    } else if (sc.ah == 0) {       // AC first: one component, one block per MCU
        int eobrun = 0;
        for (int m = 0; m < sg.mcus; ++m) {
            if (eobrun > 0) {
                --eobrun;
                continue;
            }
            int16_t *blk = scan_block(coef, im, sc, sg.first_mcu + m, 0);
            for (int k = ss; k <= se; ++k) {
                br.fill();
                int used;
                bool bad = false;
                const int rs = huff_decode(br, s_tab[0], used, bad);
                if (bad) err |= 1;
                const int r = rs >> 4, s = rs & 15;
                if (s) {
                    k += r;
                    const int v = huff_extend(br.get(s), s);
                    blk[c_natural[min(k, 63)]] = (int16_t)((unsigned)v << al);   // libjpeg's natural order ends in 63s
                } else if (r == 15) {
                    k += 15;
                } else {
                    eobrun = 1 << r;
                    if (r) eobrun += br.get(r);
                    --eobrun;
                    break;
                }
            }
        }
    } else {                       // AC refine: the block in shared memory, the next one loading meanwhile
        const int p1 = 1 << al, m1 = -p1;
        int16_t *s_blk = reinterpret_cast<int16_t *>(s_blk4);
        int eobrun = 0;
        int4 nxt[8];
        if (sg.mcus > 0) {
            const int4 *g = reinterpret_cast<const int4 *>(scan_block(coef, im, sc, sg.first_mcu, 0));
#pragma unroll
            for (int q = 0; q < 8; ++q) nxt[q] = g[q];
        }
        for (int m = 0; m < sg.mcus; ++m) {
            int16_t *blk = scan_block(coef, im, sc, sg.first_mcu + m, 0);
#pragma unroll
            for (int q = 0; q < 8; ++q) s_blk4[q] = nxt[q];
            if (m + 1 < sg.mcus) {
                const int4 *g = reinterpret_cast<const int4 *>(scan_block(coef, im, sc, sg.first_mcu + m + 1, 0));
#pragma unroll
                for (int q = 0; q < 8; ++q) nxt[q] = g[q];
            }
            unsigned long long changed = 0;
            int k = ss;
            if (eobrun == 0) {
                for (; k <= se; ++k) {
                    br.fill();
                    int used;
                    bool bad = false;
                    const int rs = huff_decode(br, s_tab[0], used, bad);
                    if (bad) err |= 1;
                    int r = rs >> 4, s = rs & 15;
                    if (s) {   // a size other than 1 is only a warning in libjpeg
                        s = br.get(1) ? p1 : m1;
                    } else if (r != 15) {
                        eobrun = 1 << r;
                        if (r) eobrun += br.get(r);
                        break;
                    }
                    // correction bits of the nonzero coefficients up to the r+1-th zero one
                    do {
                        const int pos = c_natural[k];
                        const int cur = s_blk[pos];
                        if (cur != 0) {
                            if (br.get(1) && (cur & p1) == 0) {
                                s_blk[pos] = (int16_t)(cur >= 0 ? cur + p1 : cur + m1);
                                changed |= 1ull << pos;
                            }
                        } else if (--r < 0) {
                            break;
                        }
                        ++k;
                    } while (k <= se);
                    if (s) {
                        const int pos = c_natural[min(k, 63)];
                        s_blk[pos] = (int16_t)s;
                        changed |= 1ull << pos;
                    }
                }
            }
            if (eobrun > 0) {   // the rest of the band after the end of band: correction bits only
                for (; k <= se; ++k) {
                    const int pos = c_natural[k];
                    const int cur = s_blk[pos];
                    if (cur != 0 && br.get(1) && (cur & p1) == 0) {
                        s_blk[pos] = (int16_t)(cur >= 0 ? cur + p1 : cur + m1);
                        changed |= 1ull << pos;
                    }
                }
                --eobrun;
            }
            // only this band's coefficients go back: a scan of the same level may be writing another band of the block
            while (changed) {
                const int pos = __ffsll((long long)changed) - 1;
                blk[pos] = s_blk[pos];
                changed &= changed - 1;
            }
        }
    }
    if (br.overrun()) err |= 2;
    int *st = status + 4 * sc.image;
    if (err) atomicOr(st, err);
    atomicAdd(st + 3, 1);
}

__global__ void __launch_bounds__(IDCT_THREADS) prog_idct_kernel(const uint8_t *__restrict__ blob, uint8_t *__restrict__ ws) {
    __shared__ int s_q[3][64];
    const ProgBlobHeader &H = phdr(blob);
    const ProgImg &im = pimgs(blob)[blockIdx.y];
    idct_image(im, ws + H.ws_coef + im.coef_offset, ws + H.ws_plane + im.plane_offset, s_q);
}

__global__ void __launch_bounds__(COLOR_THREADS) prog_color_kernel(const uint8_t *__restrict__ blob, const uint8_t *__restrict__ ws,
                                                                   uint8_t *__restrict__ dst) {
    const ProgBlobHeader &H = phdr(blob);
    const ProgImg &im = pimgs(blob)[blockIdx.y];
    color_image(im, ws + H.ws_plane + im.plane_offset, dst + im.dst_offset);
}

struct ProgPlan {
    Parsed p;
    ProgHook hook;
};

int parse_progressive(const uint8_t *d, size_t n, ProgPlan &pl, const char *who) {
    return parse_jpeg(d, n, pl.p, who, &pl.hook);
}

const ProgBlobHeader *check_prog_blob(const void *blob_host, const char *fn) {
    const ProgBlobHeader *H = static_cast<const ProgBlobHeader *>(blob_host);
    if (!H || H->magic != PROG_BLOB_MAGIC || H->n <= 0) {
        set_error("%s: not a descriptor blob made by k2y_jpeg_progressive_plan", fn);
        return nullptr;
    }
    return H;
}

}  // namespace
}  // namespace k2y

using namespace k2y;

extern "C" int k2y_jpeg_progressive_inspect(const unsigned char *data, size_t size, k2y_jpeg_progressive_info *info) {
    if (!data || !info) {
        set_error("k2y_jpeg_progressive_inspect: bad arguments");
        return K2Y_ERR_INVALID;
    }
    ProgPlan pl;
    const int rc = parse_progressive(data, size, pl, "k2y_jpeg_progressive_inspect");
    if (rc != K2Y_OK) return rc;
    const Parsed &p = pl.p;
    memset(info, 0, sizeof(*info));
    info->height = p.h;
    info->width = p.w;
    info->components = p.ncomp;
    info->sof_marker = p.sof;
    info->scans = pl.hook.nscans;
    info->levels = pl.hook.nlevel;
    info->gpu_decodable = p.gpu ? 1 : 0;
    snprintf(info->reason, sizeof(info->reason), "%s", p.gpu ? "" : p.reason);
    return K2Y_OK;
}

extern "C" int k2y_jpeg_progressive_plan(const unsigned char *const *files, const size_t *sizes, int n, const long long *src_offsets,
                                         const long long *dst_offsets, void *blob, size_t blob_capacity, size_t *blob_bytes) {
    if (!files || !sizes || n <= 0 || !blob_bytes || (blob && (!src_offsets || !dst_offsets))) {
        set_error("k2y_jpeg_progressive_plan: bad arguments");
        return K2Y_ERR_INVALID;
    }
    std::vector<ProgPlan> plans(n);
    long long nscan = 0, nseg = 0, ntab = 0;
    int nlevel = 0;
    for (int i = 0; i < n; ++i) {
        char who[64];
        snprintf(who, sizeof(who), "k2y_jpeg_progressive_plan: image %d", i);
        if (!files[i]) {
            set_error("%s: null file pointer", who);
            return K2Y_ERR_INVALID;
        }
        ProgPlan &pl = plans[i];
        const int rc = parse_progressive(files[i], sizes[i], pl, who);
        if (rc != K2Y_OK) return rc;
        if (!pl.p.gpu) {
            set_error("%s: not decodable on the GPU: %s", who, pl.p.reason);
            return K2Y_ERR_INVALID;
        }
        if (blob && (src_offsets[i] & 15)) {
            set_error("%s: source offset %lld is not a multiple of 16", who, src_offsets[i]);
            return K2Y_ERR_INVALID;
        }
        nlevel = std::max(nlevel, pl.hook.nlevel);
        for (const ScanRec &r : pl.hook.scans) {
            ++nscan;
            ntab += r.ntab;
        }
    }
    // geometry of every image and scan, then the segments
    const long long img_off = align16(sizeof(ProgBlobHeader));
    const long long scan_off = img_off + (long long)sizeof(ProgImg) * n;
    std::vector<ProgImg> I(n);
    std::vector<ProgScan> S;
    std::vector<ProgSeg> G;
    std::vector<JpegHuff> T;
    S.reserve(nscan);
    T.reserve(ntab);
    long long coef = 0, plane = 0, max_pixels = 0;
    int max_blocks = 0;
    for (int i = 0; i < n; ++i) {
        const Parsed &p = plans[i].p;
        ProgImg &im = I[i];
        memset(&im, 0, sizeof(im));
        im.src_offset = src_offsets ? src_offsets[i] : 0;
        im.dst_offset = dst_offsets ? dst_offsets[i] : 0;
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
        const int mcux = (p.w + 8 * hmax - 1) / (8 * hmax), mcuy = (p.h + 8 * vmax - 1) / (8 * vmax);
        int blocks = 0, pbytes = 0;
        for (int c = 0; c < p.ncomp; ++c) {
            im.bw[c] = mcux * hs[c];
            im.bh[c] = mcuy * vs[c];
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
        for (const ScanRec &r : plans[i].hook.scans) {
            ProgScan sc;
            memset(&sc, 0, sizeof(sc));
            sc.image = i;
            sc.ss = r.ss;
            sc.se = r.se;
            sc.ah = r.ah;
            sc.al = r.al;
            sc.huff_first = (int)T.size();
            sc.ntab = r.ntab;
            for (int k = 0; k < r.ntab; ++k) {
                T.emplace_back();
                derive_huff(r.tab[k], T.back());
            }
            long long mcus;
            if (r.ns == 1) {   // non-interleaved: one block per MCU over the component's own ceil(dw/8) x ceil(dh/8)
                const int c = r.comp[0];
                sc.mcux = (im.dw[c] + 7) / 8;
                mcus = (long long)sc.mcux * ((im.dh[c] + 7) / 8);
                for (int f = 0; f < 3; ++f) sc.hs[f] = sc.vs[f] = 1;
                sc.bpm = 1;
                sc.mcu_comp[0] = (uint8_t)c;
            } else {
                sc.mcux = mcux;
                mcus = (long long)mcux * mcuy;
                for (int f = 0; f < 3; ++f) {
                    sc.hs[f] = hs[f];
                    sc.vs[f] = vs[f];
                }
                int bpm = 0;
                for (int k = 0; k < r.ns; ++k) {
                    const int f = r.comp[k];
                    for (int by = 0; by < vs[f]; ++by)
                        for (int bx = 0; bx < hs[f]; ++bx) {
                            sc.mcu_comp[bpm] = (uint8_t)f;
                            sc.mcu_bx[bpm] = (uint8_t)bx;
                            sc.mcu_by[bpm] = (uint8_t)by;
                            sc.mcu_tab[bpm] = (uint8_t)k;
                            ++bpm;
                        }
                }
                sc.bpm = bpm;
            }
            const long long per = r.restart ? r.restart : mcus;
            const long long segs = (mcus + per - 1) / per;
            const size_t found = r.bounds.size() / 2;   // segments the data holds; missing ones are empty
            for (long long k = 0; k < segs; ++k) {
                ProgSeg g;
                g.scan = (int)S.size();
                g.first_mcu = (int)(k * per);
                g.mcus = (int)std::min(per, mcus - k * per);
                g.level = r.level;
                g.begin = k < (long long)found ? r.bounds[2 * k] : r.bounds.back();
                g.end = k < (long long)found ? r.bounds[2 * k + 1] : r.bounds.back();
                G.push_back(g);
            }
            S.push_back(sc);
        }
        im.coef_offset = coef;
        coef += (long long)blocks * 128;
        im.plane_offset = plane;
        plane += pbytes;
        max_blocks = std::max(max_blocks, blocks);
        max_pixels = std::max(max_pixels, (long long)p.h * p.w);
    }
    nseg = (long long)G.size();
    if (nseg > INT_MAX / 2) {
        set_error("k2y_jpeg_progressive_plan: %lld segments in one batch", nseg);
        return K2Y_ERR_INVALID;
    }
    const long long seg_off = align16(scan_off + (long long)sizeof(ProgScan) * nscan);
    const long long huff_off = align16(seg_off + (long long)sizeof(ProgSeg) * nseg);
    const long long total = huff_off + (long long)sizeof(JpegHuff) * ntab;
    *blob_bytes = (size_t)total;
    if (!blob) return K2Y_OK;
    if (blob_capacity < (size_t)total || ((uintptr_t)blob & 15)) {
        set_error("k2y_jpeg_progressive_plan: the blob needs %lld bytes at a 16-byte aligned address, got %zu", total, blob_capacity);
        return K2Y_ERR_INVALID;
    }
    uint8_t *B = static_cast<uint8_t *>(blob);
    memset(B, 0, (size_t)total);
    ProgBlobHeader &H = *reinterpret_cast<ProgBlobHeader *>(B);
    memcpy(B + img_off, I.data(), sizeof(ProgImg) * n);
    memcpy(B + scan_off, S.data(), sizeof(ProgScan) * nscan);
    ProgSeg *segs = reinterpret_cast<ProgSeg *>(B + seg_off);
    int at = 0;
    for (int l = 0; l < nlevel; ++l) {   // segments grouped by level
        H.level_seg[l] = at;
        for (const ProgSeg &g : G)
            if (g.level == l) segs[at++] = g;
    }
    H.level_seg[nlevel] = at;
    if (ntab) memcpy(B + huff_off, T.data(), sizeof(JpegHuff) * ntab);
    H.magic = PROG_BLOB_MAGIC;
    H.n = n;
    H.nscan = (int)nscan;
    H.nseg = (int)nseg;
    H.ntab = (int)ntab;
    H.nlevel = nlevel;
    H.max_blocks = max_blocks;
    H.max_pixels = max_pixels;
    H.img_off = img_off;
    H.scan_off = scan_off;
    H.seg_off = seg_off;
    H.huff_off = huff_off;
    H.blob_bytes = total;
    H.ws_coef = 0;
    H.ws_plane = align16(coef);
    H.ws_bytes = H.ws_plane + align16(plane);
    return K2Y_OK;
}

extern "C" int k2y_jpeg_progressive_workspace_bytes(const void *blob_host, size_t *bytes) {
    const ProgBlobHeader *H = check_prog_blob(blob_host, "k2y_jpeg_progressive_workspace_bytes");
    if (!H || !bytes) {
        if (H) set_error("k2y_jpeg_progressive_workspace_bytes: bad arguments");
        return K2Y_ERR_INVALID;
    }
    *bytes = (size_t)H->ws_bytes;
    return K2Y_OK;
}

extern "C" int k2y_jpeg_progressive_decode(const void *blob_host, const void *blob_dev, const unsigned char *src_dev,
                                           unsigned char *dst_dev, void *workspace_dev, size_t workspace_bytes, int32_t *status_dev,
                                           void *stream) {
    const ProgBlobHeader *H = check_prog_blob(blob_host, "k2y_jpeg_progressive_decode");
    if (!H) return K2Y_ERR_INVALID;
    if (!blob_dev || !src_dev || !dst_dev || !workspace_dev || !status_dev || ((uintptr_t)blob_dev & 15) || ((uintptr_t)src_dev & 15) ||
        ((uintptr_t)workspace_dev & 15) || workspace_bytes < (size_t)H->ws_bytes) {
        set_error("k2y_jpeg_progressive_decode: bad arguments (16-byte aligned blob, source and workspace of %lld bytes needed, "
                  "got %zu)", H->ws_bytes, workspace_bytes);
        return K2Y_ERR_INVALID;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const uint8_t *blob = static_cast<const uint8_t *>(blob_dev);
    uint8_t *ws = static_cast<uint8_t *>(workspace_dev);
    K2Y_CUDA_CHECK(cudaMemsetAsync(status_dev, 0, sizeof(int32_t) * 4 * (size_t)H->n, st));
    K2Y_CUDA_CHECK(cudaMemsetAsync(ws + H->ws_coef, 0, (size_t)(H->ws_plane - H->ws_coef), st));
    for (int l = 0; l < H->nlevel; ++l) {
        const int count = H->level_seg[l + 1] - H->level_seg[l];
        if (count > 0) prog_entropy_kernel<<<count, 1, 0, st>>>(blob, src_dev, ws, status_dev, H->level_seg[l]);
    }
    prog_idct_kernel<<<dim3((unsigned)((H->max_blocks + IDCT_THREADS - 1) / IDCT_THREADS), H->n), IDCT_THREADS, 0, st>>>(blob, ws);
    prog_color_kernel<<<dim3((unsigned)((H->max_pixels + COLOR_THREADS - 1) / COLOR_THREADS), H->n), COLOR_THREADS, 0, st>>>(blob, ws,
                                                                                                                          dst_dev);
    K2Y_CUDA_CHECK(cudaGetLastError());
    return K2Y_OK;
}
