// PNG decode on the device, in front of the batch letterbox: the pixels Helper._read_img (PIL) gives for non-interlaced
// PNGs of every colour type and depth except 16-bit greyscale.
//
// Host side: parse_png walks the chunks (CRCs of the chunks before the first IDAT, the IDAT run, IEND) and decides the route;
// k2y_png_plan writes the descriptor blob: per image its IDAT payload ranges, its zlib stream and inflated-row ranges in the
// workspace, its geometry and palette.  Device side, one launch per stage whatever the image count:
//   png_gather_kernel    one CTA per image copies the IDAT payloads into one contiguous zlib stream;
//   png_find_kernel      one CTA per 64 KiB chunk of compressed data after the first finds the first bit where a block header
//                        parses strictly (strict_header): the chunk's speculative start;
//   png_chunk_kernel     one warp per chunk decodes from its start into 16-bit symbols (a byte, or a reference into the 32 KiB
//                        before the chunk's first output) until it stands on a later chunk's start at a block boundary;
//   png_resolve_kernel   one CTA per image follows those links from the stream's start (the chain is the serial decode, since
//                        decoding from a true block boundary is deterministic), resolves the references chunk by chunk into the
//                        filtered rows and checks the Adler-32;
//   png_inflate_kernel   one thread per image whose chain did not decode it inflates the stream serially (RFC 1950/1951),
//                        stopping where zlib, as PIL drives it, stops: PIL's reads of the IDAT data bound the tail it checks
//                        (see inflate_image);
//   png_unfilter_kernel  one CTA per image undoes the row filters as a diagonal wavefront (row r handles its unit x at step
//                        x + r, so Up / Avg / Paeth always find their upper and upper-left bytes done) and writes HWC RGB at
//                        the image's output offset, with sub-byte unpacking, palette, grey replication, 16-bit high bytes and
//                        alpha dropping fused into the write.  Rows the stream never filled are decoded from zero bytes, which
//                        is what PIL's zero-initialised image holds.
// Corrupt data only sets status bits: every read stays inside the image's stream (bounds-checked bit reader) and every write
// inside its inflated rows and its output pixels.
#include <algorithm>
#include <vector>

#include "common.h"

namespace k2y {
namespace {

constexpr uint32_t PNG_BLOB_MAGIC = 0x504e4742u;   // "PNGB"
constexpr int GATHER_THREADS = 256;
constexpr int UNFILTER_THREADS = 1024;
constexpr int PNG_MAX_DIMENSION = 65535;   // rows / columns the GPU route takes (larger files go to PIL)
constexpr int FAST_BITS = 10;              // first-level Huffman lookup (longer codes are decoded canonically)
constexpr int WINDOW = 32768;
constexpr int CHUNK_BYTES = 65536;         // compressed bytes per speculative chunk (more for streams of over MAX_CHUNKS chunks)
constexpr int MAX_CHUNKS = 4096;           // chunks per image
constexpr int FIND_THREADS = 256;
constexpr int CHUNK_THREADS = 32;
constexpr int RESOLVE_THREADS = 1024;
constexpr long long CHUNK_SYMBOLS = 4LL * CHUNK_BYTES + 131072;   // output capacity of a speculative chunk (symbols)
constexpr long long MAX_RAW_BYTES = (1LL << 31) - 1;              // filtered bytes of one image the GPU takes
constexpr long long PIL_READ = 65536;      // most IDAT bytes PIL hands zlib at once (ImageFile.MAXBLOCK)
enum : int32_t { CHUNK_FINAL = 1, CHUNK_FAILED = 2 };

enum : int32_t {
    PNG_ERR_HEADER = 1,     // invalid block type, stored LEN/NLEN mismatch or invalid dynamic block header
    PNG_ERR_CODE = 2,       // invalid literal/length or distance code
    PNG_ERR_DISTANCE = 4,   // distance reaches before the start of the stream
    PNG_ERR_TRUNCATED = 8,  // the image data ends early where PIL refuses that
    PNG_ERR_ADLER = 16,     // Adler-32 mismatch
    PNG_ERR_FILTER = 32,    // filter type byte above 4
};

struct alignas(16) PngImg {
    long long stream_off, stream_len;   // zlib stream (payload of every IDAT) in the workspace
    long long raw_off, raw_len;         // filtered rows in the workspace: h * (1 + rowbytes)
    long long dst_offset;               // h * w * 3 RGB bytes in the output buffer
    int32_t h, w, color, depth, rowbytes, unit;   // unit: bytes of one wavefront step (bytes per pixel, at least 1)
    int32_t seg_first, nseg, plte_n, pad;
    long long prod_off;                 // workspace: int64 bytes inflated, int64 "the chunk chain decoded the image" flag
    long long chunk_bytes;              // compressed bytes per chunk
    int32_t chunk_first, nchunks;
    long long piece_first, npiece;      // PIL's reads of the stream: their end offsets in the blob's piece array
    uint8_t plte[768];
};

struct alignas(16) PngChunk {
    long long buf_off, cap;             // uint16 symbols of the chunk's decode in the workspace, and their capacity
    long long meta_off;                 // its ChunkMeta in the workspace
    int32_t image, index;               // image and chunk within it
};

struct alignas(16) ChunkMeta {
    long long cand;                     // bit where the chunk's decode starts: the first strict block header found, -1 none
    long long len;                      // symbols decoded
    long long end_bit;                  // bit after the final block (CHUNK_FINAL)
    int32_t next, flags;                // chunk whose candidate the decode reached at a block boundary (-1 none), CHUNK_*
};

struct alignas(16) PngSeg {
    long long src, len, dst;            // IDAT payload in the source buffer -> offset in the image's stream
    long long pad;
};

struct alignas(16) PngBlobHeader {
    uint32_t magic;
    int32_t n, nseg, nchunks;
    long long img_off, seg_off, chunk_off, blob_bytes, ws_bytes;
    long long piece_off, npieces;
};

long long align16(long long v) { return (v + 15) & ~15LL; }

uint32_t crc32_of(const uint8_t *p, size_t n) {
    static uint32_t table[256];
    static bool ready = false;
    if (!ready) {
        for (uint32_t i = 0; i < 256; ++i) {
            uint32_t c = i;
            for (int k = 0; k < 8; ++k) c = c & 1 ? 0xEDB88320u ^ (c >> 1) : c >> 1;
            table[i] = c;
        }
        ready = true;
    }
    uint32_t c = 0xFFFFFFFFu;
    for (size_t i = 0; i < n; ++i) c = table[(c ^ p[i]) & 0xFF] ^ (c >> 8);
    return c ^ 0xFFFFFFFFu;
}

uint32_t be32(const uint8_t *p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }

struct PngParsed {
    int h = 0, w = 0, color = 0, depth = 0, interlace = 0;
    int plte_n = 0;
    uint8_t plte[768] = {};
    std::vector<std::pair<long long, long long>> idat;   // (payload offset, length) in the file
    long long stream_len = 0;
    bool gpu = false;
    char reason[64] = {};
};

int channels_of(int color) { return color == 0 ? 1 : color == 2 ? 3 : color == 3 ? 1 : color == 4 ? 2 : 4; }

bool valid_depth(int color, int depth) {
    switch (color) {
        case 0: return depth == 1 || depth == 2 || depth == 4 || depth == 8 || depth == 16;
        case 3: return depth == 1 || depth == 2 || depth == 4 || depth == 8;
        case 2: case 4: case 6: return depth == 8 || depth == 16;
        default: return false;
    }
}

// K2Y_ERR_INVALID for what is not a PNG with a sound IHDR; otherwise K2Y_OK with p.gpu and p.reason.
int parse_png(const uint8_t *d, size_t size, PngParsed &p, const char *who) {
    static const uint8_t sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1A, '\n'};
    if (size < 8 + 25 || memcmp(d, sig, 8) != 0) {
        set_error("%s: not a PNG file", who);
        return K2Y_ERR_INVALID;
    }
    if (be32(d + 8) != 13 || memcmp(d + 12, "IHDR", 4) != 0 || crc32_of(d + 12, 17) != be32(d + 29)) {
        set_error("%s: the file does not start with a sound IHDR chunk", who);
        return K2Y_ERR_INVALID;
    }
    const uint8_t *ih = d + 16;
    const uint32_t w = be32(ih), h = be32(ih + 4);
    p.depth = ih[8];
    p.color = ih[9];
    p.interlace = ih[12];
    if (w == 0 || h == 0 || w > 0x7FFFFFFFu || h > 0x7FFFFFFFu || !valid_depth(p.color, p.depth) || ih[10] != 0 || ih[11] != 0 ||
        p.interlace > 1) {
        set_error("%s: invalid IHDR (%ux%u, colour type %d, depth %d)", who, w, h, p.color, p.depth);
        return K2Y_ERR_INVALID;
    }
    p.w = (int)std::min<uint32_t>(w, 0x7FFFFFFF);
    p.h = (int)std::min<uint32_t>(h, 0x7FFFFFFF);
    auto refuse = [&](const char *why) {
        snprintf(p.reason, sizeof(p.reason), "%s", why);
        p.gpu = false;
        return K2Y_OK;
    };
    if (p.interlace) return refuse("interlaced (Adam7)");
    if (p.color == 0 && p.depth == 16) return refuse("16-bit greyscale");
    if (w > (uint32_t)PNG_MAX_DIMENSION || h > (uint32_t)PNG_MAX_DIMENSION) return refuse("more than 65535 rows or columns");
    if ((long long)h * (1 + (((long long)w * channels_of(p.color) * p.depth + 7) / 8)) > MAX_RAW_BYTES)
        return refuse("more than 2 GiB of filtered image data");
    size_t pos = 33;
    bool seen_plte = false, in_idat = false, after_idat = false;
    char why[64];
    while (true) {
        if (pos + 12 > size) return refuse(p.idat.empty() ? "no IDAT chunk" : "no IEND chunk");
        const uint32_t len = be32(d + pos);
        const uint8_t *type = d + pos + 4;
        if (len > 0x7FFFFFFFu || pos + 12 + (size_t)len > size) return refuse(p.idat.empty() ? "damaged chunk before IDAT" : "no IEND chunk");
        const bool is_idat = memcmp(type, "IDAT", 4) == 0, is_iend = memcmp(type, "IEND", 4) == 0;
        if (is_iend) {
            if (p.idat.empty()) return refuse("no IDAT chunk");
            break;
        }
        if (is_idat) {
            if (after_idat) return refuse("chunk between IDAT chunks");
            in_idat = true;
            p.idat.push_back({(long long)pos + 8, (long long)len});
            p.stream_len += len;
        } else {
            if (in_idat) {
                in_idat = false;
                after_idat = true;
            }
            if (!after_idat) {
                if (crc32_of(type, 4 + (size_t)len) != be32(d + pos + 8 + len)) {
                    snprintf(why, sizeof(why), "CRC error in %.4s chunk", (const char *)type);
                    return refuse(why);
                }
                if (memcmp(type, "acTL", 4) == 0) return refuse("APNG (acTL chunk)");
                if (memcmp(type, "PLTE", 4) == 0) {
                    if (seen_plte || len == 0 || len % 3 || len > 768 || p.color == 0 || p.color == 4) return refuse("damaged PLTE chunk");
                    seen_plte = true;
                    p.plte_n = (int)(len / 3);
                    memcpy(p.plte, d + pos + 8, len);
                } else if (!(type[0] & 0x20) && memcmp(type, "IHDR", 4) != 0) {
                    snprintf(why, sizeof(why), "unknown critical chunk %.4s", (const char *)type);
                    return refuse(why);
                } else if (memcmp(type, "IHDR", 4) == 0) {
                    return refuse("second IHDR chunk");
                }
            }
        }
        pos += 12 + (size_t)len;
    }
    if (p.color == 3 && !seen_plte) return refuse("palette image without PLTE");
    // zlib header: CM = 8, CINFO <= 7, no preset dictionary, FCHECK
    uint8_t zh[2];
    int got = 0;
    for (auto &c : p.idat)
        for (long long k = 0; k < c.second && got < 2; ++k) zh[got++] = d[c.first + k];
    if (got < 2) return refuse("zlib stream shorter than its header");
    if ((zh[0] & 15) != 8 || (zh[0] >> 4) > 7 || (zh[1] & 0x20) || ((zh[0] << 8) | zh[1]) % 31) return refuse("unsupported zlib header");
    p.gpu = true;
    return K2Y_OK;
}

int row_bytes(const PngParsed &p) { return (int)(((long long)p.w * channels_of(p.color) * p.depth + 7) / 8); }

// ---------------------------------------------------------------------------------------------------------------------
// device

__global__ void __launch_bounds__(GATHER_THREADS) png_gather_kernel(const uint8_t *__restrict__ blob, const uint8_t *__restrict__ src,
                                                                    uint8_t *__restrict__ ws) {
    const PngBlobHeader &H = *reinterpret_cast<const PngBlobHeader *>(blob);
    const PngImg &im = reinterpret_cast<const PngImg *>(blob + H.img_off)[blockIdx.x];
    const PngSeg *seg = reinterpret_cast<const PngSeg *>(blob + H.seg_off) + im.seg_first;
    uint8_t *dst = ws + im.stream_off;
    for (int s = 0; s < im.nseg; ++s) {
        const uint8_t *a = src + seg[s].src;
        uint8_t *b = dst + seg[s].dst;
        for (long long k = threadIdx.x; k < seg[s].len; k += GATHER_THREADS) b[k] = a[k];
    }
    if (threadIdx.x < 8) dst[im.stream_len + threadIdx.x] = 0;    // the bit reader's look-ahead past the end reads zeros
}

struct Bits {
    const uint8_t *p;
    long long total;    // bits in the stream
    long long pos;      // bits consumed
    uint64_t buf;       // bits from `pos` on (valid: `cnt`)
    int cnt;
    long long next;     // next byte to load

    __device__ __forceinline__ void fill() {
        while (cnt <= 56) {
            // the stream is followed by 8 zero bytes in the workspace; past those the buffer is padded with zeros
            const uint64_t b = next < (total >> 3) + 8 ? __ldg(p + next) : 0;
            buf |= b << cnt;
            cnt += 8;
            ++next;
        }
    }
    __device__ __forceinline__ uint32_t peek(int n) {
        fill();
        return (uint32_t)(buf & ((1ull << n) - 1));
    }
    __device__ __forceinline__ void drop(int n) {
        buf >>= n;
        cnt -= n;
        pos += n;
    }
    __device__ __forceinline__ bool has(int n) const { return pos + n <= total; }
    // positions the reader at bit `bit` of the stream (`total` bits, followed by 8 zero bytes)
    __device__ __forceinline__ void start(const uint8_t *stream, long long total_bits, long long bit) {
        p = stream;
        total = total_bits;
        next = bit >> 3;
        pos = bit & ~7LL;
        buf = 0;
        cnt = 0;
        fill();
        drop((int)(bit & 7));
    }
    __device__ __forceinline__ void align() { drop((int)((8 - (pos & 7)) & 7)); }
};

// Canonical Huffman code: lengths 0..15 of `n` symbols.  fast[] maps the next FAST_BITS bits to (symbol << 4 | length) for codes
// of at most FAST_BITS bits, 0 otherwise (longer or unassigned codes: decoded canonically from count / sym).
struct Huff {
    uint16_t fast[1 << FAST_BITS];
    uint16_t count[16];
    uint16_t sym[288];
    uint16_t maxlen;        // longest code (0: no code)
};

// Returns 0 for a usable code, -1 for an over-subscribed one, 1 for an incomplete one (`left` > 0 codes unused).
__device__ int build_huff(Huff &hf, const uint8_t *len, int n) {
    for (int i = 0; i < 16; ++i) hf.count[i] = 0;
    for (int i = 0; i < n; ++i) hf.count[len[i]]++;
    hf.count[0] = 0;
    hf.maxlen = 0;
    for (int l = 1; l < 16; ++l)
        if (hf.count[l]) hf.maxlen = (uint16_t)l;
    int left = 1;
    for (int l = 1; l < 16; ++l) {
        left = (left << 1) - hf.count[l];
        if (left < 0) return -1;
    }
    uint16_t offs[16];
    offs[1] = 0;
    for (int l = 1; l < 15; ++l) offs[l + 1] = offs[l] + hf.count[l];
    for (int i = 0; i < n; ++i)
        if (len[i]) hf.sym[offs[len[i]]++] = (uint16_t)i;
    for (int i = 0; i < (1 << FAST_BITS); ++i) hf.fast[i] = 0;
    int code = 0, k = 0;
    for (int l = 1; l <= FAST_BITS; ++l) {
        for (int c = 0; c < hf.count[l]; ++c, ++k, ++code) {
            int rev = 0;
            for (int b = 0; b < l; ++b) rev |= ((code >> b) & 1) << (l - 1 - b);
            for (int f = rev; f < (1 << FAST_BITS); f += 1 << l) hf.fast[f] = (uint16_t)(hf.sym[k] << 4 | l);
        }
        code <<= 1;
    }
    return left > 0 ? 1 : 0;
}

// Next symbol: >= 0, -1 invalid code, -2 the code needs bits past the end of the stream.  As in zlib, a code is invalid as soon
// as the bits read rule out every code (the one-bit code's other bit, any first bit of an empty code), not only after 15 bits.
__device__ __forceinline__ int decode_sym(Bits &br, const Huff &hf) {
    const uint32_t look = br.peek(15);
    const uint16_t e = hf.fast[look & ((1 << FAST_BITS) - 1)];
    if (e) {
        const int l = e & 15;
        if (!br.has(l)) return -2;
        br.drop(l);
        return e >> 4;
    }
    int code = 0, first = 0, index = 0;
    for (int l = 1; l < 16; ++l) {
        code |= (look >> (l - 1)) & 1;
        const int c = hf.count[l];
        if (code - c < first) {
            if (!br.has(l)) return -2;
            br.drop(l);
            return hf.sym[index + (code - first)];
        }
        if (l >= hf.maxlen) return br.has(l) ? -1 : -2;
        index += c;
        first = (first + c) << 1;
        code <<= 1;
    }
    return -1;
}

__constant__ uint16_t c_lbase[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t c_lext[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t c_dbase[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073,
                                     4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t c_dext[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t c_clorder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// Reads a dynamic block header into `lit` / `dist`: 0 ok, PNG_ERR_HEADER, or -2 when the stream ends inside it.  zlib's rules:
// HLIT <= 286, HDIST <= 30, a complete code-length code, no repeat of a missing length or past the end, an end-of-block code, and
// literal/length and distance codes that are complete or a single code of one bit (an empty distance code is allowed; using it
// is an invalid distance code).
__device__ __forceinline__ int read_dynamic(Bits &br, Huff &lit, Huff &dist, uint8_t *lens) {
    if (!br.has(14)) return -2;
    const int nlen = (int)br.peek(5) + 257;
    br.drop(5);
    const int ndist = (int)br.peek(5) + 1;
    br.drop(5);
    const int ncode = (int)br.peek(4) + 4;
    br.drop(4);
    if (nlen > 286 || ndist > 30) return PNG_ERR_HEADER;
    uint8_t cl[19];
    for (int i = 0; i < 19; ++i) cl[i] = 0;
    for (int i = 0; i < ncode; ++i) {
        if (!br.has(3)) return -2;
        cl[c_clorder[i]] = (uint8_t)br.peek(3);
        br.drop(3);
    }
    const int rc = build_huff(lit, cl, 19);
    if (rc < 0 || (rc > 0 && lit.maxlen)) return PNG_ERR_HEADER;    // the code-length code must be complete
    // all zero: zlib reads every code length as a 0 of one bit, then finds no end-of-block code
    if (rc > 0) return br.has(nlen + ndist) ? PNG_ERR_HEADER : -2;
    for (int i = 0; i < nlen + ndist;) {
        const int s = decode_sym(br, lit);
        if (s == -2) return -2;
        if (s < 0) return PNG_ERR_HEADER;
        if (s < 16) {
            lens[i++] = (uint8_t)s;
            continue;
        }
        int rep, val = 0;
        if (s == 16) {
            if (!br.has(2)) return -2;      // zlib reads the repeat count before it refuses a first repeat
            if (i == 0) return PNG_ERR_HEADER;
            val = lens[i - 1];
            rep = 3 + (int)br.peek(2);
            br.drop(2);
        } else if (s == 17) {
            if (!br.has(3)) return -2;
            rep = 3 + (int)br.peek(3);
            br.drop(3);
        } else {
            if (!br.has(7)) return -2;
            rep = 11 + (int)br.peek(7);
            br.drop(7);
        }
        if (i + rep > nlen + ndist) return PNG_ERR_HEADER;
        while (rep--) lens[i++] = (uint8_t)val;
    }
    if (lens[256] == 0) return PNG_ERR_HEADER;
    int max_l = 0;
    for (int i = 0; i < nlen; ++i) max_l = max(max_l, (int)lens[i]);
    int r = build_huff(lit, lens, nlen);
    if (r < 0 || (r > 0 && max_l != 1)) return PNG_ERR_HEADER;
    max_l = 0;
    for (int i = 0; i < ndist; ++i) max_l = max(max_l, (int)lens[nlen + i]);
    r = build_huff(dist, lens + nlen, ndist);
    if (r < 0 || (r > 0 && max_l > 1)) return PNG_ERR_HEADER;
    return 0;
}

__device__ void fixed_tables(Huff &lit, Huff &dist, uint8_t *lens) {
    for (int i = 0; i < 288; ++i) lens[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8;
    build_huff(lit, lens, 288);
    for (int i = 0; i < 32; ++i) lens[i] = 5;    // codes 30 and 31 decode, and are then refused as invalid distance codes
    build_huff(dist, lens, 32);
}

// Inflates one image's zlib stream into its `total` filtered bytes, stopping where zlib stops as PIL drives it.  PIL hands zlib
// the stream one read at a time (each IDAT in pieces of at most 64 KiB from its start: `ends`) with one row of output room per
// call, and stops after the call that completes the last row.  So once the image's last byte is written, decoding goes on only
// through the rest of the read that call was fed and only until zlib would have to write another byte (a literal, a match with
// a valid distance code, or a non-empty stored block), still checking end-of-block codes, block headers, stored LEN / NLEN and
// the Adler-32; an invalid code there is an error, a distance too far back is not (zlib checks it only when it has room to
// copy).  A symbol decoded in the call that filled a row waits for the next call, which is fed the next read when that call
// used up its own; with no read left PIL finds the file truncated.  A stream that ends early leaves the rest of the image
// unwritten: PIL accepts that only when the call that wrote the last row also read the final block's Adler-32, after at least
// one row.  Status: [0] error bits, [3] bytes written.
__device__ void inflate_image(const PngImg &im, const uint8_t *stream, const long long *ends, uint8_t *out, int32_t *status,
                              long long *produced, uint8_t *win, Huff &lit, Huff &dist, uint8_t *lens) {
    Bits br;
    br.start(stream, im.stream_len * 8, 16);     // past the zlib header, which the host checked
    const long long total = im.raw_len, row = 1 + (long long)im.rowbytes;
    long long o = 0;
    int err = 0;
    uint32_t a1 = 1, a2 = 0;     // Adler-32 of everything written (bytes past `total` are never written)
    int since = 0;               // bytes added to a1 / a2 since the last modulo reduction
    auto put = [&](uint8_t b) {
        out[o] = b;
        win[o & (WINDOW - 1)] = b;
        ++o;
        a1 += b;
        a2 += a1;
        if (++since == 5552) {
            a1 %= 65521u;
            a2 %= 65521u;
            since = 0;
        }
    };
    long long pc = 0, lim = ends[0];     // the read the zlib call writing at `o` is fed, and its end in the stream
    bool stranded = false;               // a call waited for a read that does not exist
    // Before a symbol's first byte at `o` (n bytes, of which those past `total` are never written): the read its call is fed.
    auto place = [&](long long n) {
        const long long q = (br.pos + 7) >> 3;     // bytes zlib has taken in
        const bool fresh = q > lim;                 // decoded in a later read's call, which has room
        while (q > lim) lim = ends[++pc];
        const bool waits = (!fresh && o > 0 && o % row == 0) || (o / row + 1) * row < o + min(n, total - o);
        if (waits && q == lim) {
            if (pc + 1 < im.npiece) lim = ends[++pc];
            else stranded = true;
        }
    };
    // once the image is complete, nothing past the read that completed it is checked
    auto done = [&]() {
        if (o == total) br.total = min(br.total, lim * 8);
    };
    bool last = false, ended = false;     // ended: the final block and a matching Adler-32 were read
    while (!err) {
        if (last) {             // end of the stream: the Adler-32, big-endian, byte aligned
            br.align();
            if (br.has(32)) {
                uint32_t v = 0;
                for (int k = 0; k < 4; ++k) {
                    v = v << 8 | br.peek(8);
                    br.drop(8);
                }
                if (v != ((a2 % 65521u) << 16 | (a1 % 65521u))) err |= PNG_ERR_ADLER;
                ended = (br.pos >> 3) <= lim;
            }
            break;
        }
        if (!br.has(3)) break;
        last = br.peek(1);
        const int type = (int)(br.peek(3) >> 1);
        br.drop(3);
        if (type == 3) {
            err |= PNG_ERR_HEADER;
            break;
        }
        if (type == 0) {
            br.align();
            if (!br.has(32)) break;
            const uint32_t len = br.peek(16);
            br.drop(16);
            const uint32_t nlen = br.peek(16);
            br.drop(16);
            if (len != (~nlen & 0xFFFF)) {
                err |= PNG_ERR_HEADER;
                break;
            }
            if (len && o >= total) break;
            bool cut = false;      // input or image space ran out inside the stored block
            for (uint32_t k = 0; k < len; ++k) {
                if (!br.has(8) || o >= total) {
                    cut = true;
                    break;
                }
                // a stored byte is written by the call fed the read that holds it
                while ((br.pos >> 3) + 1 > lim) lim = ends[++pc];
                put((uint8_t)br.peek(8));
                br.drop(8);
                done();
            }
            if (cut) break;
            continue;
        }
        if (type == 1) {
            fixed_tables(lit, dist, lens);
        } else {
            const int r = read_dynamic(br, lit, dist, lens);
            if (r == -2) break;
            if (r) {
                err |= r;
                break;
            }
        }
        bool stop = false;
        while (true) {
            const int s = decode_sym(br, lit);
            if (s == -2) {
                stop = true;
                break;
            }
            if (s < 0 || s > 285) {
                err |= PNG_ERR_CODE;
                break;
            }
            if (s < 256) {
                if (o >= total) {
                    stop = true;
                    break;
                }
                place(1);
                put((uint8_t)s);
                done();
                continue;
            }
            if (s == 256) break;
            const int li = s - 257;
            if (!br.has(c_lext[li])) {
                stop = true;
                break;
            }
            const int length = c_lbase[li] + (int)br.peek(c_lext[li]);
            br.drop(c_lext[li]);
            const int ds = decode_sym(br, dist);
            if (ds == -2) {
                stop = true;
                break;
            }
            if (ds < 0 || ds > 29) {
                err |= PNG_ERR_CODE;
                break;
            }
            if (!br.has(c_dext[ds])) {
                stop = true;
                break;
            }
            const int d = c_dbase[ds] + (int)br.peek(c_dext[ds]);
            br.drop(c_dext[ds]);
            if (o >= total) {       // zlib checks the distance against the output only when it has room to copy
                stop = true;
                break;
            }
            if (d > o) {
                err |= PNG_ERR_DISTANCE;
                break;
            }
            place(length);
            const int n = (int)min((long long)length, total - o);
            for (int k = 0; k < n; ++k) put(win[(o - d) & (WINDOW - 1)]);
            done();
            if (n < length) {
                stop = true;
                break;
            }
        }
        if (stop) break;
    }
    // an image left incomplete decodes only when its stream ended cleanly after at least one whole row (and on a row boundary)
    if (!err && (stranded || (o < total && (!ended || o == 0 || o % row)))) err |= PNG_ERR_TRUNCATED;
    status[0] |= err;
    status[3] = (int32_t)o;     // every byte decoded serially (o < 2^31: the host refuses larger images)
    *produced = o;
}

// Reads a stored block's zero padding and LEN / NLEN behind its 3 header bits; the block's length, or -1.
__device__ long long stored_len(Bits &br) {
    const int pad = (int)((8 - (br.pos & 7)) & 7);
    if (br.peek(pad) != 0) return -1;
    br.drop(pad);
    if (!br.has(32)) return -1;
    const uint32_t v = br.peek(32);
    br.drop(32);
    return (v & 0xFFFF) == (~(v >> 16) & 0xFFFF) ? (long long)(v & 0xFFFF) : -1;
}

__device__ bool strict_dynamic(Bits &br);

// Speculative chunk search: the first bit of chunk k's range where a block header parses strictly.  Dynamic: HLIT <= 286,
// HDIST <= 30, a complete code-length code, code lengths that decode with valid repeats, an end-of-block code, a literal/length
// code that is complete (or one code of one bit) and a distance code that is complete, empty or one code of one bit.  Stored:
// zero padding to the byte boundary, LEN == ~NLEN and a header that parses behind the stored bytes.  Fixed-Huffman blocks cannot be told from noise and are never found.
__device__ bool strict_header(const uint8_t *stream, long long total, long long bit) {
    Bits br;
    br.start(stream, total, bit);
    if (!br.has(3)) return false;
    int type = (int)(br.peek(3) >> 1);
    br.drop(3);
    if (type == 2) return strict_dynamic(br);
    if (type != 0) return false;
    const long long len = stored_len(br);
    if (len < 0) return false;
    // LEN == ~NLEN alone matches one offset in 2^16 of random data: the header behind the stored bytes must parse too
    const long long after = br.pos + 8 * len;
    if (after + 3 > total) return true;
    br.start(stream, total, after);
    type = (int)(br.peek(3) >> 1);
    br.drop(3);
    if (type == 0) return stored_len(br) >= 0;
    if (type == 2) return strict_dynamic(br);
    return type == 1;
}

__device__ bool strict_dynamic(Bits &br) {
    if (!br.has(14)) return false;
    const int nlen = (int)br.peek(5) + 257;
    br.drop(5);
    const int ndist = (int)br.peek(5) + 1;
    br.drop(5);
    const int ncode = (int)br.peek(4) + 4;
    br.drop(4);
    if (nlen > 286 || ndist > 30 || !br.has(3 * ncode)) return false;
    uint8_t cl[19];
    int cnt[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 19; ++i) cl[i] = 0;
    for (int i = 0; i < ncode; ++i) {
        cl[c_clorder[i]] = (uint8_t)br.peek(3);
        br.drop(3);
    }
    for (int i = 0; i < 19; ++i) cnt[cl[i]]++;
    int left = 1;
    for (int l = 1; l < 8; ++l) left = (left << 1) - cnt[l];
    if (left != 0) return false;
    uint8_t sym[19];
    int offs[8];
    offs[1] = 0;
    for (int l = 1; l < 7; ++l) offs[l + 1] = offs[l] + cnt[l];
    for (int i = 0; i < 19; ++i)
        if (cl[i]) sym[offs[cl[i]]++] = (uint8_t)i;
    int lc[16], dc[16];
    for (int l = 0; l < 16; ++l) lc[l] = dc[l] = 0;
    int prev = -1;
    bool eob = false;
    for (int i = 0; i < nlen + ndist;) {
        // canonical decode of one code-length symbol
        const uint32_t look = br.peek(7);
        int code = 0, first = 0, index = 0, s = -1, used = 0;
        for (int l = 1; l < 8; ++l) {
            code |= (look >> (l - 1)) & 1;
            if (code - cnt[l] < first) {
                s = sym[index + code - first];
                used = l;
                break;
            }
            index += cnt[l];
            first = (first + cnt[l]) << 1;
            code <<= 1;
        }
        if (s < 0 || !br.has(used)) return false;
        br.drop(used);
        int rep = 1, val = s;
        if (s == 16) {
            if (prev < 0 || !br.has(2)) return false;
            val = prev;
            rep = 3 + (int)br.peek(2);
            br.drop(2);
        } else if (s == 17) {
            if (!br.has(3)) return false;
            val = 0;
            rep = 3 + (int)br.peek(3);
            br.drop(3);
        } else if (s == 18) {
            if (!br.has(7)) return false;
            val = 0;
            rep = 11 + (int)br.peek(7);
            br.drop(7);
        }
        if (i + rep > nlen + ndist) return false;
        for (int k = 0; k < rep; ++k, ++i) {
            if (i < nlen) {
                lc[val]++;
                if (i == 256 && val) eob = true;
            } else {
                dc[val]++;
            }
        }
        prev = val;
    }
    if (!eob) return false;
    int ll = 1, dl = 1, lmax = 0, dmax = 0;
    for (int l = 1; l < 16; ++l) {
        ll = (ll << 1) - lc[l];
        dl = (dl << 1) - dc[l];
        if (ll < 0 || dl < 0) return false;
        if (lc[l]) lmax = l;
        if (dc[l]) dmax = l;
    }
    return (ll == 0 || lmax == 1) && (dl == 0 || dmax <= 1);
}

__global__ void __launch_bounds__(FIND_THREADS) png_find_kernel(const uint8_t *__restrict__ blob, uint8_t *__restrict__ ws) {
    const PngBlobHeader &H = *reinterpret_cast<const PngBlobHeader *>(blob);
    const PngChunk &ch = reinterpret_cast<const PngChunk *>(blob + H.chunk_off)[blockIdx.x];
    const PngImg &im = reinterpret_cast<const PngImg *>(blob + H.img_off)[ch.image];
    ChunkMeta &m = *reinterpret_cast<ChunkMeta *>(ws + ch.meta_off);
    if (ch.index == 0) {
        if (threadIdx.x == 0) m.cand = 16;      // the stream's first block, behind the zlib header
        return;
    }
    __shared__ int found;
    const long long total = im.stream_len * 8;
    const long long b0 = (long long)ch.index * im.chunk_bytes * 8, b1 = min(total, b0 + im.chunk_bytes * 8);
    const uint8_t *stream = ws + im.stream_off;
    long long cand = -1;
    for (long long base = b0; base < b1 && cand < 0; base += FIND_THREADS) {
        if (threadIdx.x == 0) found = FIND_THREADS;
        __syncthreads();
        const long long bit = base + threadIdx.x;
        if (bit < b1 && strict_header(stream, total, bit)) atomicMin(&found, (int)threadIdx.x);
        __syncthreads();
        if (found < FIND_THREADS) cand = base + found;
        __syncthreads();
    }
    if (threadIdx.x == 0) m.cand = cand;
}

// One warp per chunk, lane 0 decoding: from the chunk's candidate into uint16 symbols (a byte, or 256 + w for the byte w of the
// 32 KiB before the chunk's first output), until it stands on a later chunk's candidate at a block boundary (CHUNK: next), ends
// the final block, or fails (invalid data, a distance before the window, more symbols than its capacity, the end of the
// stream).  Decoding from a true block boundary is deterministic, so a chain of such links from chunk 0 is the serial decode.
__global__ void __launch_bounds__(CHUNK_THREADS) png_chunk_kernel(const uint8_t *__restrict__ blob, uint8_t *__restrict__ ws) {
    extern __shared__ uint16_t swin[];      // WINDOW symbols
    __shared__ Huff lit, dist;
    __shared__ uint8_t lens[320];
    const PngBlobHeader &H = *reinterpret_cast<const PngBlobHeader *>(blob);
    const PngChunk *chunks = reinterpret_cast<const PngChunk *>(blob + H.chunk_off);
    const PngChunk &ch = chunks[blockIdx.x];
    const PngImg &im = reinterpret_cast<const PngImg *>(blob + H.img_off)[ch.image];
    ChunkMeta &m = *reinterpret_cast<ChunkMeta *>(ws + ch.meta_off);
    const long long p0 = m.cand;
    for (int k = threadIdx.x; k < WINDOW; k += CHUNK_THREADS) swin[k] = (uint16_t)(256 + k);
    __syncwarp();
    if (threadIdx.x) return;
    long long o = 0, end_bit = 0;
    int next = -1, flags = 0;
    if (p0 < 0) {
        flags = CHUNK_FAILED;
    } else {
        uint16_t *out = reinterpret_cast<uint16_t *>(ws + ch.buf_off);
        const long long cap = ch.cap, slack = ch.index ? WINDOW : 0;
        const PngChunk *mine = chunks + (blockIdx.x - ch.index);    // chunk 0 of the image
        Bits br;
        br.start(ws + im.stream_off, im.stream_len * 8, p0);
        int j = ch.index + 1;
        auto put = [&](uint16_t v) {
            out[o] = v;
            swin[o & (WINDOW - 1)] = v;
            ++o;
        };
        while (true) {
            while (j < im.nchunks) {
                const long long c = reinterpret_cast<const ChunkMeta *>(ws + mine[j].meta_off)->cand;
                if (c >= 0 && c >= br.pos) break;
                ++j;
            }
            if (j < im.nchunks && reinterpret_cast<const ChunkMeta *>(ws + mine[j].meta_off)->cand == br.pos) {
                next = j;
                break;
            }
            if (!br.has(3)) {
                flags = CHUNK_FAILED;
                break;
            }
            const bool last = br.peek(1);
            const int type = (int)(br.peek(3) >> 1);
            br.drop(3);
            bool bad = type == 3;
            if (type == 0) {
                br.align();
                if (!br.has(32)) {
                    flags = CHUNK_FAILED;
                    break;
                }
                const uint32_t len = br.peek(16);
                br.drop(16);
                const uint32_t nlen = br.peek(16);
                br.drop(16);
                if (len != (~nlen & 0xFFFF) || o + len > cap || !br.has(8LL * len)) {
                    flags = CHUNK_FAILED;
                    break;
                }
                for (uint32_t k = 0; k < len; ++k) {
                    put((uint16_t)br.peek(8));
                    br.drop(8);
                }
            } else if (!bad) {
                if (type == 1) fixed_tables(lit, dist, lens);
                else bad = read_dynamic(br, lit, dist, lens) != 0;
                while (!bad) {
                    const int s = decode_sym(br, lit);
                    if (s < 0 || s > 285) {
                        bad = true;
                        break;
                    }
                    if (s < 256) {
                        if (o >= cap) {
                            bad = true;
                            break;
                        }
                        put((uint16_t)s);
                        continue;
                    }
                    if (s == 256) break;
                    const int li = s - 257;
                    if (!br.has(c_lext[li])) {
                        bad = true;
                        break;
                    }
                    const int length = c_lbase[li] + (int)br.peek(c_lext[li]);
                    br.drop(c_lext[li]);
                    const int ds = decode_sym(br, dist);
                    if (ds < 0 || ds > 29 || !br.has(c_dext[ds])) {
                        bad = true;
                        break;
                    }
                    const int d = c_dbase[ds] + (int)br.peek(c_dext[ds]);
                    br.drop(c_dext[ds]);
                    if (d > o + slack || o + length > cap) {
                        bad = true;
                        break;
                    }
                    for (int k = 0; k < length; ++k) put(swin[(o - d) & (WINDOW - 1)]);
                }
            }
            if (bad) {
                flags = CHUNK_FAILED;
                break;
            }
            if (last) {
                flags = CHUNK_FINAL;
                end_bit = br.pos;
                break;
            }
        }
    }
    m.len = o;
    m.end_bit = end_bit;
    m.next = next;
    m.flags = flags;
}

// One CTA per image: follows the chain of chunk links from chunk 0.  When it ends with the final block after exactly the image's
// filtered bytes, every chunk of the chain is resolved in order into the filtered rows (a reference reads the bytes already
// resolved before the chunk) and the Adler-32 behind the final block is checked; then the image is decoded and its flag word
// set.  Otherwise (damaged or unusual streams) the serial decoder below decodes it with the complete zlib rules.
// Status: [1] chunks, [2] chunks after the first whose speculative start was confirmed.
__global__ void __launch_bounds__(RESOLVE_THREADS) png_resolve_kernel(const uint8_t *__restrict__ blob, uint8_t *__restrict__ ws,
                                                                      int32_t *status) {
    const PngBlobHeader &H = *reinterpret_cast<const PngBlobHeader *>(blob);
    const PngImg &im = reinterpret_cast<const PngImg *>(blob + H.img_off)[blockIdx.x];
    const PngChunk *chunks = reinterpret_cast<const PngChunk *>(blob + H.chunk_off) + im.chunk_first;
    long long *prod = reinterpret_cast<long long *>(ws + im.prod_off);
    int32_t *st = status + 4 * blockIdx.x;
    __shared__ int chain[MAX_CHUNKS];
    __shared__ int nchain, ok;
    __shared__ long long end_bit, longest;
    __shared__ uint32_t part_a[RESOLVE_THREADS], part_b[RESOLVE_THREADS];
    if (threadIdx.x == 0) {
        int c = 0, k = 0;
        long long total = 0, most = 0;
        ok = 0;
        while (k < MAX_CHUNKS) {
            const ChunkMeta &m = *reinterpret_cast<const ChunkMeta *>(ws + chunks[c].meta_off);
            if (m.flags & CHUNK_FAILED) break;
            chain[k++] = c;
            total += m.len;
            most = max(most, m.len);
            if (m.flags & CHUNK_FINAL) {
                ok = total == im.raw_len;
                end_bit = m.end_bit;
                break;
            }
            if (m.next <= c) break;
            c = m.next;
        }
        nchain = k;
        longest = most;
        st[1] = im.nchunks;
        st[2] = k ? k - 1 : 0;
        prod[1] = 0;
    }
    __syncthreads();
    if (!ok) return;
    uint8_t *raw = ws + im.raw_off;
    long long off = 0;
    int bad = 0;
    for (int k = 0; k < nchain; ++k) {
        const PngChunk &ch = chunks[chain[k]];
        const uint16_t *sym = reinterpret_cast<const uint16_t *>(ws + ch.buf_off);
        const long long len = reinterpret_cast<const ChunkMeta *>(ws + ch.meta_off)->len;
        for (long long i = threadIdx.x; i < len; i += RESOLVE_THREADS) {
            const uint16_t v = sym[i];
            const long long from = off - WINDOW + (v - 256);
            if (v < 256) raw[off + i] = (uint8_t)v;
            else if (from >= 0) raw[off + i] = raw[from];
            else bad = 1;       // a reference before the stream: left to the serial decoder's error rules
        }
        off += len;
        __syncthreads();
    }
    // Adler-32 of the filtered rows: per-thread runs, combined in order
    const long long T = im.raw_len, per = (T + RESOLVE_THREADS - 1) / RESOLVE_THREADS;
    const long long a0 = min(T, per * threadIdx.x), a1 = min(T, a0 + per);
    uint32_t sa = 0, sb = 0;
    for (long long i = a0; i < a1; ++i) {
        sa = (sa + raw[i]) % 65521u;
        sb = (sb + sa) % 65521u;
    }
    part_a[threadIdx.x] = sa;
    part_b[threadIdx.x] = sb;
    if (bad) atomicOr(&ok, 2);
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t A = 1, B = 0;
        for (int t = 0; t < RESOLVE_THREADS; ++t) {
            const long long n = min(T, per * (t + 1)) - min(T, per * t);
            // appending a run of n bytes with sums (a, b): B += n * A + b, A += a
            B = (uint32_t)((B + (n % 65521) * A + part_b[t]) % 65521u);
            A = (A + part_a[t]) % 65521u;
        }
        const long long at = (end_bit + 7) >> 3;
        const uint8_t *z = ws + im.stream_off;
        bool good = ok == 1 && at + 4 <= im.stream_len;
        if (good) {
            const uint32_t v = (uint32_t)z[at] << 24 | (uint32_t)z[at + 1] << 16 | (uint32_t)z[at + 2] << 8 | z[at + 3];
            good = v == (B << 16 | A);
        }
        if (good) {
            prod[0] = T;
            prod[1] = 1;
            st[3] = (int32_t)longest;
        }
    }
}

__global__ void __launch_bounds__(1) png_inflate_kernel(const uint8_t *__restrict__ blob, uint8_t *__restrict__ ws, int32_t *status) {
    __shared__ uint8_t win[WINDOW];
    __shared__ Huff lit, dist;
    __shared__ uint8_t lens[320];
    const PngBlobHeader &H = *reinterpret_cast<const PngBlobHeader *>(blob);
    const PngImg &im = reinterpret_cast<const PngImg *>(blob + H.img_off)[blockIdx.x];
    long long *prod = reinterpret_cast<long long *>(ws + im.prod_off);
    if (prod[1]) return;        // the chunk chain decoded it
    const long long *ends = reinterpret_cast<const long long *>(blob + H.piece_off) + im.piece_first;
    inflate_image(im, ws + im.stream_off, ends, ws + im.raw_off, status + 4 * blockIdx.x, prod, win, lit, dist, lens);
}

__device__ __forceinline__ uint8_t paeth(int a, int b, int c) {
    const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
    return (uint8_t)(pa <= pb && pa <= pc ? a : pb <= pc ? b : c);
}

// Writes the RGB pixels one wavefront unit of reconstructed bytes `u` (unit x of its row) covers.
__device__ void write_unit(const PngImg &im, const uint8_t *u, int x, uint8_t *o_row) {
    const int d = im.depth;
    if (d < 8) {
        const int per = 8 / d, mask = (1 << d) - 1;
        const int x0 = x * per, x1 = min(im.w, x0 + per);
        for (int px = x0; px < x1; ++px) {
            const int v = (u[0] >> (8 - d * (px - x0 + 1))) & mask;
            uint8_t *o = o_row + 3 * (long long)px;
            if (im.color == 3) {
                const bool in = v < im.plte_n;
                o[0] = in ? im.plte[3 * v] : 0;
                o[1] = in ? im.plte[3 * v + 1] : 0;
                o[2] = in ? im.plte[3 * v + 2] : 0;
            } else {
                const uint8_t g = (uint8_t)(v * (255 / mask));
                o[0] = o[1] = o[2] = g;
            }
        }
        return;
    }
    uint8_t *o = o_row + 3 * (long long)x;
    const int step = d / 8;     // 1 or 2: the high byte of each sample comes first
    switch (im.color) {
        case 0: case 4: o[0] = o[1] = o[2] = u[0]; break;
        case 3: {
            const int v = u[0];
            const bool in = v < im.plte_n;
            o[0] = in ? im.plte[3 * v] : 0;
            o[1] = in ? im.plte[3 * v + 1] : 0;
            o[2] = in ? im.plte[3 * v + 2] : 0;
            break;
        }
        default: o[0] = u[0]; o[1] = u[step]; o[2] = u[2 * step]; break;
    }
}

__global__ void __launch_bounds__(UNFILTER_THREADS) png_unfilter_kernel(const uint8_t *__restrict__ blob, uint8_t *__restrict__ ws,
                                                                        uint8_t *__restrict__ dst, int32_t *status) {
    const PngBlobHeader &H = *reinterpret_cast<const PngBlobHeader *>(blob);
    const PngImg &im = reinterpret_cast<const PngImg *>(blob + H.img_off)[blockIdx.x];
    int32_t *st = status + 4 * blockIdx.x;
    const long long row = 1 + (long long)im.rowbytes;
    const int filled = (int)min((long long)im.h, *reinterpret_cast<const long long *>(ws + im.prod_off) / row);
    uint8_t *raw = ws + im.raw_off;
    uint8_t *out = dst + im.dst_offset;
    const int unit = im.unit;
    const int units = (im.rowbytes + unit - 1) / unit;
    int bad = 0;
    for (int r = threadIdx.x; r < filled; r += UNFILTER_THREADS)
        if (raw[r * row] > 4) bad = 1;
    if (bad) atomicOr(st, PNG_ERR_FILTER);
    const uint8_t zero[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    // rows the stream never filled hold zero bytes
    for (long long k = threadIdx.x; k < (long long)(im.h - filled) * units; k += UNFILTER_THREADS) {
        const int r = filled + (int)(k / units), x = (int)(k % units);
        write_unit(im, zero, x, out + (long long)r * im.w * 3);
    }
    const int steps = units + filled - 1;
    for (int s = 0; s < steps; ++s) {
        for (int r = threadIdx.x; r < filled; r += UNFILTER_THREADS) {
            const int x = s - r;
            if (x < 0) break;
            if (x >= units) continue;
            uint8_t *cur = raw + r * row + 1;
            const uint8_t *up = r ? raw + (r - 1) * row + 1 : nullptr;
            const int f = raw[r * row];
            const int b0 = x * unit, b1 = min(im.rowbytes, b0 + unit);
            for (int b = b0; b < b1; ++b) {
                const int a = b >= unit ? cur[b - unit] : 0;
                const int u = up ? up[b] : 0;
                const int c = up && b >= unit ? up[b - unit] : 0;
                int v = cur[b];
                switch (f) {
                    case 1: v += a; break;
                    case 2: v += u; break;
                    case 3: v += (a + u) >> 1; break;
                    case 4: v += paeth(a, u, c); break;
                    default: break;
                }
                cur[b] = (uint8_t)v;
            }
            uint8_t px[8];
            for (int b = 0; b < unit; ++b) px[b] = b0 + b < im.rowbytes ? cur[b0 + b] : 0;
            write_unit(im, px, x, out + (long long)r * im.w * 3);
        }
        __syncthreads();
    }
}

const PngBlobHeader *check_blob(const void *blob_host, const char *fn) {
    const PngBlobHeader *H = static_cast<const PngBlobHeader *>(blob_host);
    if (!H || H->magic != PNG_BLOB_MAGIC || H->n <= 0) {
        set_error("%s: not a descriptor blob made by k2y_png_plan", fn);
        return nullptr;
    }
    return H;
}

}  // namespace
}  // namespace k2y

using namespace k2y;

extern "C" int k2y_png_inspect(const unsigned char *data, size_t size, k2y_png_info *info) {
    if (!data || !info) {
        set_error("k2y_png_inspect: bad arguments");
        return K2Y_ERR_INVALID;
    }
    PngParsed p;
    const int rc = parse_png(data, size, p, "k2y_png_inspect");
    if (rc != K2Y_OK) return rc;
    memset(info, 0, sizeof(*info));
    info->height = p.h;
    info->width = p.w;
    info->color_type = p.color;
    info->bit_depth = p.depth;
    info->interlace = p.interlace;
    info->idat_chunks = (int32_t)p.idat.size();
    info->stream_bytes = p.stream_len;
    info->gpu_decodable = p.gpu ? 1 : 0;
    snprintf(info->reason, sizeof(info->reason), "%s", p.gpu ? "" : p.reason);
    return K2Y_OK;
}

extern "C" int k2y_png_plan(const unsigned char *const *files, const size_t *sizes, int n, const long long *src_offsets,
                            const long long *dst_offsets, void *blob, size_t blob_capacity, size_t *blob_bytes) {
    if (!files || !sizes || n <= 0 || !blob_bytes || (blob && (!src_offsets || !dst_offsets))) {
        set_error("k2y_png_plan: bad arguments");
        return K2Y_ERR_INVALID;
    }
    std::vector<PngParsed> ps(n);
    long long nseg = 0;
    for (int i = 0; i < n; ++i) {
        char who[48];
        snprintf(who, sizeof(who), "k2y_png_plan: image %d", i);
        if (!files[i]) {
            set_error("%s: null file pointer", who);
            return K2Y_ERR_INVALID;
        }
        const int rc = parse_png(files[i], sizes[i], ps[i], who);
        if (rc != K2Y_OK) return rc;
        if (!ps[i].gpu) {
            set_error("%s: not decodable on the GPU: %s", who, ps[i].reason);
            return K2Y_ERR_INVALID;
        }
        nseg += (long long)ps[i].idat.size();
    }
    // PIL's reads: every non-empty IDAT in pieces of at most PIL_READ bytes from its start
    std::vector<long long> npiece(n, 0);
    long long npieces = 0;
    for (int i = 0; i < n; ++i) {
        for (auto &c : ps[i].idat) npiece[i] += (c.second + PIL_READ - 1) / PIL_READ;
        npieces += npiece[i];
    }
    std::vector<long long> chunk_bytes(n);
    std::vector<int> nchunks(n);
    long long nch = 0;
    for (int i = 0; i < n; ++i) {
        const long long len = ps[i].stream_len;
        chunk_bytes[i] = std::max<long long>(CHUNK_BYTES, (len + MAX_CHUNKS - 1) / MAX_CHUNKS);
        nchunks[i] = (int)std::max<long long>(1, (len + chunk_bytes[i] - 1) / chunk_bytes[i]);
        nch += nchunks[i];
    }
    const long long img_off = align16(sizeof(PngBlobHeader));
    const long long seg_off = img_off + (long long)sizeof(PngImg) * n;
    const long long chunk_off = seg_off + (long long)sizeof(PngSeg) * nseg;
    const long long piece_off = chunk_off + (long long)sizeof(PngChunk) * nch;
    const long long total = piece_off + (long long)sizeof(long long) * npieces;
    *blob_bytes = (size_t)total;
    if (!blob) return K2Y_OK;
    if (blob_capacity < (size_t)total || ((uintptr_t)blob & 15)) {
        set_error("k2y_png_plan: the blob needs %lld bytes at a 16-byte aligned address, got %zu", total, blob_capacity);
        return K2Y_ERR_INVALID;
    }
    uint8_t *B = static_cast<uint8_t *>(blob);
    memset(B, 0, (size_t)total);
    PngBlobHeader &H = *reinterpret_cast<PngBlobHeader *>(B);
    PngImg *I = reinterpret_cast<PngImg *>(B + img_off);
    PngSeg *S = reinterpret_cast<PngSeg *>(B + seg_off);
    PngChunk *C = reinterpret_cast<PngChunk *>(B + chunk_off);
    long long *P = reinterpret_cast<long long *>(B + piece_off);
    long long ws = 0, pg = 0;
    int sg = 0, cg = 0;
    for (int i = 0; i < n; ++i) {
        const PngParsed &p = ps[i];
        PngImg &im = I[i];
        im.h = p.h;
        im.w = p.w;
        im.color = p.color;
        im.depth = p.depth;
        im.rowbytes = row_bytes(p);
        im.unit = std::max(1, channels_of(p.color) * p.depth / 8);
        im.plte_n = p.plte_n;
        memcpy(im.plte, p.plte, sizeof(im.plte));
        im.dst_offset = dst_offsets[i];
        im.stream_off = ws;
        im.stream_len = p.stream_len;
        ws += align16(p.stream_len + 8);
        im.raw_off = ws;
        im.raw_len = (long long)p.h * (1 + im.rowbytes);
        ws += align16(im.raw_len);
        im.prod_off = ws;
        ws += 16;
        im.chunk_bytes = chunk_bytes[i];
        im.chunk_first = cg;
        im.nchunks = nchunks[i];
        for (int k = 0; k < nchunks[i]; ++k, ++cg) {
            C[cg].image = i;
            C[cg].index = k;
            C[cg].meta_off = ws;
            ws += sizeof(ChunkMeta);
            C[cg].cap = k ? std::min(im.raw_len, CHUNK_SYMBOLS) : im.raw_len;   // chunk 0 may have to decode the whole image
            C[cg].buf_off = ws;
            ws += align16(2 * C[cg].cap);
        }
        im.seg_first = sg;
        im.nseg = (int)p.idat.size();
        im.piece_first = pg;
        im.npiece = npiece[i];
        long long at = 0;
        for (auto &c : p.idat) {
            S[sg].src = src_offsets[i] + c.first;
            S[sg].len = c.second;
            S[sg].dst = at;
            for (long long k = 0; k < c.second; k += PIL_READ) P[pg++] = at + std::min(c.second, k + PIL_READ);
            at += c.second;
            ++sg;
        }
    }
    H.magic = PNG_BLOB_MAGIC;
    H.n = n;
    H.nseg = (int)nseg;
    H.img_off = img_off;
    H.seg_off = seg_off;
    H.chunk_off = chunk_off;
    H.nchunks = (int)nch;
    H.piece_off = piece_off;
    H.npieces = npieces;
    H.blob_bytes = total;
    H.ws_bytes = ws;
    return K2Y_OK;
}

extern "C" int k2y_png_workspace_bytes(const void *blob_host, size_t *bytes) {
    const PngBlobHeader *H = check_blob(blob_host, "k2y_png_workspace_bytes");
    if (!H || !bytes) {
        if (H) set_error("k2y_png_workspace_bytes: bad arguments");
        return K2Y_ERR_INVALID;
    }
    *bytes = (size_t)H->ws_bytes;
    return K2Y_OK;
}

extern "C" int k2y_png_decode(const void *blob_host, const void *blob_dev, const unsigned char *src_dev, unsigned char *dst_dev,
                              void *workspace_dev, size_t workspace_bytes, int32_t *status_dev, void *stream) {
    const PngBlobHeader *H = check_blob(blob_host, "k2y_png_decode");
    if (!H) return K2Y_ERR_INVALID;
    if (!blob_dev || !src_dev || !dst_dev || !workspace_dev || !status_dev || ((uintptr_t)blob_dev & 15) ||
        ((uintptr_t)workspace_dev & 15) || workspace_bytes < (size_t)H->ws_bytes) {
        set_error("k2y_png_decode: bad arguments (16-byte aligned blob and workspace of %lld bytes needed, got %zu)", H->ws_bytes,
                  workspace_bytes);
        return K2Y_ERR_INVALID;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const uint8_t *blob = static_cast<const uint8_t *>(blob_dev);
    uint8_t *ws = static_cast<uint8_t *>(workspace_dev);
    K2Y_CUDA_CHECK(cudaMemsetAsync(status_dev, 0, sizeof(int32_t) * 4 * (size_t)H->n, st));
    static bool smem_set = false;
    if (!smem_set) {
        K2Y_CUDA_CHECK(cudaFuncSetAttribute(png_chunk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, WINDOW * 2));
        smem_set = true;
    }
    png_gather_kernel<<<H->n, GATHER_THREADS, 0, st>>>(blob, src_dev, ws);
    png_find_kernel<<<H->nchunks, FIND_THREADS, 0, st>>>(blob, ws);
    png_chunk_kernel<<<H->nchunks, CHUNK_THREADS, WINDOW * 2, st>>>(blob, ws);
    png_resolve_kernel<<<H->n, RESOLVE_THREADS, 0, st>>>(blob, ws, status_dev);
    png_inflate_kernel<<<H->n, 1, 0, st>>>(blob, ws, status_dev);
    png_unfilter_kernel<<<H->n, UNFILTER_THREADS, 0, st>>>(blob, ws, dst_dev, status_dev);
    K2Y_CUDA_CHECK(cudaGetLastError());
    return K2Y_OK;
}
