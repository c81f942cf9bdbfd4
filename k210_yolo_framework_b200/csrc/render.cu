// Detection and track rendering on the GPU, pixel for pixel what draw.draw_detections (keras_inference.py:137-174 through
// PIL) and draw.draw_tracks draw: per record, in to_host order (class ascending, then record order, a later record
// overwriting an earlier one),
//   - `(h + w) // 300` one-pixel outline rings of the box, ring j = ImageDraw.rectangle([left+j, top+j, right-j, bottom-j]);
//   - the label box [origin, origin + textbbox size] filled in the record's colour;
//   - the label in black, composited through its 8-bit glyph mask as Pillow's fill_mask_L does:
//     DIV255(in * (255 - m) + ink * m) with ink 0.
// Geometry follows draw.box_geometry: floor(v + 0.5) in double on the float32 coordinates, top/left clipped at 0,
// bottom/right at h/w, the label at (left, top + 1), or (left, top - label_h) when top >= h.
//
// Detections (k2y_render_detections): the record's box, its class colour and the label "{:2d} {:.2f}".  The two decimals
// are rint(double(score) * 100) (exact for a float32, ties to even as Python formats them); the glyph masks, their offsets
// and the textbbox sizes of whole labels come from a label atlas built on the host with Pillow (render.LabelAtlas).
//
// Tracks (k2y_render_tracks): the track box and id the tracker wrote for the record (records with id < 0 are skipped), the
// colour colors[id % color_num] and the label "{:2d} #{id}".  Ids are unbounded, so the label is composed from the 12
// glyphs "0".."9", " ", "#" of a track atlas (render.TrackLabelAtlas: per glyph its mask, mask offset, textbbox and
// advance).  Glyph i starts at the integer pen sum(advance[c_j], j < i) (the atlas builder refuses fonts whose advances of
// these glyphs are fractional or kern), the label box is the union of the glyphs' textbboxes at their pens, and the mask is
// folded per pixel in string order as FreeType's bitmaps are laid into one string bitmap: t = s + DIV255(t * (255 - s)).
//
// One difference from draw.py, on purpose: where PIL raises ValueError because a ring's corners cross (left + j > right - j
// or top + j > bottom - j, e.g. a one-pixel-wide box on a large image), the kernel stops that box's rings at the first
// crossing ring and still draws its label.  A score outside [0, 1] (or NaN) is labelled with its hundredths clamped to
// 0..100, and non-finite or huge coordinates are clamped to +-2^30 before the integer geometry.
//
// Work split: one CTA per 32x8 pixel tile of one image.  The CTA walks the image's records 256 at a time: each thread
// derives one record's geometry, the records whose outline, label box or text touch the tile are compacted in order into
// shared memory, and every thread folds them over its pixel.  One launch per batch of up to RENDER_MAX_IMAGES images.  The
// two kernels are one template (render_kernel) over the label: DetLabel or TrackLabel.
#include "common.h"

#include <math.h>

namespace k2y {
namespace {

constexpr int RENDER_MAX_IMAGES = 128;
constexpr int RENDER_MAX_CLASSES = 80;
constexpr int TILE_W = 32, TILE_H = 8, RENDER_THREADS = TILE_W * TILE_H;
constexpr int LABELS_PER_CLASS = 101;          // hundredths 0..100
constexpr int ATLAS_HEADER_WORDS = 8;          // [0] classes (label atlas) or glyphs (track atlas)
constexpr int ATLAS_ENTRY_WORDS = 8;           // mask byte offset, mask w, mask h, mask x, mask y, label w, label h, 0
constexpr int TRACK_GLYPHS = 12;               // "0".."9", " ", "#"
constexpr int GLYPH_SPACE = 10, GLYPH_HASH = 11;
constexpr int TRACK_ENTRY_WORDS = 10;          // mask byte offset, mask w, mask h, mask x, mask y, textbbox l, t, r, b, advance

struct RenderImage {
    long long offset;        // packed HWC RGB
    const int32_t *atlas;    // label or track atlas of the image's font
    int32_t h, w;
};

struct RenderBatch {
    uint8_t *images;
    const int32_t *dets;                  // detections: k2y_det records [C][K][6] per image
    const int32_t *ids;                   // tracks: ids [C][K] and track boxes [C][K][4] per image
    const float *boxes;
    const int32_t *counts;
    long long det_stride, id_stride, box_stride, count_stride;   // words per image
    const uint8_t *colors;                // [color_num][3]: per class (detections) or per id % color_num (tracks)
    int C, K, color_num;
    RenderImage img[RENDER_MAX_IMAGES];
};

// What every record draws besides its text: the outline rings and the filled label box, in one colour.
struct Box {
    int top, left, bottom, right, rings;
    int ox, oy, lw, lh;
    uint32_t rgb;
};

__device__ inline int round_coord(float v) {
    double d = floor((double)v + 0.5);
    d = fmin(fmax(d, -1073741824.0), 1073741824.0);   // NaN -> -2^30
    return (int)d;
}

__device__ inline void place_box(Box &e, const float *tlbr, int lw, int lh, int h, int w, int thickness, const uint8_t *col) {
    e.lw = lw;
    e.lh = lh;
    e.top = max(0, round_coord(tlbr[0]));
    e.left = max(0, round_coord(tlbr[1]));
    e.bottom = min(h, round_coord(tlbr[2]));
    e.right = min(w, round_coord(tlbr[3]));
    e.ox = e.left;
    e.oy = e.top - h >= 0 ? e.top - e.lh : e.top + 1;
    e.rings = 0;
    if (e.right >= e.left && e.bottom >= e.top)
        e.rings = min(thickness, min((e.right - e.left) / 2 + 1, (e.bottom - e.top) / 2 + 1));
    e.rgb = (uint32_t)col[0] | ((uint32_t)col[1] << 8) | ((uint32_t)col[2] << 16);
}

struct Tile {
    int x0, y0;
    __device__ bool meets(int ax0, int ay0, int ax1, int ay1) const {
        return ax0 <= x0 + TILE_W - 1 && ax1 >= x0 && ay0 <= y0 + TILE_H - 1 && ay1 >= y0;
    }
    __device__ bool meets(const Box &e) const {
        return (e.rings > 0 && meets(e.left, e.top, e.right, e.bottom + 1)) || meets(e.ox, e.oy, e.ox + e.lw, e.oy + e.lh);
    }
};

__device__ inline bool ring_pixel(const Box &e, int x, int y, int j) {
    if (j < 0 || j >= e.rings) return false;
    const int L = e.left + j, R = e.right - j, T = e.top + j, B = e.bottom - j;
    if ((y == T || y == B) && x >= L && x <= R) return true;              // the two horizontal lines
    // PIL's vertical lines run from T + 1 to max(B - 1, T + 1): a one-row ring (T == B) also sets the pixel below its ends
    return (x == L || x == R) && y >= T + 1 && y <= max(B - 1, T + 1);
}

__device__ inline void paint_box(const Box &f, int x, int y, int &r, int &g, int &b) {
    if (f.rings > 0 && (ring_pixel(f, x, y, y - f.top) || ring_pixel(f, x, y, f.bottom - y) ||
                        ring_pixel(f, x, y, x - f.left) || ring_pixel(f, x, y, f.right - x))) {
        r = f.rgb & 255;
        g = (f.rgb >> 8) & 255;
        b = f.rgb >> 16;
    }
    if (x >= f.ox && x <= f.ox + f.lw && y >= f.oy && y <= f.oy + f.lh) {
        r = f.rgb & 255;
        g = (f.rgb >> 8) & 255;
        b = f.rgb >> 16;
    }
}

__device__ inline int div255(int a) {
    const int t = a + 128;
    return ((t >> 8) + t) >> 8;
}

__device__ inline void ink(int m, int &r, int &g, int &b) {     // fill_mask_L with ink 0
    const int mk = 255 - m;
    r = div255(r * mk);
    g = div255(g * mk);
    b = div255(b * mk);
}

// Detections: one whole-label mask per (class, hundredths) from the label atlas.
struct DetLabel {
    struct Entry {
        Box box;
        int mask_off, mw, mh, mx, my;
    };
    struct Table {};
    __device__ static void load_table(Table &, const int32_t *, int) {}
    __device__ static const uint8_t *masks(const int32_t *atlas) {
        return reinterpret_cast<const uint8_t *>(atlas + ATLAS_HEADER_WORDS + (size_t)atlas[0] * LABELS_PER_CLASS * ATLAS_ENTRY_WORDS);
    }
    __device__ static bool load(const RenderBatch &p, const RenderImage &im, const Table &, int cls, int k, int thickness,
                                const Tile &tile, Entry &e) {
        const int32_t *rec = p.dets + (long long)blockIdx.z * p.det_stride + ((long long)cls * p.K + k) * 6;
        const float *tlbr = reinterpret_cast<const float *>(rec);
        double hs = rint((double)__int_as_float(rec[4]) * 100.0);
        hs = fmin(fmax(hs, 0.0), 100.0);   // NaN -> 0
        const int32_t *a = im.atlas + ATLAS_HEADER_WORDS + (cls * LABELS_PER_CLASS + (int)hs) * ATLAS_ENTRY_WORDS;
        e.mask_off = a[0];
        e.mw = a[1];
        e.mh = a[2];
        e.mx = a[3];
        e.my = a[4];
        place_box(e.box, tlbr, a[5], a[6], im.h, im.w, thickness, p.colors + cls * 3);
        const int mx0 = e.box.ox + e.mx, my0 = e.box.oy + e.my;
        return tile.meets(e.box) || (e.mw > 0 && e.mh > 0 && tile.meets(mx0, my0, mx0 + e.mw - 1, my0 + e.mh - 1));
    }
    __device__ static void text(const Entry &f, const Table &, const uint8_t *masks, int x, int y, int &r, int &g, int &b) {
        const int u = x - (f.box.ox + f.mx), v = y - (f.box.oy + f.my);
        if (u >= 0 && u < f.mw && v >= 0 && v < f.mh) ink(masks[f.mask_off + v * f.mw + u], r, g, b);
    }
};

// Tracks: "{:2d} #{id}" composed from the track atlas's 12 glyphs, which the CTA keeps in shared memory.
struct TrackLabel {
    struct Entry {
        Box box;
        int tx0, ty0, tx1, ty1;     // the glyph masks' union, from the label origin, end exclusive
        unsigned long long codes;   // glyph i of the label in bits [4i, 4i + 4)
        int n;
    };
    struct Table {
        int32_t g[TRACK_GLYPHS][TRACK_ENTRY_WORDS];
    };
    __device__ static void load_table(Table &t, const int32_t *atlas, int tid) {
        if (tid < TRACK_GLYPHS * TRACK_ENTRY_WORDS) (&t.g[0][0])[tid] = atlas[ATLAS_HEADER_WORDS + tid];
    }
    __device__ static const uint8_t *masks(const int32_t *atlas) {
        return reinterpret_cast<const uint8_t *>(atlas + ATLAS_HEADER_WORDS + TRACK_GLYPHS * TRACK_ENTRY_WORDS);
    }
    __device__ static bool load(const RenderBatch &p, const RenderImage &im, const Table &t, int cls, int k, int thickness,
                                const Tile &tile, Entry &e) {
        const long long rk = (long long)cls * p.K + k;
        const int id = p.ids[(long long)blockIdx.z * p.id_stride + rk];
        if (id < 0) return false;
        // the label's glyphs: the class right-aligned in two columns, " #", then the id's decimal digits
        unsigned long long codes = (unsigned long long)(cls >= 10 ? cls / 10 : GLYPH_SPACE) | ((unsigned long long)(cls % 10) << 4) |
                                   (GLYPH_SPACE << 8) | (GLYPH_HASH << 12);
        unsigned long long digits = 0;
        int n = 4;
        for (unsigned v = (unsigned)id;; v /= 10) {     // least significant first, each in front of the last
            digits = (digits << 4) | (v % 10);
            ++n;
            if (v < 10) break;
        }
        e.codes = codes | (digits << 16);
        e.n = n;
        int pen = 0, l = INT_MAX, tp = INT_MAX, r = INT_MIN, b = INT_MIN;
        int x0 = INT_MAX, y0 = INT_MAX, x1 = INT_MIN, y1 = INT_MIN;
        for (int i = 0; i < n; ++i) {
            const int32_t *g = t.g[(e.codes >> (4 * i)) & 15];
            l = min(l, pen + g[5]);
            tp = min(tp, g[6]);
            r = max(r, pen + g[7]);
            b = max(b, g[8]);
            if (g[1] > 0 && g[2] > 0) {
                x0 = min(x0, pen + g[3]);
                y0 = min(y0, g[4]);
                x1 = max(x1, pen + g[3] + g[1]);
                y1 = max(y1, g[4] + g[2]);
            }
            pen += g[9];
        }
        if (x0 > x1) x0 = y0 = x1 = y1 = 0;
        e.tx0 = x0;
        e.ty0 = y0;
        e.tx1 = x1;
        e.ty1 = y1;
        place_box(e.box, p.boxes + (long long)blockIdx.z * p.box_stride + rk * 4, r - l, b - tp, im.h, im.w, thickness,
                  p.colors + (id % p.color_num) * 3);
        return tile.meets(e.box) || (x1 > x0 && y1 > y0 && tile.meets(e.box.ox + x0, e.box.oy + y0, e.box.ox + x1 - 1, e.box.oy + y1 - 1));
    }
    __device__ static void text(const Entry &f, const Table &t, const uint8_t *masks, int x, int y, int &r, int &g, int &b) {
        const int u = x - f.box.ox, v = y - f.box.oy;
        if (u < f.tx0 || u >= f.tx1 || v < f.ty0 || v >= f.ty1) return;
        int m = 0, pen = 0;
        for (int i = 0; i < f.n; ++i) {
            const int32_t *e = t.g[(f.codes >> (4 * i)) & 15];
            const int gu = u - pen - e[3], gv = v - e[4];
            if (gu >= 0 && gu < e[1] && gv >= 0 && gv < e[2]) {
                const int s = masks[e[0] + gv * e[1] + gu];
                m = s + div255(m * (255 - s));
            }
            pen += e[9];
        }
        ink(m, r, g, b);
    }
};

template <class Label>
__global__ void __launch_bounds__(RENDER_THREADS) render_kernel(const __grid_constant__ RenderBatch p) {
    using Entry = typename Label::Entry;
    __shared__ int s_pref[RENDER_MAX_CLASSES + 1];
    __shared__ Entry s_e[RENDER_THREADS];
    __shared__ int s_warp[RENDER_THREADS / 32 + 1];
    __shared__ typename Label::Table s_table;
    const RenderImage im = p.img[blockIdx.z];
    const Tile tile{(int)blockIdx.x * TILE_W, (int)blockIdx.y * TILE_H};
    if (tile.x0 >= im.w || tile.y0 >= im.h) return;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int32_t *counts = p.counts + (long long)blockIdx.z * p.count_stride;
    Label::load_table(s_table, im.atlas, tid);
    if (tid == 0) {
        int s = 0;
        for (int c = 0; c < p.C; ++c) {
            s_pref[c] = s;
            s += min(max(counts[c], 0), p.K);
        }
        s_pref[p.C] = s;
    }
    __syncthreads();
    const int total = s_pref[p.C];
    const int x = tile.x0 + (tid % TILE_W), y = tile.y0 + tid / TILE_W;
    const bool inside = x < im.w && y < im.h;
    uint8_t *px = p.images + im.offset + ((long long)y * im.w + x) * 3;
    int r = 0, g = 0, b = 0;
    if (inside) {
        r = px[0];
        g = px[1];
        b = px[2];
    }
    const int thickness = (im.h + im.w) / 300;
    const uint8_t *masks = Label::masks(im.atlas);
    for (int c0 = 0; c0 < total; c0 += RENDER_THREADS) {
        const int ri = c0 + tid;
        bool hit = false;
        Entry e;
        if (ri < total) {
            int cls = 0;
            while (cls + 1 < p.C && s_pref[cls + 1] <= ri) ++cls;
            hit = Label::load(p, im, s_table, cls, ri - s_pref[cls], thickness, tile, e);
        }
        // ordered compaction of the records that touch the tile
        const unsigned m = __ballot_sync(0xffffffffu, hit);
        if (lane == 0) s_warp[wid] = __popc(m);
        __syncthreads();
        if (tid == 0) {
            int s = 0;
            for (int w = 0; w < RENDER_THREADS / 32; ++w) {
                const int c = s_warp[w];
                s_warp[w] = s;
                s += c;
            }
            s_warp[RENDER_THREADS / 32] = s;
        }
        __syncthreads();
        if (hit) s_e[s_warp[wid] + __popc(m & ((1u << lane) - 1))] = e;
        __syncthreads();
        const int nhit = s_warp[RENDER_THREADS / 32];
        if (inside) {
            for (int i = 0; i < nhit; ++i) {
                const Entry &f = s_e[i];
                paint_box(f.box, x, y, r, g, b);
                Label::text(f, s_table, masks, x, y, r, g, b);
            }
        }
        __syncthreads();
    }
    if (inside) {
        px[0] = (uint8_t)r;
        px[1] = (uint8_t)g;
        px[2] = (uint8_t)b;
    }
}

// The image checks and the launches of up to RENDER_MAX_IMAGES images each, shared by both entry points.
template <class Label>
int launch(const char *name, RenderBatch base, int n, const long long *offsets_host, const int *hw_host, const int32_t *const *atlas_dev,
           cudaStream_t st) {
    for (int i = 0; i < n; ++i) {
        if (offsets_host[i] < 0 || hw_host[2 * i] < 1 || hw_host[2 * i + 1] < 1 || hw_host[2 * i] > 65535 || hw_host[2 * i + 1] > 65535 ||
            !atlas_dev[i]) {
            set_error("%s: image %d has offset %lld, size %dx%d and atlas %p", name, i, offsets_host[i], hw_host[2 * i],
                      hw_host[2 * i + 1], (const void *)atlas_dev[i]);
            return K2Y_ERR_INVALID;
        }
    }
    for (int g0 = 0; g0 < n; g0 += RENDER_MAX_IMAGES) {
        const int g = n - g0 < RENDER_MAX_IMAGES ? n - g0 : RENDER_MAX_IMAGES;
        RenderBatch p = base;
        if (p.dets) p.dets += p.det_stride * g0;
        if (p.ids) p.ids += p.id_stride * g0;
        if (p.boxes) p.boxes += p.box_stride * g0;
        p.counts += p.count_stride * g0;
        int th = 1, tw = 1;
        for (int i = 0; i < g; ++i) {
            RenderImage &im = p.img[i];
            im.offset = offsets_host[g0 + i];
            im.h = hw_host[2 * (g0 + i)];
            im.w = hw_host[2 * (g0 + i) + 1];
            im.atlas = atlas_dev[g0 + i];
            th = im.h > th * TILE_H ? (im.h + TILE_H - 1) / TILE_H : th;
            tw = im.w > tw * TILE_W ? (im.w + TILE_W - 1) / TILE_W : tw;
        }
        render_kernel<Label><<<dim3(tw, th, g), RENDER_THREADS, 0, st>>>(p);
        K2Y_CUDA_CHECK(cudaGetLastError());
    }
    return K2Y_OK;
}

}  // namespace
}  // namespace k2y

extern "C" int k2y_render_detections(unsigned char *images_dev, int n, const long long *offsets_host, const int *hw_host,
                                     const int32_t *const *atlas_dev, const int32_t *dets_dev, const int32_t *counts_dev,
                                     long long det_image_stride_words, long long count_image_stride_words, int class_num,
                                     int max_per_class, const unsigned char *colors_dev, void *stream) {
    using namespace k2y;
    if (!images_dev || n <= 0 || !offsets_host || !hw_host || !atlas_dev || !dets_dev || !counts_dev || !colors_dev ||
        max_per_class < 1 || det_image_stride_words < (long long)class_num * max_per_class * 6 || count_image_stride_words < class_num) {
        set_error("k2y_render_detections: bad arguments");
        return K2Y_ERR_INVALID;
    }
    if (class_num < 1 || class_num > RENDER_MAX_CLASSES) {
        set_error("k2y_render_detections: class_num %d is outside 1..%d (the colour table's classes)", class_num, RENDER_MAX_CLASSES);
        return K2Y_ERR_INVALID;
    }
    RenderBatch p;
    memset(&p, 0, sizeof(p));
    p.images = images_dev;
    p.dets = dets_dev;
    p.counts = counts_dev;
    p.det_stride = det_image_stride_words;
    p.count_stride = count_image_stride_words;
    p.colors = colors_dev;
    p.C = class_num;
    p.K = max_per_class;
    p.color_num = class_num;
    return launch<DetLabel>("k2y_render_detections", p, n, offsets_host, hw_host, atlas_dev, (cudaStream_t)stream);
}

extern "C" int k2y_render_tracks(unsigned char *images_dev, int n, const long long *offsets_host, const int *hw_host,
                                 const int32_t *const *atlas_dev, const int32_t *ids_dev, const float *boxes_dev,
                                 const int32_t *counts_dev, long long id_image_stride, long long box_image_stride_words,
                                 long long count_image_stride, int class_num, int max_per_class, const unsigned char *colors_dev,
                                 int color_num, void *stream) {
    using namespace k2y;
    if (!images_dev || n <= 0 || !offsets_host || !hw_host || !atlas_dev || !ids_dev || !boxes_dev || !counts_dev || !colors_dev ||
        max_per_class < 1 || color_num < 1 || id_image_stride < (long long)class_num * max_per_class ||
        box_image_stride_words < (long long)class_num * max_per_class * 4 || count_image_stride < class_num) {
        set_error("k2y_render_tracks: bad arguments");
        return K2Y_ERR_INVALID;
    }
    if (class_num < 1 || class_num > RENDER_MAX_CLASSES) {
        set_error("k2y_render_tracks: class_num %d is outside 1..%d (two-digit classes)", class_num, RENDER_MAX_CLASSES);
        return K2Y_ERR_INVALID;
    }
    RenderBatch p;
    memset(&p, 0, sizeof(p));
    p.images = images_dev;
    p.ids = ids_dev;
    p.boxes = boxes_dev;
    p.counts = counts_dev;
    p.id_stride = id_image_stride;
    p.box_stride = box_image_stride_words;
    p.count_stride = count_image_stride;
    p.colors = colors_dev;
    p.C = class_num;
    p.K = max_per_class;
    p.color_num = color_num;
    return launch<TrackLabel>("k2y_render_tracks", p, n, offsets_host, hw_host, atlas_dev, (cudaStream_t)stream);
}
