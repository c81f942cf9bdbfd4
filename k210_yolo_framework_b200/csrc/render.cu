// Detection rendering on the GPU, pixel for pixel what draw.draw_detections (keras_inference.py:137-174 through PIL) draws:
// per record, in to_host order (class ascending, then record order, a later record overwriting an earlier one),
//   - `(h + w) // 300` one-pixel outline rings of the box, ring j = ImageDraw.rectangle([left+j, top+j, right-j, bottom-j]);
//   - the label box [origin, origin + textbbox size] filled in the class colour;
//   - the label "{:2d} {:.2f}" in black, composited through its 8-bit glyph mask as Pillow's fill_mask_L does:
//     DIV255(in * (255 - m) + ink * m) with ink 0.
// Geometry follows draw.box_geometry: floor(v + 0.5) in double on the float32 coordinates, top/left clipped at 0,
// bottom/right at h/w, the label at (left, top + 1), or (left, top - label_h) when top >= h.  The two decimals of the label
// are rint(double(score) * 100) (exact for a float32, ties to even as Python formats them); the glyph masks, their offsets
// and the textbbox sizes come from a label atlas built on the host with Pillow (render.LabelAtlas).
//
// One difference from draw.py, on purpose: where PIL raises ValueError because a ring's corners cross (left + j > right - j
// or top + j > bottom - j, e.g. a one-pixel-wide box on a large image), the kernel stops that box's rings at the first
// crossing ring and still draws its label.  A score outside [0, 1] (or NaN) is labelled with its hundredths clamped to
// 0..100, and non-finite or huge coordinates are clamped to +-2^30 before the integer geometry.
//
// Work split: one CTA per 32x8 pixel tile of one image.  The CTA walks the image's records 256 at a time: each thread
// derives one record's geometry, the records whose outline, label box or text touch the tile are compacted in order into
// shared memory, and every thread folds them over its pixel.  One launch per batch of up to RENDER_MAX_IMAGES images.
#include "common.h"

#include <math.h>

namespace k2y {
namespace {

constexpr int RENDER_MAX_IMAGES = 128;
constexpr int RENDER_MAX_CLASSES = 80;
constexpr int TILE_W = 32, TILE_H = 8, RENDER_THREADS = TILE_W * TILE_H;
constexpr int LABELS_PER_CLASS = 101;          // hundredths 0..100
constexpr int ATLAS_HEADER_WORDS = 8;          // [0] classes
constexpr int ATLAS_ENTRY_WORDS = 8;           // mask byte offset, mask w, mask h, mask x, mask y, label w, label h, 0

struct RenderImage {
    long long offset;        // packed HWC RGB
    const int32_t *atlas;    // label atlas of the image's font
    int32_t h, w;
};

struct RenderBatch {
    uint8_t *images;
    const int32_t *dets;
    const int32_t *counts;
    long long det_stride, count_stride;   // int32 words per image
    const uint8_t *colors;                // [classes][3]
    int C, K;
    RenderImage img[RENDER_MAX_IMAGES];
};

struct Entry {
    int top, left, bottom, right, rings;
    int ox, oy, lw, lh;
    int mask_off, mw, mh, mx, my;
    uint32_t rgb;
};

__device__ inline int round_coord(float v) {
    double d = floor((double)v + 0.5);
    d = fmin(fmax(d, -1073741824.0), 1073741824.0);   // NaN -> -2^30
    return (int)d;
}

__device__ inline bool ring_pixel(const Entry &e, int x, int y, int j) {
    if (j < 0 || j >= e.rings) return false;
    const int L = e.left + j, R = e.right - j, T = e.top + j, B = e.bottom - j;
    if ((y == T || y == B) && x >= L && x <= R) return true;              // the two horizontal lines
    // PIL's vertical lines run from T + 1 to max(B - 1, T + 1): a one-row ring (T == B) also sets the pixel below its ends
    return (x == L || x == R) && y >= T + 1 && y <= max(B - 1, T + 1);
}

__device__ inline int div255(int a) {
    const int t = a + 128;
    return ((t >> 8) + t) >> 8;
}

__global__ void __launch_bounds__(RENDER_THREADS) render_kernel(RenderBatch p) {
    __shared__ int s_pref[RENDER_MAX_CLASSES + 1];
    __shared__ Entry s_e[RENDER_THREADS];
    __shared__ int s_warp[RENDER_THREADS / 32 + 1];
    const RenderImage im = p.img[blockIdx.z];
    const int x0 = blockIdx.x * TILE_W, y0 = blockIdx.y * TILE_H;
    if (x0 >= im.w || y0 >= im.h) return;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int32_t *counts = p.counts + (long long)blockIdx.z * p.count_stride;
    const int32_t *dets = p.dets + (long long)blockIdx.z * p.det_stride;
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
    const int x = x0 + (tid % TILE_W), y = y0 + tid / TILE_W;
    const bool inside = x < im.w && y < im.h;
    uint8_t *px = p.images + im.offset + ((long long)y * im.w + x) * 3;
    int r = 0, g = 0, b = 0;
    if (inside) {
        r = px[0];
        g = px[1];
        b = px[2];
    }
    const int thickness = (im.h + im.w) / 300;
    const uint8_t *masks =
        reinterpret_cast<const uint8_t *>(im.atlas + ATLAS_HEADER_WORDS + (size_t)im.atlas[0] * LABELS_PER_CLASS * ATLAS_ENTRY_WORDS);
    for (int c0 = 0; c0 < total; c0 += RENDER_THREADS) {
        const int ri = c0 + tid;
        bool hit = false;
        Entry e;
        if (ri < total) {
            int cls = 0;
            while (cls + 1 < p.C && s_pref[cls + 1] <= ri) ++cls;
            const int k = ri - s_pref[cls];
            const int32_t *rec = dets + ((long long)cls * p.K + k) * 6;
            const float ymin = __int_as_float(rec[0]), xmin = __int_as_float(rec[1]);
            const float ymax = __int_as_float(rec[2]), xmax = __int_as_float(rec[3]), score = __int_as_float(rec[4]);
            double hs = rint((double)score * 100.0);
            hs = fmin(fmax(hs, 0.0), 100.0);   // NaN -> 0
            const int32_t *a = im.atlas + ATLAS_HEADER_WORDS + (cls * LABELS_PER_CLASS + (int)hs) * ATLAS_ENTRY_WORDS;
            e.mask_off = a[0];
            e.mw = a[1];
            e.mh = a[2];
            e.mx = a[3];
            e.my = a[4];
            e.lw = a[5];
            e.lh = a[6];
            e.top = max(0, round_coord(ymin));
            e.left = max(0, round_coord(xmin));
            e.bottom = min(im.h, round_coord(ymax));
            e.right = min(im.w, round_coord(xmax));
            e.ox = e.left;
            e.oy = e.top - im.h >= 0 ? e.top - e.lh : e.top + 1;
            e.rings = 0;
            if (e.right >= e.left && e.bottom >= e.top)
                e.rings = min(thickness, min((e.right - e.left) / 2 + 1, (e.bottom - e.top) / 2 + 1));
            const uint8_t *col = p.colors + cls * 3;
            e.rgb = (uint32_t)col[0] | ((uint32_t)col[1] << 8) | ((uint32_t)col[2] << 16);
            const int tx1 = x0 + TILE_W - 1, ty1 = y0 + TILE_H - 1;
            auto meets = [&](int ax0, int ay0, int ax1, int ay1) { return ax0 <= tx1 && ax1 >= x0 && ay0 <= ty1 && ay1 >= y0; };
            hit = (e.rings > 0 && meets(e.left, e.top, e.right, e.bottom + 1)) || meets(e.ox, e.oy, e.ox + e.lw, e.oy + e.lh) ||
                  (e.mw > 0 && e.mh > 0 && meets(e.ox + e.mx, e.oy + e.my, e.ox + e.mx + e.mw - 1, e.oy + e.my + e.mh - 1));
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
                const int u = x - (f.ox + f.mx), v = y - (f.oy + f.my);
                if (u >= 0 && u < f.mw && v >= 0 && v < f.mh) {
                    const int mk = 255 - masks[f.mask_off + v * f.mw + u];
                    r = div255(r * mk);
                    g = div255(g * mk);
                    b = div255(b * mk);
                }
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
    for (int i = 0; i < n; ++i) {
        if (offsets_host[i] < 0 || hw_host[2 * i] < 1 || hw_host[2 * i + 1] < 1 || hw_host[2 * i] > 65535 || hw_host[2 * i + 1] > 65535 ||
            !atlas_dev[i]) {
            set_error("k2y_render_detections: image %d has offset %lld, size %dx%d and atlas %p", i, offsets_host[i], hw_host[2 * i],
                      hw_host[2 * i + 1], (const void *)atlas_dev[i]);
            return K2Y_ERR_INVALID;
        }
    }
    cudaStream_t st = (cudaStream_t)stream;
    for (int g0 = 0; g0 < n; g0 += RENDER_MAX_IMAGES) {
        const int g = n - g0 < RENDER_MAX_IMAGES ? n - g0 : RENDER_MAX_IMAGES;
        RenderBatch p;
        memset(&p, 0, sizeof(p));
        p.images = images_dev;
        p.dets = dets_dev + det_image_stride_words * g0;
        p.counts = counts_dev + count_image_stride_words * g0;
        p.det_stride = det_image_stride_words;
        p.count_stride = count_image_stride_words;
        p.colors = colors_dev;
        p.C = class_num;
        p.K = max_per_class;
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
        render_kernel<<<dim3(tw, th, g), RENDER_THREADS, 0, st>>>(p);
        K2Y_CUDA_CHECK(cudaGetLastError());
    }
    return K2Y_OK;
}
