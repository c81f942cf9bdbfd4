// SORT tracking of a stream's gathered detection records (oracle/sort_ref.py states every rule; this is it bit for bit).
//
// One CTA per stream, one thread per class: a class's tracks, association and Kalman filters are its thread's alone.  Each
// association is the one-thread form of warp_lsap (lsap_warp.cuh, scipy's assignment, ties included), as the threads of a
// warp serve different classes.  The classes meet once per frame in frame_loop (tracker.cuh), where the frame's births
// take their ids from one counter in (class, birth) order.  The launch walks the batch's frames in order, so one launch
// serves a batch of any length; with several streams, each CTA walks its own stream's frames on its own state.
//
// The state lives in global memory between launches (SORT_ARRAYS): the stream's header, every class's track list in
// SORT's order, and per-class scratch (the frame's detections, the tracks' predicted boxes and the assignment's work
// arrays).  A class holds at most TRACK_MAX tracks; the host refuses K (max_age + 1) > TRACK_MAX, which bounds the live
// tracks, so the list never overflows.
//
// Float64 throughout, in the oracle's operation order: every product is __dmul_rn (so nothing contracts into an FMA),
// division and sqrt are IEEE round-to-nearest.
#include <cmath>

#include "common.h"
#include "tracker.cuh"

namespace k2y {
namespace {

constexpr int TRACK_MAX = 1024;      // tracks per class (oracle/sort_ref.py MAX_TRACKS_PER_CLASS)

struct Trk {
    Filt kf;
    int id, hits, hit_streak, tsu, age, pad;
};

// Every per-class array: type, name, entries per class (k = K records, n = cap tracks).
#define SORT_ARRAYS(X)                                                                                                      \
    X(int, n_tracks, 1)                                                                                                     \
    X(Trk, trk, n)                                                                                                          \
    X(double, dbox, 4 * k)          /* the frame's detections, x1 y1 x2 y2 */                                              \
    X(double, pbox, 4 * n)          /* the tracks' predicted boxes */                                                       \
    X(int, det_k, k)                /* each detection's record */                                                           \
    X(int, mdet, k)                 /* each detection's track, -1 for none */                                              \
    X(int, born, k)                 /* the detections born, in order */

struct ClassView {
    SORT_ARRAYS(K2Y_STATE_FIELD)
    LsapWork w;
};

__device__ ClassView class_view(unsigned char *state, size_t C, int c, size_t k, size_t n) {
    ClassView v;
    size_t o = state_start();
    SORT_ARRAYS(K2Y_STATE_SLICE)
    K2Y_LSAP_ARRAYS(K2Y_STATE_SLICE, k, n)
    return v;
}

size_t state_bytes(size_t C, size_t k, size_t n) {
    size_t o = state_start();
    SORT_ARRAYS(K2Y_STATE_BYTES)
    K2Y_LSAP_ARRAYS(K2Y_STATE_BYTES, k, n)
    return o;
}

__device__ void to_z(const double *box, double *z) {
    double w = box[2] - box[0], h = box[3] - box[1];
    z[0] = box[0] + w / 2.0;
    z[1] = box[1] + h / 2.0;
    z[2] = mul(w, h);
    z[3] = w / h;
}

__device__ void update(Trk &t, const double *box) {
    double z[4];
    to_z(box, z);
    filt_update(t.kf, z);
    t.tsu = 0;
    t.hits += 1;
    t.hit_streak += 1;
}

__device__ void birth(Trk &t, const double *box) {
    double z[4];
    to_z(box, z);
    filt_init(t.kf, z);
    t.id = -1;
    t.hits = t.hit_streak = t.tsu = t.age = 0;
}

// SORT's predict of every track of the class, then its deletion of tracks whose predicted box has a NaN; returns the count
// left and puts their predicted boxes in pbox.
__device__ int predict_all(const ClassView &s, int n) {
    int w = 0;
    for (int t = 0; t < n; ++t) {
        Trk k = s.trk[t];
        sort_predict(k);
        double b[4];
        state_box(k.kf, b);
        if (b[0] != b[0] || b[1] != b[1] || b[2] != b[2] || b[3] != b[3]) continue;
        s.trk[w] = k;
        for (int q = 0; q < 4; ++q) s.pbox[4 * w + q] = b[q];
        ++w;
    }
    return w;
}

__device__ int remove_dead(const ClassView &s, int n, int max_age) {
    int w = 0;
    for (int t = 0; t < n; ++t) {
        if (s.trk[t].tsu > max_age) continue;
        if (w != t) s.trk[w] = s.trk[t];
        ++w;
    }
    return w;
}

__device__ void emit_box(const Trk &t, float *out) {
    double b[4];
    state_box(t.kf, b);
    write_box(out, b);
}

// The batch is read in place from the parameters (__grid_constant__), as the callbacks take it by reference.
__global__ void __launch_bounds__(1024) track_update_kernel(unsigned char *state, const __grid_constant__ Batch bt, int cap,
                                                            int max_age, int min_hits, double iou_thresh) {
    if (!stream_has_frames(bt)) return;
    state += (size_t)blockIdx.x * bt.stride;
    const int c = threadIdx.x, C = bt.C, K = bt.K;
    const bool active = c < C;
    const ClassView s = class_view(state, C, active ? c : 0, K, cap);
    int n = active ? *s.n_tracks : 0, nb = 0;
    auto empty = [&](long long count, long long) {
        for (long long e = 0; e < count; ++e) {
            n = predict_all(s, n);
            n = remove_dead(s, n, max_age);
        }
    };
    auto frame = [&](int f, long long fc, int *births) {
        nb = 0;
        if (!active) return;
        const int32_t *rec;
        const int cnt = bt.records(f, c, rec);
        int32_t *ids = bt.ids(f, c);
        float *obox = bt.boxes(f, c);
        bt.clear(f, c, 0, 1);
        n = predict_all(s, n);
        int D = 0;
        for (int k = 0; k < cnt; ++k) {
            double ymin = __int_as_float(rec[6 * k]), xmin = __int_as_float(rec[6 * k + 1]);
            double ymax = __int_as_float(rec[6 * k + 2]), xmax = __int_as_float(rec[6 * k + 3]);
            if (xmax - xmin > 0 && ymax - ymin > 0) {
                double *d = s.dbox + 4 * D;
                d[0] = xmin; d[1] = ymin; d[2] = xmax; d[3] = ymax;
                s.det_k[D++] = k;
            }
        }
        for (int d = 0; d < D; ++d) s.mdet[d] = -1;
        if (n > 0 && D > 0) {
            // SORT's shortcut: every row and column of (iou > thresh) has at most one entry, and some entry is set
            int row_max = 0, col_max = 0;
            int *col_cnt = s.w.row4col;         // free until the assignment
            for (int j = 0; j < n; ++j) col_cnt[j] = 0;
            for (int d = 0; d < D; ++d) {
                int above = 0;
                for (int j = 0; j < n; ++j) {
                    if (sort_iou(s.dbox + 4 * d, s.pbox + 4 * j) > iou_thresh) {
                        ++above;
                        s.mdet[d] = j;
                        int cnt_j = ++col_cnt[j];
                        col_max = cnt_j > col_max ? cnt_j : col_max;
                    }
                }
                row_max = above > row_max ? above : row_max;
            }
            if (!(row_max == 1 && col_max == 1))
                warp_lsap<1>(D, n, [&](int i, int j) { return -sort_iou(s.dbox + 4 * i, s.pbox + 4 * j); }, s.w, s.mdet);
        }
        const bool early = fc <= min_hits;
        for (int d = 0; d < D; ++d)
            if (s.mdet[d] < 0) s.born[nb++] = d;
        for (int d = 0; d < D; ++d) {
            int j = s.mdet[d];
            if (j < 0) continue;
            if (sort_iou(s.dbox + 4 * d, s.pbox + 4 * j) < iou_thresh) {
                s.born[nb++] = d;
                continue;
            }
            Trk &t = s.trk[j];
            update(t, s.dbox + 4 * d);
            if (t.hit_streak >= min_hits || early) {
                ids[s.det_k[d]] = t.id;
                emit_box(t, obox + 4 * s.det_k[d]);
            }
        }
        n = remove_dead(s, n, max_age);
        nb = nb < cap - n ? nb : cap - n;       // never binds: at most cap tracks are alive (see the top of this file)
        for (int b = 0; b < nb; ++b) {
            Trk &t = s.trk[n + b];
            birth(t, s.dbox + 4 * s.born[b]);
            if (0 >= min_hits || early) emit_box(t, obox + 4 * s.det_k[s.born[b]]);
        }
        births[c] = nb;
    };
    auto emit = [&](int f, long long fc, const int *, const int *base) {
        if (!active) return;
        int32_t *ids = bt.ids(f, c);
        for (int b = 0; b < nb; ++b) {
            Trk &t = s.trk[n + b];
            t.id = base[c] + 1 + b;
            if (0 >= min_hits || fc <= min_hits) ids[s.det_k[s.born[b]]] = t.id;
        }
        n += nb;
    };
    frame_loop(state, bt, (long long)max_age + 1, empty, frame, emit);
    if (active) *s.n_tracks = n;
}

int track_cap(int K, int max_age) { return (int)((long long)K * (max_age + 1)); }

bool track_args_ok(const char *fn, int C, int K, int max_age) {
    if (C < 1 || C > 1024 || K < 1 || max_age < 0 || (long long)K * (max_age + 1) > TRACK_MAX) {
        set_error("%s: class_num %d (1..1024), max_per_class %d (>= 1) and max_age %d (>= 0) with max_per_class x (max_age + 1) "
                  "<= %d tracks per class", fn, C, K, max_age, TRACK_MAX);
        return false;
    }
    return true;
}

}  // namespace
}  // namespace k2y

using namespace k2y;

extern "C" int k2y_track_state_bytes(int class_num, int max_per_class, int max_age, size_t *bytes) {
    if (!bytes || !track_args_ok("k2y_track_state_bytes", class_num, max_per_class, max_age)) {
        if (!bytes) set_error("k2y_track_state_bytes: null output");
        return K2Y_ERR_INVALID;
    }
    *bytes = state_bytes(class_num, max_per_class, track_cap(max_per_class, max_age));
    return K2Y_OK;
}

extern "C" int k2y_track_update_streams(void *state_dev, int n_streams, size_t state_stride, const k2y_det *dets_dev,
                                        const int32_t *counts_dev, long long row_stride_words, const int32_t *rows_dev,
                                        const long long *positions_dev, const int32_t *streams_dev, int n_frames, int class_num,
                                        int max_per_class, int max_age, int min_hits, double iou_thresh, int32_t *ids_out_dev,
                                        float *boxes_out_dev, void *stream) {
    const char *fn = "k2y_track_update";
    const Batch bt{(const int32_t *)dets_dev, counts_dev, rows_dev, positions_dev, row_stride_words, n_frames, class_num,
                   max_per_class, ids_out_dev, boxes_out_dev, streams_dev, n_streams, state_stride};
    if (!track_args_ok(fn, class_num, max_per_class, max_age) ||
        !batch_ok(fn, state_dev, bt, state_bytes(class_num, max_per_class, track_cap(max_per_class, max_age))))
        return K2Y_ERR_INVALID;
    if (min_hits < 0 || !(iou_thresh >= 0.0 && iou_thresh <= 1.0)) {
        set_error("%s: min_hits < 0 or iou_thresh outside [0, 1]", fn);
        return K2Y_ERR_INVALID;
    }
    if (n_frames == 0) return K2Y_OK;
    const int threads = (class_num + 31) / 32 * 32;
    track_update_kernel<<<n_streams, threads, 0, (cudaStream_t)stream>>>((unsigned char *)state_dev, bt,
                                                                         track_cap(max_per_class, max_age), max_age, min_hits,
                                                                         iou_thresh);
    K2Y_CUDA_CHECK(cudaGetLastError());
    return K2Y_OK;
}

extern "C" int k2y_track_update(void *state_dev, const k2y_det *dets_dev, const int32_t *counts_dev, long long row_stride_words,
                                const int32_t *rows_dev, const long long *positions_dev, int n_frames, int class_num,
                                int max_per_class, int max_age, int min_hits, double iou_thresh, int32_t *ids_out_dev,
                                float *boxes_out_dev, void *stream) {
    return k2y_track_update_streams(state_dev, 1, 0, dets_dev, counts_dev, row_stride_words, rows_dev, positions_dev, nullptr,
                                    n_frames, class_num, max_per_class, max_age, min_hits, iou_thresh, ids_out_dev, boxes_out_dev,
                                    stream);
}
