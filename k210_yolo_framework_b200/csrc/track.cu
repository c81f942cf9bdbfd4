// SORT tracking of a stream's gathered detection records (oracle/sort_ref.py states every rule; this is it bit for bit).
//
// One CTA per stream, one thread per class: a class's tracks, association and Kalman filters are its thread's alone, and
// the classes meet once per frame, where the frame's births take their ids from one counter in (class, birth) order through
// a prefix over the CTA.  The launch walks the batch's frames in order, so one launch serves a batch of any length.
//
// The state lives in global memory between launches (track_layout): the stream's frame count, last position and ids taken,
// every class's track list in SORT's order, and per-class scratch (the frame's detections, the tracks' predicted boxes and
// the assignment's work arrays).  A class holds at most TRACK_MAX tracks; the host refuses K (max_age + 1) > TRACK_MAX, which
// bounds the live tracks, so the list never overflows.
//
// Float64 throughout, in the oracle's operation order: every product is __dmul_rn (so nothing contracts into an FMA),
// division and sqrt are IEEE round-to-nearest.
#include <cmath>

#include "common.h"

namespace k2y {
namespace {

constexpr int TRACK_MAX = 1024;      // tracks per class (oracle/sort_ref.py MAX_TRACKS_PER_CLASS)

struct Trk {
    double blk[3][5];       // (p, v, P_pp, P_pv, P_vv) of cx, cy and s
    double r, pr;           // r and its variance
    int id, hits, streak, tsu, age, pad;
};

struct TrackHeader {
    long long frame_count, last_pos;
    int ids_taken, started;
};

struct Layout {
    size_t n_tracks, tracks, dbox, pbox, u, v, spc, det_k, col4row, sr, path, row4col, sc, remaining, mdet, born, total;
};

__host__ __device__ inline size_t take(size_t &o, size_t bytes) {
    size_t at = o;
    o = (o + bytes + 255) & ~(size_t)255;
    return at;
}

__host__ __device__ inline Layout track_layout(int C, int K, int cap) {
    Layout L;
    size_t o = 0;
    take(o, sizeof(TrackHeader));
    L.n_tracks = take(o, sizeof(int) * C);
    L.tracks = take(o, sizeof(Trk) * C * cap);
    L.dbox = take(o, sizeof(double) * 4 * C * K);
    L.pbox = take(o, sizeof(double) * 4 * C * cap);
    L.u = take(o, sizeof(double) * C * K);
    L.v = take(o, sizeof(double) * C * cap);
    L.spc = take(o, sizeof(double) * C * cap);
    L.det_k = take(o, sizeof(int) * C * K);
    L.col4row = take(o, sizeof(int) * C * K);
    L.sr = take(o, sizeof(int) * C * K);
    L.path = take(o, sizeof(int) * C * cap);
    L.row4col = take(o, sizeof(int) * C * cap);
    L.sc = take(o, sizeof(int) * C * cap);
    L.remaining = take(o, sizeof(int) * C * cap);
    L.mdet = take(o, sizeof(int) * C * K);
    L.born = take(o, sizeof(int) * C * K);
    L.total = o;
    return L;
}

__device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
// numpy's maximum / minimum: a NaN in either operand is the result
__device__ __forceinline__ double mx(double a, double b) { return (a >= b || a != a) ? a : b; }
__device__ __forceinline__ double mn(double a, double b) { return (a <= b || a != a) ? a : b; }

__device__ double iou(const double *d, const double *t) {
    double w = mx(0.0, mn(d[2], t[2]) - mx(d[0], t[0]));
    double h = mx(0.0, mn(d[3], t[3]) - mx(d[1], t[1]));
    double wh = mul(w, h);
    double uni = (mul(d[2] - d[0], d[3] - d[1]) + mul(t[2] - t[0], t[3] - t[1])) - wh;
    return uni > 0 ? wh / uni : 0.0;
}

__device__ void predict2(double *b, double qp, double qv) {
    double t = b[3] + b[4];
    b[0] = b[0] + b[1];
    b[2] = ((b[2] + b[3]) + t) + qp;
    b[3] = t;
    b[4] = b[4] + qv;
}

__device__ void update2(double *b, double z, double R) {
    double p = b[0], v = b[1], a = b[2], pv = b[3], d = b[4];
    double y = z - p, S = a + R;
    double k0 = a / S, k1 = pv / S;
    double c = 1.0 - k0;
    double m = pv - mul(k1, a), n = d - mul(k1, pv), rk0 = mul(R, k0);
    b[0] = p + mul(k0, y);
    b[1] = v + mul(k1, y);
    b[2] = mul(mul(c, a), c) + mul(rk0, k0);
    b[3] = mul(c, m) + mul(rk0, k1);
    b[4] = (n - mul(k1, m)) + mul(mul(R, k1), k1);
}

__device__ void to_z(const double *box, double *z) {
    double w = box[2] - box[0], h = box[3] - box[1];
    z[0] = box[0] + w / 2.0;
    z[1] = box[1] + h / 2.0;
    z[2] = mul(w, h);
    z[3] = w / h;
}

__device__ void state_box(const Trk &t, double *box) {
    double w = sqrt(mul(t.blk[2][0], t.r));
    double h = t.blk[2][0] / w;
    box[0] = t.blk[0][0] - w / 2.0;
    box[1] = t.blk[1][0] - h / 2.0;
    box[2] = t.blk[0][0] + w / 2.0;
    box[3] = t.blk[1][0] + h / 2.0;
}

__device__ void predict(Trk &t) {
    if (t.blk[2][1] + t.blk[2][0] <= 0) t.blk[2][1] = mul(t.blk[2][1], 0.0);
    predict2(t.blk[0], 1.0, 0.01);
    predict2(t.blk[1], 1.0, 0.01);
    predict2(t.blk[2], 1.0, 1e-4);
    t.pr = t.pr + 1.0;
    t.age += 1;
    if (t.tsu > 0) t.streak = 0;
    t.tsu += 1;
}

__device__ void update(Trk &t, const double *box) {
    double z[4];
    to_z(box, z);
    update2(t.blk[0], z[0], 1.0);
    update2(t.blk[1], z[1], 1.0);
    update2(t.blk[2], z[2], 10.0);
    double S = t.pr + 10.0, k = t.pr / S, c = 1.0 - k;
    t.r = t.r + mul(k, z[3] - t.r);
    t.pr = mul(mul(c, t.pr), c) + mul(mul(10.0, k), k);
    t.tsu = 0;
    t.hits += 1;
    t.streak += 1;
}

__device__ void birth(Trk &t, const double *box) {
    double z[4];
    to_z(box, z);
    for (int b = 0; b < 3; ++b) {
        t.blk[b][0] = z[b];
        t.blk[b][1] = 0.0;
        t.blk[b][2] = 10.0;
        t.blk[b][3] = 0.0;
        t.blk[b][4] = 10000.0;
    }
    t.r = z[3];
    t.pr = 10.0;
    t.id = -1;
    t.hits = t.streak = t.tsu = t.age = 0;
}

// One class's view of the state.
struct ClassState {
    Trk *trk;
    double *dbox, *pbox, *u, *v, *spc;
    int *det_k, *col4row, *sr, *path, *row4col, *sc, *remaining, *mdet, *born;
};

// scipy's linear_sum_assignment of cost(i, j) = -iou(det i, track j) over D detections and T tracks (oracle/sort_ref.py
// lsap): mdet[d] = the track assigned to detection d, -1 for none.
__device__ void lsap(const ClassState &s, int D, int T) {
    const bool tr = T < D;
    const int nr = tr ? T : D, nc = tr ? D : T;
    auto cost = [&](int i, int j) { return tr ? -iou(s.dbox + 4 * j, s.pbox + 4 * i) : -iou(s.dbox + 4 * i, s.pbox + 4 * j); };
    for (int d = 0; d < D; ++d) s.mdet[d] = -1;
    for (int i = 0; i < nr; ++i) { s.u[i] = 0.0; s.col4row[i] = -1; }
    for (int j = 0; j < nc; ++j) { s.v[j] = 0.0; s.path[j] = -1; s.row4col[j] = -1; }
    for (int cur = 0; cur < nr; ++cur) {
        for (int i = 0; i < nr; ++i) s.sr[i] = 0;
        for (int j = 0; j < nc; ++j) { s.sc[j] = 0; s.spc[j] = INFINITY; s.remaining[j] = nc - j - 1; }
        int num = nc, i = cur, sink = -1;
        double min_val = 0.0;
        while (sink == -1) {
            int index = -1;
            double lowest = INFINITY;
            s.sr[i] = 1;
            const double ui = s.u[i];
            for (int it = 0; it < num; ++it) {
                int j = s.remaining[it];
                double r = ((min_val + cost(i, j)) - ui) - s.v[j];
                double pj = s.spc[j];
                if (r < pj) {
                    s.path[j] = i;
                    s.spc[j] = pj = r;
                }
                if (pj < lowest || (pj == lowest && s.row4col[j] == -1)) {
                    lowest = pj;
                    index = it;
                }
            }
            min_val = lowest;
            int j = s.remaining[index];
            if (s.row4col[j] == -1) sink = j;
            else i = s.row4col[j];
            s.sc[j] = 1;
            s.remaining[index] = s.remaining[--num];
        }
        s.u[cur] += min_val;
        for (int r = 0; r < nr; ++r)
            if (s.sr[r] && r != cur) s.u[r] += min_val - s.spc[s.col4row[r]];
        for (int j = 0; j < nc; ++j)
            if (s.sc[j]) s.v[j] -= min_val - s.spc[j];
        int j = sink;
        while (true) {
            int r = s.path[j];
            s.row4col[j] = r;
            int t = s.col4row[r];
            s.col4row[r] = j;
            j = t;
            if (r == cur) break;
        }
    }
    for (int r = 0; r < nr; ++r) {
        if (tr) s.mdet[s.col4row[r]] = r;
        else s.mdet[r] = s.col4row[r];
    }
}

// SORT's predict of every track of the class, then its deletion of tracks whose predicted box has a NaN; returns the count
// left and puts their predicted boxes in pbox.
__device__ int predict_all(const ClassState &s, int n) {
    int w = 0;
    for (int t = 0; t < n; ++t) {
        Trk k = s.trk[t];
        predict(k);
        double b[4];
        state_box(k, b);
        if (b[0] != b[0] || b[1] != b[1] || b[2] != b[2] || b[3] != b[3]) continue;
        s.trk[w] = k;
        for (int q = 0; q < 4; ++q) s.pbox[4 * w + q] = b[q];
        ++w;
    }
    return w;
}

__device__ int remove_dead(const ClassState &s, int n, int max_age) {
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
    state_box(t, b);
    out[0] = (float)b[1];
    out[1] = (float)b[0];
    out[2] = (float)b[3];
    out[3] = (float)b[2];
}

__global__ void __launch_bounds__(1024) track_update_kernel(
    unsigned char *state, const int32_t *dets, const int32_t *counts, long long row_stride, const int32_t *rows,
    const long long *positions, int n_frames, int C, int K, int cap, int max_age, int min_hits, double iou_thresh, int32_t *ids_out,
    float *boxes_out) {
    __shared__ int s_births[1024];
    __shared__ int s_base[1024];
    __shared__ int s_total;
    const int c = threadIdx.x;
    const bool active = c < C;
    const Layout L = track_layout(C, K, cap);
    TrackHeader *hdr = reinterpret_cast<TrackHeader *>(state);
    int *n_tracks = reinterpret_cast<int *>(state + L.n_tracks);
    ClassState s;
    const int cc = active ? c : 0;
    s.trk = reinterpret_cast<Trk *>(state + L.tracks) + (size_t)cc * cap;
    s.dbox = reinterpret_cast<double *>(state + L.dbox) + (size_t)cc * 4 * K;
    s.pbox = reinterpret_cast<double *>(state + L.pbox) + (size_t)cc * 4 * cap;
    s.u = reinterpret_cast<double *>(state + L.u) + (size_t)cc * K;
    s.v = reinterpret_cast<double *>(state + L.v) + (size_t)cc * cap;
    s.spc = reinterpret_cast<double *>(state + L.spc) + (size_t)cc * cap;
    s.det_k = reinterpret_cast<int *>(state + L.det_k) + (size_t)cc * K;
    s.col4row = reinterpret_cast<int *>(state + L.col4row) + (size_t)cc * K;
    s.sr = reinterpret_cast<int *>(state + L.sr) + (size_t)cc * K;
    s.path = reinterpret_cast<int *>(state + L.path) + (size_t)cc * cap;
    s.row4col = reinterpret_cast<int *>(state + L.row4col) + (size_t)cc * cap;
    s.sc = reinterpret_cast<int *>(state + L.sc) + (size_t)cc * cap;
    s.remaining = reinterpret_cast<int *>(state + L.remaining) + (size_t)cc * cap;
    s.mdet = reinterpret_cast<int *>(state + L.mdet) + (size_t)cc * K;
    s.born = reinterpret_cast<int *>(state + L.born) + (size_t)cc * K;

    long long fc = hdr->frame_count, last = hdr->last_pos;
    int taken = hdr->ids_taken, started = hdr->started;
    int n = active ? n_tracks[c] : 0;
    for (int f = 0; f < n_frames; ++f) {
        const long long pos = positions[f];
        // a jump of g positions is g - 1 updates without detections; after max_age + 1 of them no track is left
        long long gap = started && pos > last + 1 ? pos - last - 1 : 0;
        long long empty = gap < (long long)max_age + 1 ? gap : (long long)max_age + 1;
        for (long long e = 0; e < empty; ++e) {
            n = predict_all(s, n);
            n = remove_dead(s, n, max_age);
        }
        fc += gap + 1;
        last = pos;
        started = 1;
        int nb = 0;
        if (active) {
            const int32_t *rec = dets + rows[f] * row_stride + (long long)c * K * 6;
            int cnt = counts[rows[f] * row_stride + c];
            cnt = cnt < 0 ? 0 : (cnt > K ? K : cnt);
            int32_t *ids = ids_out + ((long long)f * C + c) * K;
            float *obox = boxes_out + (((long long)f * C + c) * K) * 4;
            for (int k = 0; k < K; ++k) {
                ids[k] = -1;
                for (int q = 0; q < 4; ++q) obox[4 * k + q] = 0.f;
            }
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
                for (int j = 0; j < n; ++j) s.row4col[j] = 0;
                for (int d = 0; d < D; ++d) {
                    int above = 0;
                    for (int j = 0; j < n; ++j) {
                        if (iou(s.dbox + 4 * d, s.pbox + 4 * j) > iou_thresh) {
                            ++above;
                            s.mdet[d] = j;
                            int cnt_j = ++s.row4col[j];
                            col_max = cnt_j > col_max ? cnt_j : col_max;
                        }
                    }
                    row_max = above > row_max ? above : row_max;
                }
                if (!(row_max == 1 && col_max == 1)) lsap(s, D, n);
            }
            const bool early = fc <= min_hits;
            for (int d = 0; d < D; ++d)
                if (s.mdet[d] < 0) s.born[nb++] = d;
            for (int d = 0; d < D; ++d) {
                int j = s.mdet[d];
                if (j < 0) continue;
                if (iou(s.dbox + 4 * d, s.pbox + 4 * j) < iou_thresh) {
                    s.born[nb++] = d;
                    continue;
                }
                Trk &t = s.trk[j];
                update(t, s.dbox + 4 * d);
                if (t.streak >= min_hits || early) {
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
            s_births[c] = nb;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            int acc = 0;
            for (int q = 0; q < C; ++q) {
                s_base[q] = acc;
                acc += s_births[q];
            }
            s_total = acc;
        }
        __syncthreads();
        if (active) {
            int32_t *ids = ids_out + ((long long)f * C + c) * K;
            for (int b = 0; b < nb; ++b) {
                Trk &t = s.trk[n + b];
                t.id = taken + 1 + s_base[c] + b;
                if (0 >= min_hits || fc <= min_hits) ids[s.det_k[s.born[b]]] = t.id;
            }
            n += nb;
        }
        taken += s_total;
        __syncthreads();        // s_births / s_base / s_total are rewritten by the next frame
    }
    if (active) n_tracks[c] = n;
    if (threadIdx.x == 0) {
        hdr->frame_count = fc;
        hdr->last_pos = last;
        hdr->ids_taken = taken;
        hdr->started = started;
    }
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
    *bytes = track_layout(class_num, max_per_class, track_cap(max_per_class, max_age)).total;
    return K2Y_OK;
}

extern "C" int k2y_track_update(void *state_dev, const k2y_det *dets_dev, const int32_t *counts_dev, long long row_stride_words,
                                const int32_t *rows_dev, const long long *positions_dev, int n_frames, int class_num,
                                int max_per_class, int max_age, int min_hits, double iou_thresh, int32_t *ids_out_dev,
                                float *boxes_out_dev, void *stream) {
    const char *fn = "k2y_track_update";
    if (!track_args_ok(fn, class_num, max_per_class, max_age)) return K2Y_ERR_INVALID;
    if (!state_dev || !dets_dev || !counts_dev || !rows_dev || !positions_dev || !ids_out_dev || !boxes_out_dev || n_frames < 0 ||
        min_hits < 0 || !(iou_thresh >= 0.0 && iou_thresh <= 1.0)) {
        set_error("%s: null pointer, n_frames < 0, min_hits < 0 or iou_thresh outside [0, 1]", fn);
        return K2Y_ERR_INVALID;
    }
    if (row_stride_words < (long long)class_num * max_per_class * 6) {
        set_error("%s: row stride %lld words is smaller than one row's records", fn, row_stride_words);
        return K2Y_ERR_INVALID;
    }
    if (n_frames == 0) return K2Y_OK;
    const int threads = (class_num + 31) / 32 * 32;
    track_update_kernel<<<1, threads, 0, (cudaStream_t)stream>>>(
        (unsigned char *)state_dev, (const int32_t *)dets_dev, counts_dev, row_stride_words, rows_dev, positions_dev, n_frames,
        class_num, max_per_class, track_cap(max_per_class, max_age), max_age, min_hits, iou_thresh, ids_out_dev, boxes_out_dev);
    K2Y_CUDA_CHECK(cudaGetLastError());
    return K2Y_OK;
}
