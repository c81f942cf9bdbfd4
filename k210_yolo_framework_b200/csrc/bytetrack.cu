// ByteTrack tracking of a stream's gathered detection records (oracle/bytetrack_ref.py states every rule; this is it bit for
// bit).
//
// One CTA per stream, one warp per class (the warps stride over the classes when there are more): a class's track lists,
// associations and Kalman filters are its warp's alone.  The lanes predict and update the tracks, compact the ordered lists
// with ballots, and solve each association with warp_lsap (lsap_warp.cuh, scipy's assignment, ties included), whose cost
// functor computes the IoU costs on the fly.  The classes meet once per frame in frame_loop (tracker.cuh), where the
// frame's births take their ids from one counter in (class, birth) order.  The launch walks the batch's frames in order.
//
// The state lives in global memory between launches (BT_ARRAYS): the stream's header, and per class its two lists, tracked
// then lost, in one of two track buffers (each frame's rebuild writes the other), plus per-class scratch.  Each buffer
// holds cap = K (max(B, 1) + 2) tracks, the bound oracle/bytetrack_ref.py derives for the tracks of a class within a frame;
// the host refuses a setting where it passes BT_MAX.
//
// Float64 throughout, in the oracle's operation order: every product is __dmul_rn (so nothing contracts into an FMA),
// division and sqrt are IEEE round-to-nearest.
#include <cmath>

#include "common.h"
#include "tracker.cuh"

namespace k2y {
namespace {

constexpr int BT_MAX = 4096;                       // tracks per class (track.py BYTETRACK_MAX_TRACKS_PER_CLASS)
constexpr double W_P = 1.0 / 20, W_V = 1.0 / 160;
constexpr double LOW_THRESH = 0.1, SECOND_THRESH = 0.5, UNCONFIRMED_THRESH = 0.7, DUPLICATE_THRESH = 0.15;
constexpr int TRACKED = 1, LOST = 2, REMOVED = 3;
constexpr int BT_WARPS = 8, BT_THREADS = BT_WARPS * 32;    // 148 registers a thread, no spills (at 16 warps, 128 spill)

struct BTrk {
    double m[8];            // x, y, a, h, then their velocities
    double P[4][3];         // per block (x, y, a, h): P_pp, P_pv, P_vv
    int id, state, activated, frame_id, start_frame, rec;
};

struct BDet {
    double tlwh[4], tlbr[4], score;
    int k, pad;
};

__host__ __device__ inline int bt_cap(int K, int B) { return K * ((B > 1 ? B : 1) + 2); }

// Every per-class array: type, name, entries per class (k = K records, n = cap tracks).
#define BT_ARRAYS(X)                                                                                                        \
    X(int, lists, 4)                /* n_tracked, n_lost, buffer */                                                         \
    X(BTrk, trk, 2 * n)             /* the two track buffers */                                                             \
    X(BTrk, born, k)                                                                                                        \
    X(BDet, high, k)                                                                                                        \
    X(BDet, low, k)                                                                                                         \
    X(int, pool, n) X(int, unc, n) X(int, rest, n) X(int, match, n) X(int, nlist, n) X(int, drop, n)                        \
    X(int, left, k) X(int, hm, k)                                                                                           \
    X(double, pbox, 4 * n) X(double, ubox, 4 * n) X(double, nbox, 4 * n)

struct ClassView {
    BT_ARRAYS(K2Y_STATE_FIELD)
    LsapWork w;
};

__device__ ClassView class_view(unsigned char *state, size_t C, int c, size_t k, size_t n) {
    ClassView v;
    size_t o = state_start();
    BT_ARRAYS(K2Y_STATE_SLICE)
    K2Y_LSAP_ARRAYS(K2Y_STATE_SLICE, n, n)
    return v;
}

size_t state_bytes(size_t C, size_t k, size_t n) {
    size_t o = state_start();
    BT_ARRAYS(K2Y_STATE_BYTES)
    K2Y_LSAP_ARRAYS(K2Y_STATE_BYTES, n, n)
    return o;
}

// Cython's min / max: the second operand when it compares below / above the first
__device__ __forceinline__ double cmin(double a, double b) { return b < a ? b : a; }
__device__ __forceinline__ double cmax(double a, double b) { return b > a ? b : a; }

// cython_bbox.bbox_overlaps of box a (a track's tlbr) and query box b, 0 where the union is not > 0
__device__ double iou(const double *a, const double *b) {
    const double iw = (cmin(a[2], b[2]) - cmax(a[0], b[0])) + 1.0;
    if (iw > 0) {
        const double ih = (cmin(a[3], b[3]) - cmax(a[1], b[1])) + 1.0;
        if (ih > 0) {
            const double inter = mul(iw, ih);
            const double ua = (mul((a[2] - a[0]) + 1.0, (a[3] - a[1]) + 1.0) + mul((b[2] - b[0]) + 1.0, (b[3] - b[1]) + 1.0)) - inter;
            return ua > 0 ? inter / ua : 0.0;
        }
    }
    return 0.0;
}

__device__ __forceinline__ double cost(const double *t, const BDet &d, bool fuse) {
    const double c = 1.0 - iou(t, d.tlbr);
    return fuse ? 1.0 - mul(1.0 - c, d.score) : c;
}

__device__ void tlbr(const BTrk &t, double *b) {
    const double w = mul(t.m[2], t.m[3]);
    const double x1 = t.m[0] - w / 2.0, y1 = t.m[1] - t.m[3] / 2.0;
    b[0] = x1;
    b[1] = y1;
    b[2] = w + x1;
    b[3] = t.m[3] + y1;
}

__device__ void initiate(BTrk &t, const BDet &d, int f, int birth) {
    const double x1 = d.tlwh[0], y1 = d.tlwh[1], w = d.tlwh[2], h = d.tlwh[3];
    t.m[0] = x1 + w / 2.0;
    t.m[1] = y1 + h / 2.0;
    t.m[2] = w / h;
    t.m[3] = h;
    for (int b = 4; b < 8; ++b) t.m[b] = 0.0;
    const double sp = mul(mul(2.0, W_P), h), sv = mul(mul(10.0, W_V), h);
    for (int b = 0; b < 4; ++b) {
        t.P[b][0] = b == 2 ? mul(1e-2, 1e-2) : mul(sp, sp);
        t.P[b][1] = 0.0;
        t.P[b][2] = b == 2 ? mul(1e-5, 1e-5) : mul(sv, sv);
    }
    t.id = -(birth + 1);            // the birth's place in the class; its id once the frame's prefix is known
    t.state = TRACKED;
    t.activated = f == 1;
    t.frame_id = t.start_frame = f;
    t.rec = d.k;
}

__device__ void predict(BTrk &t) {
    if (t.state != TRACKED) t.m[7] = 0.0;
    const double qp = mul(W_P, t.m[3]), qv = mul(W_V, t.m[3]);
    for (int b = 0; b < 4; ++b) {
        const double Qp = b == 2 ? mul(1e-2, 1e-2) : mul(qp, qp), Qv = b == 2 ? mul(1e-5, 1e-5) : mul(qv, qv);
        const double a = t.P[b][0], pv = t.P[b][1], d = t.P[b][2];
        const double s = pv + d;
        t.m[b] = t.m[b] + t.m[4 + b];
        t.P[b][0] = ((a + pv) + s) + Qp;
        t.P[b][1] = s;
        t.P[b][2] = d + Qv;
    }
}

__device__ void update(BTrk &t, const BDet &d, int f) {
    const double x1 = d.tlwh[0], y1 = d.tlwh[1], w = d.tlwh[2], h = d.tlwh[3];
    const double z[4] = {x1 + w / 2.0, y1 + h / 2.0, w / h, h};
    const double r = mul(W_P, t.m[3]);
    for (int b = 0; b < 4; ++b) {
        const double R = b == 2 ? mul(1e-1, 1e-1) : mul(r, r);
        const double a = t.P[b][0], pv = t.P[b][1], dd = t.P[b][2];
        const double S = a + R, L = sqrt(S);
        const double k0 = (a / L) / L, k1 = (pv / L) / L;
        const double y = z[b] - t.m[b];
        t.m[b] = t.m[b] + mul(k0, y);
        t.m[4 + b] = t.m[4 + b] + mul(k1, y);
        const double ks0 = mul(k0, S), ks1 = mul(k1, S);
        t.P[b][0] = a - mul(ks0, k0);
        t.P[b][1] = pv - mul(ks0, k1);
        t.P[b][2] = dd - mul(ks1, k1);
    }
    t.frame_id = f;
    t.state = TRACKED;
    t.activated = 1;
    t.rec = d.k;
}

// 1 high, 2 low, 0 not a detection (oracle/bytetrack_ref.py ``detections``); fills d for a detection
__device__ int load_det(const int32_t *rec, int k, double track_thresh, BDet &d) {
    const double ymin = __int_as_float(rec[6 * k]), xmin = __int_as_float(rec[6 * k + 1]);
    const double ymax = __int_as_float(rec[6 * k + 2]), xmax = __int_as_float(rec[6 * k + 3]);
    if (!(isfinite(ymin) && isfinite(xmin) && isfinite(ymax) && isfinite(xmax))) return 0;
    const double w = xmax - xmin, h = ymax - ymin;
    if (!(w > 0 && h > 0)) return 0;
    const double s = __int_as_float(rec[6 * k + 4]);
    const int kind = s > track_thresh ? 1 : (LOW_THRESH < s && s < track_thresh ? 2 : 0);
    d.tlwh[0] = xmin; d.tlwh[1] = ymin; d.tlwh[2] = w; d.tlwh[3] = h;
    d.tlbr[0] = xmin; d.tlbr[1] = ymin; d.tlbr[2] = w + xmin; d.tlbr[3] = h + ymin;
    d.score = s;
    d.k = k;
    return kind;
}

// oracle/bytetrack_ref.py ``assign``: match[i] = the column of row i whose cost is < thresh in the assignment of
// min(cost - thresh, 0), else -1.  Warp-wide.
template <class Cost>
__device__ void assign(int nr, int nc, const Cost &c, double thresh, const LsapWork &w, int *match) {
    const int lane = threadIdx.x & 31;
    if (nr == 0) return;
    if (nc == 0) {
        for (int i = lane; i < nr; i += 32) match[i] = -1;
        __syncwarp();
        return;
    }
    auto reduced = [&](int i, int j) {
        const double x = c(i, j) - thresh;
        return 0.0 < x ? 0.0 : x;
    };
    warp_lsap(nr, nc, reduced, w, match);
    for (int i = lane; i < nr; i += 32) {
        const int j = match[i];
        if (j >= 0 && !(c(i, j) < thresh)) match[i] = -1;
    }
    __syncwarp();
}

struct Setting {
    double track_thresh, match_thresh, det_thresh;
    int buffer, cap;
    bool fuse;
};

// One update of one class at frame id f (oracle/bytetrack_ref.py ``ByteTrack._step``), over its records rec[0..cnt) (none
// for an update without detections).  Leaves the new lists in the other buffer, births with ids -(b + 1); returns the
// births.  Warp-wide.
__device__ int class_step(const ClassView &s, int f, const int32_t *rec, int cnt, const Setting &st) {
    const int lane = threadIdx.x & 31;
    const int nt = s.lists[0], nl = s.lists[1], buf = s.lists[2];
    BTrk *in = s.trk + (size_t)buf * st.cap, *out = s.trk + (size_t)(buf ^ 1) * st.cap;
    BDet tmp;
    const int nh = compact(cnt, [&](int k) { return load_det(rec, k, st.track_thresh, tmp) == 1; },
                           [&](int k, int at) { load_det(rec, k, st.track_thresh, s.high[at]); });
    const int nlo = compact(cnt, [&](int k) { return load_det(rec, k, st.track_thresh, tmp) == 2; },
                            [&](int k, int at) { load_det(rec, k, st.track_thresh, s.low[at]); });
    // 1. unconfirmed, and the pool = active + lost, predicted
    const int na = compact(nt, [&](int i) { return in[i].activated != 0; }, [&](int i, int at) { s.pool[at] = i; });
    const int nu = compact(nt, [&](int i) { return in[i].activated == 0; }, [&](int i, int at) { s.unc[at] = i; });
    const int np = na + nl;
    for (int i = lane; i < nl; i += 32) s.pool[na + i] = nt + i;
    for (int j = lane; j < nh; j += 32) s.hm[j] = 0;
    __syncwarp();
    for (int i = lane; i < np; i += 32) {
        BTrk &t = in[s.pool[i]];
        predict(t);
        tlbr(t, s.pbox + 4 * i);
    }
    for (int i = lane; i < nu; i += 32) tlbr(in[s.unc[i]], s.ubox + 4 * i);
    __syncwarp();
    // 2. pool x high detections; a Lost track matched is re-activated
    assign(np, nh, [&](int i, int j) { return cost(s.pbox + 4 * i, s.high[j], st.fuse); }, st.match_thresh, s.w, s.match);
    for (int i = lane; i < np; i += 32) {
        const int j = s.match[i];
        if (j >= 0) {
            update(in[s.pool[i]], s.high[j], f);
            s.hm[j] = 1;
        }
    }
    __syncwarp();
    // 3. the unmatched active rows x low detections; the rows left become Lost
    const int nr = compact(na, [&](int i) { return s.match[i] < 0; }, [&](int i, int at) { s.rest[at] = i; });
    assign(nr, nlo, [&](int i, int j) { return cost(s.pbox + 4 * s.rest[i], s.low[j], false); }, SECOND_THRESH, s.w, s.match);
    for (int i = lane; i < nr; i += 32) {
        BTrk &t = in[s.pool[s.rest[i]]];
        const int j = s.match[i];
        if (j >= 0) update(t, s.low[j], f);
        else t.state = LOST;
    }
    __syncwarp();
    // 4. unconfirmed x the high detections left; the unconfirmed left are removed
    const int nleft = compact(nh, [&](int j) { return s.hm[j] == 0; }, [&](int j, int at) { s.left[at] = j; });
    assign(nu, nleft, [&](int i, int j) { return cost(s.ubox + 4 * i, s.high[s.left[j]], st.fuse); }, UNCONFIRMED_THRESH, s.w,
           s.match);
    for (int i = lane; i < nu; i += 32) {
        BTrk &t = in[s.unc[i]];
        const int j = s.match[i];
        if (j >= 0) {
            update(t, s.high[s.left[j]], f);
            s.hm[s.left[j]] = 1;
        } else {
            t.state = REMOVED;
        }
    }
    __syncwarp();
    // 5. births
    const int nb = compact(nleft, [&](int j) { return s.hm[s.left[j]] == 0 && s.high[s.left[j]].score >= st.det_thresh; },
                           [&](int j, int at) { initiate(s.born[at], s.high[s.left[j]], f, at); });
    // 6, 7. tracked = still Tracked + births + re-activated; lost = old lost still Lost and within the buffer + newly lost.
    // nlist holds each entry's source: i >= 0 is in[i], -(b + 1) is births[b].
    int *nl_ = s.nlist;
    const int a = compact(nt, [&](int i) { return in[i].state == TRACKED; }, [&](int i, int at) { nl_[at] = i; });
    for (int b = lane; b < nb; b += 32) nl_[a + b] = -(b + 1);
    const int r = compact(nl, [&](int i) { return in[nt + i].state == TRACKED; }, [&](int i, int at) { nl_[a + nb + at] = nt + i; });
    const int ntn = a + nb + r;
    const int d = compact(nl, [&](int i) { const BTrk &t = in[nt + i]; return t.state == LOST && !(f - t.frame_id > st.buffer); },
                          [&](int i, int at) { nl_[ntn + at] = nt + i; });
    const int e = compact(nt, [&](int i) { return in[i].state == LOST; }, [&](int i, int at) { nl_[ntn + d + at] = i; });
    const int nln = d + e;
    auto src = [&](int q) -> const BTrk & { const int x = nl_[q]; return x >= 0 ? in[x] : s.born[-x - 1]; };
    for (int q = lane; q < ntn + nln; q += 32) {
        tlbr(src(q), s.nbox + 4 * q);
        s.drop[q] = 0;
    }
    __syncwarp();
    // 8. duplicates between tracked and lost
    for (int p = 0; p < ntn; ++p) {
        const BTrk &A = src(p);
        const int ta = A.frame_id - A.start_frame;
        for (int q = lane; q < nln; q += 32) {
            if (1.0 - iou(s.nbox + 4 * p, s.nbox + 4 * (ntn + q)) < DUPLICATE_THRESH) {
                const BTrk &Bq = src(ntn + q);
                if (ta > Bq.frame_id - Bq.start_frame) s.drop[ntn + q] = 1;
                else s.drop[p] = 1;
            }
        }
    }
    __syncwarp();
    const int nt2 = compact(ntn, [&](int q) { return s.drop[q] == 0; }, [&](int q, int at) { out[at] = src(q); });
    const int nl2 = compact(nln, [&](int q) { return s.drop[ntn + q] == 0; }, [&](int q, int at) { out[nt2 + at] = src(ntn + q); });
    if (lane == 0) {
        s.lists[0] = nt2;
        s.lists[1] = nl2;
        s.lists[2] = buf ^ 1;
    }
    __syncwarp();
    return nb;
}

// The batch and the setting are read in place from the parameters (__grid_constant__), as the callbacks take them by
// reference.
__global__ void __launch_bounds__(BT_THREADS, 1) bytetrack_update_kernel(unsigned char *state, const __grid_constant__ Batch bt,
                                                                         const __grid_constant__ Setting st) {
    __shared__ ClassView s_view[BT_WARPS];      // the warp's class, in shared memory to keep its pointers out of registers
    if (!stream_has_frames(bt)) return;
    state += (size_t)blockIdx.x * bt.stride;
    const int lane = threadIdx.x & 31;
    ClassView &s = s_view[threadIdx.x >> 5];
    auto view = [&](int c) { return class_view(state, bt.C, c, bt.K, st.cap); };
    auto empty = [&](long long n, long long fc) {
        for_each_class(bt.C, s, view, [&](int) {
            for (long long e = 0; e < n; ++e) class_step(s, (int)(fc + 1 + e), nullptr, 0, st);
        });
    };
    auto frame = [&](int f, long long fc, int *births) {
        for_each_class(bt.C, s, view, [&](int c) {
            const int32_t *rec;
            const int cnt = bt.records(f, c, rec);
            const int nb = class_step(s, (int)fc, rec, cnt, st);
            if (lane == 0) births[c] = nb;
        });
    };
    auto emit = [&](int f, long long, const int *, const int *base) {
        for_each_class(bt.C, s, view, [&](int c) {
            bt.clear(f, c, lane, 32);
            __syncwarp();
            int32_t *ids = bt.ids(f, c);
            float *obox = bt.boxes(f, c);
            BTrk *trk = s.trk + (size_t)s.lists[2] * st.cap;
            for (int i = lane; i < s.lists[0]; i += 32) {
                BTrk &t = trk[i];
                if (t.id < 0) t.id = base[c] - t.id;
                if (t.activated) {
                    double b[4];
                    tlbr(t, b);
                    ids[t.rec] = t.id;
                    write_box(obox + 4 * t.rec, b);
                }
            }
            __syncwarp();
        });
    };
    frame_loop(state, bt, (long long)st.buffer + 2, empty, frame, emit);
}

bool bt_args_ok(const char *fn, int C, int K, int B) {
    if (C < 1 || C > 1024 || K < 1 || B < 0 || (long long)K * ((B > 1 ? B : 1) + 2) > BT_MAX) {
        set_error("%s: class_num %d (1..1024), max_per_class %d (>= 1) and track_buffer %d (>= 0) with max_per_class x "
                  "(max(track_buffer, 1) + 2) <= %d tracks per class", fn, C, K, B, BT_MAX);
        return false;
    }
    return true;
}

}  // namespace
}  // namespace k2y

using namespace k2y;

extern "C" int k2y_bytetrack_state_bytes(int class_num, int max_per_class, int track_buffer, size_t *bytes) {
    if (!bytes) {
        set_error("k2y_bytetrack_state_bytes: null output");
        return K2Y_ERR_INVALID;
    }
    if (!bt_args_ok("k2y_bytetrack_state_bytes", class_num, max_per_class, track_buffer)) return K2Y_ERR_INVALID;
    *bytes = state_bytes(class_num, max_per_class, bt_cap(max_per_class, track_buffer));
    return K2Y_OK;
}

extern "C" int k2y_bytetrack_update_streams(void *state_dev, int n_streams, size_t state_stride, const k2y_det *dets_dev,
                                            const int32_t *counts_dev, long long row_stride_words, const int32_t *rows_dev,
                                            const long long *positions_dev, const int32_t *streams_dev, int n_frames,
                                            int class_num, int max_per_class, double track_thresh, double match_thresh,
                                            int track_buffer, int fuse_score, int32_t *ids_out_dev, float *boxes_out_dev,
                                            void *stream) {
    const char *fn = "k2y_bytetrack_update";
    const Batch bt{(const int32_t *)dets_dev, counts_dev, rows_dev, positions_dev, row_stride_words, n_frames, class_num,
                   max_per_class, ids_out_dev, boxes_out_dev, streams_dev, n_streams, state_stride};
    if (!bt_args_ok(fn, class_num, max_per_class, track_buffer) ||
        !batch_ok(fn, state_dev, bt, state_bytes(class_num, max_per_class, bt_cap(max_per_class, track_buffer))))
        return K2Y_ERR_INVALID;
    if (!(track_thresh >= 0.0 && track_thresh <= 1.0) || !(match_thresh >= 0.0 && match_thresh <= 1.0)) {
        set_error("%s: track_thresh or match_thresh outside [0, 1]", fn);
        return K2Y_ERR_INVALID;
    }
    if (n_frames == 0) return K2Y_OK;
    Setting st;
    st.track_thresh = track_thresh;
    st.match_thresh = match_thresh;
    st.det_thresh = track_thresh + 0.1;
    st.buffer = track_buffer;
    st.cap = bt_cap(max_per_class, track_buffer);
    st.fuse = fuse_score != 0;
    const int threads = (class_num < BT_WARPS ? class_num : BT_WARPS) * 32;
    bytetrack_update_kernel<<<n_streams, threads, 0, (cudaStream_t)stream>>>((unsigned char *)state_dev, bt, st);
    K2Y_CUDA_CHECK(cudaGetLastError());
    return K2Y_OK;
}

extern "C" int k2y_bytetrack_update(void *state_dev, const k2y_det *dets_dev, const int32_t *counts_dev, long long row_stride_words,
                                    const int32_t *rows_dev, const long long *positions_dev, int n_frames, int class_num,
                                    int max_per_class, double track_thresh, double match_thresh, int track_buffer, int fuse_score,
                                    int32_t *ids_out_dev, float *boxes_out_dev, void *stream) {
    return k2y_bytetrack_update_streams(state_dev, 1, 0, dets_dev, counts_dev, row_stride_words, rows_dev, positions_dev, nullptr,
                                        n_frames, class_num, max_per_class, track_thresh, match_thresh, track_buffer, fuse_score,
                                        ids_out_dev, boxes_out_dev, stream);
}
