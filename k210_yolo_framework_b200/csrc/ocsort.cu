// OC-SORT tracking of a stream's gathered detection records (oracle/ocsort_ref.py states every rule; this is it bit for
// bit).
//
// One CTA per stream, one warp per class (the warps stride over the classes when there are more), as bytetrack.cu.  The
// lanes predict the tracks, update the matched ones (a re-found track replays its ORU path, at most max_age + 1 steps, on its
// lane) and keep the ordered lists with ballots.  The filter and the IoU are SORT's (tracker.cuh).  Each association is one
// warp_lsap (lsap_warp.cuh): round 1's cost -(iou + angle) is worked out once per pair into scratch, the IoU of rounds 2 and
// 3 in the cost functor.  The classes meet once per frame in frame_loop (tracker.cuh), where the births take their ids from
// one counter in (class, birth) order.
//
// The state lives in global memory between launches (OC_ARRAYS): the stream's header, and per class its track list (slot
// numbers in list order), cap = K (max_age + 1) track slots, the bound oracle/ocsort_ref.py derives, and scratch, round 1's
// K x cap cost matrix among it.  The host refuses a setting where cap passes OC_MAX.
//
// Float64 throughout, in the oracle's operation order: every product is __dmul_rn (so nothing contracts into an FMA),
// division and sqrt are IEEE round-to-nearest, and acos is fdlibm's, as the oracle restates it.
#include <cmath>

#include "common.h"
#include "tracker.cuh"

namespace k2y {
namespace {

constexpr int OC_MAX = 4096;                      // tracks per class (track.py OCSORT_MAX_TRACKS_PER_CLASS)
constexpr int DT_MAX = 8;                         // delta_t, the ring of observations each track keeps
constexpr double LOW_THRESH = 0.1;
constexpr int OC_WARPS = 8, OC_THREADS = OC_WARPS * 32;

struct OTrk {
    Filt kf, frozen;
    double last_z[4];                // the observation history's last z
    double last_obs[5];              // (x1, y1, x2, y2, score) or the sentinel
    double ring[DT_MAX][5];          // observations at age ring_age[a % delta_t]
    double vel[2];                   // (dy, dx), 0 until set
    double pb[4];                    // this frame's predicted box
    int ring_age[DT_MAX];
    int id, hits, hit_streak, tsu, age, observed, has_frozen, n_hist, last_i;
};

struct ODet {
    double b[5];                     // x1, y1, x2, y2, score
    int k, pad;
};

__host__ __device__ inline int oc_cap(int K, int max_age) { return K * (max_age + 1); }

// Every per-class array: type, name, entries per class (k = K records, n = cap track slots).
#define OC_ARRAYS(X)                                                                                                        \
    X(int, n, 1)                    /* the list's length */                                                                 \
    X(int, ord, n) X(int, ord2, n)  /* the list: slot numbers in list order */                                              \
    X(OTrk, trk, n)                                                                                                         \
    X(ODet, high, k) X(ODet, low, k)                                                                                        \
    X(double, pbox, 4 * n)                                                                                                  \
    X(double, prev, 5 * n)          /* k-previous centre (cx, cy), valid, velocity (dy, dx) */                              \
    X(double, cost, k * n)          /* round 1's cost matrix */                                                             \
    X(int, colc, n) X(int, rowp, k) X(int, match, n) X(int, dflag, k) X(int, tflag, n) X(int, ud, k) X(int, ut, n)          \
    X(int, owner, k) X(int, born, k) X(int, freel, n)

struct ClassView {
    OC_ARRAYS(K2Y_STATE_FIELD)
    LsapWork w;
};

__device__ ClassView class_view(unsigned char *state, size_t C, int c, size_t k, size_t n) {
    ClassView v;
    size_t o = state_start();
    OC_ARRAYS(K2Y_STATE_SLICE)
    K2Y_LSAP_ARRAYS(K2Y_STATE_SLICE, n, n)
    return v;
}

size_t state_bytes(size_t C, size_t k, size_t n) {
    size_t o = state_start();
    OC_ARRAYS(K2Y_STATE_BYTES)
    K2Y_LSAP_ARRAYS(K2Y_STATE_BYTES, n, n)
    return o;
}

// -- fdlibm's __ieee754_acos (oracle/ocsort_ref.py ``acos``) ---------------------------------------------------------------
constexpr double PI = 3.14159265358979311600e+00, PIO2_HI = 1.57079632679489655800e+00, PIO2_LO = 6.12323399573676603587e-17;

__device__ double acos_pq(double z) {
    const double p = mul(z, 1.66666666666666657415e-01 +
                               mul(z, -3.25565818622400915405e-01 +
                                          mul(z, 2.01212532134862925881e-01 +
                                                     mul(z, -4.00555345006794114027e-02 +
                                                                mul(z, 7.91534994289814532176e-04 +
                                                                           mul(z, 3.47933107596021167570e-05))))));
    const double q = 1.0 + mul(z, -2.40339491173441421878e+00 +
                                      mul(z, 2.02094576023350569471e+00 +
                                                 mul(z, -6.88283971605453293030e-01 + mul(z, 7.70381505559019352791e-02))));
    return p / q;
}

__device__ double fd_acos(double x) {
    const long long u = __double_as_longlong(x);
    const int hx = (int)(u >> 32);
    const unsigned lx = (unsigned)(u & 0xffffffffLL);
    const int ix = hx & 0x7fffffff;
    if (ix >= 0x3ff00000) {
        if (((unsigned)(ix - 0x3ff00000) | lx) == 0) return hx > 0 ? 0.0 : PI + mul(2.0, PIO2_LO);
        return CUDART_NAN;
    }
    if (ix < 0x3fe00000) {
        if (ix <= 0x3c600000) return PIO2_HI + PIO2_LO;
        const double r = acos_pq(mul(x, x));
        return PIO2_HI - (x - (PIO2_LO - mul(x, r)));
    }
    if (hx < 0) {
        const double z = mul(1.0 + x, 0.5);
        const double s = sqrt(z);
        const double r = acos_pq(z);
        const double w = mul(r, s) - PIO2_LO;
        return PI - mul(2.0, s + w);
    }
    const double z = mul(1.0 - x, 0.5);
    const double s = sqrt(z);
    const double df = __hiloint2double(__double2hiint(s), 0);
    const double c = (z - mul(df, df)) / (s + df);
    const double r = acos_pq(z);
    const double w = mul(r, s) + c;
    return mul(2.0, df + w);
}

// -- the filter: SORT's (tracker.cuh), fed OC-SORT's z ----------------------------------------------------------------
__device__ void to_z(const double *b, double *z) {
    const double w = b[2] - b[0], h = b[3] - b[1];
    z[0] = b[0] + w / 2.0;
    z[1] = b[1] + h / 2.0;
    z[2] = mul(w, h);
    z[3] = w / (h + 1e-6);
}

// -- boxes -----------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double sum5(const double *o) { return (((o[0] + o[1]) + o[2]) + o[3]) + o[4]; }

// the unit (dy, dx) from centre (cx1, cy1) to (cx2, cy2)
__device__ void direction(double cx1, double cy1, double cx2, double cy2, double &uy, double &ux) {
    const double dy = cy2 - cy1, dx = cx2 - cx1;
    const double norm = sqrt(mul(dy, dy) + mul(dx, dx)) + 1e-6;
    uy = dy / norm;
    ux = dx / norm;
}

struct Setting {
    double iou_thresh, det_thresh, inertia;
    int max_age, min_hits, delta_t, use_byte, cap;
};

// -- a track ---------------------------------------------------------------------------------------------------------------
__device__ void birth(OTrk &t, const ODet &d, int b) {
    double z[4];
    to_z(d.b, z);
    filt_init(t.kf, z);
    for (int q = 0; q < 5; ++q) t.last_obs[q] = -1.0;
    for (int q = 0; q < DT_MAX; ++q) t.ring_age[q] = -1;
    t.vel[0] = t.vel[1] = 0.0;
    t.id = -(b + 1);                // the birth's place in the class; its id once the frame's prefix is known
    t.hits = t.hit_streak = t.tsu = t.age = 0;
    t.observed = t.has_frozen = t.n_hist = 0;
    t.last_i = -1;
}

// SORT's tracker predict; leaves the predicted box in t.pb.
__device__ void predict(OTrk &t) {
    sort_predict(t);
    state_box(t.kf, t.pb);
}

// k_previous_obs: the observation at age - dt for the first dt from delta_t down to 1, else last_obs
__device__ const double *k_previous(const OTrk &t, int delta_t) {
    for (int dt = delta_t; dt >= 1; --dt) {
        const int a = t.age - dt;
        if (a >= 0 && t.ring_age[a % delta_t] == a) return t.ring[a % delta_t];
    }
    return t.last_obs;
}

// The filter's update with z, or without (z null): freeze on a loss, ORU on the re-find.
__device__ void filt_observe(OTrk &t, const double *z) {
    const int i = t.n_hist++;
    if (!z) {
        if (t.observed) {
            t.frozen = t.kf;
            t.has_frozen = 1;
            t.observed = 0;
        }
        return;
    }
    if (!t.observed && t.has_frozen) {
        t.kf = t.frozen;
        t.has_frozen = 0;
        const double gap = (double)(i - t.last_i);
        const double x1 = t.last_z[0], y1 = t.last_z[1], s1 = t.last_z[2], r1 = t.last_z[3];
        const double w1 = sqrt(mul(s1, r1)), h1 = sqrt(s1 / r1);
        const double w2 = sqrt(mul(z[2], z[3])), h2 = sqrt(z[2] / z[3]);
        const double dx = (z[0] - x1) / gap, dy = (z[1] - y1) / gap, dw = (w2 - w1) / gap, dh = (h2 - h1) / gap;
        const int steps = i - t.last_i;
        double vz[4];
        for (int k = 0; k < steps; ++k) {
            const double f = (double)(k + 1);
            const double w = w1 + mul(f, dw), h = h1 + mul(f, dh);
            vz[0] = x1 + mul(f, dx);
            vz[1] = y1 + mul(f, dy);
            vz[2] = mul(w, h);
            vz[3] = w / h;
            filt_update(t.kf, vz);
            if (k != steps - 1) filt_predict(t.kf);
        }
        for (int q = 0; q < 4; ++q) t.last_z[q] = vz[q];
    } else {
        for (int q = 0; q < 4; ++q) t.last_z[q] = z[q];
    }
    t.last_i = i;
    t.observed = 1;
    filt_update(t.kf, z);
}

// A matched update with detection d (oracle/ocsort_ref.py ``_Track.update``).
__device__ void observe(OTrk &t, const ODet &d, int delta_t) {
    if (sum5(t.last_obs) >= 0) {
        const double *p = k_previous(t, delta_t);
        direction((p[0] + p[2]) / 2.0, (p[1] + p[3]) / 2.0, (d.b[0] + d.b[2]) / 2.0, (d.b[1] + d.b[3]) / 2.0, t.vel[0], t.vel[1]);
    }
    for (int q = 0; q < 5; ++q) t.last_obs[q] = d.b[q];
    const int slot = t.age % delta_t;
    for (int q = 0; q < 5; ++q) t.ring[slot][q] = d.b[q];
    t.ring_age[slot] = t.age;
    t.tsu = 0;
    t.hits += 1;
    t.hit_streak += 1;
    double z[4];
    to_z(d.b, z);
    filt_observe(t, z);
}

// 1 high, 2 low, 0 neither (oracle/ocsort_ref.py ``detections``); fills d for both
__device__ int load_det(const int32_t *rec, int k, const Setting &st, ODet &d) {
    const double ymin = __int_as_float(rec[6 * k]), xmin = __int_as_float(rec[6 * k + 1]);
    const double ymax = __int_as_float(rec[6 * k + 2]), xmax = __int_as_float(rec[6 * k + 3]);
    if (!(isfinite(ymin) && isfinite(xmin) && isfinite(ymax) && isfinite(xmax))) return 0;
    if (!(xmax - xmin > 0 && ymax - ymin > 0)) return 0;
    const double s = __int_as_float(rec[6 * k + 4]);
    const int kind = s > st.det_thresh ? 1 : (st.use_byte && LOW_THRESH < s && s < st.det_thresh ? 2 : 0);
    d.b[0] = xmin; d.b[1] = ymin; d.b[2] = xmax; d.b[3] = ymax; d.b[4] = s;
    d.k = k;
    return kind;
}

__device__ double warp_max(double v) {
    for (int o = 16; o > 0; o >>= 1) {
        const double x = __shfl_xor_sync(0xffffffffu, v, o);
        v = x > v ? x : v;
    }
    return v;
}

__device__ int warp_sum(int v) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Rounds 2 and 3 (oracle/ocsort_ref.py ``_rematch``): when the largest IoU of the nr x nc pairs is > thresh, match[i] = the
// column of row i in lsap(-iou) when that pair's iou is not < thresh, else -1; returns false (match untouched) otherwise.
// Warp-wide.
template <class Iou>
__device__ bool rematch(int nr, int nc, const Iou &io, double thresh, const LsapWork &w, int *match) {
    const int lane = threadIdx.x & 31;
    double best = -CUDART_INF;
    for (int x = lane; x < nr * nc; x += 32) {
        const double v = io(x / nc, x % nc);
        best = v > best ? v : best;
    }
    if (!(warp_max(best) > thresh)) return false;
    warp_lsap(nr, nc, [&](int i, int j) { return -io(i, j); }, w, match);
    for (int i = lane; i < nr; i += 32) {
        const int j = match[i];
        if (j >= 0 && io(i, j) < thresh) match[i] = -1;
    }
    __syncwarp();
    return true;
}

// One update of one class at frame count fc (oracle/ocsort_ref.py ``OcSort._step``) over its records rec[0..cnt) (none
// for an update without detections).  Births get ids -(b + 1) and their slots in s.born; owner[k] is the slot record k
// updated or created, else -1.  Returns the births.  Warp-wide.
__device__ int class_step(const ClassView &s, const int32_t *rec, int cnt, int K, const Setting &st) {
    const int lane = threadIdx.x & 31;
    const int cap = st.cap;
    OTrk *trk = s.trk;
    int *ord = s.ord;
    for (int k = lane; k < K; k += 32) s.owner[k] = -1;
    // predict; a track whose predicted box has a NaN is deleted
    const int n0 = *s.n;
    for (int i = lane; i < n0; i += 32) predict(trk[ord[i]]);
    __syncwarp();
    const int T = compact(n0, [&](int i) { const double *b = trk[ord[i]].pb; return !(b[0] != b[0] || b[1] != b[1] || b[2] != b[2] || b[3] != b[3]); },
                          [&](int i, int at) { s.ord2[at] = ord[i]; });
    for (int j = lane; j < T; j += 32) {
        ord[j] = s.ord2[j];
        const OTrk &t = trk[ord[j]];
        for (int q = 0; q < 4; ++q) s.pbox[4 * j + q] = t.pb[q];
        const double *p = k_previous(t, st.delta_t);
        double *pv = s.prev + 5 * j;
        pv[0] = (p[0] + p[2]) / 2.0;
        pv[1] = (p[1] + p[3]) / 2.0;
        pv[2] = p[4] < 0 ? 0.0 : 1.0;
        pv[3] = t.vel[0];
        pv[4] = t.vel[1];
    }
    ODet tmp;
    const int D = compact(cnt, [&](int k) { return load_det(rec, k, st, tmp) == 1; }, [&](int k, int at) { load_det(rec, k, st, s.high[at]); });
    const int NL = st.use_byte ? compact(cnt, [&](int k) { return load_det(rec, k, st, tmp) == 2; },
                                         [&](int k, int at) { load_det(rec, k, st, s.low[at]); })
                               : 0;
    // round 1: high detections x predicted tracks, by IoU and the direction term
    for (int d = lane; d < D; d += 32) s.dflag[d] = 0;          // 0 untouched, 1 matched, 2 dropped
    for (int j = lane; j < T; j += 32) s.tflag[j] = 0;          // 1 touched by round 1's pairs
    __syncwarp();
    if (D > 0 && T > 0) {
        for (int j = lane; j < T; j += 32) s.colc[j] = 0;
        int rowmax = 0;
        for (int d = 0; d < D; ++d) {
            const double *db = s.high[d].b;
            double *crow = s.cost + (size_t)d * cap;
            int cntd = 0, pick = -1;
            for (int j = lane; j < T; j += 32) {
                const double v = sort_iou(db, s.pbox + 4 * j);
                crow[j] = v;
                if (v > st.iou_thresh) {
                    ++cntd;
                    ++s.colc[j];
                    pick = j;
                }
            }
            const int tot = warp_sum(cntd);
            const unsigned who = __ballot_sync(0xffffffffu, pick >= 0);
            const int p = who ? __shfl_sync(0xffffffffu, pick, __ffs(who) - 1) : -1;
            if (lane == 0) s.rowp[d] = tot == 1 ? p : -1;
            rowmax = tot > rowmax ? tot : rowmax;
        }
        int colmax = 0;
        for (int j = lane; j < T; j += 32) colmax = s.colc[j] > colmax ? s.colc[j] : colmax;
        for (int o = 16; o > 0; o >>= 1) {
            const int x = __shfl_xor_sync(0xffffffffu, colmax, o);
            colmax = x > colmax ? x : colmax;
        }
        __syncwarp();
        if (rowmax == 1 && colmax == 1) {
            for (int d = lane; d < D; d += 32) s.match[d] = s.rowp[d];
        } else {
            for (int d = 0; d < D; ++d) {
                const ODet &dt = s.high[d];
                const double cx = (dt.b[0] + dt.b[2]) / 2.0, cy = (dt.b[1] + dt.b[3]) / 2.0;
                double *crow = s.cost + (size_t)d * cap;
                for (int j = lane; j < T; j += 32) {
                    const double *pv = s.prev + 5 * j;
                    double uy, ux;
                    direction(pv[0], pv[1], cx, cy, uy, ux);
                    double c = mul(pv[4], ux) + mul(pv[3], uy);
                    c = c < -1.0 ? -1.0 : (c > 1.0 ? 1.0 : c);
                    const double a = (PI / 2.0 - fabs(fd_acos(c))) / PI;
                    const double ang = mul(mul(mul(pv[2], a), st.inertia), dt.b[4]);
                    crow[j] = -(crow[j] + ang);
                }
            }
            __syncwarp();
            warp_lsap(D, T, [&](int i, int j) { return s.cost[(size_t)i * cap + j]; }, s.w, s.match);
        }
        for (int d = lane; d < D; d += 32) {
            const int j = s.match[d];
            if (j >= 0) {
                s.tflag[j] = 1;
                s.dflag[d] = sort_iou(s.high[d].b, s.pbox + 4 * j) < st.iou_thresh ? 2 : 1;
            }
        }
        __syncwarp();
        for (int d = lane; d < D; d += 32)
            if (s.dflag[d] == 1) {
                const int slot = ord[s.match[d]];
                observe(trk[slot], s.high[d], st.delta_t);
                s.owner[s.high[d].k] = slot;
            }
        __syncwarp();
    }
    // unmatched, in SORT's order: untouched ascending, then the dropped pairs' in match order
    int nud = compact(D, [&](int d) { return s.dflag[d] == 0; }, [&](int d, int at) { s.ud[at] = d; });
    nud += compact(D, [&](int d) { return s.dflag[d] == 2; }, [&](int d, int at) { s.ud[nud + at] = d; });
    int nut = compact(T, [&](int j) { return s.tflag[j] == 0; }, [&](int j, int at) { s.ut[at] = j; });
    nut += compact(D, [&](int d) { return s.dflag[d] == 2; }, [&](int d, int at) { s.ut[nut + at] = s.match[d]; });
    // round 2 (BYTE): low detections x the unmatched tracks' predicted boxes
    if (NL > 0 && nut > 0) {
        const bool ran = rematch(NL, nut, [&](int i, int j) { return sort_iou(s.low[i].b, s.pbox + 4 * s.ut[j]); },
                                 st.iou_thresh, s.w, s.match);
        if (ran) {
            for (int j = lane; j < T; j += 32) s.tflag[j] = 0;          // 1 unmatched, 2 taken here
            __syncwarp();
            for (int j = lane; j < nut; j += 32) s.tflag[s.ut[j]] = 1;
            __syncwarp();
            for (int i = lane; i < NL; i += 32) {
                const int j = s.match[i];
                if (j >= 0) {
                    const int slot = ord[s.ut[j]];
                    observe(trk[slot], s.low[i], st.delta_t);
                    s.owner[s.low[i].k] = slot;
                    s.tflag[s.ut[j]] = 2;
                }
            }
            __syncwarp();
            nut = compact(T, [&](int j) { return s.tflag[j] == 1; }, [&](int j, int at) { s.ut[at] = j; });
        }
    }
    // round 3 (OCR): the unmatched high detections x the unmatched tracks' last observations
    if (nud > 0 && nut > 0) {
        const auto io = [&](int i, int j) { return sort_iou(s.high[s.ud[i]].b, trk[ord[s.ut[j]]].last_obs); };
        const bool ran = rematch(nud, nut, io, st.iou_thresh, s.w, s.match);
        if (ran) {
            for (int j = lane; j < T; j += 32) s.tflag[j] = 0;
            for (int d = lane; d < D; d += 32) s.dflag[d] = 0;
            __syncwarp();
            for (int j = lane; j < nut; j += 32) s.tflag[s.ut[j]] = 1;
            for (int i = lane; i < nud; i += 32) s.dflag[s.ud[i]] = 1;
            __syncwarp();
            for (int i = lane; i < nud; i += 32) {
                const int j = s.match[i];
                if (j >= 0) {
                    const int slot = ord[s.ut[j]];
                    observe(trk[slot], s.high[s.ud[i]], st.delta_t);
                    s.owner[s.high[s.ud[i]].k] = slot;
                    s.tflag[s.ut[j]] = 2;
                    s.dflag[s.ud[i]] = 2;
                }
            }
            __syncwarp();
            nud = compact(D, [&](int d) { return s.dflag[d] == 1; }, [&](int d, int at) { s.ud[at] = d; });
            nut = compact(T, [&](int j) { return s.tflag[j] == 1; }, [&](int j, int at) { s.ut[at] = j; });
        }
    }
    for (int j = lane; j < nut; j += 32) filt_observe(trk[ord[s.ut[j]]], nullptr);
    __syncwarp();
    // the dead go, then the births are appended in list order, each in a free slot
    const int n1 = compact(T, [&](int i) { return trk[ord[i]].tsu <= st.max_age; }, [&](int i, int at) { s.ord2[at] = ord[i]; });
    for (int j = lane; j < cap; j += 32) s.tflag[j] = 0;
    __syncwarp();
    for (int i = lane; i < n1; i += 32) {
        ord[i] = s.ord2[i];
        s.tflag[ord[i]] = 1;
    }
    __syncwarp();
    compact(cap, [&](int j) { return s.tflag[j] == 0; }, [&](int j, int at) { s.freel[at] = j; });
    for (int b = lane; b < nud; b += 32) {
        const int slot = s.freel[b];
        const ODet &d = s.high[s.ud[b]];
        birth(trk[slot], d, b);
        ord[n1 + b] = slot;
        s.born[b] = slot;
        s.owner[d.k] = slot;
    }
    __syncwarp();
    if (lane == 0) *s.n = n1 + nud;
    __syncwarp();
    return nud;
}

// The batch and the setting are read in place from the parameters (__grid_constant__), as the callbacks take them by
// reference.
__global__ void __launch_bounds__(OC_THREADS, 1) ocsort_update_kernel(unsigned char *state, const __grid_constant__ Batch bt,
                                                                      const __grid_constant__ Setting st) {
    __shared__ ClassView s_view[OC_WARPS];      // the warp's class, in shared memory to keep its pointers out of registers
    const int lane = threadIdx.x & 31, K = bt.K;
    ClassView &s = s_view[threadIdx.x >> 5];
    auto view = [&](int c) { return class_view(state, bt.C, c, K, st.cap); };
    auto empty = [&](long long n, long long) {
        for_each_class(bt.C, s, view, [&](int) {
            for (long long e = 0; e < n; ++e) class_step(s, nullptr, 0, K, st);
        });
    };
    auto frame = [&](int f, long long, int *births) {
        for_each_class(bt.C, s, view, [&](int c) {
            const int32_t *rec;
            const int cnt = bt.records(f, c, rec);
            const int nb = class_step(s, rec, cnt, K, st);
            if (lane == 0) births[c] = nb;
        });
    };
    auto emit = [&](int f, long long fc, const int *births, const int *base) {
        for_each_class(bt.C, s, view, [&](int c) {
            for (int b = lane; b < births[c]; b += 32) {
                OTrk &t = s.trk[s.born[b]];
                t.id = base[c] - t.id;
            }
            __syncwarp();
            int32_t *ids = bt.ids(f, c);
            float *obox = bt.boxes(f, c);
            for (int k = lane; k < K; k += 32) {
                int id = -1;
                double b[4] = {0.0, 0.0, 0.0, 0.0};
                const int slot = s.owner[k];
                if (slot >= 0) {
                    const OTrk &t = s.trk[slot];
                    if (t.tsu < 1 && (t.hit_streak >= st.min_hits || fc <= st.min_hits)) {
                        id = t.id;
                        if (sum5(t.last_obs) >= 0) {
                            for (int q = 0; q < 4; ++q) b[q] = t.last_obs[q];
                        } else {
                            state_box(t.kf, b);
                        }
                    }
                }
                ids[k] = id;
                write_box(obox + 4 * k, b);
            }
            __syncwarp();
        });
    };
    frame_loop(state, bt, (long long)st.max_age + 1, empty, frame, emit);
}

bool oc_args_ok(const char *fn, int C, int K, int max_age, int delta_t) {
    if (C < 1 || C > 1024 || K < 1 || max_age < 0 || delta_t < 1 || delta_t > DT_MAX ||
        (long long)K * (max_age + 1LL) > OC_MAX) {
        set_error("%s: class_num %d (1..1024), max_per_class %d (>= 1), max_age %d (>= 0) and delta_t %d (1..%d) with "
                  "max_per_class x (max_age + 1) <= %d tracks per class", fn, C, K, max_age, delta_t, DT_MAX, OC_MAX);
        return false;
    }
    return true;
}

}  // namespace
}  // namespace k2y

using namespace k2y;

extern "C" int k2y_ocsort_state_bytes(int class_num, int max_per_class, int max_age, int delta_t, size_t *bytes) {
    if (!bytes) {
        set_error("k2y_ocsort_state_bytes: null output");
        return K2Y_ERR_INVALID;
    }
    if (!oc_args_ok("k2y_ocsort_state_bytes", class_num, max_per_class, max_age, delta_t)) return K2Y_ERR_INVALID;
    *bytes = state_bytes(class_num, max_per_class, oc_cap(max_per_class, max_age));
    return K2Y_OK;
}

extern "C" int k2y_ocsort_update(void *state_dev, const k2y_det *dets_dev, const int32_t *counts_dev, long long row_stride_words,
                                 const int32_t *rows_dev, const long long *positions_dev, int n_frames, int class_num,
                                 int max_per_class, double det_thresh, int max_age, int min_hits, double iou_thresh, int delta_t,
                                 double inertia, int use_byte, int32_t *ids_out_dev, float *boxes_out_dev, void *stream) {
    const char *fn = "k2y_ocsort_update";
    const Batch bt{(const int32_t *)dets_dev, counts_dev, rows_dev, positions_dev, row_stride_words, n_frames, class_num,
                   max_per_class, ids_out_dev, boxes_out_dev};
    if (!oc_args_ok(fn, class_num, max_per_class, max_age, delta_t) || !batch_ok(fn, state_dev, bt)) return K2Y_ERR_INVALID;
    if (min_hits < 0 || !(det_thresh >= 0.0 && det_thresh <= 1.0) || !(iou_thresh >= 0.0 && iou_thresh <= 1.0) ||
        !(inertia >= 0.0 && inertia <= 1.0)) {
        set_error("%s: min_hits < 0, or det_thresh, iou_thresh or inertia outside [0, 1]", fn);
        return K2Y_ERR_INVALID;
    }
    if (n_frames == 0) return K2Y_OK;
    Setting st;
    st.iou_thresh = iou_thresh;
    st.det_thresh = det_thresh;
    st.inertia = inertia;
    st.max_age = max_age;
    st.min_hits = min_hits;
    st.delta_t = delta_t;
    st.use_byte = use_byte != 0;
    st.cap = oc_cap(max_per_class, max_age);
    const int threads = (class_num < OC_WARPS ? class_num : OC_WARPS) * 32;
    ocsort_update_kernel<<<1, threads, 0, (cudaStream_t)stream>>>((unsigned char *)state_dev, bt, st);
    K2Y_CUDA_CHECK(cudaGetLastError());
    return K2Y_OK;
}
