// MOTChallenge tracking evaluation on the device: CLEAR MOT and the identity metrics, by the protocol of oracle/mot_ref.py
// (TrackEval's MotChallenge2DBox preprocessing, CLEAR and Identity), counts equal and float64 sums equal bit for bit.
//
// Per sequence: the gt is uploaded once (k2y_mot_add_sequence); each update compacts the person records with a track id
// of a batch of frames into per-frame tracker slots (k2y_mot_update).  k2y_mot_result then runs, per sequence:
//   relabel   the tracker ids to dense indices (a table indexed by id, cleared again afterwards);
//   stage A   one warp per frame: the IoU of the frame's gt rows with its tracker rows, distractor removal (an assignment
//             only where a distractor row has a positive entry, none where the positives are isolated), the kept tracker
//             rows, the potential-match counts (integer atomics), and the frame's first CLEAR assignment with no bonus;
//   stage B   CLEAR by rounds: one warp per frame whose predecessor's matches changed re-solves with the bonus taken from
//             them, until nothing changes (oracle/mot_ref.py shows this equals the sequential loop); frames of isolated
//             positives take them directly in stage A and are never solved again;
//   stage C   per gt id over its frames: IDSW, Frag, MT / PT / ML; per frame TP / FP / FN and the IoU sum in row order,
//             then MOTP_sum over the frames in order, serially;
//   stage D   IDTP: one warp solves the maximum-weight matching of the potential-match counts (an exact assignment on
//             the dense gt id x tracker id matrix; the value is unique).
// With k2y_mot_result_ex, HOTA (oracle/mot_hota_ref.py) follows on stage A's kept rows: tracker ids ranked by sorted id,
// per-frame row / column sums, potential-match sums per gt id in frame order, one assignment per frame of its score matrix,
// per-pair match counts, and the association sums in numpy's pairwise order over the non-zero pairs.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <map>
#include <vector>

#include "common.h"
#include "lsap_warp.cuh"

using namespace k2y;

namespace {

constexpr int CAP = K2Y_MOT_MAX_ROWS;            // gt rows and tracker rows of one frame
constexpr int MAX_ID = K2Y_MOT_MAX_TRACK_ID;     // tracker ids are < MAX_ID
constexpr long long MAX_PAIRS = 1LL << 28;       // gt ids x tracker ids of one sequence
constexpr double EPS = 2.220446049250313e-16;    // np.finfo(float).eps
constexpr double HALF_M = 0.5 - EPS;             // 0.5 - eps, as numpy rounds it

enum Ctr { TP, FP, FN, IDSW, FRAG, MT, PT, ML, IDTP, TRK_ROWS, N_CTR };

struct Seq {
    int L = 0, G = 0, T = 0;    // frames, kept gt ids, tracker ids
    // gt, sorted by frame: boxes (left, top, w, h), class, dense id (-1: not kept), per-frame offsets
    double *gbox = nullptr;
    int *gcls = nullptr, *gid = nullptr, *goff = nullptr;
    // kept gt rows per frame (row indices, offsets), and per gt id its (frame, position in the frame's kept list)
    int *kidx = nullptr, *koff = nullptr, *idoff = nullptr, *idframe = nullptr, *idpos = nullptr;
    // tracker slots [L][CAP]: id and box; tn[L] rows per frame (-1: no update gave the frame)
    int *tid = nullptr, *tn = nullptr;
    double *tbox = nullptr;
    // frame state: kept tracker slots and count, flags (1 effective, 2 isolated), predecessor, matches [2][L][CAP],
    // changed [2][L], IoU sum
    int *tkeep = nullptr, *tkn = nullptr, *flags = nullptr, *pred = nullptr, *match = nullptr, *changed = nullptr;
    double *fsum = nullptr;
    unsigned long long *ctr = nullptr;    // [N_CTR]
    double *motp = nullptr;
};

struct Dev {
    int *n = nullptr;           // [0] tracker ids seen, [1] frames changed in a round, [2] frames solved in a round
    unsigned *status = nullptr;
    int *tmap = nullptr;        // [MAX_ID]: dense index of a tracker id, -1 elsewhere
    unsigned *hbits = nullptr;  // [MAX_ID / 32]: HOTA's kept tracker ids as bits, cleared after each sequence
    long long *hwpre = nullptr; // [MAX_ID / 32 + 1]: kept ids in the words before each word (the sorted rank's base)
};

__device__ __forceinline__ double box_iou(const double *a, const double *b) {
    const double ax2 = __dadd_rn(a[0], a[2]), ay2 = __dadd_rn(a[1], a[3]);
    const double bx2 = __dadd_rn(b[0], b[2]), by2 = __dadd_rn(b[1], b[3]);
    double inter = __dmul_rn(fmax(fmin(ax2, bx2) - fmax(a[0], b[0]), 0.0), fmax(fmin(ay2, by2) - fmax(a[1], b[1]), 0.0));
    const double a1 = __dmul_rn(ax2 - a[0], ay2 - a[1]);
    const double a2 = __dmul_rn(bx2 - b[0], by2 - b[1]);
    double uni = __dsub_rn(__dadd_rn(a1, a2), inter);
    if (a1 <= EPS || a2 <= EPS || uni <= EPS) inter = 0.0;
    if (uni <= EPS) uni = 1.0;
    return inter / uni;
}

struct WarpSmem {
    double u[CAP], v[CAP], spc[CAP];
    int path[CAP], col4row[CAP], row4col[CAP], remaining[CAP], match[CAP], bonus[CAP], cnt_r[CAP], cnt_c[CAP];
    unsigned char SR[CAP], SC[CAP], removed[CAP];
};

__device__ LsapWork smem_work(WarpSmem &s) {
    return LsapWork{s.u, s.v, s.spc, s.path, s.col4row, s.row4col, s.remaining, s.SR, s.SC};
}

// distractor matching: -S with S zeroed below 0.5 - eps; rows are every gt row of the frame, columns its tracker slots
struct DistractorCost {
    const double *gbox, *tbox;
    __device__ double operator()(int i, int j) const {
        const double s = box_iou(gbox + 4 * i, tbox + 4 * j);
        return s >= HALF_M ? -s : -0.0;
    }
};

// CLEAR: -(1000 * [tracker id == bonus] + IoU), 0 below 0.5 - eps; rows the kept gt rows, columns the kept tracker slots
struct ClearCost {
    const double *gbox, *tbox;
    const int *kidx, *tkeep, *tid, *bonus;
    __device__ double operator()(int i, int j) const {
        const int t = tkeep[j];
        const double s = box_iou(gbox + 4 * kidx[i], tbox + 4 * t);
        if (!(s >= HALF_M)) return -0.0;
        return tid[t] == bonus[i] ? -(1000.0 + s) : -s;
    }
};

// Counts each row's and column's positive entries (IoU >= 0.5 - eps) into s.cnt_r / s.cnt_c; true when none exceeds 1.
template <class Pos>
__device__ bool positives_isolated(int nr, int nc, const Pos &pos, WarpSmem &s) {
    const int lane = threadIdx.x & 31;
    for (int i = lane; i < CAP; i += 32) s.cnt_r[i] = s.cnt_c[i] = 0;
    __syncwarp();
    for (int e = lane; e < nr * nc; e += 32) {
        const int i = e / nc, j = e % nc;
        if (pos(i, j)) {
            atomicAdd(&s.cnt_r[i], 1);
            atomicAdd(&s.cnt_c[j], 1);
        }
    }
    __syncwarp();
    int bad = 0;
    for (int i = lane; i < nr; i += 32) bad |= s.cnt_r[i] > 1;
    for (int j = lane; j < nc; j += 32) bad |= s.cnt_c[j] > 1;
    return !__any_sync(0xffffffffu, bad);
}

// CLEAR's pairs of frame f into s.match (column or -1 per kept gt row): the positives when isolated, else the assignment.
__device__ void clear_solve(const Seq &q, int f, int ng, int nt, bool iso, WarpSmem &s) {
    const int lane = threadIdx.x & 31;
    const int *kidx = q.kidx + q.koff[f], *tkeep = q.tkeep + (size_t)f * CAP;
    const double *tbox = q.tbox + (size_t)f * CAP * 4;
    ClearCost cost{q.gbox, tbox, kidx, tkeep, q.tid + (size_t)f * CAP, s.bonus};
    if (iso) {
        for (int i = lane; i < ng; i += 32) {
            int m = -1;
            for (int j = 0; j < nt; ++j)
                if (cost(i, j) < 0.0) m = j;
            s.match[i] = m;
        }
        __syncwarp();
        return;
    }
    warp_lsap(ng, nt, cost, smem_work(s), s.match);
    for (int i = lane; i < ng; i += 32)
        if (s.match[i] >= 0 && !(-cost(i, s.match[i]) > EPS)) s.match[i] = -1;
    __syncwarp();
}

struct CompactArgs {
    const int32_t *counts, *ids;
    const float *boxes;
    long long count_stride, id_stride, box_stride;
    const long long *positions;
    int C, K, person;
    Seq q;
    unsigned *status;
};

// One warp per frame of the update: the person records with a track id, in record order, into the frame's slots.
__global__ void __launch_bounds__(32) mot_compact_kernel(CompactArgs a) {
    const int n = blockIdx.x, lane = threadIdx.x;
    const long long f = a.positions[n];
    int cnt = a.counts[n * a.count_stride + a.person];
    if (cnt < 0 || cnt > a.K) {
        if (lane == 0) atomicOr(a.status, K2Y_MOT_BAD_COUNT);
        cnt = cnt < 0 ? 0 : a.K;
    }
    int base = 0;
    unsigned bad = 0;
    for (int k0 = 0; k0 < cnt; k0 += 32) {
        const int k = k0 + lane;
        int id = -1;
        float y0 = 0, x0 = 0, y1 = 0, x1 = 0;
        if (k < cnt) {
            id = a.ids[n * a.id_stride + (long long)a.person * a.K + k];
            const float *b = a.boxes + n * a.box_stride + ((long long)a.person * a.K + k) * 4;
            y0 = b[0], x0 = b[1], y1 = b[2], x1 = b[3];
        }
        const unsigned take = __ballot_sync(0xffffffffu, id >= 0);
        const int slot = base + __popc(take & ((1u << lane) - 1));
        if (id >= 0) {
            if (id >= MAX_ID) bad |= K2Y_MOT_BAD_ID;
            if (!(isfinite(y0) && isfinite(x0) && isfinite(y1) && isfinite(x1))) bad |= K2Y_MOT_BAD_BOX;
            if (slot < CAP) {
                a.q.tid[f * CAP + slot] = id;
                double *t = a.q.tbox + (f * CAP + slot) * 4;
                t[0] = (double)x0 + 1.0;
                t[1] = (double)y0 + 1.0;
                t[2] = (double)x1 - (double)x0;
                t[3] = (double)y1 - (double)y0;
            }
        }
        base += __popc(take);
    }
    bad = __reduce_or_sync(0xffffffffu, bad);
    if (base > CAP) bad |= K2Y_MOT_TOO_MANY_ROWS;
    if (lane == 0) {
        if (bad) atomicOr(a.status, bad);
        a.q.tn[f] = base > CAP ? CAP : base;
    }
}

// Dense tracker indices: the first thread to see an id takes the next index.
__global__ void mot_relabel_kernel(Seq q, int *tmap, int *n_ids) {
    const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (e >= (long long)q.L * CAP) return;
    const int f = (int)(e / CAP), j = (int)(e % CAP);
    if (j >= q.tn[f]) return;
    const int id = q.tid[e];
    if (id >= 0 && id < MAX_ID && atomicCAS(&tmap[id], -1, -2) == -1) tmap[id] = atomicAdd(n_ids, 1);
}

__global__ void mot_unlabel_kernel(Seq q, int *tmap) {
    const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (e >= (long long)q.L * CAP) return;
    const int f = (int)(e / CAP), j = (int)(e % CAP);
    const int id = q.tid[e];
    if (j < q.tn[f] && id >= 0 && id < MAX_ID) tmap[id] = -1;
}

struct StageArgs {
    Seq q;
    int benchmark, round;
    const int *tmap;
    int *pairs;            // [G][T] potential-match counts
    int *n;
    unsigned *status;
};

// Stage A, one warp per frame.
__global__ void __launch_bounds__(32) mot_stage_a_kernel(StageArgs a) {
    __shared__ WarpSmem s;
    const Seq &q = a.q;
    const int f = blockIdx.x, lane = threadIdx.x;
    const int g0 = q.goff[f], ng_all = q.goff[f + 1] - g0;
    const int nt_all = q.tn[f] < 0 ? 0 : q.tn[f];
    const int *tid = q.tid + (size_t)f * CAP;
    const double *tbox = q.tbox + (size_t)f * CAP * 4;
    const double *gbox = q.gbox + (size_t)g0 * 4;
    // a tracker id twice in the frame
    int dup = 0;
    for (int e = lane; e < nt_all * nt_all; e += 32) {
        const int i = e / nt_all, j = e % nt_all;
        dup |= i < j && tid[i] == tid[j];
    }
    if (__any_sync(0xffffffffu, dup) && lane == 0) atomicOr(a.status, K2Y_MOT_REPEATED_ID);
    // distractor removal
    for (int j = lane; j < CAP; j += 32) s.removed[j] = 0;
    __syncwarp();
    if (a.benchmark != 15 && ng_all > 0 && nt_all > 0) {
        const int *gcls = q.gcls + g0;
        auto distractor = [&](int c) { return c == 2 || c == 7 || c == 8 || c == 12 || (a.benchmark == 20 && c == 6); };
        int any = 0;
        for (int e = lane; e < ng_all * nt_all; e += 32) {
            const int i = e / nt_all, j = e % nt_all;
            any |= distractor(gcls[i]) && box_iou(gbox + 4 * i, tbox + 4 * j) >= HALF_M;
        }
        if (__any_sync(0xffffffffu, any)) {
            DistractorCost cost{gbox, tbox};
            auto pos = [&](int i, int j) { return cost(i, j) < 0.0; };
            if (positives_isolated(ng_all, nt_all, pos, s)) {
                for (int i = lane; i < ng_all; i += 32) {
                    s.match[i] = -1;
                    for (int j = 0; j < nt_all; ++j)
                        if (pos(i, j)) s.match[i] = j;
                }
                __syncwarp();
            } else {
                warp_lsap(ng_all, nt_all, cost, smem_work(s), s.match);
            }
            for (int i = lane; i < ng_all; i += 32) {
                const int j = s.match[i];
                if (j >= 0 && -cost(i, j) > EPS && distractor(gcls[i])) s.removed[j] = 1;
            }
            __syncwarp();
        }
    }
    // the kept tracker slots, in order
    int *tkeep = q.tkeep + (size_t)f * CAP;
    int nt = 0;
    for (int j0 = 0; j0 < nt_all; j0 += 32) {
        const int j = j0 + lane;
        const bool keep = j < nt_all && !s.removed[j];
        const unsigned b = __ballot_sync(0xffffffffu, keep);
        if (keep) tkeep[nt + __popc(b & ((1u << lane) - 1))] = j;
        nt += __popc(b);
    }
    __syncwarp();
    const int ng = q.koff[f + 1] - q.koff[f];
    const int *kidx = q.kidx + q.koff[f];
    const bool eff = ng > 0 && nt > 0;
    // potential matches (IoU >= 0.5) of the kept rows
    if (eff && a.pairs) {
        for (int e = lane; e < ng * nt; e += 32) {
            const int i = e / nt, j = tkeep[e % nt];
            if (tid[j] < MAX_ID && box_iou(q.gbox + 4 * kidx[i], tbox + 4 * j) >= 0.5)
                atomicAdd(&a.pairs[(long long)q.gid[kidx[i]] * q.T + a.tmap[tid[j]]], 1);
        }
    }
    int flags = eff ? 1 : 0;
    if (eff) {
        for (int i = lane; i < ng; i += 32) s.bonus[i] = -1;
        __syncwarp();
        ClearCost cost{q.gbox, tbox, kidx, tkeep, tid, s.bonus};
        auto pos = [&](int i, int j) { return cost(i, j) < 0.0; };
        const bool iso = positives_isolated(ng, nt, pos, s);
        flags |= iso ? 2 : 0;
        clear_solve(q, f, ng, nt, iso, s);
        int *m0 = q.match + (size_t)f * CAP, *m1 = q.match + ((size_t)q.L + f) * CAP;
        for (int i = lane; i < ng; i += 32) m0[i] = m1[i] = s.match[i];
        if (lane == 0 && !iso) atomicAdd(&a.n[2], 1);
    }
    if (lane == 0) {
        q.tkn[f] = nt;
        q.flags[f] = flags;
        q.changed[f] = eff;
        q.changed[q.L + f] = 0;
        atomicAdd(&q.ctr[TRK_ROWS], (unsigned long long)nt);
    }
}

// The previous effective frame of every frame (one thread).
__global__ void mot_link_kernel(Seq q) {
    int p = -1;
    for (int f = 0; f < q.L; ++f) {
        q.pred[f] = p;
        if (q.flags[f] & 1) p = f;
    }
}

// Stage B, round r >= 1: one warp per effective frame that is not of isolated positives.
__global__ void __launch_bounds__(32) mot_round_kernel(StageArgs a) {
    __shared__ WarpSmem s;
    const Seq &q = a.q;
    const int f = blockIdx.x, lane = threadIdx.x;
    const int fl = q.flags[f];
    const int rd = (a.round - 1) & 1, wr = a.round & 1;
    if (!(fl & 1) || (fl & 2)) {        // never solved again: never changes
        if (lane == 0) q.changed[(size_t)wr * q.L + f] = 0;
        return;
    }
    const int ng = q.koff[f + 1] - q.koff[f];
    const int *prev = q.match + ((size_t)rd * q.L + f) * CAP;
    int *next = q.match + ((size_t)wr * q.L + f) * CAP;
    const int p = q.pred[f];
    if (p < 0 || !q.changed[(size_t)rd * q.L + p]) {
        for (int i = lane; i < ng; i += 32) next[i] = prev[i];
        if (lane == 0) q.changed[(size_t)wr * q.L + f] = 0;
        return;
    }
    // the bonus of each kept gt row: the tracker id its gt id was matched to at the predecessor
    const int *kidx = q.kidx + q.koff[f], *pk = q.kidx + q.koff[p];
    const int png = q.koff[p + 1] - q.koff[p];
    const int *pm = q.match + ((size_t)rd * q.L + p) * CAP;
    for (int i = lane; i < ng; i += 32) {
        const int g = q.gid[kidx[i]];
        int b = -1;
        for (int k = 0; k < png; ++k)
            if (q.gid[pk[k]] == g && pm[k] >= 0) b = q.tid[(size_t)p * CAP + q.tkeep[(size_t)p * CAP + pm[k]]];
        s.bonus[i] = b;
    }
    __syncwarp();
    clear_solve(q, f, ng, q.tkn[f], false, s);
    int diff = 0;
    for (int i = lane; i < ng; i += 32) {
        diff |= s.match[i] != prev[i];
        next[i] = s.match[i];
    }
    diff = __any_sync(0xffffffffu, diff);
    if (lane == 0) {
        q.changed[(size_t)wr * q.L + f] = diff;
        atomicAdd(&a.n[2], 1);
        if (diff) atomicAdd(&a.n[1], 1);
    }
}

// Stage C per frame: TP / FP / FN and the IoU sum of the matches in row order.
__global__ void mot_frame_kernel(Seq q, int final_buf) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= q.L) return;
    const int ng = q.koff[f + 1] - q.koff[f], nt = q.tkn[f];
    double sum = 0.0;
    if (ng == 0) {
        atomicAdd(&q.ctr[FP], (unsigned long long)nt);
    } else if (nt == 0) {
        atomicAdd(&q.ctr[FN], (unsigned long long)ng);
    } else {
        const int *m = q.match + ((size_t)final_buf * q.L + f) * CAP;
        const int *kidx = q.kidx + q.koff[f];
        int tp = 0;
        for (int i = 0; i < ng; ++i)
            if (m[i] >= 0) {
                sum = __dadd_rn(sum, box_iou(q.gbox + 4 * kidx[i], q.tbox + ((size_t)f * CAP + q.tkeep[(size_t)f * CAP + m[i]]) * 4));
                ++tp;
            }
        atomicAdd(&q.ctr[TP], (unsigned long long)tp);
        atomicAdd(&q.ctr[FN], (unsigned long long)(ng - tp));
        atomicAdd(&q.ctr[FP], (unsigned long long)(nt - tp));
    }
    q.fsum[f] = sum;
}

__global__ void mot_motp_kernel(Seq q) {
    double s = 0.0;
    for (int f = 0; f < q.L; ++f) s = __dadd_rn(s, q.fsum[f]);
    *q.motp = s;
}

// Stage C per gt id: IDSW, Frag and MT / PT / ML over its frames in order.
__global__ void mot_id_kernel(Seq q, int final_buf) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= q.G) return;
    int present = 0, matched = 0, idsw = 0, frag = 0, last_t = -1, last_f = -1;
    for (int k = q.idoff[g]; k < q.idoff[g + 1]; ++k) {
        const int f = q.idframe[k];
        ++present;
        if (q.tkn[f] == 0) continue;
        const int m = q.match[((size_t)final_buf * q.L + f) * CAP + q.idpos[k]];
        if (m < 0) continue;
        const int t = q.tid[(size_t)f * CAP + q.tkeep[(size_t)f * CAP + m]];
        ++matched;
        if (last_t >= 0 && last_t != t) ++idsw;
        if (last_f < 0 || last_f != q.pred[f]) ++frag;
        last_t = t;
        last_f = f;
    }
    const double ratio = (double)matched / (double)present;
    atomicAdd(&q.ctr[IDSW], (unsigned long long)idsw);
    if (frag > 1) atomicAdd(&q.ctr[FRAG], (unsigned long long)(frag - 1));
    atomicAdd(&q.ctr[ratio > 0.8 ? MT : ratio >= 0.2 ? PT : ML], 1ULL);
}

struct IdtpCost {
    const int *pairs;
    int T;
    __device__ double operator()(int i, int j) const { return -(double)pairs[(long long)i * T + j]; }
};

// Stage D: IDTP, one warp.
__global__ void __launch_bounds__(32) mot_idtp_kernel(Seq q, const int *pairs, LsapWork w, int *match) {
    IdtpCost cost{pairs, q.T};
    warp_lsap(q.G, q.T, cost, w, match);
    long long s = 0;
    for (int i = threadIdx.x; i < q.G; i += 32)
        if (match[i] >= 0) s += pairs[(long long)i * q.T + match[i]];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) q.ctr[IDTP] = (unsigned long long)s;
}

// ---- HOTA (oracle/mot_hota_ref.py), on stage A's kept rows -------------------------------------------------------------
constexpr int NA = K2Y_MOT_HOTA_ALPHAS;
constexpr int NW = MAX_ID / 32;                  // words of the kept-tracker-id bitmap
// np.arange(0.05, 0.99, 0.05); a match counts at alpha a when IoU >= alpha - eps
__constant__ double c_alpha[NA] = {0.05, 0.1, 0.15000000000000002, 0.2, 0.25, 0.3, 0.35000000000000003, 0.4, 0.45, 0.5,
                                   0.55, 0.6000000000000001, 0.6500000000000001, 0.7000000000000001, 0.7500000000000001,
                                   0.8, 0.8500000000000001, 0.9000000000000001, 0.9500000000000001};

struct Hota {
    // per frame slot [L][CAP]: row sums (pairwise) and column sums (sequential) of S, positive entries per row, the sorted
    // rank of each kept tracker row, and each kept gt row's HOTA match (column or -1) and level (the alphas it counts at)
    double *rsum, *csum;
    int *rowcnt, *trank, *hm, *hl;
    int *msize, *ftp, *tc, *gcnt, *gdist;      // [L] ng * nt, [L][NA] matches, [T] frames per tracker rank, [G] x 2
    long long *moff, *gseg, *poff;             // exclusive prefixes of msize, gcnt, gdist (with the total at the end)
    double *floc, *M;                          // [L][NA] IoU sums; score matrices gas * S, [moff[L]]
    // entries: one per (frame, kept gt row, kept tracker row) with S > 0, by gt id and then frame
    int *et, *ef, *eij;                        // tracker rank, frame, i * CAP + j
    double *ev, *es;                           // sim_iou, S
    unsigned char *efirst, *elvl;              // first entry of its (gt id, tracker rank) in the gt id's list; HOTA level
    // pairs (gt id, tracker rank) with an entry, by position g * T + t
    long long *ppos;
    int *pgc, *ptc, *pmc;                      // gt id's and tracker's frame counts, [P][NA] match counts
    long long *cnt;                            // [3][NA] TP, FN, FP
    double *sum;                               // [4][NA] LocA, AssA, AssRe, AssPr sums
    int Th;                                    // kept tracker ids
};

// Exclusive prefix of in(0..n-1) into out[0..n], out[n] the total; one block of 1024 threads.
struct PopcIn {
    const unsigned *w;
    __device__ long long operator()(int k) const { return __popc(w[k]); }
};
struct IntIn {
    const int *p;
    __device__ long long operator()(int k) const { return p[k]; }
};
template <class In>
__global__ void __launch_bounds__(1024) hota_scan_kernel(In in, int n, long long *out) {
    __shared__ long long part[1024];
    const int t = threadIdx.x, per = (n + 1023) / 1024, b = min(n, t * per), e = min(n, b + per);
    long long s = 0;
    for (int k = b; k < e; ++k) s += in(k);
    part[t] = s;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
        const long long v = t >= o ? part[t - o] : 0;
        __syncthreads();
        part[t] += v;
        __syncthreads();
    }
    long long run = part[t] - s;
    for (int k = b; k < e; ++k) {
        out[k] = run;
        run += in(k);
    }
    if (t == 1023) out[n] = part[1023];
}

// The kept tracker ids as bits, then each kept row's rank among them (np.unique's index) and its tracker's frame count.
__global__ void hota_mark_kernel(Seq q, unsigned *bits) {
    const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (e >= (long long)q.L * CAP) return;
    const int f = (int)(e / CAP), j = (int)(e % CAP);
    if (j >= q.tkn[f]) return;
    const int id = q.tid[(size_t)f * CAP + q.tkeep[e]];
    if (id >= 0 && id < MAX_ID) atomicOr(&bits[id >> 5], 1u << (id & 31));
}

__global__ void hota_rank_kernel(Seq q, const unsigned *bits, const long long *wpre, Hota h) {
    const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (e >= (long long)q.L * CAP) return;
    const int f = (int)(e / CAP), j = (int)(e % CAP);
    if (j >= q.tkn[f]) return;
    const int id = q.tid[(size_t)f * CAP + q.tkeep[e]];
    const int r = id >= 0 && id < MAX_ID ? (int)(wpre[id >> 5] + __popc(bits[id >> 5] & ((1u << (id & 31)) - 1u))) : 0;
    h.trank[e] = r;
    atomicAdd(&h.tc[r], 1);
}

// numpy's pairwise sum of v(lo .. lo + n - 1): 8 interleaved accumulators up to 128 elements, split at n / 2 rounded down
// to a multiple of 8 above (D levels, enough for CAP).
template <class V>
__device__ double pw_leaf(const V &v, int lo, int n) {
    if (n < 8) {
        double r = 0.0;
        for (int k = 0; k < n; ++k) r += v(lo + k);
        return r;
    }
    double r0 = v(lo), r1 = v(lo + 1), r2 = v(lo + 2), r3 = v(lo + 3), r4 = v(lo + 4), r5 = v(lo + 5), r6 = v(lo + 6),
           r7 = v(lo + 7);
    int i = 8;
    for (; i < n - n % 8; i += 8) {
        r0 += v(lo + i), r1 += v(lo + i + 1), r2 += v(lo + i + 2), r3 += v(lo + i + 3);
        r4 += v(lo + i + 4), r5 += v(lo + i + 5), r6 += v(lo + i + 6), r7 += v(lo + i + 7);
    }
    double res = ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7));
    for (; i < n; ++i) res += v(lo + i);
    return res;
}

template <int D, class V>
__device__ double pw_dense(const V &v, int lo, int n) {
    if constexpr (D == 0) {
        return pw_leaf(v, lo, n);
    } else {
        if (n <= 128) return pw_leaf(v, lo, n);
        int n2 = n / 2;
        n2 -= n2 % 8;
        return pw_dense<D - 1>(v, lo, n2) + pw_dense<D - 1>(v, lo + n2, n - n2);
    }
}
static_assert(CAP <= 1024, "pw_dense<4> covers rows of up to 1024 elements");

// One warp per frame: S.sum(1) (pairwise) and S.sum(0) (sequential) of the kept rows, positives per row, ng * nt.
__global__ void __launch_bounds__(32) hota_frame_sums_kernel(Seq q, Hota h) {
    const int f = blockIdx.x, lane = threadIdx.x;
    const int ng = q.koff[f + 1] - q.koff[f], nt = q.tkn[f];
    const int *kidx = q.kidx + q.koff[f], *tkeep = q.tkeep + (size_t)f * CAP;
    const double *tbox = q.tbox + (size_t)f * CAP * 4;
    for (int i = lane; i < ng; i += 32) {
        const double *g = q.gbox + 4 * kidx[i];
        auto S = [&](int j) { return box_iou(g, tbox + 4 * tkeep[j]); };
        int c = 0;
        for (int j = 0; j < nt; ++j) c += S(j) > 0.0;
        h.rsum[(size_t)f * CAP + i] = 0.0 + pw_dense<4>(S, 0, nt);
        h.rowcnt[(size_t)f * CAP + i] = c;
    }
    for (int j = lane; j < nt; j += 32) {
        double s = 0.0;
        for (int i = 0; i < ng; ++i) s += box_iou(q.gbox + 4 * kidx[i], tbox + 4 * tkeep[j]);
        h.csum[(size_t)f * CAP + j] = s;
    }
    if (lane == 0) h.msize[f] = ng * nt;
}

// Entries per gt id: the positive S of its rows over its frames.
__global__ void hota_gcount_kernel(Seq q, Hota h) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= q.G) return;
    int n = 0;
    for (int k = q.idoff[g]; k < q.idoff[g + 1]; ++k) n += h.rowcnt[(size_t)q.idframe[k] * CAP + q.idpos[k]];
    h.gcnt[g] = n;
}

// One warp per gt id: its entries in frame order, with sim_iou = S / ((colsum + rowsum) - S) where that is > eps.
__global__ void __launch_bounds__(32) hota_gather_kernel(Seq q, Hota h) {
    const int g = blockIdx.x, lane = threadIdx.x;
    long long base = h.gseg[g];
    for (int k = q.idoff[g]; k < q.idoff[g + 1]; ++k) {
        const int f = q.idframe[k], i = q.idpos[k], nt = q.tkn[f];
        const double *gb = q.gbox + 4 * q.kidx[q.koff[f] + i];
        const double rs = h.rsum[(size_t)f * CAP + i];
        for (int j0 = 0; j0 < nt; j0 += 32) {
            const int j = j0 + lane;
            const double s = j < nt ? box_iou(gb, q.tbox + ((size_t)f * CAP + q.tkeep[(size_t)f * CAP + j]) * 4) : 0.0;
            const unsigned b = __ballot_sync(0xffffffffu, s > 0.0);
            if (s > 0.0) {
                const long long e = base + __popc(b & ((1u << lane) - 1u));
                const double den = (h.csum[(size_t)f * CAP + j] + rs) - s;
                h.et[e] = h.trank[(size_t)f * CAP + j];
                h.ev[e] = den > EPS ? s / den : 0.0;
                h.es[e] = s;
                h.ef[e] = f;
                h.eij[e] = i * CAP + j;
            }
            base += __popc(b);
        }
    }
}

// One warp per gt id: pmc[g, t] = the entries' sim_iou summed in frame order, gas = pmc / ((gc + tc) - pmc), and each
// entry's score gas * S into its frame's matrix; which entries come first for their tracker, and how many pairs.
__global__ void __launch_bounds__(32) hota_pmc_kernel(Seq q, Hota h) {
    const int g = blockIdx.x, lane = threadIdx.x;
    const long long b = h.gseg[g], end = h.gseg[g + 1];
    const double gc = (double)(q.idoff[g + 1] - q.idoff[g]);
    int firsts = 0;
    for (long long e = b + lane; e < end; e += 32) {
        const int t = h.et[e];
        double pmc = 0.0;
        bool first = true;
        for (long long e2 = b; e2 < end; ++e2)
            if (h.et[e2] == t) {
                pmc += h.ev[e2];
                first &= e2 >= e;
            }
        const double gas = pmc / ((gc + (double)h.tc[t]) - pmc);
        const int f = h.ef[e], ij = h.eij[e];
        h.M[h.moff[f] + (long long)(ij / CAP) * q.tkn[f] + ij % CAP] = __dmul_rn(gas, h.es[e]);
        h.efirst[e] = first;
        firsts += first;
    }
    firsts = __reduce_add_sync(0xffffffffu, firsts);
    if (lane == 0) h.gdist[g] = firsts;
}

struct ScoreCost {
    const double *m;
    int nt;
    __device__ double operator()(int i, int j) const { return -m[i * nt + j]; }
};

// One warp per frame with gt and tracker rows: lsap(-score) once (or the positives when they are isolated), each row's
// match and level, then per alpha the matches and their IoU sum in row order.
__global__ void __launch_bounds__(32) hota_frame_kernel(Seq q, Hota h) {
    __shared__ WarpSmem s;
    const int f = blockIdx.x, lane = threadIdx.x;
    const int ng = q.koff[f + 1] - q.koff[f], nt = q.tkn[f];
    if (ng == 0 || nt == 0) {
        if (lane < NA) {
            h.ftp[f * NA + lane] = 0;
            h.floc[f * NA + lane] = 0.0;
        }
        return;
    }
    const double *M = h.M + h.moff[f];
    ScoreCost cost{M, nt};
    auto pos = [&](int i, int j) { return M[i * nt + j] > 0.0; };
    if (positives_isolated(ng, nt, pos, s)) {
        for (int i = lane; i < ng; i += 32) {
            int m = -1;
            for (int j = 0; j < nt; ++j)
                if (pos(i, j)) m = j;
            s.match[i] = m;
        }
        __syncwarp();
    } else {
        warp_lsap(ng, nt, cost, smem_work(s), s.match);
    }
    const int *kidx = q.kidx + q.koff[f], *tkeep = q.tkeep + (size_t)f * CAP;
    for (int i = lane; i < ng; i += 32) {
        const int j = s.match[i];
        int lvl = 0;
        double v = 0.0;
        if (j >= 0 && pos(i, j)) {
            v = box_iou(q.gbox + 4 * kidx[i], q.tbox + ((size_t)f * CAP + tkeep[j]) * 4);
            for (int a = 0; a < NA; ++a) lvl += v >= c_alpha[a] - EPS;
        }
        h.hm[(size_t)f * CAP + i] = lvl > 0 ? j : -1;
        h.hl[(size_t)f * CAP + i] = lvl;
        s.u[i] = v;
        s.cnt_r[i] = lvl;
    }
    __syncwarp();
    if (lane < NA) {
        int tp = 0;
        double loc = 0.0;
        for (int i = 0; i < ng; ++i)
            if (s.cnt_r[i] > lane) {
                ++tp;
                loc += s.u[i];
            }
        h.ftp[f * NA + lane] = tp;
        h.floc[f * NA + lane] = loc;
    }
}

// TP / FN / FP per alpha, and LocA_sum over the frames in order (one lane per alpha).
__global__ void hota_total_kernel(Seq q, Hota h) {
    const int a = threadIdx.x;
    if (a >= NA) return;
    long long tp = 0, fn = 0, fp = 0;
    double loc = 0.0;
    for (int f = 0; f < q.L; ++f) {
        const int ng = q.koff[f + 1] - q.koff[f], nt = q.tkn[f];
        if (ng == 0) {
            fp += nt;
        } else if (nt == 0) {
            fn += ng;
        } else {
            const int m = h.ftp[f * NA + a];
            tp += m;
            fn += ng - m;
            fp += nt - m;
            loc += h.floc[f * NA + a];
        }
    }
    h.cnt[a] = tp;
    h.cnt[NA + a] = fn;
    h.cnt[2 * NA + a] = fp;
    h.sum[a] = loc;
}

// One warp per gt id: each pair's position (its tracker's rank among the gt id's trackers) and its match count per alpha.
__global__ void __launch_bounds__(32) hota_pairs_kernel(Seq q, Hota h) {
    const int g = blockIdx.x, lane = threadIdx.x;
    const long long b = h.gseg[g], end = h.gseg[g + 1];
    for (long long e = b + lane; e < end; e += 32) {
        const int f = h.ef[e], ij = h.eij[e];
        const size_t r = (size_t)f * CAP + ij / CAP;
        h.elvl[e] = h.hm[r] == ij % CAP ? (unsigned char)h.hl[r] : 0;
    }
    __syncwarp();
    for (long long e = b + lane; e < end; e += 32) {
        if (!h.efirst[e]) continue;
        const int t = h.et[e];
        int rank = 0, m[NA];
#pragma unroll
        for (int a = 0; a < NA; ++a) m[a] = 0;
        for (long long e2 = b; e2 < end; ++e2) {
            const int t2 = h.et[e2];
            rank += h.efirst[e2] && t2 < t;
            if (t2 == t) {
                const int lv = h.elvl[e2];
#pragma unroll
                for (int a = 0; a < NA; ++a) m[a] += lv > a;
            }
        }
        const long long p = h.poff[g] + rank;
        h.ppos[p] = (long long)g * h.Th + t;
        h.pgc[p] = q.idoff[g + 1] - q.idoff[g];
        h.ptc[p] = h.tc[t];
#pragma unroll
        for (int a = 0; a < NA; ++a) h.pmc[p * NA + a] = m[a];
    }
}

// mc * (mc / den) of pair p for sum `kind` (0 AssA, 1 AssRe, 2 AssPr) at alpha a.
__device__ __forceinline__ double ass_value(const Hota &h, long long p, int kind, int a) {
    const double m = (double)h.pmc[p * NA + a], gc = (double)h.pgc[p], tc = (double)h.ptc[p];
    const double den = kind == 0 ? fmax(1.0, (gc + tc) - m) : fmax(1.0, kind == 1 ? gc : tc);
    return __dmul_rn(m, m / den);
}

// The association sums: numpy's pairwise sum over the dense G x T array, walked over the sorted pairs (zeros are neutral,
// so empty subtrees are skipped).  One warp; lane l computes sums l and l + 32 of the 3 x NA, all on one walk.
__global__ void __launch_bounds__(32) hota_assoc_kernel(Hota h, int G, long long n) {
    constexpr int DEPTH = 64;
    __shared__ long long s_lo[DEPTH], s_n[DEPTH];
    __shared__ int s_st[DEPTH];
    __shared__ double s_left[DEPTH][2][32];
    const int lane = threadIdx.x;
    const long long P = h.poff[G];
    const int c1 = lane + 32 < 3 * NA ? lane + 32 : lane;
    const int k0 = lane / NA, a0 = lane % NA, k1 = c1 / NA, a1 = c1 % NA;
    if (lane == 0) {
        s_lo[0] = 0;
        s_n[0] = n;
        s_st[0] = 0;
    }
    __syncwarp();
    int sp = 0;
    long long k = 0;
    double v0 = 0.0, v1 = 0.0;
    while (true) {
        const long long lo = s_lo[sp], len = s_n[sp];
        const int st = s_st[sp];
        long long n2 = len / 2;
        n2 -= n2 % 8;
        if (st == 0 && !(k >= P || h.ppos[k] >= lo + len) && len > 128) {
            __syncwarp();
            if (lane == 0) {
                s_st[sp] = 1;
                s_lo[sp + 1] = lo;
                s_n[sp + 1] = n2;
                s_st[sp + 1] = 0;
            }
            ++sp;
            __syncwarp();
            continue;
        }
        if (st == 1) {
            s_left[sp][0][lane] = v0;
            s_left[sp][1][lane] = v1;
            __syncwarp();
            if (lane == 0) {
                s_st[sp] = 2;
                s_lo[sp + 1] = lo + n2;
                s_n[sp + 1] = len - n2;
                s_st[sp + 1] = 0;
            }
            ++sp;
            __syncwarp();
            continue;
        }
        if (st == 2) {
            v0 = s_left[sp][0][lane] + v0;
            v1 = s_left[sp][1][lane] + v1;
        } else if (k >= P || h.ppos[k] >= lo + len) {
            v0 = v1 = 0.0;
        } else {        // a leaf with pairs: numpy's 8 accumulators over the block, the remainder after them
            const long long nb = len - len % 8;
            double r0[8], r1[8], x0 = 0.0, x1 = 0.0;
#pragma unroll
            for (int c = 0; c < 8; ++c) r0[c] = r1[c] = 0.0;
            bool tree = false;
            for (; k < P && h.ppos[k] < lo + len; ++k) {
                const long long d = h.ppos[k] - lo;
                const double y0 = ass_value(h, k, k0, a0), y1 = ass_value(h, k, k1, a1);
                if (d < nb) {
                    const int c = (int)(d & 7);
#pragma unroll
                    for (int u = 0; u < 8; ++u)
                        if (u == c) {
                            r0[u] += y0;
                            r1[u] += y1;
                        }
                    continue;
                }
                if (!tree) {
                    x0 = ((r0[0] + r0[1]) + (r0[2] + r0[3])) + ((r0[4] + r0[5]) + (r0[6] + r0[7]));
                    x1 = ((r1[0] + r1[1]) + (r1[2] + r1[3])) + ((r1[4] + r1[5]) + (r1[6] + r1[7]));
                    tree = true;
                }
                x0 += y0;
                x1 += y1;
            }
            if (!tree) {
                x0 = ((r0[0] + r0[1]) + (r0[2] + r0[3])) + ((r0[4] + r0[5]) + (r0[6] + r0[7]));
                x1 = ((r1[0] + r1[1]) + (r1[2] + r1[3])) + ((r1[4] + r1[5]) + (r1[6] + r1[7]));
            }
            v0 = x0;
            v1 = x1;
        }
        if (sp == 0) break;
        --sp;
    }
    h.sum[NA + lane] = 0.0 + v0;
    if (lane + 32 < 3 * NA) h.sum[NA + lane + 32] = 0.0 + v1;
}

template <class T>
cudaError_t dalloc(T **p, size_t n) {
    return cudaMalloc((void **)p, std::max<size_t>(n, 1) * sizeof(T));
}

template <class T>
cudaError_t upload(T **p, const std::vector<T> &v) {
    cudaError_t e = dalloc(p, v.size());
    if (e == cudaSuccess && !v.empty()) e = cudaMemcpy(*p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice);
    return e;
}

void free_seq(Seq &q) {
    void *ps[] = {q.gbox, q.gcls, q.gid, q.goff, q.kidx, q.koff, q.idoff, q.idframe, q.idpos, q.tid, q.tn, q.tbox,
                  q.tkeep, q.tkn, q.flags, q.pred, q.match, q.changed, q.fsum, q.ctr, q.motp};
    for (void *p : ps) cudaFree(p);
    q = Seq();
}

struct DeviceGuard {
    int old = -1;
    explicit DeviceGuard(int d) {
        cudaGetDevice(&old);
        cudaSetDevice(d);
    }
    ~DeviceGuard() {
        if (old >= 0) cudaSetDevice(old);
    }
};

}  // namespace

struct k2y_mot {
    int device = 0, benchmark = 17;
    cudaEvent_t done = nullptr;         // the handle's last operation, so successive calls on different streams stay ordered
    std::vector<Seq> seqs;
    std::vector<long long> gt_rows;      // kept gt rows per sequence
    Dev d;
};

extern "C" int k2y_mot_create(int benchmark, int device, k2y_mot **out) {
    if (!out || (benchmark != 15 && benchmark != 16 && benchmark != 17 && benchmark != 20)) {
        set_error("k2y_mot_create: benchmark must be 15, 16, 17 or 20");
        return K2Y_ERR_INVALID;
    }
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || device < 0 || device >= n) {
        cudaGetLastError();
        set_error("k2y_mot_create: no CUDA device %d", device);
        return K2Y_ERR_CUDA;
    }
    DeviceGuard g(device);
    k2y_mot *h = new k2y_mot();
    h->device = device;
    h->benchmark = benchmark;
    cudaError_t e = dalloc(&h->d.n, 4);
    if (e == cudaSuccess) e = dalloc(&h->d.status, 1);
    if (e == cudaSuccess) e = dalloc(&h->d.tmap, MAX_ID);
    if (e == cudaSuccess) e = cudaMemset(h->d.tmap, 0xff, sizeof(int) * (size_t)MAX_ID);
    if (e == cudaSuccess) e = dalloc(&h->d.hbits, MAX_ID / 32);
    if (e == cudaSuccess) e = dalloc(&h->d.hwpre, MAX_ID / 32 + 1);
    if (e == cudaSuccess) e = cudaMemset(h->d.hbits, 0, sizeof(unsigned) * (MAX_ID / 32));
    if (e == cudaSuccess) e = cudaMemset(h->d.status, 0, sizeof(unsigned));
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->done, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) {
        set_error("k2y_mot_create: %s", cudaGetErrorString(e));
        k2y_mot_destroy(h);
        return K2Y_ERR_CUDA;
    }
    *out = h;
    return K2Y_OK;
}

extern "C" int k2y_mot_destroy(k2y_mot *h) {
    if (!h) return K2Y_OK;
    DeviceGuard g(h->device);
    if (h->done) cudaEventSynchronize(h->done);
    for (Seq &q : h->seqs) free_seq(q);
    cudaFree(h->d.n);
    cudaFree(h->d.status);
    cudaFree(h->d.tmap);
    cudaFree(h->d.hbits);
    cudaFree(h->d.hwpre);
    if (h->done) cudaEventDestroy(h->done);
    delete h;
    return K2Y_OK;
}

extern "C" int k2y_mot_add_sequence(k2y_mot *h, const double *gt_host, long long n_gt, int seq_length, int *index) {
    if (!h || (n_gt > 0 && !gt_host) || n_gt < 0 || seq_length < 1 || !index) {
        set_error("k2y_mot_add_sequence: bad arguments");
        return K2Y_ERR_INVALID;
    }
    const int L = seq_length;
    std::vector<std::vector<int>> by_frame(L);
    for (long long r = 0; r < n_gt; ++r) {
        const double *row = gt_host + 8 * r;
        const double fr = row[0];
        if (!(fr >= 1 && fr <= L && fr == std::floor(fr))) {
            set_error("k2y_mot_add_sequence: gt row %lld has frame %g, outside 1..%d", r, fr, L);
            return K2Y_ERR_INVALID;
        }
        by_frame[(int)fr - 1].push_back((int)r);
    }
    std::vector<double> gbox;
    std::vector<int> gcls, gid, goff(L + 1, 0), kidx, koff(L + 1, 0);
    std::map<double, int> ids;
    for (int f = 0; f < L; ++f) {
        if ((int)by_frame[f].size() > CAP) {
            set_error("k2y_mot_add_sequence: frame %d has %d gt rows, more than %d", f + 1, (int)by_frame[f].size(), CAP);
            return K2Y_ERR_INVALID;
        }
        for (int r : by_frame[f]) {
            const double *row = gt_host + 8 * (long long)r;
            const bool keep = row[6] != 0 && (h->benchmark == 15 || row[7] == 1);
            if (keep) ids.emplace(row[1], 0);
        }
    }
    int G = 0;
    for (auto &kv : ids) kv.second = G++;
    std::vector<std::vector<std::pair<int, int>>> per_id(G);
    for (int f = 0; f < L; ++f) {
        goff[f] = (int)gcls.size();
        koff[f] = (int)kidx.size();
        for (int r : by_frame[f]) {
            const double *row = gt_host + 8 * (long long)r;
            const bool keep = row[6] != 0 && (h->benchmark == 15 || row[7] == 1);
            const int local = (int)gcls.size();
            gbox.insert(gbox.end(), row + 2, row + 6);
            gcls.push_back((int)row[7]);
            gid.push_back(keep ? ids[row[1]] : -1);
            if (keep) {
                per_id[gid.back()].push_back({f, (int)kidx.size() - koff[f]});
                kidx.push_back(local);
            }
        }
    }
    goff[L] = (int)gcls.size();
    koff[L] = (int)kidx.size();
    std::vector<int> idoff(G + 1, 0), idframe, idpos;
    for (int g = 0; g < G; ++g) {
        idoff[g] = (int)idframe.size();
        for (auto &fp : per_id[g]) {
            idframe.push_back(fp.first);
            idpos.push_back(fp.second);
        }
    }
    idoff[G] = (int)idframe.size();
    DeviceGuard dg(h->device);
    if (cudaEventSynchronize(h->done) != cudaSuccess) {
        set_error("k2y_mot_add_sequence: %s", cudaGetErrorString(cudaGetLastError()));
        return K2Y_ERR_CUDA;
    }
    Seq q;
    q.L = L;
    q.G = G;
    const size_t slots = (size_t)L * CAP;
    cudaError_t e = upload(&q.gbox, gbox);
    if (e == cudaSuccess) e = upload(&q.gcls, gcls);
    if (e == cudaSuccess) e = upload(&q.gid, gid);
    if (e == cudaSuccess) e = upload(&q.goff, goff);
    if (e == cudaSuccess) e = upload(&q.kidx, kidx);
    if (e == cudaSuccess) e = upload(&q.koff, koff);
    if (e == cudaSuccess) e = upload(&q.idoff, idoff);
    if (e == cudaSuccess) e = upload(&q.idframe, idframe);
    if (e == cudaSuccess) e = upload(&q.idpos, idpos);
    if (e == cudaSuccess) e = dalloc(&q.tid, slots);
    if (e == cudaSuccess) e = dalloc(&q.tbox, slots * 4);
    if (e == cudaSuccess) e = dalloc(&q.tn, L);
    if (e == cudaSuccess) e = dalloc(&q.tkeep, slots);
    if (e == cudaSuccess) e = dalloc(&q.tkn, L);
    if (e == cudaSuccess) e = dalloc(&q.flags, L);
    if (e == cudaSuccess) e = dalloc(&q.pred, L);
    if (e == cudaSuccess) e = dalloc(&q.match, 2 * slots);
    if (e == cudaSuccess) e = dalloc(&q.changed, 2 * (size_t)L);
    if (e == cudaSuccess) e = dalloc(&q.fsum, L);
    if (e == cudaSuccess) e = dalloc(&q.ctr, N_CTR);
    if (e == cudaSuccess) e = dalloc(&q.motp, 1);
    if (e == cudaSuccess) e = cudaMemset(q.tn, 0xff, sizeof(int) * L);     // no frame given yet
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) {
        set_error("k2y_mot_add_sequence: %s", cudaGetErrorString(e));
        free_seq(q);
        return K2Y_ERR_CUDA;
    }
    *index = (int)h->seqs.size();
    h->seqs.push_back(q);
    h->gt_rows.push_back((long long)kidx.size());
    return K2Y_OK;
}

extern "C" int k2y_mot_update(k2y_mot *h, int seq, const int32_t *counts_dev, const int32_t *ids_dev, const float *boxes_dev,
                              long long count_stride, long long id_stride, long long box_stride, int n_frames,
                              const long long *positions_dev, int class_num, int max_per_class, int person_class,
                              void *stream) {
    if (!h || seq < 0 || seq >= (int)h->seqs.size() || n_frames < 0 || class_num < 1 || max_per_class < 1 ||
        person_class < 0 || person_class >= class_num ||
        (n_frames > 0 && (!counts_dev || !ids_dev || !boxes_dev || !positions_dev))) {
        set_error("k2y_mot_update: bad arguments");
        return K2Y_ERR_INVALID;
    }
    if (n_frames == 0) return K2Y_OK;
    DeviceGuard g(h->device);
    CompactArgs a{counts_dev, ids_dev, boxes_dev, count_stride, id_stride, box_stride, positions_dev,
                  class_num, max_per_class, person_class, h->seqs[seq], h->d.status};
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaStreamWaitEvent(st, h->done, 0);
    if (e == cudaSuccess) {
        mot_compact_kernel<<<n_frames, 32, 0, st>>>(a);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaEventRecord(h->done, st);
    if (e != cudaSuccess) {
        set_error("k2y_mot_update: %s", cudaGetErrorString(e));
        return K2Y_ERR_CUDA;
    }
    return K2Y_OK;
}

// The scratch of one sequence's evaluation.  On every exit the tracker ids' entries of the relabel table are cleared
// again (a later result() relies on a clean table) and the buffers are freed, after the stream's work on them.
struct EvalScratch {
    k2y_mot *h;
    const Seq &q;
    cudaStream_t st;
    bool relabeled = false;
    int *pairs = nullptr, *di = nullptr;
    double *dd = nullptr;
    unsigned char *db = nullptr;
    EvalScratch(k2y_mot *h_, const Seq &q_, cudaStream_t st_) : h(h_), q(q_), st(st_) {}
    ~EvalScratch() {
        if (relabeled) mot_unlabel_kernel<<<(int)(((long long)q.L * CAP + 255) / 256), 256, 0, st>>>(q, h->d.tmap);
        cudaStreamSynchronize(st);
        cudaFree(pairs);
        cudaFree(dd);
        cudaFree(di);
        cudaFree(db);
    }
};

// Runs the stages of one sequence; its counters and MOTP_sum stay on the device.
static cudaError_t evaluate_seq(k2y_mot *h, Seq &q, cudaStream_t st, int *host_n, int *rounds, long long *solved) {
    const int L = q.L;
    EvalScratch x(h, q, st);
    cudaError_t e = cudaMemsetAsync(q.ctr, 0, sizeof(unsigned long long) * N_CTR, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(h->d.n, 0, sizeof(int) * 4, st);
    if (e != cudaSuccess) return e;
    mot_relabel_kernel<<<(int)(((long long)L * CAP + 255) / 256), 256, 0, st>>>(q, h->d.tmap, h->d.n);
    x.relabeled = true;
    if ((e = cudaMemcpyAsync(host_n, h->d.n, sizeof(int), cudaMemcpyDeviceToHost, st)) != cudaSuccess) return e;
    if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return e;
    q.T = host_n[0];
    const bool identity = (long long)q.G * q.T <= MAX_PAIRS;
    if (identity && q.G > 0 && q.T > 0) {
        if ((e = dalloc(&x.pairs, (size_t)q.G * q.T)) != cudaSuccess) return e;
        if ((e = cudaMemsetAsync(x.pairs, 0, sizeof(int) * (size_t)q.G * q.T, st)) != cudaSuccess) return e;
    }
    StageArgs a{q, h->benchmark, 0, h->d.tmap, x.pairs, h->d.n, h->d.status};
    mot_stage_a_kernel<<<L, 32, 0, st>>>(a);
    mot_link_kernel<<<1, 1, 0, st>>>(q);
    if ((e = cudaMemcpyAsync(host_n, h->d.n, sizeof(int) * 4, cudaMemcpyDeviceToHost, st)) != cudaSuccess) return e;
    if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return e;
    *solved = host_n[2];
    int r = 0, any_eff = 0;
    {
        std::vector<int> fl(L);
        if ((e = cudaMemcpy(fl.data(), q.flags, sizeof(int) * L, cudaMemcpyDeviceToHost)) != cudaSuccess) return e;
        for (int v : fl) any_eff |= v & 1;
    }
    *rounds = any_eff ? 1 : 0;
    while (any_eff) {
        ++r;
        if ((e = cudaMemsetAsync(h->d.n + 1, 0, sizeof(int) * 2, st)) != cudaSuccess) return e;
        a.round = r;
        mot_round_kernel<<<L, 32, 0, st>>>(a);
        if ((e = cudaMemcpyAsync(host_n, h->d.n, sizeof(int) * 4, cudaMemcpyDeviceToHost, st)) != cudaSuccess) return e;
        if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return e;
        if (host_n[2] > 0) ++*rounds;
        *solved += host_n[2];
        if (host_n[1] == 0) break;
    }
    const int fin = r & 1;
    mot_frame_kernel<<<(L + 127) / 128, 128, 0, st>>>(q, fin);
    mot_motp_kernel<<<1, 1, 0, st>>>(q);
    if (q.G > 0) mot_id_kernel<<<(q.G + 127) / 128, 128, 0, st>>>(q, fin);
    if (x.pairs) {
        const int n = std::max(q.G, q.T);
        if ((e = dalloc(&x.dd, 3 * (size_t)n)) != cudaSuccess || (e = dalloc(&x.di, 5 * (size_t)n)) != cudaSuccess ||
            (e = dalloc(&x.db, 2 * (size_t)n)) != cudaSuccess)
            return e;
        LsapWork w{x.dd, x.dd + n, x.dd + 2 * n, x.di, x.di + n, x.di + 2 * n, x.di + 3 * n, x.db, x.db + n};
        mot_idtp_kernel<<<1, 32, 0, st>>>(q, x.pairs, w, x.di + 4 * n);
    }
    return cudaGetLastError();
}

// HOTA of one sequence after its CLEAR stages, on stage A's kept slots: counts [3][NA] and sums [4][NA] to the host.
struct HotaScratch {
    cudaStream_t st;
    std::vector<void *> ps;
    explicit HotaScratch(cudaStream_t s) : st(s) {}
    template <class T>
    cudaError_t alloc(T **p, size_t n) {
        cudaError_t e = dalloc(p, n);
        if (e == cudaSuccess) ps.push_back(*p);
        return e;
    }
    ~HotaScratch() {
        cudaStreamSynchronize(st);
        for (void *p : ps) cudaFree(p);
    }
};

static cudaError_t hota_seq(k2y_mot *hd, const Seq &q, cudaStream_t st, long long *cnt_host, double *sum_host) {
    const int L = q.L, G = q.G;
    const size_t slots = (size_t)L * CAP;
    const int blocks = (int)((slots + 255) / 256);
    HotaScratch x(st);
    Hota h{};
    cudaError_t e = cudaSuccess;
    auto ok = [&](cudaError_t r) { return (e = r) == cudaSuccess; };
    if (!(ok(x.alloc(&h.rsum, slots)) && ok(x.alloc(&h.csum, slots)) && ok(x.alloc(&h.rowcnt, slots)) &&
          ok(x.alloc(&h.trank, slots)) && ok(x.alloc(&h.hm, slots)) && ok(x.alloc(&h.hl, slots)) &&
          ok(x.alloc(&h.msize, L)) && ok(x.alloc(&h.ftp, (size_t)L * NA)) && ok(x.alloc(&h.floc, (size_t)L * NA)) &&
          ok(x.alloc(&h.tc, std::max(q.T, 1))) && ok(x.alloc(&h.gcnt, G)) && ok(x.alloc(&h.gdist, G)) &&
          ok(x.alloc(&h.moff, (size_t)L + 1)) && ok(x.alloc(&h.gseg, (size_t)G + 1)) && ok(x.alloc(&h.poff, (size_t)G + 1)) &&
          ok(x.alloc(&h.cnt, 3 * NA)) && ok(x.alloc(&h.sum, 4 * NA)) &&
          ok(cudaMemsetAsync(h.tc, 0, sizeof(int) * std::max(q.T, 1), st))))
        return e;
    hota_mark_kernel<<<blocks, 256, 0, st>>>(q, hd->d.hbits);
    hota_scan_kernel<<<1, 1024, 0, st>>>(PopcIn{hd->d.hbits}, NW, hd->d.hwpre);
    hota_rank_kernel<<<blocks, 256, 0, st>>>(q, hd->d.hbits, hd->d.hwpre, h);
    if (!ok(cudaMemsetAsync(hd->d.hbits, 0, sizeof(unsigned) * NW, st))) return e;
    hota_frame_sums_kernel<<<L, 32, 0, st>>>(q, h);
    if (G > 0) hota_gcount_kernel<<<(G + 127) / 128, 128, 0, st>>>(q, h);
    hota_scan_kernel<<<1, 1024, 0, st>>>(IntIn{h.gcnt}, G, h.gseg);
    hota_scan_kernel<<<1, 1024, 0, st>>>(IntIn{h.msize}, L, h.moff);
    long long sizes[3];       // entries, score matrix elements, kept tracker ids
    if (!(ok(cudaMemcpyAsync(sizes, h.gseg + G, sizeof(long long), cudaMemcpyDeviceToHost, st)) &&
          ok(cudaMemcpyAsync(sizes + 1, h.moff + L, sizeof(long long), cudaMemcpyDeviceToHost, st)) &&
          ok(cudaMemcpyAsync(sizes + 2, hd->d.hwpre + NW, sizeof(long long), cudaMemcpyDeviceToHost, st)) &&
          ok(cudaStreamSynchronize(st))))
        return e;
    const size_t E = (size_t)sizes[0];
    h.Th = (int)sizes[2];
    if (!(ok(x.alloc(&h.et, E)) && ok(x.alloc(&h.ef, E)) && ok(x.alloc(&h.eij, E)) && ok(x.alloc(&h.ev, E)) &&
          ok(x.alloc(&h.es, E)) && ok(x.alloc(&h.efirst, E)) && ok(x.alloc(&h.elvl, E)) && ok(x.alloc(&h.ppos, E)) &&
          ok(x.alloc(&h.pgc, E)) && ok(x.alloc(&h.ptc, E)) && ok(x.alloc(&h.pmc, E * NA)) &&
          ok(x.alloc(&h.M, (size_t)sizes[1])) && ok(cudaMemsetAsync(h.M, 0, sizeof(double) * (size_t)sizes[1], st))))
        return e;
    if (G > 0) {
        hota_gather_kernel<<<G, 32, 0, st>>>(q, h);
        hota_pmc_kernel<<<G, 32, 0, st>>>(q, h);
    }
    hota_scan_kernel<<<1, 1024, 0, st>>>(IntIn{h.gdist}, G, h.poff);
    hota_frame_kernel<<<L, 32, 0, st>>>(q, h);
    hota_total_kernel<<<1, 32, 0, st>>>(q, h);
    if (G > 0) hota_pairs_kernel<<<G, 32, 0, st>>>(q, h);
    hota_assoc_kernel<<<1, 32, 0, st>>>(h, G, (long long)G * h.Th);
    if (!(ok(cudaGetLastError()) &&
          ok(cudaMemcpyAsync(cnt_host, h.cnt, sizeof(long long) * 3 * NA, cudaMemcpyDeviceToHost, st)) &&
          ok(cudaMemcpyAsync(sum_host, h.sum, sizeof(double) * 4 * NA, cudaMemcpyDeviceToHost, st))))
        return e;
    return cudaStreamSynchronize(st);
}

extern "C" int k2y_mot_result_ex(k2y_mot *h, long long *counts_host, double *motp_sum_host, int *rounds_host,
                                 long long *solved_host, long long *hota_counts_host, double *hota_sums_host,
                                 unsigned *status_host, void *stream) {
    if (!h || (!h->seqs.empty() && (!counts_host || !motp_sum_host || !rounds_host || !solved_host)) || !status_host ||
        (!hota_counts_host != !hota_sums_host)) {
        set_error("k2y_mot_result: null pointer");
        return K2Y_ERR_INVALID;
    }
    DeviceGuard g(h->device);
    cudaStream_t st = (cudaStream_t)stream;
    *status_host = 0;
    int host_n[4];
    cudaError_t e = cudaStreamWaitEvent(st, h->done, 0);
    for (size_t s = 0; s < h->seqs.size() && e == cudaSuccess; ++s) {
        Seq &q = h->seqs[s];
        e = evaluate_seq(h, q, st, host_n, rounds_host + s, solved_host + s);
        long long c[N_CTR];
        if (e == cudaSuccess) e = cudaMemcpyAsync(c, q.ctr, sizeof(c), cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaMemcpyAsync(motp_sum_host + s, q.motp, sizeof(double), cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) break;
        long long *o = counts_host + K2Y_MOT_FIELDS * s;
        for (int k = 0; k < 9; ++k) o[k] = c[k];        // TP FP FN IDSW Frag MT PT ML IDTP
        o[9] = h->gt_rows[s];
        o[10] = c[TRK_ROWS];
        o[11] = q.T;
        if ((long long)q.G * q.T > MAX_PAIRS) *status_host |= K2Y_MOT_TOO_MANY_IDS;
        else if (hota_counts_host)
            e = hota_seq(h, q, st, hota_counts_host + 3 * NA * s, hota_sums_host + 4 * NA * s);
        if (e != cudaSuccess) break;
    }
    unsigned st_dev = 0;
    if (e == cudaSuccess) e = cudaMemcpyAsync(&st_dev, h->d.status, sizeof(unsigned), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaEventRecord(h->done, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) {
        set_error("k2y_mot_result: %s", cudaGetErrorString(e));
        return K2Y_ERR_CUDA;
    }
    *status_host = st_dev | (*status_host & K2Y_MOT_TOO_MANY_IDS);
    return K2Y_OK;
}

extern "C" int k2y_mot_result(k2y_mot *h, long long *counts_host, double *motp_sum_host, int *rounds_host,
                              long long *solved_host, unsigned *status_host, void *stream) {
    return k2y_mot_result_ex(h, counts_host, motp_sum_host, rounds_host, solved_host, nullptr, nullptr, status_host, stream);
}
