// What the GPU trackers (track.cu, bytetrack.cu, ocsort.cu) share: the state's layout, the float64 product that never
// contracts into an FMA, the ordered ballot compaction, SORT's IoU and block Kalman filter (oracle/sort_ref.py), and the
// stream's frame loop, which hands out the births' ids.  What differs between the trackers (their z, which records they
// keep, their association) stays in their own files.
#pragma once

#include <cstddef>

#include "common.h"
#include "lsap_warp.cuh"

namespace k2y {

// Reserves `bytes` at offset o (256-byte aligned slices) and returns where they start.
__host__ __device__ inline size_t take(size_t &o, size_t bytes) {
    size_t at = o;
    o = (o + bytes + 255) & ~(size_t)255;
    return at;
}

// The stream's frame count, last position and ids taken: the first bytes of every tracker's state.
struct StreamHeader {
    long long frame_count, last_pos;
    int ids_taken, started;
};

// A tracker's state is the header, then each per-class array as C consecutive slices of its per-class entries.  A tracker
// lists its arrays once, as X(type, name, entries per class), and these expand the list: K2Y_STATE_FIELD into its class
// view's fields, K2Y_STATE_SLICE into class c's view (device) and K2Y_STATE_BYTES into the state's bytes (host).  The two
// walks advance an offset o from state_start(); the entries per class are a product, such as 4 * k.
#define K2Y_STATE_FIELD(T, name, per) T *name;
#define K2Y_STATE_SLICE(T, name, per) v.name = reinterpret_cast<T *>(state + take(o, sizeof(T) * C * (per))) + c * per;
#define K2Y_STATE_BYTES(T, name, per) take(o, sizeof(T) * C * (per));

// The assignment solver's arrays, as a class view's LsapWork w: `rows` entries for the rows, `cols` for the columns (the
// smaller and the larger side of the problems the tracker solves).
#define K2Y_LSAP_ARRAYS(X, rows, cols)                                                                                       \
    X(double, w.u, rows) X(double, w.v, cols) X(double, w.spc, cols) X(int, w.path, cols) X(int, w.col4row, rows)           \
    X(int, w.row4col, cols) X(int, w.remaining, cols) X(unsigned char, w.SR, rows) X(unsigned char, w.SC, cols)

// The offset of the first per-class array.
__host__ __device__ inline size_t state_start() {
    size_t o = 0;
    take(o, sizeof(StreamHeader));
    return o;
}

__device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }

// numpy's maximum / minimum: a NaN in either operand is the result
__device__ __forceinline__ double mx(double a, double b) { return (a >= b || a != a) ? a : b; }
__device__ __forceinline__ double mn(double a, double b) { return (a <= b || a != a) ? a : b; }

// SORT's iou_batch for one pair (oracle/sort_ref.py ``iou``), 0 where the union is not > 0
__device__ inline double sort_iou(const double *d, const double *t) {
    const double w = mx(0.0, mn(d[2], t[2]) - mx(d[0], t[0]));
    const double h = mx(0.0, mn(d[3], t[3]) - mx(d[1], t[1]));
    const double wh = mul(w, h);
    const double uni = (mul(d[2] - d[0], d[3] - d[1]) + mul(t[2] - t[0], t[3] - t[1])) - wh;
    return uni > 0 ? wh / uni : 0.0;
}

// Calls emit(i, at) for the i in [0, n) with keep(i), at counting them in order from 0; returns their count.  Warp-wide.
template <class Keep, class Emit>
__device__ int compact(int n, const Keep &keep, const Emit &emit) {
    const int lane = threadIdx.x & 31;
    int base = 0;
    for (int i0 = 0; i0 < n; i0 += 32) {
        const int i = i0 + lane;
        const bool k = i < n && keep(i);
        const unsigned b = __ballot_sync(0xffffffffu, k);
        if (k) emit(i, base + __popc(b & ((1u << lane) - 1u)));
        base += __popc(b);
    }
    __syncwarp();
    return base;
}

// The walk of the warp-per-class trackers over the classes: the warps stride over them, and for each class c the warp's
// view slot (in shared memory, which keeps the view's pointers out of registers) is set to view(c) before body(c) runs.
// Warp-wide.
template <class View, class MakeView, class Body>
__device__ void for_each_class(int C, View &slot, const MakeView &view, const Body &body) {
    for (int c = threadIdx.x >> 5; c < C; c += blockDim.x >> 5) {
        __syncwarp();
        if ((threadIdx.x & 31) == 0) slot = view(c);
        __syncwarp();
        body(c);
    }
}

// -- SORT's filter in block form (oracle/sort_ref.py): (p, v, P_pp, P_pv, P_vv) of cx, cy, s, and (r, P_rr) ---------------
struct Filt {
    double b[3][5];
    double r[2];
};

__device__ inline void filt_init(Filt &f, const double *z) {
    for (int q = 0; q < 3; ++q) {
        f.b[q][0] = z[q];
        f.b[q][1] = 0.0;
        f.b[q][2] = 10.0;
        f.b[q][3] = 0.0;
        f.b[q][4] = 10000.0;
    }
    f.r[0] = z[3];
    f.r[1] = 10.0;
}

// The predict and update of one block (p, v, P_pp, P_pv, P_vv)
__device__ inline void blk_predict(double *b, double qv) {
    const double t = b[3] + b[4];
    b[0] = b[0] + b[1];
    b[2] = ((b[2] + b[3]) + t) + 1.0;
    b[3] = t;
    b[4] = b[4] + qv;
}

__device__ inline void blk_update(double *b, double z, double R) {
    const double p = b[0], v = b[1], a = b[2], pv = b[3], d = b[4];
    const double y = z - p, S = a + R;
    const double k0 = a / S, k1 = pv / S;
    const double c = 1.0 - k0;
    const double m = pv - mul(k1, a), n = d - mul(k1, pv), rk0 = mul(R, k0);
    b[0] = p + mul(k0, y);
    b[1] = v + mul(k1, y);
    b[2] = mul(mul(c, a), c) + mul(rk0, k0);
    b[3] = mul(c, m) + mul(rk0, k1);
    b[4] = (n - mul(k1, m)) + mul(mul(R, k1), k1);
}

__device__ inline void filt_predict(Filt &f) {
    blk_predict(f.b[0], 0.01);
    blk_predict(f.b[1], 0.01);
    blk_predict(f.b[2], 1e-4);
    f.r[1] = f.r[1] + 1.0;
}

__device__ inline void filt_update(Filt &f, const double *z) {
    blk_update(f.b[0], z[0], 1.0);
    blk_update(f.b[1], z[1], 1.0);
    blk_update(f.b[2], z[2], 10.0);
    const double S = f.r[1] + 10.0, k = f.r[1] / S, c = 1.0 - k;
    f.r[0] = f.r[0] + mul(k, z[3] - f.r[0]);
    f.r[1] = mul(mul(c, f.r[1]), c) + mul(mul(10.0, k), k);
}

__device__ inline void state_box(const Filt &f, double *o) {
    const double cx = f.b[0][0], cy = f.b[1][0], s = f.b[2][0];
    const double w = sqrt(mul(s, f.r[0]));
    const double h = s / w;
    o[0] = cx - w / 2.0;
    o[1] = cy - h / 2.0;
    o[2] = cx + w / 2.0;
    o[3] = cy + h / 2.0;
}

// SORT's tracker predict, for a track with a filter kf and the counters age, hit_streak and tsu (time since update): the
// `vs *= 0` quirk on the scale's velocity, the filter's predict, then the counters.
template <class Track>
__device__ void sort_predict(Track &t) {
    double *sb = t.kf.b[2];
    if (sb[1] + sb[0] <= 0) sb[1] = mul(sb[1], 0.0);
    filt_predict(t.kf);
    t.age += 1;
    if (t.tsu > 0) t.hit_streak = 0;
    t.tsu += 1;
}

// -- the stream ------------------------------------------------------------------------------------------------------------
// A batch of frames in a gathered record block (dets [.., C, K, 6] and counts [.., C], row_stride words a row), and the
// outputs ids [n_frames, C, K] and boxes [n_frames, C, K, 4].  The frames may belong to n_streams streams, whose states lie
// `stride` bytes apart: frame f is stream streams[f] (every frame is stream 0 when streams is null).
struct Batch {
    const int32_t *dets, *counts, *rows;
    const long long *positions;
    long long row_stride;
    int n_frames, C, K;
    int32_t *ids_out;
    float *boxes_out;
    const int32_t *streams;
    int n_streams;
    size_t stride;

    __device__ int stream(int f) const { return streams ? streams[f] : 0; }
    // the first frame from f on of the CTA's stream, blockIdx.x; n_frames when there is none
    __device__ int next_frame(int f) const {
        while (f < n_frames && stream(f) != (int)blockIdx.x) ++f;
        return f;
    }

    // class c's records in frame f and their count, clamped to [0, K]
    __device__ int records(int f, int c, const int32_t *&rec) const {
        const long long row = rows[f] * row_stride;
        rec = dets + row + (long long)c * K * 6;
        const int n = counts[row + c];
        return n < 0 ? 0 : (n > K ? K : n);
    }
    __device__ int32_t *ids(int f, int c) const { return ids_out + ((long long)f * C + c) * K; }
    __device__ float *boxes(int f, int c) const { return boxes_out + ((long long)f * C + c) * K * 4; }
    // class c's outputs of frame f, the entries first, first + step, ..., cleared: id -1, box 0
    __device__ void clear(int f, int c, int first, int step) const {
        int32_t *id = ids(f, c);
        float *box = boxes(f, c);
        for (int k = first; k < K; k += step) {
            id[k] = -1;
            for (int q = 0; q < 4; ++q) box[4 * k + q] = 0.f;
        }
    }
};

// Box (x1, y1, x2, y2) as the records' float32 (y1, x1, y2, x2).
__device__ inline void write_box(float *o, const double *b) {
    o[0] = (float)b[1];
    o[1] = (float)b[0];
    o[2] = (float)b[3];
    o[3] = (float)b[2];
}

// The checks every tracker's update makes of its batch; false, with the error set, for a null pointer, n_frames < 0, a
// row stride below one row's records, n_streams < 1, or (with several streams) a state stride below one stream's
// state_bytes or not a multiple of 256.
inline bool batch_ok(const char *fn, const void *state, const Batch &b, size_t state_bytes) {
    if (!state || !b.dets || !b.counts || !b.rows || !b.positions || !b.ids_out || !b.boxes_out || b.n_frames < 0) {
        set_error("%s: null pointer or n_frames < 0", fn);
        return false;
    }
    if (b.row_stride < (long long)b.C * b.K * 6) {
        set_error("%s: row stride %lld words is smaller than one row's records", fn, b.row_stride);
        return false;
    }
    if (b.n_streams < 1 || (b.n_streams > 1 && (b.stride < state_bytes || b.stride % 256 != 0))) {
        set_error("%s: n_streams %d (>= 1) and, with several, a state stride of %zu bytes (a multiple of 256, >= the %zu "
                  "bytes of one stream's state)", fn, b.n_streams, b.stride, state_bytes);
        return false;
    }
    return true;
}

// Whether the batch has a frame of the CTA's stream, blockIdx.x; a kernel returns at once when it has none, leaving that
// stream's state as it is, and else works on the state at blockIdx.x * stride.  CTA 0 first clears the outputs of the
// frames whose stream lies outside [0, n_streams).  Block-wide.  Not inlined: inlined, it costs SORT's kernel (held to 64
// registers) spills in its frame loop.
__device__ __noinline__ inline bool stream_has_frames(const Batch &bt) {
    if (blockIdx.x == 0 && bt.streams) {
        for (long long i = threadIdx.x; i < (long long)bt.n_frames * bt.C; i += blockDim.x) {
            const int f = (int)(i / bt.C), s = bt.streams[f];
            if (s < 0 || s >= bt.n_streams) bt.clear(f, (int)(i % bt.C), 0, 1);
        }
    }
    int mine = 0;
    for (int f = threadIdx.x; f < bt.n_frames && !mine; f += blockDim.x) mine = bt.stream(f) == (int)blockIdx.x;
    return __syncthreads_or(mine);
}

// The stream's frame loop, run by the whole CTA over the batch's frames of its stream, blockIdx.x, in batch order; `state`
// is that stream's.  A jump of g positions is g - 1 updates without detections, and after max_empty of
// them no track is left; then the frame runs, and its births take their ids from the stream's one counter in (class,
// birth) order.  The tracker's callbacks:
//  - empty(n, fc): n updates without detections, the first at frame count fc + 1;
//  - frame(f, fc, births): frame f at frame count fc, storing class c's births in births[c];
//  - emit(f, fc, births, base): frame f's outputs; class c's births are ids base[c] + 1, base[c] + 2, ...
template <class Empty, class Frame, class Emit>
__device__ void frame_loop(unsigned char *state, const Batch &bt, long long max_empty, const Empty &empty, const Frame &frame,
                           const Emit &emit) {
    __shared__ int s_births[1024];
    __shared__ int s_base[1024];
    __shared__ StreamHeader s_hdr;      // the header as the frames advance it, in shared memory to keep it out of registers
    StreamHeader *hdr = reinterpret_cast<StreamHeader *>(state);
    if (threadIdx.x == 0) s_hdr = *hdr;
    __syncthreads();
    for (int f = bt.next_frame(0); f < bt.n_frames; f = bt.next_frame(f + 1)) {
        const long long pos = bt.positions[f], last = s_hdr.last_pos;
        const long long gap = s_hdr.started && pos > last + 1 ? pos - last - 1 : 0;
        empty(gap < max_empty ? gap : max_empty, s_hdr.frame_count);
        const long long fc = s_hdr.frame_count + gap + 1;
        frame(f, fc, s_births);
        __syncthreads();
        if (threadIdx.x == 0) {
            int acc = s_hdr.ids_taken;
            for (int q = 0; q < bt.C; ++q) {
                s_base[q] = acc;
                acc += s_births[q];
            }
            s_hdr.frame_count = fc;
            s_hdr.last_pos = pos;
            s_hdr.ids_taken = acc;
            s_hdr.started = 1;
        }
        __syncthreads();
        emit(f, fc, s_births, s_base);
        __syncthreads();        // s_births / s_base / s_hdr are rewritten by the next frame
    }
    if (threadIdx.x == 0) *hdr = s_hdr;
}

}  // namespace k2y
