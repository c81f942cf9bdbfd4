// scipy's linear_sum_assignment (Crouse's shortest augmenting path as scipy implements it), run by a group of W threads,
// a warp (W = 32) or one thread (W = 1): the row and column of every pair equal scipy's, ties included (oracle/sort_ref.py
// ``lsap`` restates the algorithm).  The column scan of each step is spread over the group; its pick is reduced over the
// warp with scipy's tie rule: the lowest reduced cost, among equal costs the last unassigned column in scan order, else the
// first column.  Every other step is the first thread's.  The one-thread form has no warp-collective operation, so the
// threads of a warp may each solve their own problem with divergent control flow.
#pragma once

#include <math_constants.h>

// Per-group state: u / col4row / SR of min(nr, nc) rows, the rest of max(nr, nc) columns.  Shared or global memory.
struct LsapWork {
    double *u, *v, *spc;
    int *path, *col4row, *row4col, *remaining;
    unsigned char *SR, *SC;
};

// Solves the nr0 x nc0 problem of cost(i, j) (transposed when nc0 < nr0, as scipy does) and writes match[i] = the column
// of row i, or -1 for a row left out (only when nr0 > nc0).  Every thread of the group calls it; match is complete after
// it returns.
template <int W = 32, class Cost>
__device__ void warp_lsap(int nr0, int nc0, const Cost &cost, LsapWork w, int *match) {
    static_assert(W == 32 || W == 1, "a warp or one thread");
    auto sync = [] {
        if constexpr (W == 32) __syncwarp();
    };
    const int lane = W == 32 ? threadIdx.x & 31 : 0;
    const bool tr = nc0 < nr0;
    const int nr = tr ? nc0 : nr0, nc = tr ? nr0 : nc0;
    for (int i = lane; i < nr; i += W) {
        w.u[i] = 0.0;
        w.col4row[i] = -1;
    }
    for (int j = lane; j < nc; j += W) {
        w.v[j] = 0.0;
        w.path[j] = -1;
        w.row4col[j] = -1;
    }
    sync();
    for (int cur = 0; cur < nr; ++cur) {
        for (int j = lane; j < nc; j += W) {
            w.spc[j] = CUDART_INF;
            w.SC[j] = 0;
            w.remaining[j] = nc - j - 1;
        }
        for (int i = lane; i < nr; i += W) w.SR[i] = 0;
        sync();
        int i = cur, sink = -1, num = nc;
        double min_val = 0.0;
        while (sink == -1) {
            if (lane == 0) w.SR[i] = 1;
            const double ui = w.u[i];
            double best = CUDART_INF;
            int key = 0x7fffffff;       // unassigned: num - 1 - it (the last wins), assigned: nc + it (the first wins)
            for (int it = lane; it < num; it += W) {
                const int j = w.remaining[it];
                const double c = tr ? cost(j, i) : cost(i, j);
                const double r = ((min_val + c) - ui) - w.v[j];
                if (r < w.spc[j]) {
                    w.path[j] = i;
                    w.spc[j] = r;
                }
                const double s = w.spc[j];
                const int k = w.row4col[j] == -1 ? num - 1 - it : nc + it;
                if (s < best || (s == best && k < key)) {
                    best = s;
                    key = k;
                }
            }
            if constexpr (W == 32) {
                for (int o = 16; o > 0; o >>= 1) {
                    const double ob = __shfl_xor_sync(0xffffffffu, best, o);
                    const int ok = __shfl_xor_sync(0xffffffffu, key, o);
                    if (ob < best || (ob == best && ok < key)) {
                        best = ob;
                        key = ok;
                    }
                }
            }
            const int index = key >= nc ? key - nc : num - 1 - key;
            min_val = best;
            sync();
            const int j = w.remaining[index];
            const int rj = w.row4col[j];
            if (rj == -1) sink = j;
            else i = rj;
            sync();
            if (lane == 0) {
                w.SC[j] = 1;
                w.remaining[index] = w.remaining[num - 1];
            }
            --num;
            sync();
        }
        for (int r = lane; r < nr; r += W)
            if (r == cur) w.u[r] += min_val;
            else if (w.SR[r]) w.u[r] += min_val - w.spc[w.col4row[r]];
        for (int j = lane; j < nc; j += W)
            if (w.SC[j]) w.v[j] -= min_val - w.spc[j];
        sync();
        if (lane == 0) {
            int j = sink;
            while (true) {
                const int r = w.path[j];
                w.row4col[j] = r;
                const int t = w.col4row[r];
                w.col4row[r] = j;
                j = t;
                if (r == cur) break;
            }
        }
        sync();
    }
    if (tr) {
        for (int r = lane; r < nr0; r += W) match[r] = w.row4col[r];
    } else {
        for (int r = lane; r < nr0; r += W) match[r] = w.col4row[r];
    }
    sync();
}
