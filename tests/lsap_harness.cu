// Test-only harness around warp_lsap (csrc/lsap_warp.cuh): one warp per problem, a dense float64 cost matrix per problem,
// match[i] = the column of row i or -1.  Two kernels, for the two places the library keeps the solver's state:
//  - lsap_global: LsapWork in global memory, sized per problem (as the evaluator's IDTP solve);
//  - lsap_shared: LsapWork in a shared block of K2Y_MOT_MAX_ROWS entries per array (as the evaluator's per-frame solves).
// Built by tests/test_gpu_lsap.py into a temporary directory; not part of the library.
#include <cstdint>

#include "k210_yolo_b200.h"
#include "lsap_warp.cuh"

namespace {

constexpr int CAP = K2Y_MOT_MAX_ROWS;

struct DenseCost {
    const double *c;
    int nc;
    __device__ double operator()(int i, int j) const { return c[(long long)i * nc + j]; }
};

struct SharedWork {
    double u[CAP], v[CAP], spc[CAP];
    int path[CAP], col4row[CAP], row4col[CAP], remaining[CAP];
    unsigned char SR[CAP], SC[CAP];
};

// woff[p]: the problem's first entry in each per-entry array of the global workspace (entries = max(nr, nc)).
__global__ void __launch_bounds__(32) lsap_global(const double *cost, const long long *coff, const int *nr, const int *nc,
                                                  const long long *woff, double *wd, int *wi, unsigned char *wb, long long wn,
                                                  int *match, const long long *moff) {
    const int p = blockIdx.x;
    const long long o = woff[p];
    LsapWork w{wd + o, wd + wn + o, wd + 2 * wn + o, wi + o, wi + wn + o, wi + 2 * wn + o, wi + 3 * wn + o, wb + o, wb + wn + o};
    warp_lsap(nr[p], nc[p], DenseCost{cost + coff[p], nc[p]}, w, match + moff[p]);
}

__global__ void __launch_bounds__(32) lsap_shared(const double *cost, const long long *coff, const int *nr, const int *nc,
                                                  int *match, const long long *moff) {
    __shared__ SharedWork s;
    const int p = blockIdx.x;
    LsapWork w{s.u, s.v, s.spc, s.path, s.col4row, s.row4col, s.remaining, s.SR, s.SC};
    warp_lsap(nr[p], nc[p], DenseCost{cost + coff[p], nc[p]}, w, match + moff[p]);
}

}  // namespace

// Solves n problems on `stream`: problem p is the nr[p] x nc[p] row-major matrix at cost + coff[p], its rows' columns go to
// match + moff[p].  shared != 0 runs lsap_shared (every max(nr, nc) <= K2Y_MOT_MAX_ROWS); otherwise lsap_global with
// workspace arrays wd [3 wn], wi [4 wn], wb [2 wn] and offsets woff.  Returns the launch's cudaError_t.
extern "C" int lsap_harness_run(int n, int shared, const double *cost, const long long *coff, const int *nr, const int *nc,
                                const long long *woff, double *wd, int *wi, unsigned char *wb, long long wn, int *match,
                                const long long *moff, void *stream) {
    if (n <= 0) return 0;
    if (shared)
        lsap_shared<<<n, 32, 0, (cudaStream_t)stream>>>(cost, coff, nr, nc, match, moff);
    else
        lsap_global<<<n, 32, 0, (cudaStream_t)stream>>>(cost, coff, nr, nc, woff, wd, wi, wb, wn, match, moff);
    return (int)cudaGetLastError();
}
