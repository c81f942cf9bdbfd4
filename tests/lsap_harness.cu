// Test-only harness around warp_lsap (csrc/lsap_warp.cuh): a dense float64 cost matrix per problem, match[i] = the column
// of row i or -1.  Three kernels, for the solver's two widths and the two places the library keeps its state:
//  - lsap_global: one warp per problem, LsapWork in global memory, sized per problem (as the evaluator's IDTP solve);
//  - lsap_shared: one warp per problem, LsapWork in a shared block of K2Y_MOT_MAX_ROWS entries per array (as the
//    evaluator's per-frame solves);
//  - lsap_thread: one thread per problem, 32 problems to a warp, LsapWork in global memory (as SORT's per-class solves).
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

// The workspace arrays wd [3 wn], wi [4 wn], wb [2 wn] from entry o on.
__device__ LsapWork global_work(double *wd, int *wi, unsigned char *wb, long long wn, long long o) {
    return LsapWork{wd + o, wd + wn + o, wd + 2 * wn + o, wi + o, wi + wn + o, wi + 2 * wn + o, wi + 3 * wn + o, wb + o, wb + wn + o};
}

// woff[p]: the problem's first entry in each per-entry array of the global workspace (entries = max(nr, nc)).
__global__ void __launch_bounds__(32) lsap_global(const double *cost, const long long *coff, const int *nr, const int *nc,
                                                  const long long *woff, double *wd, int *wi, unsigned char *wb, long long wn,
                                                  int *match, const long long *moff) {
    const int p = blockIdx.x;
    warp_lsap(nr[p], nc[p], DenseCost{cost + coff[p], nc[p]}, global_work(wd, wi, wb, wn, woff[p]), match + moff[p]);
}

__global__ void __launch_bounds__(32) lsap_shared(const double *cost, const long long *coff, const int *nr, const int *nc,
                                                  int *match, const long long *moff) {
    __shared__ SharedWork s;
    const int p = blockIdx.x;
    LsapWork w{s.u, s.v, s.spc, s.path, s.col4row, s.row4col, s.remaining, s.SR, s.SC};
    warp_lsap(nr[p], nc[p], DenseCost{cost + coff[p], nc[p]}, w, match + moff[p]);
}

__global__ void __launch_bounds__(32) lsap_thread(int n, const double *cost, const long long *coff, const int *nr, const int *nc,
                                                  const long long *woff, double *wd, int *wi, unsigned char *wb, long long wn,
                                                  int *match, const long long *moff) {
    const int p = blockIdx.x * 32 + threadIdx.x;
    if (p >= n) return;
    warp_lsap<1>(nr[p], nc[p], DenseCost{cost + coff[p], nc[p]}, global_work(wd, wi, wb, wn, woff[p]), match + moff[p]);
}

}  // namespace

// Solves n problems on `stream`: problem p is the nr[p] x nc[p] row-major matrix at cost + coff[p], its rows' columns go to
// match + moff[p].  mode 1 runs lsap_shared (every max(nr, nc) <= K2Y_MOT_MAX_ROWS); mode 0 lsap_global and mode 2
// lsap_thread, with workspace arrays wd [3 wn], wi [4 wn], wb [2 wn] and offsets woff.  Returns the launch's cudaError_t.
extern "C" int lsap_harness_run(int n, int mode, const double *cost, const long long *coff, const int *nr, const int *nc,
                                const long long *woff, double *wd, int *wi, unsigned char *wb, long long wn, int *match,
                                const long long *moff, void *stream) {
    if (n <= 0) return 0;
    if (mode == 1)
        lsap_shared<<<n, 32, 0, (cudaStream_t)stream>>>(cost, coff, nr, nc, match, moff);
    else if (mode == 2)
        lsap_thread<<<(n + 31) / 32, 32, 0, (cudaStream_t)stream>>>(n, cost, coff, nr, nc, woff, wd, wi, wb, wn, match, moff);
    else
        lsap_global<<<n, 32, 0, (cudaStream_t)stream>>>(cost, coff, nr, nc, woff, wd, wi, wb, wn, match, moff);
    return (int)cudaGetLastError();
}
