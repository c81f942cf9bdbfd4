// Small helpers of the warp-per-class trackers (bytetrack.cu, ocsort.cu): the state layout's aligned slices, the float64
// product that never contracts into an FMA, and the ordered ballot compaction.
#pragma once

#include <cstddef>

namespace k2y {

// Reserves `bytes` at offset o (256-byte aligned slices) and returns where they start.
__host__ __device__ inline size_t take(size_t &o, size_t bytes) {
    size_t at = o;
    o = (o + bytes + 255) & ~(size_t)255;
    return at;
}

__device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }

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

}  // namespace k2y
