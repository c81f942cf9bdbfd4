// Hopper tensor-core (wgmma) convolution path — interface used by net.cu.
#pragma once
#include "common.h"

namespace k2y {

// Weights re-packed for the tensor-core kernels: B operand, K-major [Npad][Kpad] fp32, split into a
// tf32-exact "hi" plane and the fp32 remainder "lo" (for the 3xTF32 scheme).
struct TcWeights {
    float *d_hi = nullptr;
    float *d_lo = nullptr;
    unsigned short *d_bh = nullptr;  // bf16x3: bf16(w) and bf16(w - hi) planes, K-major [Npad][Kpad64]
    unsigned short *d_bm = nullptr;
    int K = 0, N = 0, Kpad = 0, Kpad64 = 0, Npad = 0;
};

int tc_pack(TcWeights &w, const float *kernel_kn, int K, int N);  // kernel_kn: [K][N] row-major (Keras HWIO flattened)
void tc_free(TcWeights &w);
bool tc_supported(const ConvArgs &a, const TcWeights &w);
size_t tc_scratch_bound(const ConvArgs &a, const TcWeights &w);           // split-K scratch a net must provide for this layer
int tc_launch_count(const ConvArgs &a, const TcWeights &w, int math_mode);  // kernels one launch_conv_tc issues
cudaError_t launch_conv_tc(const ConvArgs &a, const TcWeights &w, int math_mode, cudaStream_t st);

}  // namespace k2y
