// Shared declarations for libk210yolo_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <string>

#include "../../include/k210_yolo_b200.h"

namespace k2y {

void set_error(const char *fmt, ...);

// libjpeg-turbo's JPEG_MAX_DIMENSION: it (and so PIL) refuses to write or read a frame with more rows or columns.
constexpr int JPEG_MAX_DIMENSION = 65500;

#define K2Y_CUDA_CHECK(expr)                                                                     \
    do {                                                                                         \
        cudaError_t _e = (expr);                                                                 \
        if (_e != cudaSuccess) {                                                                 \
            k2y::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
            return K2Y_ERR_CUDA;                                                                 \
        }                                                                                        \
    } while (0)

enum Act : int { ACT_NONE = 0, ACT_LEAKY = 1, ACT_RELU = 2, ACT_RELU6 = 3 };

// One dense convolution (1x1 or 3x3) as an implicit GEMM over NHWC fp32 activations:
//   dst[b,oy,ox,n] = act( scale[n] * sum_{ky,kx,ci} in[b, oy*s-pad_t+ky, ox*s-pad_l+kx, ci] * w[(ky,kx,ci), n] + shift[n] ) (+ residual)
// where `in` is the channel-concatenation of src0 (optionally nearest-upsampled x2) and src1.
struct ConvArgs {
    const float *src0;
    const float *src1;      // nullptr when there is no concat
    const float *residual;  // nullptr when there is no Add
    float *dst;
    const float *w;         // [K][N] row-major, K = kh*kw*(C0+C1) ordered (ky,kx,ci)  (== Keras HWIO flattened)
    const float *scale;     // [N]
    const float *shift;     // [N]
    int B, H, W;            // logical input extent (after upsampling src0)
    int C0, C1;
    int up0;                // src0 stored at (H/2, W/2)
    int OH, OW, N;
    int kh, kw, stride, pad_t, pad_l;
    int act;
    float alpha;
    // first layer only: uint8 pixels + per-image maximum; the kernel feeds x = u8 / max  (tools/utils.py:405 `img / np.max(img)`)
    const unsigned char *src_u8 = nullptr;
    const int *img_max = nullptr;
    // host copies of w / scale / shift (first conv: passed to the kernel BY VALUE, i.e. through the constant bank)
    const float *w_host = nullptr, *scale_host = nullptr, *shift_host = nullptr;
    // caller-owned scratch for split-K partials (one per net, so nets on different streams never share it); null = the
    // per-device default of the single-layer test hook
    float *tc_scratch = nullptr;
    size_t tc_scratch_bytes = 0;
    // SM budget of the persistent tensor-core kernels (tile planner + grid size); 0 = the whole device.  A net that shares the
    // GPU with other nets in flight (LanedPipeline) plans for its share, so that the lanes' kernels run side by side instead of
    // queueing behind each other's one-CTA-per-SM grids
    int sm_limit = 0;
};

struct DwArgs {
    const float *src;
    float *dst;
    const float *w;      // [9][C]
    const float *scale;  // [C]
    const float *shift;  // [C]
    int B, H, W, C, OH, OW, stride, pad_t, pad_l;
    int act;
    float alpha;
};

struct PoolArgs {
    const float *src;
    float *dst;
    int B, H, W, C, OH, OW, stride;  // 2x2 window, SAME (pads bottom/right with -inf)
};

// fp32 CUDA-core kernels (conv_simt.cu)
cudaError_t launch_conv_simt(const ConvArgs &a, cudaStream_t st);
cudaError_t launch_dwconv(const DwArgs &a, cudaStream_t st);
cudaError_t launch_maxpool(const PoolArgs &a, cudaStream_t st);
cudaError_t launch_image_max_u8(const unsigned char *x, int batch, size_t bytes_per_image, int *max_out, cudaStream_t st);

// Programmatic dependent launch: every kernel of a step is launched with programmaticStreamSerializationAllowed and calls
// pdl_wait() before it touches anything a predecessor wrote or may still read (returns once the preceding grid has
// completed and flushed).  The next kernel is launched as each grid's CTAs exit, before the grid's completion and flush,
// which hides the launch gap.  No kernel triggers its dependents earlier (griddepcontrol.launch_dependents): the next
// kernel's CTAs would then be placed as soon as any SM had room and wait there, and a persistent tensor-core CTA holds a
// whole SM's shared memory while it waits, so with several nets in flight (LanedPipeline) one lane's waiting CTAs took the
// SMs another lane's running kernels could use (cfg 2 at two lanes ran 0.913-0.919 ms per step with the early trigger,
// 0.784-0.787 without, on an H100 80GB HBM3 SXM at 700 W).  K2Y_NO_PDL=1 falls back to plain stream order.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
bool pdl_enabled();

template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

__device__ __forceinline__ float apply_act(float v, int act, float alpha) {
    if (act == ACT_LEAKY) return v >= 0.f ? v : v * alpha;
    if (act == ACT_RELU) return fmaxf(v, 0.f);
    if (act == ACT_RELU6) return fminf(fmaxf(v, 0.f), 6.f);
    return v;
}

}  // namespace k2y
