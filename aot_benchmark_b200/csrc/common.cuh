// Shared helpers for libaotb200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>

#define AOTB_OK 0
#define AOTB_ERR_ARG (-1)
#define AOTB_ERR_CUDA (-2)
#define AOTB_ERR_UNSUPPORTED (-3)

namespace aotb {

void set_error(const char* fmt, ...);
void count_launches(int n);

inline int check_launch(const char* what, int n_kernels = 1) {
    count_launches(n_kernels);
    cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) {
        cudaGetLastError();  // clear the sticky launch error
        set_error("%s: %s", what, cudaGetErrorString(e));
        return AOTB_ERR_CUDA;
    }
    return AOTB_OK;
}

#define AOTB_REQUIRE(cond, ...)               \
    do {                                      \
        if (!(cond)) {                        \
            ::aotb::set_error(__VA_ARGS__);   \
            return AOTB_ERR_ARG;              \
        }                                     \
    } while (0)

static inline int cdiv(int a, int b) { return (a + b - 1) / b; }

// ---- programmatic dependent launch (PDL): when enabled every kernel of this library is launched with the
// programmatic-stream-serialization attribute; kernels call pdl_trigger() at once (the next kernel in the stream may
// start its prologue) and pdl_wait() before their first read of data produced by the previous kernel.
bool pdl_enabled();

// cluster_z > 1 launches thread-block clusters of (1, 1, cluster_z) CTAs (grid.z must be a multiple of it).
template <typename... KArgs, typename... Args>
inline void launch_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, int cluster_z,
                           Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[2];
    int n = 0;
    if (pdl_enabled()) {
        attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[n].val.programmaticStreamSerializationAllowed = 1;
        ++n;
    }
    if (cluster_z > 1) {
        attr[n].id = cudaLaunchAttributeClusterDimension;
        attr[n].val.clusterDim.x = 1;
        attr[n].val.clusterDim.y = 1;
        attr[n].val.clusterDim.z = (unsigned)cluster_z;
        ++n;
    }
    cfg.attrs = attr;
    cfg.numAttrs = n;
    cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}
template <typename... KArgs, typename... Args>
inline void launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
    launch_cluster(kernel, grid, block, smem, st, 1, args...);
}

__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_sync() { pdl_trigger(); pdl_wait(); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// activation codes shared by several entry points
enum Act { ACT_NONE = 0, ACT_RELU = 1, ACT_GELU = 2, ACT_SILU = 3, ACT_RELU6 = 4, ACT_HSWISH = 5 };

// h_sigmoid(v) = relu6(v + 3) / 6 with a true division, as networks/encoders/mobilenetv3.py:33-39 computes it
__device__ __forceinline__ float hsigmoid(float v) { return fminf(fmaxf(v + 3.f, 0.f), 6.f) / 6.f; }

__device__ __forceinline__ float apply_act(float v, int act) {
    switch (act) {
        case ACT_RELU: return fmaxf(v, 0.f);
        case ACT_GELU: return 0.5f * v * (1.f + erff(v * 0.70710678118654752440f));  // exact erf GELU (basic.py:32)
        case ACT_SILU: return v / (1.f + expf(-v));                                   // x*sigmoid(x) (attention.py:585)
        case ACT_RELU6: return fminf(fmaxf(v, 0.f), 6.f);
        default: return v;
    }
}

// h_swish = v * h_sigmoid(v) (mobilenetv3.py:42-48) stays out of apply_act, so every kernel that existed before it compiles
// exactly as before.  The kernels MobileNetV3 runs take it as a template flag (fp32 conv finish, depthwise conv: HS selects the
// instantiation, so the existing ones are unchanged) or as a runtime code (gate scale, apply_act_hs); the tensor-core conv and
// GroupNorm reject ACT_HSWISH at their entry points.
template <bool HS>
__device__ __forceinline__ float apply_act_or_hswish(float v, int act) {
    return HS ? v * hsigmoid(v) : apply_act(v, act);
}
__device__ __forceinline__ float apply_act_hs(float v, int act) {
    return act == ACT_HSWISH ? v * hsigmoid(v) : apply_act(v, act);
}

}  // namespace aotb
