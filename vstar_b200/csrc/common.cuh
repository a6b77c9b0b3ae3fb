// Shared device/host helpers for the vstar_b200 sm_90a kernels.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#define VSB_OK 0
#define VSB_ERR_ARG -1
#define VSB_ERR_CUDA -2
#define VSB_ERR_UNSUPPORTED -3

void vsb_set_error(const char* fmt, ...);
int vsb_batch_invariant();   // see api.cu
int vsb_gemm_forced_bn();    // force_bn of vsb_gemm_set_tuning (gemm_tcgen05.cu)

#define VSB_CHECK_ARG(cond, ...)                 \
  do {                                           \
    if (!(cond)) {                               \
      vsb_set_error(__VA_ARGS__);                \
      return VSB_ERR_ARG;                        \
    }                                            \
  } while (0)

#define VSB_CUDA(call)                                                          \
  do {                                                                          \
    cudaError_t _e = (call);                                                    \
    if (_e != cudaSuccess) {                                                    \
      vsb_set_error("%s:%d CUDA error %s", __FILE__, __LINE__, cudaGetErrorString(_e)); \
      return VSB_ERR_CUDA;                                                      \
    }                                                                           \
  } while (0)

#define VSB_LAUNCH_CHECK() VSB_CUDA(cudaGetLastError())

typedef __nv_bfloat16 bf16;

__device__ __forceinline__ float bf2f(bf16 x) { return __bfloat162float(x); }
__device__ __forceinline__ bf16 f2bf(float x) { return __float2bfloat16_rn(x); }
// round-trip through bf16 (mimics the reference's per-op bf16 rounding)
__device__ __forceinline__ float rbf(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}

// ---------------------------------------------------------------- element types of the kernels that run in bf16 or f16
// T = bf16 (the VSM and the default VQA engine) or half (the SEAL VQA LLM in fp16, the reference's dtype).  The templated
// kernels take every conversion from here, so their bf16 instantiations are the code they were before the f16 variants.
#define VSB_PTX_BF16 "bf16"
#define VSB_PTX_F16 "f16"
template <typename T>
struct ElemT;
template <>
struct ElemT<bf16> {
  static constexpr bool is_f16 = false;
  static constexpr CUtensorMapDataType tma = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;   // wgmma / mma.sync operand type: VSB_PTX_BF16
  static __device__ __forceinline__ float to_f(bf16 x) { return bf2f(x); }
  static __device__ __forceinline__ bf16 from_f(float x) { return f2bf(x); }
  static __device__ __forceinline__ float round(float x) { return rbf(x); }
  static __device__ __forceinline__ uint32_t pack2(float lo, float hi) { return pack_bf16x2(lo, hi); }
  static __device__ __forceinline__ float2 unpack2(uint32_t u) { return unpack_bf16x2(u); }
};
template <>
struct ElemT<half> {
  static constexpr bool is_f16 = true;
  static constexpr CUtensorMapDataType tma = CU_TENSOR_MAP_DATA_TYPE_FLOAT16;    // wgmma / mma.sync operand type: VSB_PTX_F16
  static __device__ __forceinline__ float to_f(half x) { return __half2float(x); }
  static __device__ __forceinline__ half from_f(float x) { return __float2half_rn(x); }
  static __device__ __forceinline__ float round(float x) { return __half2float(__float2half_rn(x)); }
  static __device__ __forceinline__ uint32_t pack2(float lo, float hi) {
    __half2 v = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
  }
  static __device__ __forceinline__ float2 unpack2(uint32_t u) {
    __half2 v = *reinterpret_cast<__half2*>(&u);
    return __half22float2(v);
  }
};

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
__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// block-wide sum for blockDim.x <= 1024 (multiple of 32); `red` = 32 floats of smem
__device__ __forceinline__ float block_sum(float v, float* red) {
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  float r = (lane < nw) ? red[lane] : 0.f;
  r = warp_sum(r);
  return r;
}

// one MUFU op; |err| ~ 5e-4 absolute, well below the bf16 rounding applied to every result that uses it
__device__ __forceinline__ float tanh_approx_f(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// x * sigmoid(1.702 x) = 0.5 x (1 + tanh(0.851 x))  -- 1 MUFU instead of ex2 + rcp (the GEMM epilogue is MUFU-bound for short K)
__device__ __forceinline__ float quick_gelu_f(float x) {
  const float h = 0.5f * x;
  return fmaf(h, tanh_approx_f(0.851f * x), h);
}
__device__ __forceinline__ float gelu_erf_f(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }
// x * sigmoid(x) = 0.5 x (1 + tanh(0.5 x))
__device__ __forceinline__ float silu_f(float x) {
  const float h = 0.5f * x;
  return fmaf(h, tanh_approx_f(h), h);
}
__device__ __forceinline__ float sigmoid_f(float x) { return 1.f / (1.f + __expf(-x)); }

// ---------------------------------------------------------------- programmatic dependent launch (decode chain)
// A decode step is ~260 kernels of a few microseconds each on one stream; the gap between dependent kernels (drain, launch,
// CTA scheduling) is as long as many of the kernels.  Kernels launched with vsb_launch_pdl may become resident while their
// predecessor is still running; pdl_prologue() - the FIRST statement of such a kernel - lets the successor do the same and
// then blocks until the predecessor grid has completed and its writes are visible (griddepcontrol.wait), so nothing is read
// or written early.
__device__ __forceinline__ void pdl_prologue() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
}

template <typename... KArgs, typename... Args>
static inline cudaError_t vsb_launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, int cluster_x,
                                         Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int n = 0;
  attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[n].val.programmaticStreamSerializationAllowed = 1;
  ++n;
  if (cluster_x > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster_x;
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

static inline int vsb_num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}
