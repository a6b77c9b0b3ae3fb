// Skinny GEMM for decode-sized problems (M <= 8 rows): C[M,N] = epi(A[M,K] . W[N,K]^T + bias) (+ residual).
//
// With one to eight activation rows every weight byte is used for <= 16 flops, so the problem is HBM-bound: the job is
// to stream W once at full bandwidth (Vicuna-7B decode reads 13.5 GB of weights per token; SURVEY.md §8d "secondary (HBM)
// bounds").  A 128-row tensor-core tile wastes >= 94 % of the tensor core here and, worse, leaves most SMs without enough
// loads in flight.  This kernel keeps the machine full of
// outstanding 16-byte loads instead:
//   * one warp owns two adjacent weight rows (= two output columns; for the interleaved gate/up matrix exactly one SwiGLU
//     output) and strides over K with 16 B per lane => every load instruction of a warp covers 512 contiguous bytes of a row;
//   * 8 such loads per row are issued back to back before the first FMA (8 KB in flight per warp), bypassing L1
//     allocation so the weights do not wash the activation rows out of L1;
//   * the M activation rows are re-read through L1 (they are at most 8 x 22 KB and shared by all warps of the SM);
//   * fp32 accumulation in the same k order for every column, butterfly reduction at the end, and the same epilogue
//     semantics as the wgmma kernel (bias -> activation / SwiGLU -> + residual -> bf16 / fp32, output-row remap).
// Algorithmic bytes per launch: 2*N*K (weights) + 2*M*K + 2*M*N.
#include "common.cuh"
#include "vstar_b200.h"

namespace {

template <typename T>
struct SkinnyParams {
  const T* A;
  const T* W;
  void* C;
  const T* bias;
  const void* residual;
  long long lda, ldw, ldc, ldr;
  int M, N, K;
  int epilogue, out_fp32;
  int rows_per_group;
  long long group_stride, group_offset;
};

__device__ __forceinline__ uint4 ld_stream16(const void* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}

template <typename T>
__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
  if constexpr (ElemT<T>::is_f16) {
    // f16 -> fp32 needs a real conversion (cvt) per element
    float2 t;
    t = ElemT<T>::unpack2(u.x); f[0] = t.x; f[1] = t.y;
    t = ElemT<T>::unpack2(u.y); f[2] = t.x; f[3] = t.y;
    t = ElemT<T>::unpack2(u.z); f[4] = t.x; f[5] = t.y;
    t = ElemT<T>::unpack2(u.w); f[6] = t.x; f[7] = t.y;
  } else {
    // bf16 -> fp32 is a 16-bit shift: low half = element 0
    f[0] = __uint_as_float(u.x << 16); f[1] = __uint_as_float(u.x & 0xffff0000u);
    f[2] = __uint_as_float(u.y << 16); f[3] = __uint_as_float(u.y & 0xffff0000u);
    f[4] = __uint_as_float(u.z << 16); f[5] = __uint_as_float(u.z & 0xffff0000u);
    f[6] = __uint_as_float(u.w << 16); f[7] = __uint_as_float(u.w & 0xffff0000u);
  }
}

constexpr int SK_THREADS = 256;
constexpr int SK_UNROLL = 8;      // 16 B loads in flight per lane and weight row

template <int MT, typename T>
__global__ void __launch_bounds__(SK_THREADS) gemm_skinny_kernel(const SkinnyParams<T> p) {
  using E = ElemT<T>;
  pdl_prologue();
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * SK_THREADS + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * SK_THREADS) >> 5;
  const int npairs = (p.N + 1) >> 1;
  const int kchunks = p.K >> 3;                 // K % 8 == 0 (checked on the host)
  const uint4 zero = make_uint4(0u, 0u, 0u, 0u);

  for (int pair = warp; pair < npairs; pair += nwarps) {
    const int n0 = pair * 2;
    const bool has1 = (n0 + 1 < p.N);
    const uint4* w0 = reinterpret_cast<const uint4*>(p.W + (long long)n0 * p.ldw);
    const uint4* w1 = reinterpret_cast<const uint4*>(p.W + (long long)(has1 ? n0 + 1 : n0) * p.ldw);
    float acc[MT][2];
#pragma unroll
    for (int m = 0; m < MT; ++m) acc[m][0] = acc[m][1] = 0.f;

    for (int c0 = lane; c0 < kchunks; c0 += 32 * SK_UNROLL) {
      uint4 wa[SK_UNROLL], wb[SK_UNROLL];
#pragma unroll
      for (int u = 0; u < SK_UNROLL; ++u) {
        const int c = c0 + u * 32;
        const bool ok = c < kchunks;
        wa[u] = ok ? ld_stream16(w0 + c) : zero;
        wb[u] = ok ? ld_stream16(w1 + c) : zero;
      }
#pragma unroll
      for (int u = 0; u < SK_UNROLL; ++u) {
        const int c = c0 + u * 32;
        if (c < kchunks) {
          float fa[8], fb[8];
          unpack8<T>(wa[u], fa);
          unpack8<T>(wb[u], fb);
#pragma unroll
          for (int m = 0; m < MT; ++m) {
            if (m < p.M) {
              const uint4 av = __ldg(reinterpret_cast<const uint4*>(p.A + (long long)m * p.lda) + c);
              float x[8];
              unpack8<T>(av, x);
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                acc[m][0] = fmaf(x[i], fa[i], acc[m][0]);
                acc[m][1] = fmaf(x[i], fb[i], acc[m][1]);
              }
            }
          }
        }
      }
    }
    // butterfly: every lane ends with the full sums
#pragma unroll
    for (int m = 0; m < MT; ++m) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        acc[m][0] += __shfl_xor_sync(0xffffffffu, acc[m][0], o);
        acc[m][1] += __shfl_xor_sync(0xffffffffu, acc[m][1], o);
      }
    }
    // lane 2m + c finishes output (m, n0 + c)
    float mine = 0.f;
#pragma unroll
    for (int m = 0; m < MT; ++m) {
      if (lane == 2 * m) mine = acc[m][0];
      if (lane == 2 * m + 1) mine = acc[m][1];
    }
    const int m = lane >> 1, c = lane & 1;
    const int n = n0 + c;
    const bool valid = (m < p.M) && (m < MT) && (n < p.N);
    if (valid && p.bias != nullptr) mine += E::to_f(p.bias[n]);
    const float up = __shfl_down_sync(0xffffffffu, mine, 1);        // SwiGLU: odd column = up_j
    if (!valid) continue;
    const long long orow = (long long)(m / p.rows_per_group) * p.group_stride + p.group_offset + (m % p.rows_per_group);
    if (p.epilogue == VSB_EPI_SWIGLU) {
      if (c == 0) reinterpret_cast<T*>(p.C)[orow * p.ldc + (n0 >> 1)] = E::from_f(silu_f(mine) * up);
      continue;
    }
    if (p.epilogue == VSB_EPI_QUICK_GELU) mine = quick_gelu_f(mine);
    else if (p.epilogue == VSB_EPI_RELU) mine = fmaxf(mine, 0.f);
    else if (p.epilogue == VSB_EPI_GELU) mine = gelu_erf_f(mine);
    if (p.out_fp32) {
      if (p.residual) mine += reinterpret_cast<const float*>(p.residual)[orow * p.ldr + n];
      reinterpret_cast<float*>(p.C)[orow * p.ldc + n] = mine;
    } else {
      if (p.residual) mine += E::to_f(reinterpret_cast<const T*>(p.residual)[orow * p.ldr + n]);
      reinterpret_cast<T*>(p.C)[orow * p.ldc + n] = E::from_f(mine);
    }
  }
}


// ---------------------------------------------------------------- M <= 16: same weight-streaming structure on mma.sync
// From three activation rows on, the scalar kernel above is bound by its FMA / unpack instructions.  The wgmma tile kernel
// is no better here: its 64-wide k-blocks fetch 128 B per weight row per TMA box, a DRAM-hostile pattern when nothing is
// reused.  This variant keeps the streaming access
// pattern and lets the tensor core do the arithmetic with W as the 16-row A operand of mma.sync.m16n8k16 and the (<= 8 per
// n-tile) activation rows as the B operand:
//   * a block owns 16 weight rows; its 8 warps interleave over K in steps of 32 (each lane loads 16 B = 8 consecutive k of
//     rows g and g+8, so a block round covers 512 contiguous bytes of every row; 4 rounds are in flight);
//   * the k order inside an MMA is permuted consistently for A and B (lane t's 16 bytes feed k-slots {2t,2t+1,2t+8,2t+9} of
//     two MMAs), which is legal because the contraction is order-free and makes every global load a 16-byte vector;
//   * the warp's accumulators already hold complete dot products over its k-steps; the 8 warps are summed through shared memory.
#define VSB_MMA_16816(TY)                                                                                                         \
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32." TY "." TY ".f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};" \
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])                                                                \
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1))
template <typename T>
__device__ __forceinline__ void mma_16816(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  if constexpr (ElemT<T>::is_f16) VSB_MMA_16816(VSB_PTX_F16);
  else VSB_MMA_16816(VSB_PTX_BF16);
}

constexpr int SM_ROWS = 16;       // weight rows per block
constexpr int SM_WARPS = 8;
constexpr int SM_UNROLL = 4;

template <int NT, typename T>      // n-tiles of 8 activation rows: M <= 8 * NT
__global__ void __launch_bounds__(SM_WARPS * 32) gemm_skinny_mma_kernel(const SkinnyParams<T> p) {
  using E = ElemT<T>;
  pdl_prologue();
  __shared__ float red[SM_WARPS][NT][SM_ROWS][8 + 1];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int ksteps = (p.K + 31) >> 5;
  const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
  const int ngroups = (p.N + SM_ROWS - 1) / SM_ROWS;

  for (int grp = blockIdx.x; grp < ngroups; grp += gridDim.x) {
    const int n0 = grp * SM_ROWS;
    const bool r0ok = (n0 + g) < p.N, r1ok = (n0 + g + 8) < p.N;
    const T* w0 = p.W + (long long)(r0ok ? n0 + g : 0) * p.ldw + t * 8;
    const T* w1 = p.W + (long long)(r1ok ? n0 + g + 8 : 0) * p.ldw + t * 8;
    const T* arow[NT];
    bool aok[NT];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      aok[nt] = (nt * 8 + g) < p.M;
      arow[nt] = p.A + (long long)(aok[nt] ? nt * 8 + g : 0) * p.lda + t * 8;
    }
    float c[NT][4];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) c[nt][0] = c[nt][1] = c[nt][2] = c[nt][3] = 0.f;

    for (int s0 = warp; s0 < ksteps; s0 += SM_WARPS * SM_UNROLL) {
      uint4 wa[SM_UNROLL], wb[SM_UNROLL];
#pragma unroll
      for (int u = 0; u < SM_UNROLL; ++u) {
        const int k = (s0 + u * SM_WARPS) * 32;
        const bool ok = (k + t * 8) < p.K;              // K % 8 == 0: a 16-byte vector is either fully inside or outside
        wa[u] = (ok && r0ok) ? ld_stream16(w0 + k) : zero;
        wb[u] = (ok && r1ok) ? ld_stream16(w1 + k) : zero;
      }
#pragma unroll
      for (int u = 0; u < SM_UNROLL; ++u) {
        const int k = (s0 + u * SM_WARPS) * 32;
        const bool ok = (k + t * 8) < p.K;
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
          const uint4 av = (ok && aok[nt]) ? __ldg(reinterpret_cast<const uint4*>(arow[nt] + k)) : zero;
          mma_16816<T>(c[nt], wa[u].x, wb[u].x, wa[u].y, wb[u].y, av.x, av.y);
          mma_16816<T>(c[nt], wa[u].z, wb[u].z, wa[u].w, wb[u].w, av.z, av.w);
        }
      }
    }
    // accumulator layout: c0 (row g, m 2t), c1 (row g, m 2t+1), c2 (row g+8, m 2t), c3 (row g+8, m 2t+1)
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      red[warp][nt][g][2 * t] = c[nt][0];
      red[warp][nt][g][2 * t + 1] = c[nt][1];
      red[warp][nt][g + 8][2 * t] = c[nt][2];
      red[warp][nt][g + 8][2 * t + 1] = c[nt][3];
    }
    __syncthreads();
    // thread -> (m, row pair): 8 row pairs x 8*NT activation rows
    for (int idx = threadIdx.x; idx < 8 * 8 * NT; idx += SM_WARPS * 32) {
      const int rp = idx & 7, m = idx >> 3;
      const int nt = m >> 3, mi = m & 7;
      float v0 = 0.f, v1 = 0.f;
#pragma unroll
      for (int w = 0; w < SM_WARPS; ++w) {
        v0 += red[w][nt][2 * rp][mi];
        v1 += red[w][nt][2 * rp + 1][mi];
      }
      const int na = n0 + 2 * rp, nb = na + 1;
      if (m < p.M && na < p.N) {
        if (p.bias != nullptr) {
          v0 += E::to_f(p.bias[na]);
          if (nb < p.N) v1 += E::to_f(p.bias[nb]);
        }
        const long long orow = (long long)(m / p.rows_per_group) * p.group_stride + p.group_offset + (m % p.rows_per_group);
        if (p.epilogue == VSB_EPI_SWIGLU) {
          reinterpret_cast<T*>(p.C)[orow * p.ldc + (na >> 1)] = E::from_f(silu_f(v0) * v1);
        } else {
          float vv[2] = {v0, v1};
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int n = na + e;
            if (n >= p.N) break;
            float x = vv[e];
            if (p.epilogue == VSB_EPI_QUICK_GELU) x = quick_gelu_f(x);
            else if (p.epilogue == VSB_EPI_RELU) x = fmaxf(x, 0.f);
            else if (p.epilogue == VSB_EPI_GELU) x = gelu_erf_f(x);
            if (p.out_fp32) {
              if (p.residual) x += reinterpret_cast<const float*>(p.residual)[orow * p.ldr + n];
              reinterpret_cast<float*>(p.C)[orow * p.ldc + n] = x;
            } else {
              if (p.residual) x += E::to_f(reinterpret_cast<const T*>(p.residual)[orow * p.ldr + n]);
              reinterpret_cast<T*>(p.C)[orow * p.ldc + n] = E::from_f(x);
            }
          }
        }
      }
    }
    __syncthreads();                                    // red is reused by the next row group
  }
}

}  // namespace

// called by vsb_gemm_bf16 / vsb_gemm_f16 (gemm_tcgen05.cu), K % 8 == 0, arguments already validated there.
// variant 1: CUDA-core kernel (M <= 8); variant 2: mma.sync kernel (M <= 16)
template <typename T>
int vsb_gemm_skinny_launch(int variant, const void* A, long long lda, const void* W, long long ldw, void* C, long long ldc, int M, int N,
                           int K, const void* bias, const void* residual, long long ldr, int epilogue, int out_fp32, int rows_per_group,
                           long long group_stride, long long group_offset, cudaStream_t stream) {
  SkinnyParams<T> p;
  p.A = reinterpret_cast<const T*>(A);
  p.W = reinterpret_cast<const T*>(W);
  p.C = C;
  p.bias = reinterpret_cast<const T*>(bias);
  p.residual = residual;
  p.lda = lda; p.ldw = ldw; p.ldc = ldc; p.ldr = ldr;
  p.M = M; p.N = N; p.K = K;
  p.epilogue = epilogue;
  p.out_fp32 = out_fp32;
  p.rows_per_group = rows_per_group;
  p.group_stride = group_stride;
  p.group_offset = group_offset;
  if (variant == 2) {
    const int ngroups = (N + SM_ROWS - 1) / SM_ROWS;
    const int blocks2 = ngroups < vsb_num_sms() * 8 ? ngroups : vsb_num_sms() * 8;
    if (M <= 8) VSB_CUDA(vsb_launch_pdl(gemm_skinny_mma_kernel<1, T>, dim3(blocks2), dim3(SM_WARPS * 32), 0, stream, 1, p));
    else VSB_CUDA(vsb_launch_pdl(gemm_skinny_mma_kernel<2, T>, dim3(blocks2), dim3(SM_WARPS * 32), 0, stream, 1, p));
    return VSB_OK;
  }
  const int npairs = (N + 1) / 2;
  const int warps_per_block = SK_THREADS / 32;
  int blocks = (npairs + warps_per_block - 1) / warps_per_block;
  const int cap = vsb_num_sms() * 8;                    // grid-stride beyond 8 resident blocks per SM
  if (blocks > cap) blocks = cap;
  if (M <= 1) VSB_CUDA(vsb_launch_pdl(gemm_skinny_kernel<1, T>, dim3(blocks), dim3(SK_THREADS), 0, stream, 1, p));
  else if (M <= 2) VSB_CUDA(vsb_launch_pdl(gemm_skinny_kernel<2, T>, dim3(blocks), dim3(SK_THREADS), 0, stream, 1, p));
  else if (M <= 4) VSB_CUDA(vsb_launch_pdl(gemm_skinny_kernel<4, T>, dim3(blocks), dim3(SK_THREADS), 0, stream, 1, p));
  else VSB_CUDA(vsb_launch_pdl(gemm_skinny_kernel<8, T>, dim3(blocks), dim3(SK_THREADS), 0, stream, 1, p));
  return VSB_OK;
}
template int vsb_gemm_skinny_launch<bf16>(int, const void*, long long, const void*, long long, void*, long long, int, int, int, const void*,
                                          const void*, long long, int, int, int, long long, long long, cudaStream_t);
template int vsb_gemm_skinny_launch<half>(int, const void*, long long, const void*, long long, void*, long long, int, int, int, const void*,
                                          const void*, long long, int, int, int, long long, long long, cudaStream_t);
