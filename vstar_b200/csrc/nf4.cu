// NF4 weights of the SEAL VQA LLM in its 4-bit mode (the reference's load_4bit: bitsandbytes NF4 with double-quantised
// scales, fp16 compute; LLaVA/llava/model/builder.py:26-43).
//
// Format of one weight tensor W [N, K] (K % 64 == 0), written from bitsandbytes' published NF4 / double-quant algorithm
// (oracle/nf4_oracle.py is the same format in numpy):
//   * blocks of 64 consecutive row-major values, absmax_b = max |w| (fp32); code = index of the NF4 table entry nearest to
//     w * (1 / absmax_b) (fp32 reciprocal, ties to the lower code; an all-zero block gets the 0.0 code);
//   * two codes per byte, the first element in the high nibble: codes u8 [N, K/2];
//   * double quant of the absmax: offset = mean(absmax) (computed by the caller), c = absmax - offset in groups of 256,
//     absmax2 = max |c|, q8 = nearest entry of the signed 8-bit dynamic map to c * (1 / absmax2); the stored fp32 scale of a
//     block is map[q8] * absmax2 + offset (product and sum rounded separately);
//   * a weight dequantises to f16(nf4[code] * scale) (fp32 product, one rounding).
//
// GEMM C = epi(A . deq(W)^T + bias) (+ residual), the semantics of vsb_gemm_f16:
//   * small M (decode, option scoring): weight-streaming kernels in the style of gemm_skinny.cu that read 16-byte vectors of
//     codes and dequantise in registers (NF4 table in shared memory): a CUDA-core FMA kernel (M <= 8) and an mma.sync
//     m16n8k16 kernel (M <= 32).  Algorithmic bytes per launch: N*K/2 (codes) + N*K/16 (scales) + 2*M*K + 2*M*N;
//   * larger M: deq(W) into a caller-provided f16 scratch, then vsb_gemm_f16 (every tile epilogue unchanged).
#include "common.cuh"
#include "vstar_b200.h"

// largest M the auto dispatch gives the mma.sync streaming kernel; above it the dequant + wgmma tile path is faster
// (tools/bench_vqa_nf4.py measures the crossover at 7B shapes)
#define NF4_SKINNY_MAX_M 32

namespace {

__constant__ float c_nf4[16] = {-1.0f, -0.6961928009986877f, -0.5250730514526367f, -0.39491748809814453f,
                                -0.28444138169288635f, -0.18477343022823334f, -0.09105003625154495f, 0.0f,
                                0.07958029955625534f, 0.16093020141124725f, 0.24611230194568634f, 0.33791524171829224f,
                                0.44070982131767273f, 0.5626170039176941f, 0.7229568362236023f, 1.0f};

// index of the entry of tab[0..n) nearest to v; ties (equal fp32 distances) go to the lower index
__device__ __forceinline__ int nearest(float v, const float* tab, int n) {
  int best = 0;
  float bd = fabsf(__fsub_rn(v, tab[0]));
  for (int i = 1; i < n; ++i) {
    const float d = fabsf(__fsub_rn(v, tab[i]));
    if (d < bd) { bd = d; best = i; }
  }
  return best;
}

__device__ __forceinline__ float inv_or_zero(float a) { return a > 0.f ? __frcp_rn(a) : 0.f; }

// one warp per 64-value block: lane l quantises elements 2l, 2l+1 and writes byte l of the block
__global__ void nf4_quantize_kernel(const half* __restrict__ W, long long nblocks, uint8_t* __restrict__ codes, float* __restrict__ absmax) {
  __shared__ float tab[16];
  if (threadIdx.x < 16) tab[threadIdx.x] = c_nf4[threadIdx.x];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long b = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); b < nblocks; b += nwarps) {
    const float2 w = __half22float2(reinterpret_cast<const __half2*>(W + b * 64)[lane]);
    const float am = warp_max(fmaxf(fabsf(w.x), fabsf(w.y)));
    const float inv = inv_or_zero(am);
    const int c0 = nearest(__fmul_rn(w.x, inv), tab, 16), c1 = nearest(__fmul_rn(w.y, inv), tab, 16);
    codes[b * 32 + lane] = (uint8_t)((c0 << 4) | c1);
    if (lane == 0) absmax[b] = am;
  }
}

// one warp per group of 256 scales (8 per lane)
__global__ void nf4_double_quant_kernel(const float* __restrict__ absmax, long long n, const float* __restrict__ offset_p,
                                        const float* __restrict__ dmap, float* __restrict__ scales) {
  __shared__ float map[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) map[i] = dmap[i];
  __syncthreads();
  const float offset = *offset_p;
  const int lane = threadIdx.x & 31;
  const long long ngroups = (n + 255) / 256;
  const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long gi = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); gi < ngroups; gi += nwarps) {
    float c[8];
    float m = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const long long i = gi * 256 + j * 32 + lane;
      c[j] = i < n ? __fsub_rn(absmax[i], offset) : 0.f;
      m = fmaxf(m, fabsf(c[j]));
    }
    const float am2 = warp_max(m);
    const float inv = inv_or_zero(am2);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const long long i = gi * 256 + j * 32 + lane;
      if (i < n) scales[i] = __fadd_rn(__fmul_rn(map[nearest(__fmul_rn(c[j], inv), map, 256)], am2), offset);
    }
  }
}

// two codes (one byte) -> f16x2, element order (high nibble = first element = low half)
__device__ __forceinline__ uint32_t deq2(uint32_t byte, float s, const float* tab) {
  return ElemT<half>::pack2(__fmul_rn(tab[(byte >> 4) & 15], s), __fmul_rn(tab[byte & 15], s));
}

// thread -> 16 codes (8 bytes) -> 32 bytes of f16
__global__ void nf4_dequant_kernel(const uint8_t* __restrict__ codes, const float* __restrict__ scales, int N, int K, half* __restrict__ out,
                                   long long ldo) {
  __shared__ float tab[16];
  pdl_prologue();
  if (threadIdx.x < 16) tab[threadIdx.x] = c_nf4[threadIdx.x];
  __syncthreads();
  const int per_row = K / 16;
  const long long total = (long long)N * per_row;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / per_row;
    const int c = (int)(i - r * per_row);
    const uint2 v = __ldg(reinterpret_cast<const uint2*>(codes) + i);
    const float s = __ldg(scales + (i >> 2));                // 16 codes of a 64-block: 4 threads per scale
    uint4 o0, o1;
    o0.x = deq2(v.x, s, tab); o0.y = deq2(v.x >> 8, s, tab); o0.z = deq2(v.x >> 16, s, tab); o0.w = deq2(v.x >> 24, s, tab);
    o1.x = deq2(v.y, s, tab); o1.y = deq2(v.y >> 8, s, tab); o1.z = deq2(v.y >> 16, s, tab); o1.w = deq2(v.y >> 24, s, tab);
    uint4* dst = reinterpret_cast<uint4*>(out + r * ldo + (long long)c * 16);
    dst[0] = o0;
    dst[1] = o1;
  }
}

struct Nf4Params {
  const half* A;
  const uint8_t* codes;
  const float* scales;
  void* C;
  const half* bias;
  const void* residual;
  long long lda, ldc, ldr;
  int M, N, K;
  int epilogue, out_fp32;
  int rows_per_group;
  long long group_stride, group_offset;
};

__device__ __forceinline__ uint4 ld_stream16(const void* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}

// epilogue of output (m, n) .. shared by both streaming kernels; same semantics as the f16 skinny / tile kernels
__device__ __forceinline__ void store_out(const Nf4Params& p, int m, int n, float v) {
  const long long orow = (long long)(m / p.rows_per_group) * p.group_stride + p.group_offset + (m % p.rows_per_group);
  if (p.epilogue == VSB_EPI_QUICK_GELU) v = quick_gelu_f(v);
  else if (p.epilogue == VSB_EPI_RELU) v = fmaxf(v, 0.f);
  else if (p.epilogue == VSB_EPI_GELU) v = gelu_erf_f(v);
  if (p.out_fp32) {
    if (p.residual) v += reinterpret_cast<const float*>(p.residual)[orow * p.ldr + n];
    reinterpret_cast<float*>(p.C)[orow * p.ldc + n] = v;
  } else {
    if (p.residual) v += __half2float(reinterpret_cast<const half*>(p.residual)[orow * p.ldr + n]);
    reinterpret_cast<half*>(p.C)[orow * p.ldc + n] = __float2half_rn(v);
  }
}
// the pair (n0, n0+1) = (gate_j, up_j) of an interleaved SwiGLU weight, or two independent columns
__device__ __forceinline__ void store_pair(const Nf4Params& p, int m, int n0, float v0, float v1) {
  if (p.bias != nullptr) {
    v0 += __half2float(p.bias[n0]);
    if (n0 + 1 < p.N) v1 += __half2float(p.bias[n0 + 1]);
  }
  if (p.epilogue == VSB_EPI_SWIGLU) {
    const long long orow = (long long)(m / p.rows_per_group) * p.group_stride + p.group_offset + (m % p.rows_per_group);
    reinterpret_cast<half*>(p.C)[orow * p.ldc + (n0 >> 1)] = __float2half_rn(silu_f(v0) * v1);
    return;
  }
  store_out(p, m, n0, v0);
  if (n0 + 1 < p.N) store_out(p, m, n0 + 1, v1);
}

// ---------------------------------------------------------------- M <= 8: CUDA cores
// One warp owns two weight rows; every lane loads 16 B of codes (32 weights, half a scale block) of each row per step, with
// NK_UNROLL steps in flight.  Activation rows come through L1 (__ldg) as four 16-byte vectors per step.
constexpr int NK_THREADS = 256;
constexpr int NK_UNROLL = 4;

__device__ __forceinline__ void deq8_f32(uint32_t w, float s, const float* tab, float* f) {
#pragma unroll
  for (int b = 0; b < 4; ++b) {
    const float2 t = ElemT<half>::unpack2(deq2(w >> (8 * b), s, tab));
    f[2 * b] = t.x;
    f[2 * b + 1] = t.y;
  }
}

template <int MT>
__global__ void __launch_bounds__(NK_THREADS) gemm_nf4_fma_kernel(const Nf4Params p) {
  __shared__ float tab[16];
  pdl_prologue();
  if (threadIdx.x < 16) tab[threadIdx.x] = c_nf4[threadIdx.x];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * NK_THREADS + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * NK_THREADS) >> 5;
  const int npairs = (p.N + 1) >> 1;
  const int kchunks = p.K >> 5;                    // 32 weights = 16 bytes of codes
  const long long rowb = p.K >> 1;
  const uint4 zero = make_uint4(0u, 0u, 0u, 0u);

  for (int pair = warp; pair < npairs; pair += nwarps) {
    const int n0 = pair * 2;
    const int n1 = (n0 + 1 < p.N) ? n0 + 1 : n0;
    const uint4* w0 = reinterpret_cast<const uint4*>(p.codes + (long long)n0 * rowb);
    const uint4* w1 = reinterpret_cast<const uint4*>(p.codes + (long long)n1 * rowb);
    const float* s0 = p.scales + (long long)n0 * (p.K >> 6);
    const float* s1 = p.scales + (long long)n1 * (p.K >> 6);
    float acc[MT][2];
#pragma unroll
    for (int m = 0; m < MT; ++m) acc[m][0] = acc[m][1] = 0.f;

    for (int c0 = lane; c0 < kchunks; c0 += 32 * NK_UNROLL) {
      uint4 wa[NK_UNROLL], wb[NK_UNROLL];
      float sa[NK_UNROLL], sb[NK_UNROLL];
#pragma unroll
      for (int u = 0; u < NK_UNROLL; ++u) {
        const int c = c0 + u * 32;
        const bool ok = c < kchunks;
        wa[u] = ok ? ld_stream16(w0 + c) : zero;
        wb[u] = ok ? ld_stream16(w1 + c) : zero;
        sa[u] = ok ? __ldg(s0 + (c >> 1)) : 0.f;
        sb[u] = ok ? __ldg(s1 + (c >> 1)) : 0.f;
      }
#pragma unroll
      for (int u = 0; u < NK_UNROLL; ++u) {
        const int c = c0 + u * 32;
        if (c < kchunks) {
          const uint32_t ua[4] = {wa[u].x, wa[u].y, wa[u].z, wa[u].w};
          const uint32_t ub[4] = {wb[u].x, wb[u].y, wb[u].z, wb[u].w};
#pragma unroll
          for (int q = 0; q < 4; ++q) {                     // 8 weights per 32-bit word of codes
            float fa[8], fb[8];
            deq8_f32(ua[q], sa[u], tab, fa);
            deq8_f32(ub[q], sb[u], tab, fb);
#pragma unroll
            for (int m = 0; m < MT; ++m) {
              if (m < p.M) {
                const uint4 av = __ldg(reinterpret_cast<const uint4*>(p.A + (long long)m * p.lda + (long long)c * 32) + q);
                const uint32_t aw[4] = {av.x, av.y, av.z, av.w};
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                  const float2 x = ElemT<half>::unpack2(aw[i]);
                  acc[m][0] = fmaf(x.x, fa[2 * i], acc[m][0]);
                  acc[m][0] = fmaf(x.y, fa[2 * i + 1], acc[m][0]);
                  acc[m][1] = fmaf(x.x, fb[2 * i], acc[m][1]);
                  acc[m][1] = fmaf(x.y, fb[2 * i + 1], acc[m][1]);
                }
              }
            }
          }
        }
      }
    }
#pragma unroll
    for (int m = 0; m < MT; ++m) {
      acc[m][0] = warp_sum(acc[m][0]);
      acc[m][1] = warp_sum(acc[m][1]);
    }
    // lane m finishes row m of both columns
#pragma unroll
    for (int m = 0; m < MT; ++m)
      if (lane == m && m < p.M) store_pair(p, m, n0, acc[m][0], acc[m][1]);
  }
}

// ---------------------------------------------------------------- M <= 32: mma.sync m16n8k16
// A block owns 16 weight rows (the A operand of the MMA); its 8 warps interleave over K in steps of 128: lane (g, t) loads
// 16 B of codes = 32 consecutive k of rows g and g+8, dequantises them in registers and feeds 8 MMAs, taking k-slots
// {2t, 2t+1, 2t+8, 2t+9} of MMA j from its weights 4j..4j+3 (the same permutation on the activation side: the contraction
// is order-free).  The activation rows (<= 8 per n-tile) are the B operand; the 8 warps are summed through shared memory.
constexpr int NM_ROWS = 16;
constexpr int NM_WARPS = 8;
constexpr int NM_UNROLL = 2;

__device__ __forceinline__ void mma_f16(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

template <int NT>      // n-tiles of 8 activation rows: M <= 8 * NT
__global__ void __launch_bounds__(NM_WARPS * 32) gemm_nf4_mma_kernel(const Nf4Params p) {
  __shared__ float tab[16];
  __shared__ float red[NM_WARPS][NT][NM_ROWS][8 + 1];
  pdl_prologue();
  if (threadIdx.x < 16) tab[threadIdx.x] = c_nf4[threadIdx.x];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int ksteps = (p.K + 127) >> 7;
  const long long rowb = p.K >> 1;
  const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
  const int ngroups = (p.N + NM_ROWS - 1) / NM_ROWS;

  for (int grp = blockIdx.x; grp < ngroups; grp += gridDim.x) {
    const int n0 = grp * NM_ROWS;
    const bool r0ok = (n0 + g) < p.N, r1ok = (n0 + g + 8) < p.N;
    const long long ra = r0ok ? n0 + g : 0, rb = r1ok ? n0 + g + 8 : 0;
    const uint8_t* w0 = p.codes + ra * rowb + t * 16;
    const uint8_t* w1 = p.codes + rb * rowb + t * 16;
    const float* s0 = p.scales + ra * (p.K >> 6);
    const float* s1 = p.scales + rb * (p.K >> 6);
    const half* arow[NT];
    bool aok[NT];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      aok[nt] = (nt * 8 + g) < p.M;
      arow[nt] = p.A + (long long)(aok[nt] ? nt * 8 + g : 0) * p.lda + t * 32;
    }
    float c[NT][4];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) c[nt][0] = c[nt][1] = c[nt][2] = c[nt][3] = 0.f;

    for (int s0i = warp; s0i < ksteps; s0i += NM_WARPS * NM_UNROLL) {
      uint4 wa[NM_UNROLL], wb[NM_UNROLL];
      float sa[NM_UNROLL], sb[NM_UNROLL];
#pragma unroll
      for (int u = 0; u < NM_UNROLL; ++u) {
        const int k = (s0i + u * NM_WARPS) * 128;
        const bool ok = (k + t * 32) < p.K;             // K % 32 == 0: a 32-weight chunk is fully inside or outside
        wa[u] = (ok && r0ok) ? ld_stream16(w0 + (k >> 1)) : zero;
        wb[u] = (ok && r1ok) ? ld_stream16(w1 + (k >> 1)) : zero;
        sa[u] = (ok && r0ok) ? __ldg(s0 + ((k + t * 32) >> 6)) : 0.f;
        sb[u] = (ok && r1ok) ? __ldg(s1 + ((k + t * 32) >> 6)) : 0.f;
      }
#pragma unroll
      for (int u = 0; u < NM_UNROLL; ++u) {
        const int k = (s0i + u * NM_WARPS) * 128;
        const bool ok = (k + t * 32) < p.K;
        const uint32_t ua[4] = {wa[u].x, wa[u].y, wa[u].z, wa[u].w};
        const uint32_t ub[4] = {wb[u].x, wb[u].y, wb[u].z, wb[u].w};
        uint32_t da[16], db[16];                         // f16x2 of weights (2i, 2i+1) of rows g and g+8
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          da[i] = deq2(ua[i >> 2] >> (8 * (i & 3)), sa[u], tab);
          db[i] = deq2(ub[i >> 2] >> (8 * (i & 3)), sb[u], tab);
        }
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
          uint4 av[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) av[q] = (ok && aok[nt]) ? __ldg(reinterpret_cast<const uint4*>(arow[nt] + k) + q) : zero;
          const uint32_t* aw = reinterpret_cast<const uint32_t*>(av);
#pragma unroll
          for (int j = 0; j < 8; ++j) mma_f16(c[nt], da[2 * j], db[2 * j], da[2 * j + 1], db[2 * j + 1], aw[2 * j], aw[2 * j + 1]);
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
    for (int idx = threadIdx.x; idx < 8 * 8 * NT; idx += NM_WARPS * 32) {
      const int rp = idx & 7, m = idx >> 3;
      const int nt = m >> 3, mi = m & 7;
      float v0 = 0.f, v1 = 0.f;
#pragma unroll
      for (int w = 0; w < NM_WARPS; ++w) {
        v0 += red[w][nt][2 * rp][mi];
        v1 += red[w][nt][2 * rp + 1][mi];
      }
      const int na = n0 + 2 * rp;
      if (m < p.M && na < p.N) store_pair(p, m, na, v0, v1);
    }
    __syncthreads();                                    // red is reused by the next row group
  }
}

int dequant_launch(const void* codes, const void* scales, int N, int K, void* out, long long ldo, cudaStream_t stream) {
  const long long total = (long long)N * (K / 16);
  long long blocks = (total + 255) / 256;
  const long long cap = (long long)vsb_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  VSB_CUDA(vsb_launch_pdl(nf4_dequant_kernel, dim3((unsigned)blocks), dim3(256), 0, stream, 1, reinterpret_cast<const uint8_t*>(codes),
                          reinterpret_cast<const float*>(scales), N, K, reinterpret_cast<half*>(out), ldo));
  return VSB_OK;
}

}  // namespace

// kernel variant of an NF4 GEMM with M rows: 1 / 2 = streaming kernels, 0 = dequant + wgmma tile, -1 = forced variant cannot
// take M.  Honours vsb_gemm_set_tuning (1 / 2 force a streaming kernel, a tile width forces the tile path) and batch invariance.
int vsb_nf4_variant(int M) {
  const int f = vsb_gemm_forced_bn();
  if (f == 1) return M <= 8 ? 1 : -1;
  if (f == 2) return M <= 32 ? 2 : -1;
  if (f != 0 || vsb_batch_invariant()) return 0;
  if (M == 1) return 1;
  return M <= NF4_SKINNY_MAX_M ? 2 : 0;
}

extern "C" int vsb_nf4_quantize(const void* w, int N, int K, void* codes, void* absmax, void* stream) {
  VSB_CHECK_ARG(w && codes && absmax && N > 0 && K > 0, "vsb_nf4_quantize: null pointer or bad shape");
  VSB_CHECK_ARG(K % 64 == 0, "vsb_nf4_quantize: K = %d is not a multiple of the 64-value block", K);
  VSB_CHECK_ARG((reinterpret_cast<uintptr_t>(w) & 3) == 0, "vsb_nf4_quantize: w must be 4-byte aligned");
  const long long nblocks = (long long)N * (K / 64);
  long long blocks = (nblocks + 7) / 8;
  const long long cap = (long long)vsb_num_sms() * 32;
  if (blocks > cap) blocks = cap;
  nf4_quantize_kernel<<<(unsigned)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const half*>(w), nblocks, reinterpret_cast<uint8_t*>(codes), reinterpret_cast<float*>(absmax));
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

extern "C" int vsb_nf4_double_quant(const void* absmax, long long n, const void* offset, const void* dmap, void* scales, void* stream) {
  VSB_CHECK_ARG(absmax && offset && dmap && scales && n > 0, "vsb_nf4_double_quant: null pointer or empty input");
  const long long ngroups = (n + 255) / 256;
  long long blocks = (ngroups + 7) / 8;
  const long long cap = (long long)vsb_num_sms() * 32;
  if (blocks > cap) blocks = cap;
  nf4_double_quant_kernel<<<(unsigned)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float*>(absmax), n, reinterpret_cast<const float*>(offset), reinterpret_cast<const float*>(dmap),
      reinterpret_cast<float*>(scales));
  VSB_LAUNCH_CHECK();
  return VSB_OK;
}

extern "C" int vsb_nf4_dequant(const void* codes, const void* scales, int N, int K, void* out, long long ldo, void* stream) {
  VSB_CHECK_ARG(codes && scales && out && N > 0 && K > 0, "vsb_nf4_dequant: null pointer or bad shape");
  VSB_CHECK_ARG(K % 64 == 0, "vsb_nf4_dequant: K = %d is not a multiple of the 64-value block", K);
  VSB_CHECK_ARG(ldo >= K && ldo % 8 == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0 && (reinterpret_cast<uintptr_t>(codes) & 7) == 0,
                "vsb_nf4_dequant: out needs ldo >= K, ldo %% 8 == 0 and 16-byte alignment, codes 8-byte alignment");
  return dequant_launch(codes, scales, N, K, out, ldo, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int vsb_gemm_nf4(const void* A, long long lda, const void* codes, const void* scales, void* C, long long ldc, int M, int N,
                                int K, const void* bias, const void* residual, long long ldr, int epilogue, int out_fp32, int rows_per_group,
                                long long group_stride, long long group_offset, void* deq_scratch, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  VSB_CHECK_ARG(A && codes && scales && C, "vsb_gemm_nf4: null pointer");
  VSB_CHECK_ARG(M > 0 && N > 0 && K > 0, "vsb_gemm_nf4: bad shape M=%d N=%d K=%d", M, N, K);
  VSB_CHECK_ARG(K % 64 == 0, "vsb_gemm_nf4: K = %d is not a multiple of the 64-value block", K);
  VSB_CHECK_ARG(lda % 8 == 0 && lda >= K, "vsb_gemm_nf4: lda must be >= K and a multiple of 8, got %lld", lda);
  VSB_CHECK_ARG((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(codes) & 15) == 0 &&
                    (reinterpret_cast<uintptr_t>(scales) & 3) == 0,
                "vsb_gemm_nf4: A / codes must be 16-byte aligned");
  VSB_CHECK_ARG(epilogue >= VSB_EPI_NONE && epilogue <= VSB_EPI_SWIGLU, "vsb_gemm_nf4: bad epilogue %d", epilogue);
  VSB_CHECK_ARG(!(epilogue == VSB_EPI_SWIGLU && (out_fp32 || residual || (N & 1))), "vsb_gemm_nf4: SwiGLU epilogue is f16, no residual, even N");
  const int variant = vsb_nf4_variant(M);
  VSB_CHECK_ARG(variant >= 0, "vsb_gemm_nf4: streaming kernel forced but M=%d too large", M);
  if (variant == 0) {
    VSB_CHECK_ARG(deq_scratch != nullptr && (reinterpret_cast<uintptr_t>(deq_scratch) & 15) == 0,
                  "vsb_gemm_nf4: M=%d takes the dequant + tile path, which needs a 16-byte aligned f16 scratch of N*K elements", M);
    const int r = dequant_launch(codes, scales, N, K, deq_scratch, K, stream);
    if (r) return r;
    return vsb_gemm_f16(A, lda, deq_scratch, K, C, ldc, M, N, K, bias, residual, ldr, epilogue, out_fp32, rows_per_group, group_stride,
                        group_offset, stream_);
  }
  Nf4Params p;
  p.A = reinterpret_cast<const half*>(A);
  p.codes = reinterpret_cast<const uint8_t*>(codes);
  p.scales = reinterpret_cast<const float*>(scales);
  p.C = C;
  p.bias = reinterpret_cast<const half*>(bias);
  p.residual = residual;
  p.lda = lda; p.ldc = ldc; p.ldr = ldr;
  p.M = M; p.N = N; p.K = K;
  p.epilogue = epilogue;
  p.out_fp32 = out_fp32;
  if (rows_per_group <= 0) {
    rows_per_group = M;
    group_stride = 0;
    group_offset = 0;
  }
  p.rows_per_group = rows_per_group;
  p.group_stride = group_stride;
  p.group_offset = group_offset;
  if (variant == 2) {
    const int ngroups = (N + NM_ROWS - 1) / NM_ROWS;
    const int blocks = ngroups < vsb_num_sms() * 8 ? ngroups : vsb_num_sms() * 8;
    if (M <= 8) VSB_CUDA(vsb_launch_pdl(gemm_nf4_mma_kernel<1>, dim3(blocks), dim3(NM_WARPS * 32), 0, stream, 1, p));
    else if (M <= 16) VSB_CUDA(vsb_launch_pdl(gemm_nf4_mma_kernel<2>, dim3(blocks), dim3(NM_WARPS * 32), 0, stream, 1, p));
    else VSB_CUDA(vsb_launch_pdl(gemm_nf4_mma_kernel<4>, dim3(blocks), dim3(NM_WARPS * 32), 0, stream, 1, p));
    return VSB_OK;
  }
  const int npairs = (N + 1) / 2;
  int blocks = (npairs + NK_THREADS / 32 - 1) / (NK_THREADS / 32);
  if (blocks > vsb_num_sms() * 8) blocks = vsb_num_sms() * 8;
  if (M <= 1) VSB_CUDA(vsb_launch_pdl(gemm_nf4_fma_kernel<1>, dim3(blocks), dim3(NK_THREADS), 0, stream, 1, p));
  else if (M <= 2) VSB_CUDA(vsb_launch_pdl(gemm_nf4_fma_kernel<2>, dim3(blocks), dim3(NK_THREADS), 0, stream, 1, p));
  else if (M <= 4) VSB_CUDA(vsb_launch_pdl(gemm_nf4_fma_kernel<4>, dim3(blocks), dim3(NK_THREADS), 0, stream, 1, p));
  else VSB_CUDA(vsb_launch_pdl(gemm_nf4_fma_kernel<8>, dim3(blocks), dim3(NK_THREADS), 0, stream, 1, p));
  return VSB_OK;
}
